"""Host-side mirror of /root/reference/src/adaptive_classifier/models.py (Example, AdaptiveHead, ModelConfig).

Same names, constructor arguments, defaults, state_dict keys and seeding side effects; the arithmetic of
AdaptiveHead.forward runs in the hand-written CUDA head kernels behind the C ABI (csrc/head.cu).
"""
from __future__ import annotations

import logging
from dataclasses import dataclass
from typing import Any, Dict, Optional

import torch
import torch.nn as nn

from . import _cabi

logger = logging.getLogger(__name__)


@dataclass
class Example:
    """Represents a single training example (models.py:9-28)."""
    text: str
    label: str
    embedding: Optional[torch.Tensor] = None

    def to_dict(self) -> Dict[str, Any]:
        return {
            "text": self.text,
            "label": self.label,
            "embedding": self.embedding.tolist() if self.embedding is not None else None,
        }

    @classmethod
    def from_dict(cls, data: Dict[str, Any]) -> "Example":
        embedding = torch.tensor(data["embedding"]) if data["embedding"] is not None else None
        return cls(text=data["text"], label=data["label"], embedding=embedding)


def _linears(seq: nn.Sequential):
    return [m for m in seq if isinstance(m, nn.Linear)]


class _CudaHeadMixin:
    """Shared plumbing: expose the nn.Linear parameters of `self.model` as the C-ABI parameter block."""

    _act = _cabi.AC_ACT_LOGITS

    def _param_dict(self) -> Dict[str, torch.Tensor]:
        lins = _linears(self.model)
        if len(lins) != 3:
            raise _cabi.AdaptiveB200Error(
                f"the CUDA head kernels implement the reference's 3-layer head (got {len(lins)} Linear layers)")
        out = {}
        for i, lin in enumerate(lins):
            for nm, t in ((f"W{i}", lin.weight), (f"b{i}", lin.bias)):
                if not t.is_cuda:
                    raise _cabi.AdaptiveB200Error("adaptive head parameters must live on the GPU (no CPU path)")
                if not t.data.is_contiguous():
                    t.data = t.data.contiguous()
                out[nm] = t.data
        return out

    def _forward_cuda(self, x: torch.Tensor, act: int) -> torch.Tensor:
        if x.dim() == 1:
            x = x.unsqueeze(0)
        p = self._param_dict()
        dev = p["W0"].device
        x = x.to(device=dev, dtype=torch.float32).contiguous()
        if self.training:
            raise _cabi.AdaptiveB200Error(
                "train-mode forward is fused into ac_head_train_step; call .eval() for inference")
        return _cabi.head_forward(x, p, act)


class AdaptiveHead(_CudaHeadMixin, nn.Module):
    """Neural network head with stable initialization and deterministic behavior (models.py:30-98)."""

    def __init__(self, input_dim: int, num_classes: int, hidden_dims: Optional[list] = None):
        super().__init__()
        if hidden_dims is None:
            hidden_dims = [input_dim]
        layers = []
        prev_dim = input_dim
        for dim in hidden_dims:
            linear = nn.Linear(prev_dim, dim)
            torch.manual_seed(42)   # global-RNG side effect kept on purpose (models.py:51)
            nn.init.kaiming_uniform_(linear.weight, mode="fan_in", nonlinearity="relu")
            nn.init.zeros_(linear.bias)
            layers.extend([linear, nn.ReLU(), nn.Dropout(0.1)])
            prev_dim = dim
        output_layer = nn.Linear(prev_dim, num_classes)
        torch.manual_seed(42)       # models.py:64
        nn.init.xavier_uniform_(output_layer.weight)
        nn.init.zeros_(output_layer.bias)
        layers.append(output_layer)
        self.model = nn.Sequential(*layers)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """[B, C] logits; a 1-D input gets a batch dimension (models.py:71-80)."""
        return self._forward_cuda(x, _cabi.AC_ACT_LOGITS)

    def update_num_classes(self, num_classes: int):
        """Grow the output layer preserving existing rows (models.py:82-98)."""
        current_weight = self.model[-1].weight
        current_bias = self.model[-1].bias
        if num_classes > current_weight.size(0):
            new_layer = nn.Linear(current_weight.size(1), num_classes)
            torch.manual_seed(42)   # models.py:89
            nn.init.xavier_uniform_(new_layer.weight)
            nn.init.zeros_(new_layer.bias)
            new_layer = new_layer.to(current_weight.device)
            with torch.no_grad():
                new_layer.weight[: current_weight.size(0)] = current_weight
                new_layer.bias[: current_weight.size(0)] = current_bias
            self.model[-1] = new_layer


class ModelConfig:
    """Configuration for the adaptive classifier (models.py:100-196); same keys and defaults."""

    _DEFAULTS = [
        ("max_length", 512), ("batch_size", 32), ("learning_rate", 0.001), ("warmup_steps", 0),
        ("max_examples_per_class", 1000), ("prototype_update_frequency", 100), ("similarity_threshold", 0.6),
        ("ewc_lambda", 100.0), ("num_representative_examples", 5),
        ("epochs", 10), ("early_stopping_patience", 3), ("min_examples_per_class", 3),
        ("prototype_weight", 0.7), ("neural_weight", 0.3), ("min_confidence", 0.1),
        ("device_map", "auto"), ("quantization", None), ("gradient_checkpointing", False),
        ("enable_strategic_mode", False), ("cost_function_type", "separable"), ("strategic_lambda", 0.1),
        ("cost_coefficients", None), ("strategic_training_frequency", 10),
        ("strategic_blend_regular_weight", 0.6), ("strategic_blend_strategic_weight", 0.4),
        ("strategic_robust_proto_weight", 0.8), ("strategic_robust_head_weight", 0.2),
        ("strategic_prediction_proto_weight", 0.5), ("strategic_prediction_head_weight", 0.5),
    ]

    def __init__(self, config: Optional[Dict[str, Any]] = None):
        self.config = config or {}
        for key, default in self._DEFAULTS:
            if key == "cost_coefficients":
                default = {}
            setattr(self, key, self.config.get(key, default))

    def update(self, **kwargs):
        for key, value in kwargs.items():
            if hasattr(self, key):
                setattr(self, key, value)
            else:
                logger.warning(f"Unknown configuration parameter: {key}")

    def to_dict(self) -> Dict[str, Any]:
        return {key: getattr(self, key) for key, _ in self._DEFAULTS}
