"""Host-side mirror of /root/reference/src/adaptive_classifier/strategic.py (strategic classification).

Same class names, constructors, errors and `compute_cost` as the reference.  The best-response search -- the reference's 50
separate head forwards per sample (strategic.py:74-123) -- runs on the H100 in csrc/strategic.cu against the classifier's own
head, and the strategic loss (strategic.py:200-242) inside the training kernel (AC_LOSS_CE_STRATEGIC).  A best response for an
arbitrary Python callable is not provided: `compute_best_response` takes the head's parameter block, not a function.
"""
from __future__ import annotations

import logging
from abc import ABC, abstractmethod
from typing import Dict, List, Optional, Union

import torch

from . import _cabi

logger = logging.getLogger(__name__)


def candidate_table(x: torch.Tensor) -> torch.Tensor:
    """The reference's `_generate_candidates(x, 50)` (strategic.py:104-123) for D >= 5: x, then x with x_i += delta for
    i = 0..3 and every delta of linspace(-2, 2, 10), then i = 4 with the first 9 deltas.  No random candidate is reached and no
    RNG is consumed.  [50, D] fp32, on x's device."""
    if x.dim() != 1 or x.shape[0] < 5:
        raise ValueError("the candidate table needs a 1-D embedding with at least 5 features")
    deltas = torch.linspace(-2.0, 2.0, 10)
    rows = [x.clone()]
    for i in range(5):
        for delta in deltas:
            if len(rows) == _cabi.AC_STRATEGIC_CANDIDATES:
                break
            c = x.clone()
            c[i] += delta.to(c.device)
            rows.append(c)
    return torch.stack(rows)


class StrategicCostFunction(ABC):
    """Abstract base class for strategic cost functions (strategic.py:11-38)."""

    cost_kind: int

    @abstractmethod
    def compute_cost(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        pass

    def device_coefficients(self, D: int, device) -> tuple:
        """(c1, c2) as fp32 [D] on `device` for the search kernel, copied once per (D, device, coefficient tensors).  Raises
        ValueError when the coefficients cannot be applied to a D-dimensional fp32 embedding -- the cases where the reference's
        torch.dot raises: a wrong length, or any dtype other than float32 (the embeddings' dtype; torch.dot requires both
        vectors to have the same one)."""
        c1, c2 = torch.as_tensor(self.c1), torch.as_tensor(self.c2)
        key = (D, str(device), id(c1), c1._version, id(c2), c2._version)
        cached = self.__dict__.get("_device_cache")
        if cached is not None and cached[0] == key:
            return cached[1]
        for c in (c1, c2):
            if c.dim() != 1 or c.shape[0] != D:
                raise ValueError(f"cost coefficients of shape {tuple(c.shape)} do not match embeddings of dimension {D}")
            if c.dtype != torch.float32:
                raise ValueError(f"cost coefficients of dtype {c.dtype} differ from the embeddings' torch.float32")
        out = (c1.to(device=device).contiguous(), c2.to(device=device).contiguous())
        self._device_cache = (key, out, c1, c2)          # c1 / c2 kept alive: their ids stay theirs while cached
        return out

    def compute_best_response(self, x: torch.Tensor, head_params: Dict[str, torch.Tensor], *, dropout_p: float = 0.0,
                              seed: int = 0, step: int = 0):
        """Best responses of the rows of x [B, D] (CUDA) against the adaptive head whose parameter block is `head_params`
        (AdaptiveHead._param_dict()).  Returns (choice int32 [B], utility fp32 [B], rows [B, D])."""
        c1, c2 = self.device_coefficients(x.shape[-1], x.device)
        return _cabi.strategic_best_response(x, head_params, self.cost_kind, c1, c2, dropout_p=dropout_p, seed=seed, step=step)


class SeparableCostFunction(StrategicCostFunction):
    """c(x, y) = max{0, c2(y) - c1(x)} (strategic.py:41-102)."""

    cost_kind = _cabi.AC_COST_SEPARABLE

    def __init__(self, c1_coefficients: Union[Dict[str, float], torch.Tensor], c2_coefficients: Union[Dict[str, float], torch.Tensor],
                 feature_names: Optional[List[str]] = None):
        if isinstance(c1_coefficients, dict) and isinstance(c2_coefficients, dict):
            if feature_names is None:
                raise ValueError("feature_names required when using dict coefficients")
            self.c1 = torch.tensor([c1_coefficients.get(name, 0.0) for name in feature_names])
            self.c2 = torch.tensor([c2_coefficients.get(name, 0.0) for name in feature_names])
            self.feature_names = feature_names
        else:
            self.c1 = c1_coefficients if isinstance(c1_coefficients, torch.Tensor) else torch.tensor(c1_coefficients)
            self.c2 = c2_coefficients if isinstance(c2_coefficients, torch.Tensor) else torch.tensor(c2_coefficients)
            self.feature_names = feature_names

    def compute_cost(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        c1_x = torch.dot(self.c1, x)
        c2_y = torch.dot(self.c2, y)
        return torch.relu(c2_y - c1_x)


class LinearCostFunction(SeparableCostFunction):
    """c(x, y) = <alpha, y - x>_+ (strategic.py:126-155)."""

    cost_kind = _cabi.AC_COST_LINEAR

    def __init__(self, alpha: Union[Dict[str, float], torch.Tensor], feature_names: Optional[List[str]] = None):
        if isinstance(alpha, dict):
            if feature_names is None:
                raise ValueError("feature_names required when using dict coefficients")
            alpha_tensor = torch.tensor([alpha.get(name, 0.0) for name in feature_names])
        else:
            alpha_tensor = alpha if isinstance(alpha, torch.Tensor) else torch.tensor(alpha)
        super().__init__(alpha_tensor, alpha_tensor, feature_names)
        self.alpha = alpha_tensor

    def compute_cost(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        diff = y - x
        cost = torch.dot(self.alpha, diff)
        return torch.relu(cost)


class CostFunctionFactory:
    """strategic.py:158-186."""

    @staticmethod
    def create_cost_function(cost_type: str, cost_coefficients: Dict[str, float], feature_names: Optional[List[str]] = None,
                             **kwargs) -> StrategicCostFunction:
        if cost_type == "linear":
            return LinearCostFunction(cost_coefficients, feature_names)
        elif cost_type == "separable":
            c2_coefficients = kwargs.get("c2_coefficients", cost_coefficients)
            return SeparableCostFunction(cost_coefficients, c2_coefficients, feature_names)
        else:
            raise ValueError(f"Unknown cost function type: {cost_type}")


class StrategicOptimizer:
    """strategic.py:189-242.  The strategic loss itself runs inside the training kernel (AdaptiveClassifier._strategic_training_step)."""

    def __init__(self, cost_function: StrategicCostFunction):
        self.cost_function = cost_function


class StrategicEvaluator:
    """strategic.py:273-358."""

    def __init__(self, cost_function: StrategicCostFunction):
        self.cost_function = cost_function

    def evaluate_robustness(self, head, test_embeddings: torch.Tensor, test_labels: torch.Tensor,
                            gaming_levels: List[float] = [0.0, 0.5, 1.0]) -> Dict[str, float]:
        """head: the classifier's AdaptiveHead (eval mode).  One best-response search over all embeddings serves every level;
        which rows game is decided per level and row by one global torch.rand(1) draw, in the reference's order."""
        params = head._param_dict()
        dev = params["W0"].device
        X = test_embeddings.to(device=dev, dtype=torch.float32).contiguous()
        _, _, br = self.cost_function.compute_best_response(X, params)
        labels = test_labels.to(dev)
        results = {}
        for level in gaming_levels:
            game = torch.tensor([torch.rand(1).item() < level for _ in range(X.shape[0])], dtype=torch.bool, device=dev)
            strategic_embeddings = torch.where(game[:, None], br, X)
            logits = _cabi.head_forward(strategic_embeddings, params, _cabi.AC_ACT_LOGITS)
            predictions = torch.argmax(logits, dim=-1)
            accuracy = (predictions == labels).float().mean().item()
            results[f"accuracy_gaming_{level}"] = accuracy
        results["robustness_score"] = results["accuracy_gaming_0.0"] - results["accuracy_gaming_1.0"]
        results["relative_robustness"] = results["accuracy_gaming_1.0"] / results["accuracy_gaming_0.0"]
        return results
