"""Host-side mirror of /root/reference/src/adaptive_classifier/ewc.py (EWC).

Same constructor and `ewc_loss(batch_size)`; Fisher accumulation and the penalty run in csrc/head.cu
(ac_head_grad with fisher accumulation, ac_ewc_penalty).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn as nn

from . import _cabi


class EWC:
    """Elastic Weight Consolidation (ewc.py:7-115)."""

    def __init__(self, model: nn.Module, dataset: torch.utils.data.Dataset, device: str = "cuda",
                 ewc_lambda: float = 100.0):
        self.model = model
        self.device = device
        self.ewc_lambda = ewc_lambda
        # theta* snapshot (ewc.py:30-34)
        self.old_params = {n: p.data.clone() for n, p in model.named_parameters() if p.requires_grad}
        self.fisher_info = self._compute_fisher(dataset)

    # name maps between nn.Module parameter names and the C-ABI block
    def _blocks(self):
        names = [n for n, p in self.model.named_parameters() if p.requires_grad]
        if len(names) != 6:
            raise _cabi.AdaptiveB200Error("EWC on the CUDA path supports the reference's 3-layer head only")
        return names

    def _as_block(self, tensors: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        names = self._blocks()
        keys = ["W0", "b0", "W1", "b1", "W2", "b2"]
        return {k: tensors[n].contiguous() for k, n in zip(keys, names)}

    def _compute_fisher(self, dataset) -> Dict[str, torch.Tensor]:
        """ewc.py:39-94: eval mode, batches of 32 shuffled with the global RNG, labels sampled from the
        model's own softmax (multinomial), fisher += grad(mean NLL)^2 / n_batches."""
        params = {n: p for n, p in self.model.named_parameters() if p.requires_grad}
        fisher = {n: torch.zeros_like(p.data) for n, p in params.items()}
        self.model.eval()
        loader = torch.utils.data.DataLoader(dataset, batch_size=32, shuffle=True)
        n_batches = len(loader)
        pblock = self._as_block({n: p.data for n, p in params.items()})
        fblock = self._as_block(fisher)
        dev = pblock["W0"].device
        sigmoid_head = getattr(self.model, "_act", _cabi.AC_ACT_LOGITS) == _cabi.AC_ACT_SIGMOID
        for batch_embeddings, _batch_labels in loader:
            x = batch_embeddings.to(device=dev, dtype=torch.float32).contiguous()
            logits = _cabi.head_forward(x, pblock, _cabi.AC_ACT_LOGITS)
            # the reference feeds the module OUTPUT to softmax: for the multilabel head that output is
            # already sigmoid(logits) (multilabel.py:41-44), kept as is
            outputs = torch.sigmoid(logits) if sigmoid_head else logits
            probs = torch.softmax(outputs, dim=1)
            sampled = torch.multinomial(probs, 1).squeeze(-1)
            if sigmoid_head:
                raise _cabi.AdaptiveB200Error("Fisher for the sigmoid head is not implemented on the CUDA path")
            _cabi.head_grad(x, sampled, pblock, loss_kind=_cabi.AC_LOSS_CE, fisher=fblock,
                            inv_n_batches=1.0 / n_batches)
        names = self._blocks()
        for k, n in zip(["W0", "b0", "W1", "b1", "W2", "b2"], names):
            fisher[n] = fblock[k]
        return fisher

    def ewc_loss(self, batch_size: Optional[int] = None) -> torch.Tensor:
        """ewc.py:96-115: lambda * sum_n sum(F_n * (theta_n - theta*_n)^2) [/ batch_size]."""
        params = {n: p.data for n, p in self.model.named_parameters() if p.requires_grad}
        out = _cabi.ewc_penalty(self._as_block(params), self._as_block(self.fisher_info),
                                self._as_block(self.old_params), self.ewc_lambda, batch_size)
        return out[0]
