"""Multi-label front end on top of the H100 hot path.

Behavioural mirror of /root/reference/src/adaptive_classifier/multilabel.py (MultiLabelAdaptiveHead :15-68,
MultiLabelAdaptiveClassifier :71-426): sigmoid head, per-label / size-adaptive thresholds, min/max number of
predictions, BCE training on multi-hot targets.  The sigmoid epilogue and the BCE optimizer step are the
AC_ACT_SIGMOID / AC_LOSS_BCE variants of csrc/head.cu; everything threshold-related is host logic and is kept
table-driven here.
"""
from __future__ import annotations

import logging
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _cabi
from .classifier import AdaptiveClassifier
from .models import _CudaHeadMixin

logger = logging.getLogger(__name__)

# multilabel.py:113-130: the more labels exist, the lower an individual sigmoid score tends to be
_SIZE_SCALE: Sequence[Tuple[int, float]] = ((2, 1.0), (5, 0.8), (10, 0.6), (20, 0.4))
_SIZE_SCALE_MANY = 0.2
# multilabel.py:280-307: rare labels get a lower bar, very common ones a higher bar (share of stored examples)
_RARE, _UNCOMMON, _COMMON = (0.05, 0.3), (0.10, 0.5), (0.30, 1.2)


class MultiLabelAdaptiveHead(_CudaHeadMixin, nn.Module):
    """Three-layer head whose forward returns sigmoid probabilities; layers keep torch's default (unseeded) init."""

    _act = _cabi.AC_ACT_SIGMOID

    def __init__(self, input_dim: int, num_classes: int, hidden_dims: List[int] = None):
        super().__init__()
        widths = [input_dim] + list(hidden_dims if hidden_dims is not None else [input_dim // 2])
        blocks: List[nn.Module] = []
        for fan_in, fan_out in zip(widths[:-1], widths[1:]):
            blocks += [nn.Linear(fan_in, fan_out), nn.ReLU(), nn.Dropout(0.1)]
        blocks.append(nn.Linear(widths[-1], num_classes))
        self.model = nn.Sequential(*blocks)
        self.num_classes = num_classes

    def forward(self, x):
        return self._forward_cuda(x, _cabi.AC_ACT_SIGMOID)

    def update_num_classes(self, new_num_classes: int):
        """Append output rows (Xavier weights, zero bias) and keep the trained ones bit for bit."""
        old = self.model[-1]
        extra = new_num_classes - self.num_classes
        if extra <= 0:
            return
        grown = nn.Linear(old.in_features, new_num_classes)      # default init first (same RNG consumption order
        fresh_w = torch.empty((extra, old.in_features))          #  as the reference), then Xavier for the new rows
        nn.init.xavier_uniform_(fresh_w)
        with torch.no_grad():
            grown.weight.copy_(torch.cat([old.weight.detach().cpu(), fresh_w], dim=0))
            grown.bias.copy_(torch.cat([old.bias.detach().cpu(), torch.zeros(extra)], dim=0))
        self.model[-1] = grown.to(old.weight.device)
        self.num_classes = new_num_classes


class MultiLabelAdaptiveClassifier(AdaptiveClassifier):
    """AdaptiveClassifier that may return several labels per text."""

    def __init__(self, model_name: str, device: Optional[str] = None, config: Optional[Dict[str, Any]] = None,
                 seed: int = 42, default_threshold: float = 0.5, min_predictions: int = 1,
                 max_predictions: Optional[int] = None, use_onnx="auto", trust_remote_code: bool = False):
        # use_onnx / trust_remote_code are accepted so that the generic load path can construct this class
        # (the reference's signature lacks them: SURVEY.md section 8(f) N1)
        super().__init__(model_name, device, config, seed, use_onnx=use_onnx, trust_remote_code=trust_remote_code)
        self.default_threshold = default_threshold
        self.min_predictions = min_predictions
        self.max_predictions = max_predictions
        self.label_thresholds: Dict[str, float] = {}
        self.adaptive_head = None

    # ------------------------------------------------------------------ head plumbing
    def _initialize_adaptive_head(self):
        dims = [self.embedding_dim, self.embedding_dim // 2]
        self.adaptive_head = MultiLabelAdaptiveHead(self.embedding_dim, len(self.label_to_id), hidden_dims=dims).to(self.device)

    def _sigmoid_probs(self, emb: torch.Tensor) -> torch.Tensor:
        self.adaptive_head.eval()
        return _cabi.head_forward(emb.contiguous(), self.adaptive_head._param_dict(), _cabi.AC_ACT_SIGMOID)

    def _head_probs(self, emb):
        # the inherited blend applies softmax to whatever the head module returns; for this head that is the sigmoid
        # vector (multilabel.py:41-44 feeding classifier.py:435)
        return None if self.adaptive_head is None else torch.softmax(self._sigmoid_probs(emb), dim=1)

    # ------------------------------------------------------------------ thresholds
    def _get_adaptive_threshold(self, num_labels: int) -> float:
        for limit, scale in _SIZE_SCALE:
            if num_labels <= limit:
                return self.default_threshold * scale
        return self.default_threshold * _SIZE_SCALE_MANY

    def _update_label_thresholds(self):
        sizes = {label: len(items) for label, items in self.memory.examples.items()}
        total = sum(sizes.values())
        if not total:
            return
        for label, n in sizes.items():
            share = n / total
            if share < _RARE[0]:
                factor = _RARE[1]
            elif share < _UNCOMMON[0]:
                factor = _UNCOMMON[1]
            elif share > _COMMON[0]:
                factor = _COMMON[1]
            else:
                factor = 1.0
            self.label_thresholds[label] = self.default_threshold * factor

    # ------------------------------------------------------------------ prediction
    def predict_multilabel(self, text: str, threshold: Optional[float] = None,
                           max_labels: Optional[int] = None) -> List[Tuple[str, float]]:
        if not text:
            raise ValueError("Empty input text")
        n_labels = len(self.label_to_id)
        if n_labels == 0:
            return []
        bar = self._get_adaptive_threshold(n_labels) if threshold is None else threshold
        cap = max_labels or self.max_predictions
        emb = self._embed_device([text])

        if self.adaptive_head is None:
            # no trained head yet: prototype neighbours above the bar (multilabel.py:189-200)
            k = min(n_labels, cap) if cap else n_labels
            return [(lab, s) for lab, s in self.memory.get_nearest_prototypes_batch(emb, k)[0] if s >= bar]

        probs = self._sigmoid_probs(emb)[0].cpu()
        known = min(probs.numel(), len(self.id_to_label))
        names = [self.id_to_label[i] for i in range(known)]
        bars = torch.tensor([self.label_thresholds.get(n, bar) for n in names], dtype=torch.float64)
        p = probs[:known]
        picked = torch.nonzero(p.double() >= bars).flatten().tolist()   # compared in double like `prob.item() >= threshold`
        picked.sort(key=lambda i: p[i].item(), reverse=True)           # stable: ties keep label-id order
        result = [(names[i], p[i].item()) for i in picked]
        if cap and len(result) > cap:
            result = result[:cap]
        short = self.min_predictions - len(result)
        if short > 0:
            # back-fill with the best-scoring labels even though they are below their bar (multilabel.py:202-227)
            have = {lab for lab, _ in result}
            vals, idx = torch.topk(probs, min(self.min_predictions, len(self.id_to_label)))
            spare = [(self.id_to_label[i], v) for v, i in zip(vals.tolist(), idx.tolist())
                     if i < len(self.id_to_label) and self.id_to_label[i] not in have]
            result = sorted(result + spare[:short], key=lambda t: t[1], reverse=True)
        return result

    def predict(self, text: str, k: int = 5) -> List[Tuple[str, float]]:
        found = self.predict_multilabel(text, max_labels=k)
        return found[:k] if found else super().predict(text, k)

    # ------------------------------------------------------------------ training
    def add_examples(self, texts: List[str], labels: List[List[str]]):
        if not texts or not labels:
            raise ValueError("Empty input lists")
        if len(texts) != len(labels):
            raise ValueError("Mismatched text and label lists")
        pairs = [(t, lab) for t, labs in zip(texts, labels) for lab in (labs or [])]   # one example per (text, label)
        if pairs:
            super().add_examples([t for t, _ in pairs], [lab for _, lab in pairs])
        self._update_label_thresholds()

    def _train_adaptive_head(self, epochs: int = 10):
        """BCE on multi-hot targets, one row per distinct text (multilabel.py:309-413); no LR scheduler."""
        rows: Dict[str, Tuple[torch.Tensor, set]] = {}
        for label, items in self.memory.examples.items():
            for ex in items:
                if ex.text in rows:
                    rows[ex.text][1].add(label)
                elif ex.embedding is not None:
                    rows[ex.text] = (ex.embedding, {label})
        if not rows:
            return
        n_cls = len(self.label_to_id)
        X = torch.stack([emb for emb, _ in rows.values()]).to(self.device, dtype=torch.float32)
        Y = torch.zeros((len(rows), n_cls), dtype=torch.float32)
        for r, (_, labs) in enumerate(rows.values()):
            Y[r, [self.label_to_id[l] for l in labs if l in self.label_to_id]] = 1.0
        X = F.normalize(X, p=2, dim=1)
        self._loss_kind = _cabi.AC_LOSS_BCE
        try:
            self._run_epochs(X, Y.to(self.device), epochs=epochs, batch_size=min(32, X.shape[0]), use_scheduler=False)
        finally:
            self._loss_kind = _cabi.AC_LOSS_CE
        self.train_steps += 1

    def _train_new_classes(self, old_head, new_classes):
        # The reference inherits the single-label routine here and thereby applies CrossEntropyLoss to sigmoid outputs
        # (SURVEY.md Appendix A.10).  The CUDA head kernels have no CE-on-probabilities step; the multi-label path
        # retrains with its BCE loop instead (documented deviation, DESIGN.md section 8).
        self._train_adaptive_head()

    def get_label_statistics(self) -> Dict[str, Any]:
        stats = super().get_example_statistics()
        stats.update(label_thresholds=dict(self.label_thresholds),
                     adaptive_threshold=self._get_adaptive_threshold(len(self.label_to_id)),
                     default_threshold=self.default_threshold, min_predictions=self.min_predictions,
                     max_predictions=self.max_predictions)
        return stats
