"""Host-side mirror of /root/reference/src/adaptive_classifier/classifier.py (AdaptiveClassifier).

Drop-in for the predict()/predict_batch()/add_examples() hot path: same method names, arguments, return
types, label-id rules, blending formulas and error behaviour (citations inline).  All arithmetic runs on
the H100 through the C ABI: encoder (csrc/encoder.cu), prototype kNN (csrc/knn_*.cu), adaptive head +
AdamW/EWC (csrc/head.cu).  HuggingFace is used for checkpoint/tokenizer IO only.

Strategic mode (classifier.py:1573-1823, strategic.py) is supported: the best-response search runs in csrc/strategic.cu and the
strategic training step in the training kernel (AC_LOSS_CE_STRATEGIC); the label blends stay host dicts.
Out of scope (SURVEY.md section 2): ONNX export/ORT inference (use_onnx is accepted and ignored), Hub push.  Persistence keeps
the reference's on-disk format (persistence.py).
"""
from __future__ import annotations

import copy
import logging
import threading
from typing import Any, Dict, List, Optional, Set, Tuple, Union

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _cabi
from .ewc import EWC
from .memory import PrototypeMemory
from .models import AdaptiveHead, Example, ModelConfig
from .strategic import CostFunctionFactory, StrategicEvaluator, StrategicOptimizer

logger = logging.getLogger(__name__)


def dataloader_epoch_permutation(gen: torch.Generator, n: int) -> torch.Tensor:
    """The index order one epoch of the reference's `DataLoader(dataset, shuffle=True, generator=gen)` yields
    (classifier.py:315-320, :1453-1459), reproduced draw for draw from the same generator:
      1. `_BaseDataLoaderIter.__init__` draws an int64 `_base_seed` when the epoch's iterator is created,
      2. `RandomSampler.__iter__` draws `randperm(n)` -- the epoch's order,
      3. on exhaustion it draws a second `randperm(n)` whose `[:num_samples % n]` (empty) slice is discarded.
    Pinned against a real DataLoader in tests/test_host_logic_cpu.py and against the reference run's recorded batches
    (tests/golden/golden_training.npz)."""
    torch.empty((), dtype=torch.int64).random_(generator=gen)
    perm = torch.randperm(n, generator=gen)
    torch.randperm(n, generator=gen)
    return perm


class AdaptiveClassifier:
    """A flexible classifier that can adapt to new classes and examples (classifier.py:27)."""

    _loss_kind = _cabi.AC_LOSS_CE
    _dropout_p = 0.1              # nn.Dropout(0.1) of the reference head (models.py:59); parity tests replay with 0

    def __init__(self, model_name: str, device: Optional[str] = None, config: Optional[Dict[str, Any]] = None,
                 seed: int = 42, use_onnx: Optional[Union[bool, str]] = "auto", trust_remote_code: bool = False):
        torch.manual_seed(seed)                                   # classifier.py:52
        self.config = ModelConfig(config)
        if device is not None and not str(device).startswith("cuda"):
            raise _cabi.AdaptiveB200Error(
                f"device={device!r}: adaptive_classifier_b200 runs on H100 GPUs only (no CPU fallback)")
        if not torch.cuda.is_available():
            raise _cabi.AdaptiveB200Error("no CUDA device: adaptive_classifier_b200 has no CPU fallback")
        _cabi.check(_cabi.load_library().ac_device_check(), "ac_device_check")
        self.device = device or "cuda"
        self.use_onnx = False                                      # north_star: no ONNX dispatch
        self.model_name = model_name

        from transformers import AutoModel, AutoTokenizer
        hf = AutoModel.from_pretrained(model_name, trust_remote_code=trust_remote_code)
        hf.eval()
        self.model = hf                                            # kept on the host for .config / save()
        self.tokenizer = AutoTokenizer.from_pretrained(model_name, trust_remote_code=trust_remote_code)
        self._max_tokens = int(self.config.config.get("b200_max_tokens", 65536))
        with torch.cuda.device(torch.device(self.device)):
            self.encoder = _cabi.Encoder.from_hf(hf, max_tokens=self._max_tokens, device=self.device)
            # WordPiece tokenizers of the BERT shape, byte-level BPE tokenizers (RoBERTa, ModernBERT, EuroBERT) and Unigram
            # tokenizers of the XLM-RoBERTa shape run on the device with identical ids; every other one stays on the host, and so
            # does one whose tables or handle cannot be built
            whys = []
            self.device_tokenizer = None
            for kind in (_cabi.WordPieceTokenizer, _cabi.BPETokenizer, _cabi.UnigramTokenizer):
                try:
                    self.device_tokenizer, why = kind.from_hf(self.tokenizer, device=self.device)
                except (_cabi.AdaptiveB200Error, ValueError) as e:
                    self.device_tokenizer, why = None, f"building the device tokenizer failed: {e}"
                if self.device_tokenizer is not None:
                    break
                whys.append(f"{kind.__name__}: {why}")
        if self.device_tokenizer is None:
            logger.debug(f"tokenization stays on the host: {'; '.join(whys)}")

        self.embedding_dim = getattr(self.model.config, "hidden_size", None) or self.model.config.dim
        self.memory = PrototypeMemory(self.embedding_dim, config=self.config)
        self.adaptive_head = None
        self.label_to_id = {}
        self.id_to_label = {}
        self.train_steps = 0
        self.training_history = {}
        self.strategic_cost_function = None
        self.strategic_optimizer = None
        self.strategic_evaluator = None
        if self.config.enable_strategic_mode:
            self._initialize_strategic_components()

    def _initialize_strategic_components(self):
        """classifier.py:1573-1592: an empty / missing coefficient set logs a warning and leaves strategic mode off; a failing
        factory call (dict coefficients without feature names, an unknown cost type) is logged and disables it."""
        try:
            if self.config.cost_coefficients:
                self.strategic_cost_function = CostFunctionFactory.create_cost_function(
                    cost_type=self.config.cost_function_type, cost_coefficients=self.config.cost_coefficients)
                self.strategic_optimizer = StrategicOptimizer(self.strategic_cost_function)
                self.strategic_evaluator = StrategicEvaluator(self.strategic_cost_function)
                logger.info(f"Initialized strategic mode with {self.config.cost_function_type} cost function")
            else:
                logger.warning("Strategic mode enabled but no cost coefficients provided")
        except Exception as e:
            logger.error(f"Failed to initialize strategic components: {e}")
            self.config.enable_strategic_mode = False

    @property
    def strategic_mode(self) -> bool:
        """classifier.py:1594-1600."""
        return self.config.enable_strategic_mode and self.strategic_cost_function is not None

    @property
    def _device_lock(self):
        """The encoder handle owns ONE activation workspace and ctypes releases the GIL during every C call: two threads
        calling predict() / add_examples() on one classifier would interleave kernel launches on the same buffers.  All device
        work of a classifier is therefore serialised by this re-entrant lock (the reference's PyTorch forward is safe under the
        same usage; PrototypeMemory has its own lock)."""
        lk = self.__dict__.get("_dev_lock")
        if lk is None:
            lk = self.__dict__.setdefault("_dev_lock", threading.RLock())
        return lk

    # ------------------------------------------------------------------------------------------ E
    def _tokenize(self, texts: List[str]):
        inputs = self.tokenizer(texts, max_length=self.config.max_length, truncation=True, padding=True,
                                return_tensors="pt")          # classifier.py:1259-1265
        ids = inputs["input_ids"].to(torch.int32)
        mask = inputs["attention_mask"].to(torch.int32)
        tt = inputs.get("token_type_ids")
        return ids, mask, (tt.to(torch.int32) if tt is not None else None)

    def _embed_ids_device(self, ids: torch.Tensor, mask: Optional[torch.Tensor], tt: Optional[torch.Tensor]) -> torch.Tensor:
        """ids/mask [B,S] int32 (host or device) -> unit CLS rows [B,H] on the device; chunks the batch so that
        B*S stays inside the encoder workspace."""
        B, S = ids.shape
        per = max(1, self._max_tokens // S)
        outs = []
        with self._device_lock, torch.cuda.device(torch.device(self.device)):
            for b0 in range(0, B, per):
                sl = slice(b0, min(B, b0 + per))
                i = ids[sl].to(self.device, non_blocking=True).contiguous()
                m = mask[sl].to(self.device, non_blocking=True).contiguous() if mask is not None else None
                t = tt[sl].to(self.device, non_blocking=True).contiguous() if tt is not None else None
                outs.append(self.encoder.forward_cls(i, m, t))
            return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    def _embed_device(self, texts: List[str]) -> torch.Tensor:
        tok = getattr(self, "device_tokenizer", None)
        if tok is not None and texts and self.config.max_length >= 2:
            with self._device_lock, torch.cuda.device(torch.device(self.device)):
                out = tok(texts, self.config.max_length)
            if out is not None:
                return self._embed_ids_device(*out)
        ids, mask, tt = self._tokenize(texts)
        return self._embed_ids_device(ids, mask, tt)

    def _get_embeddings(self, texts: List[str]) -> List[torch.Tensor]:
        """classifier.py:1249-1282: list of CPU tensors, L2-normalised CLS rows."""
        emb = self._embed_device(texts).cpu()
        return [e for e in emb]

    # ------------------------------------------------------------------------------------------ add_examples
    def add_examples(self, texts: List[str], labels: List[str]):
        """classifier.py:132-200."""
        if not texts or not labels:
            raise ValueError("Empty input lists")
        if len(texts) != len(labels):
            raise ValueError("Mismatched text and label lists")
        has_existing_classes = len(self.label_to_id) > 0
        new_classes = set(labels) - set(self.label_to_id.keys())
        is_adding_new_classes = len(new_classes) > 0
        for label in sorted(new_classes):                      # sorted ids, appended (classifier.py:146-150)
            idx = len(self.label_to_id)
            self.label_to_id[label] = idx
            self.id_to_label[idx] = label

        emb_dev = self._embed_device(texts)                      # unit CLS rows stay on the device for the memory update
        embeddings = [e for e in emb_dev.cpu()]                  # the reference's contract: CPU tensors on the Example objects
        examples = [Example(t, l, e) for t, e, l in zip(texts, embeddings, labels)]
        self.memory.add_examples_batch(examples, labels, device_rows=emb_dev)
        for label in labels:
            self.training_history[label] = self.training_history.get(label, 0) + 1

        is_incremental_learning = is_adding_new_classes and has_existing_classes
        if is_incremental_learning:
            old_head = copy.deepcopy(self.adaptive_head) if self.adaptive_head is not None else None
            num_classes = len(self.label_to_id)
            self.adaptive_head.update_num_classes(num_classes)
            self.adaptive_head = self.adaptive_head.to(self.device)
            self._train_new_classes(old_head, new_classes)
        else:
            if self.adaptive_head is None:
                self._initialize_adaptive_head()
            elif is_adding_new_classes:
                self.adaptive_head.update_num_classes(len(self.label_to_id))
                self.adaptive_head = self.adaptive_head.to(self.device)
            self._train_adaptive_head()
            if self.strategic_mode and self.train_steps % self.config.strategic_training_frequency == 0:   # classifier.py:194-197
                self._perform_strategic_training()
        self.memory._rebuild_index()                           # classifier.py:200

    def _initialize_adaptive_head(self):
        """classifier.py:1238-1247."""
        num_classes = len(self.label_to_id)
        hidden_dims = [self.embedding_dim, self.embedding_dim // 2]
        self.adaptive_head = AdaptiveHead(self.embedding_dim, num_classes, hidden_dims=hidden_dims).to(self.device)

    # ------------------------------------------------------------------------------------------ training
    def _head_blocks(self):
        p = self.adaptive_head._param_dict()
        m = {k: torch.zeros_like(v) for k, v in p.items()}
        v = {k: torch.zeros_like(t) for k, t in p.items()}
        return p, m, v

    def _run_epochs(self, X: torch.Tensor, Y: torch.Tensor, *, epochs: int, batch_size: int, use_scheduler: bool,
                    ewc=None, ewc_zero_term: bool = False):
        """Shared optimizer loop of classifier.py:322-365 / :1484-1520: shuffled batches from
        torch.Generator().manual_seed(42) consumed exactly like the reference's DataLoader (dataloader_epoch_permutation), fresh AdamW,
        optional ReduceLROnPlateau(0.5, patience 2), early stopping patience 3."""
        n = X.shape[0]
        with self._device_lock:
            return self._run_epochs_locked(X, Y, n, epochs, batch_size, use_scheduler, ewc)

    def _run_epochs_locked(self, X, Y, n, epochs, batch_size, use_scheduler, ewc):
        p, m, v = self._head_blocks()
        gen = torch.Generator().manual_seed(42)
        lr = 0.001
        best_loss, patience_counter, patience = float("inf"), 0, 3
        sched_best, sched_bad = float("inf"), 0
        step = 0
        n_batches = (n + batch_size - 1) // batch_size
        seed = int(torch.initial_seed() & 0x7FFFFFFF)
        trace = {"loss": [], "ewc": [], "gnorm": [], "steps_per_epoch": [], "lr": []}
        self.adaptive_head.train()
        for epoch in range(epochs):
            perm = dataloader_epoch_permutation(gen, n)        # the index lists the reference's DataLoader yields
            step_stats = torch.zeros((n_batches, 3), dtype=torch.float32, device=X.device)
            total, nb = _cabi.head_train_epoch(X, Y, perm, p, m, v, first_step=step + 1, batch=batch_size,
                                               loss_kind=self._loss_kind, lr=lr, dropout_p=self._dropout_p, seed=seed, ewc=ewc,
                                               step_stats=step_stats)
            step += nb
            st = step_stats.cpu()                               # the epoch's one host sync (the reference syncs per step: loss.item())
            trace["loss"] += st[:, 0].tolist()
            trace["ewc"] += st[:, 1].tolist()
            trace["gnorm"] += st[:, 2].tolist()
            trace["steps_per_epoch"].append(nb)
            trace["lr"].append(lr)
            # `total_loss += loss.item()` then `/ len(loader)` (classifier.py:353-355, :1507-1509): a Python float sum in step order
            avg_loss = sum(float(a) + float(b) for a, b in zip(st[:, 0].tolist(), st[:, 1].tolist())) / n_batches
            if use_scheduler:                                   # ReduceLROnPlateau(mode=min, factor .5, patience 2, rel 1e-4)
                if avg_loss < sched_best * (1 - 1e-4):
                    sched_best, sched_bad = avg_loss, 0
                else:
                    sched_bad += 1
                if sched_bad > 2:
                    lr, sched_bad = lr * 0.5, 0
            if avg_loss < best_loss:
                best_loss, patience_counter = avg_loss, 0
            else:
                patience_counter += 1
                if patience_counter >= patience:
                    logger.debug(f"Early stopping at epoch {epoch + 1}")
                    break
        self.last_training_trace = trace
        self.adaptive_head.eval()

    def _training_matrix(self):
        """classifier.py:1438-1450: all stored examples sorted by label then text; embeddings re-normalised.  The rows are
        gathered from the memory's device-resident class stores (no re-upload of the whole memory per call)."""
        parts, all_labels = [], []
        for label in sorted(self.memory.examples.keys()):
            exs = self.memory.examples[label]
            if not exs:
                continue
            order = sorted(range(len(exs)), key=lambda i: exs[i].text)            # Python's stable sort, as the reference
            rows = self.memory.class_rows_device(label)
            parts.append(rows.index_select(0, torch.tensor(order, dtype=torch.int64, device=rows.device)))
            all_labels += [self.label_to_id[exs[i].label] for i in order]
        X = (parts[0] if len(parts) == 1 else torch.cat(parts, 0)).to(self.device, dtype=torch.float32)
        X = F.normalize(X, p=2, dim=1)
        Y = torch.tensor(all_labels, dtype=torch.long, device=self.device)
        return X, Y

    def _train_adaptive_head(self, epochs: int = 10):
        """classifier.py:1428-1522."""
        if not self.memory.examples:
            return
        X, Y = self._training_matrix()
        self._run_epochs(X, Y, epochs=epochs, batch_size=min(32, X.shape[0]), use_scheduler=True)
        self.train_steps += 1

    def _train_new_classes(self, old_head: Optional[nn.Module], new_classes: Set[str]):
        """classifier.py:202-367: class-balanced resampling (global unseeded np.random), EWC built on the
        deep-copied old head.  In the reference the EWC term is identically 0 and carries no gradient to the
        live head (SURVEY.md section 0.5); that behaviour is reproduced by default.  config['b200_live_ewc']=True
        binds Fisher/theta* of the old head to the live head's first C_old output rows instead."""
        if not self.memory.examples:
            return
        all_embeddings, all_labels = [], []
        examples_per_class = {label: len(ex) for label, ex in self.memory.examples.items()}
        min_examples = min(examples_per_class.values())
        num_classes = len(examples_per_class)
        target = max(5, min(10, min_examples * 2))
        if num_classes > 20:                                   # classifier.py:222-243
            for label, examples in self.memory.examples.items():
                num_samples = min(len(examples), target * 2 if label in new_classes else target)
                indices = np.random.choice(len(examples), size=num_samples, replace=num_samples > len(examples))
                for idx in indices:
                    all_embeddings.append(examples[idx].embedding)
                    all_labels.append(self.label_to_id[label])
        else:                                                  # classifier.py:244-271
            for label, examples in self.memory.examples.items():
                weight = 2.0 if label in new_classes else min_examples / examples_per_class[label]
                num_samples = max(min_examples, int(len(examples) * weight))
                indices = np.random.choice(len(examples), size=num_samples, replace=num_samples > len(examples))
                for idx in indices:
                    all_embeddings.append(examples[idx].embedding)
                    all_labels.append(self.label_to_id[label])
        X = torch.stack(all_embeddings).to(self.device, dtype=torch.float32)
        Y = torch.tensor(all_labels, dtype=torch.long, device=self.device)

        ewc_arg = None
        if old_head is not None:                               # classifier.py:279-303
            old_embeddings, old_labels = [], []
            old_label_to_id = {label: idx for idx, label in enumerate(self.id_to_label.values())
                               if label not in new_classes}
            for label, examples in self.memory.examples.items():
                if label not in new_classes:
                    for example in examples[:5]:
                        old_embeddings.append(example.embedding)
                        old_labels.append(old_label_to_id[label])
            if old_embeddings:
                old_dataset = torch.utils.data.TensorDataset(torch.stack(old_embeddings),
                                                             torch.tensor(old_labels, dtype=torch.long))
                ewc = EWC(old_head, old_dataset, device=self.device, ewc_lambda=5.0)
                if self.config.config.get("b200_live_ewc", False):
                    ewc_arg = (ewc._as_block(ewc.fisher_info), ewc._as_block(ewc.old_params), 5.0,
                               old_head.model[-1].weight.shape[0])
                # default: the reference's term evaluates to exactly 0 with no gradient -> nothing to add
        self._run_epochs(X, Y, epochs=15, batch_size=32, use_scheduler=False, ewc=ewc_arg)
        self.train_steps += 1

    # ------------------------------------------------------------------------------------------ predict
    def predict(self, text: str, k: int = 5) -> List[Tuple[str, float]]:
        """classifier.py:392-413."""
        if not text:
            raise ValueError("Empty input text")
        if not self.strategic_mode:
            return self._predict_regular(text, k)
        return self._predict_dual(text, k)

    def _head_probs(self, emb: torch.Tensor) -> Optional[torch.Tensor]:
        if self.adaptive_head is None:
            return None
        with self._device_lock:
            self.adaptive_head.eval()
            return _cabi.head_forward(emb.contiguous(), self.adaptive_head._param_dict(), _cabi.AC_ACT_SOFTMAX)

    def _predict_regular(self, text: str, k: int = 5, emb: Optional[torch.Tensor] = None) -> List[Tuple[str, float]]:
        """classifier.py:415-480: prototype scores over ALL classes, head softmax over all classes,
        per-label weights from training_history (<10 -> 0.3/0.7 else 0.7/0.3), renormalise, top k.
        emb: the text's unit CLS row when the caller has it already."""
        if emb is None:
            emb = self._embed_device([text])
        max_classes = len(self.id_to_label) if self.id_to_label else k
        proto_preds = self.memory.get_nearest_prototypes_batch(emb, max_classes)[0]
        head_preds = []
        probs = self._head_probs(emb)
        if probs is not None:
            values, indices = _cabi.topk_desc(probs[:1], min(len(self.id_to_label), probs.shape[1]))   # classifier.py:438
            values, indices = values[0].cpu().tolist(), indices[0].cpu().tolist()
            head_preds = [(self.id_to_label[i], v) for v, i in zip(values, indices)]
        combined_scores = {}
        for label, score in proto_preds:
            weight = 0.3 if self.training_history.get(label, 0) < 10 else 0.7
            combined_scores[label] = score * weight
        for label, score in head_preds:
            weight = 0.7 if self.training_history.get(label, 0) < 10 else 0.3
            combined_scores[label] = combined_scores.get(label, 0) + score * weight
        predictions = sorted(combined_scores.items(), key=lambda x: x[1], reverse=True)
        total = sum(score for _, score in predictions)
        if total > 0:
            predictions = [(label, score / total) for label, score in predictions]
        return predictions[:k]

    # ------------------------------------------------------------------------------------------ strategic mode
    def _perform_strategic_training(self):
        """classifier.py:369-390: every stored example in memory order (label insertion order, then list order), embeddings as
        stored (not re-normalised)."""
        if not self.strategic_mode or not self.memory.examples:
            return
        all_embeddings, all_labels = [], []
        for label in self.memory.examples:
            for example in self.memory.examples[label]:
                all_embeddings.append(example.embedding)
                all_labels.append(self.label_to_id[label])
        if all_embeddings:
            X = torch.stack(all_embeddings).to(self.device, dtype=torch.float32)
            Y = torch.tensor(all_labels, dtype=torch.long, device=self.device)
            self._strategic_training_step(X, Y)

    def _strategic_training_step(self, all_embeddings: torch.Tensor, all_labels: torch.Tensor):
        """classifier.py:1602-1647: 5 epochs of DataLoader(batch min(16, N), shuffle, manual_seed(42)) batches, fresh
        AdamW(lr = learning_rate / 2, wd 0.01), clip 1.0, loss = strategic_loss (strategic.py:200-242) with the best responses
        searched in train mode.  All steps run in one library call (ac_head_train_strategic) with no host synchronisation;
        the per-step (loss, 0, grad norm) stay on the device in `last_strategic_trace`."""
        if not self.strategic_mode or self.adaptive_head is None:
            return
        cost = self.strategic_cost_function
        n = all_embeddings.shape[0]
        gen = torch.Generator().manual_seed(42)
        perms = torch.cat([dataloader_epoch_permutation(gen, n) for _ in range(5)])
        with self._device_lock:
            X = all_embeddings.to(self.device, dtype=torch.float32).contiguous()
            c1, c2 = cost.device_coefficients(X.shape[1], X.device)
            p, m, v = self._head_blocks()
            self.adaptive_head.train()
            self.last_strategic_trace = _cabi.head_train_strategic(
                X, all_labels, perms, p, m, v, cost_kind=cost.cost_kind, c1=c1, c2=c2, lr=self.config.learning_rate * 0.5,
                strategic_lambda=self.config.strategic_lambda, dropout_p=self._dropout_p, seed=int(torch.initial_seed() & 0x7FFFFFFF))
            self.adaptive_head.eval()

    def _best_response(self, emb: torch.Tensor) -> torch.Tensor:
        """Best responses of the rows of emb [B, D] (device) against the eval-mode head; with no head every candidate has
        the same score (the reference's uniform 1/C) and the cost-free x itself wins."""
        if self.adaptive_head is None:
            return emb
        with self._device_lock:
            self.adaptive_head.eval()
            _, _, br = self.strategic_cost_function.compute_best_response(emb.contiguous(), self.adaptive_head._param_dict())
            return br

    def _coefficients_usable(self, what: str) -> bool:
        """The reference's torch.dot raises for coefficients of the wrong length or a non-floating dtype and its predict
        methods fall back to regular prediction; here that is decided before anything is launched."""
        try:
            self.strategic_cost_function.device_coefficients(self.embedding_dim, self.device)
            return True
        except ValueError as e:
            logger.warning(f"{what} prediction failed: {e}. Falling back to regular prediction.")
            return False

    def _predict_dual(self, text: str, k: int = 5) -> List[Tuple[str, float]]:
        """classifier.py:482-522: 0.6 regular + 0.4 strategic over the union of labels.  The text is embedded once."""
        emb = self._embed_device([text])
        regular_preds = self._predict_regular(text, k, emb)
        strategic_preds = self.predict_strategic(text, k, emb)
        blended_scores = {}
        regular_weight = self.config.strategic_blend_regular_weight
        strategic_weight = self.config.strategic_blend_strategic_weight
        for label, score in regular_preds:
            blended_scores[label] = score * regular_weight
        for label, score in strategic_preds:
            blended_scores[label] = blended_scores.get(label, 0) + score * strategic_weight
        blended_predictions = sorted(blended_scores.items(), key=lambda x: x[1], reverse=True)
        total = sum(score for _, score in blended_predictions)
        if total > 0:
            blended_predictions = [(label, score / total) for label, score in blended_predictions]
        return blended_predictions[:k]

    def predict_strategic(self, text: str, k: int = 5, emb: Optional[torch.Tensor] = None) -> List[Tuple[str, float]]:
        """classifier.py:1649-1694: predict on the best response of the text's embedding."""
        if not self.strategic_mode:
            return self._predict_regular(text, k, emb)
        if emb is None:
            emb = self._embed_device([text])
        if not self._coefficients_usable("Strategic"):
            return self._predict_regular(text, k, emb)
        return self._predict_from_embedding(self._best_response(emb), k, strategic=True)

    def predict_robust(self, text: str, k: int = 5) -> List[Tuple[str, float]]:
        """classifier.py:1696-1721: prototype-heavy blend (0.8 / 0.2) on the unmodified embedding."""
        if not self.strategic_mode:
            return self._predict_regular(text, k)
        emb = self._embed_device([text])
        if not self._coefficients_usable("Robust"):
            return self._predict_regular(text, k, emb)
        return self._predict_from_embedding(emb, k, robust=True)

    def _predict_from_embedding(self, embedding: torch.Tensor, k: int = 5, robust: bool = False,
                                strategic: bool = False) -> List[Tuple[str, float]]:
        """classifier.py:1723-1795: k nearest prototypes (softmax over the k returned), head softmax top min(k, C), fixed
        weights of the mode, renormalise, top k.  embedding: [1, D] on the device."""
        proto_preds = self.memory.get_nearest_prototypes(embedding, k=k)
        head_preds = []
        probs = self._head_probs(embedding)
        if probs is not None:
            values, indices = _cabi.topk_desc(probs[:1], min(k, len(self.id_to_label)))
            values, indices = values[0].cpu().tolist(), indices[0].cpu().tolist()
            head_preds = [(self.id_to_label[i], v) for v, i in zip(values, indices)]
        combined_scores = {}
        if self.strategic_mode and robust:
            proto_weight = self.config.strategic_robust_proto_weight
            head_weight = self.config.strategic_robust_head_weight
        elif self.strategic_mode and strategic:
            proto_weight = self.config.strategic_prediction_proto_weight
            head_weight = self.config.strategic_prediction_head_weight
        else:
            proto_weight = self.config.prototype_weight
            head_weight = self.config.neural_weight
        for label, score in proto_preds:
            combined_scores[label] = score * proto_weight
        for label, score in head_preds:
            combined_scores[label] = combined_scores.get(label, 0) + score * head_weight
        predictions = sorted(combined_scores.items(), key=lambda x: x[1], reverse=True)
        total = sum(score for _, score in predictions)
        if total > 0:
            predictions = [(label, score / total) for label, score in predictions]
        return predictions[:k]

    def evaluate_strategic_robustness(self, test_texts: List[str], test_labels: List[str],
                                      gaming_levels: List[float] = [0.0, 0.5, 1.0]) -> Dict[str, float]:
        """classifier.py:1797-1823."""
        if not self.strategic_mode:
            raise ValueError("Strategic mode not enabled")
        test_embeddings = self._embed_device(test_texts)
        test_label_indices = torch.tensor([self.label_to_id[label] for label in test_labels])
        with self._device_lock:
            self.adaptive_head.eval()
            return self.strategic_evaluator.evaluate_robustness(self.adaptive_head, test_embeddings, test_label_indices,
                                                                gaming_levels)

    def predict_batch(self, texts: List[str], k: int = 5, batch_size: int = 32) -> List[List[Tuple[str, float]]]:
        """classifier.py:1308-1388: top-k prototype search (softmax over the k returned), head top-k, fixed
        0.7/0.3 blend.  The per-embedding Python loop of the reference is replaced by batched device calls;
        only the final dict blend stays on the host."""
        if not texts:
            raise ValueError("Empty input batch")
        all_predictions = []
        for i in range(0, len(texts), batch_size):
            emb = self._embed_device(texts[i : i + batch_size])
            all_predictions.extend(self._predict_from_device_embeddings(emb, k))
        return all_predictions

    def _predict_from_device_embeddings(self, emb: torch.Tensor, k: int) -> List[List[Tuple[str, float]]]:
        proto = self.memory.get_nearest_prototypes_batch(emb, k)
        head_vals = head_idx = None
        probs = self._head_probs(emb)
        if probs is not None:
            kk = min(k, len(self.id_to_label))
            hv, hi = _cabi.topk_desc(probs, kk)                   # classifier.py:1347-1350
            head_vals, head_idx = hv.cpu().tolist(), hi.cpu().tolist()
        out = []
        for b in range(emb.shape[0]):
            combined_scores = {}
            for label, score in proto[b]:
                combined_scores[label] = score * 0.7
            if head_vals is not None:
                for v, j in zip(head_vals[b], head_idx[b]):
                    label = self.id_to_label[j]
                    combined_scores[label] = combined_scores.get(label, 0) + v * 0.3
            predictions = sorted(combined_scores.items(), key=lambda x: x[1], reverse=True)
            total = sum(score for _, score in predictions)
            if total > 0:
                predictions = [(label, score / total) for label, score in predictions]
            out.append(predictions[:k])
        return out

    def predict_batch_ids(self, ids: torch.Tensor, mask: Optional[torch.Tensor] = None, k: int = 5):
        """Pre-tokenised entry (SURVEY.md section 8(f) N3): ids [B,S] int32 on host or device."""
        return self._predict_from_device_embeddings(self._embed_ids_device(ids, mask, None), k)

    # ------------------------------------------------------------------------------------------ misc API
    def to(self, device: str) -> "AdaptiveClassifier":
        if not str(device).startswith("cuda"):
            raise _cabi.AdaptiveB200Error("adaptive_classifier_b200 runs on H100 GPUs only")
        if torch.device(device) != torch.device(self.device) and torch.device(device).index not in (None, torch.device(self.device).index):
            # the encoder handle and the prototype index live on the device they were built on
            raise _cabi.AdaptiveB200Error(f"moving a built classifier from {self.device} to {device} is not supported: construct it "
                                          f"with device={device!r}")
        self.device = device
        if self.adaptive_head is not None:
            self.adaptive_head = self.adaptive_head.to(device)
        return self

    def get_memory_stats(self) -> Dict[str, Any]:
        return self.memory.get_stats()

    def get_example_statistics(self) -> Dict[str, Any]:
        """classifier.py:1284-1306."""
        stats = {
            "total_examples": sum(len(exs) for exs in self.memory.examples.values()),
            "examples_per_class": {label: len(exs) for label, exs in self.memory.examples.items()},
            "num_classes": len(self.label_to_id),
            "train_steps": self.train_steps,
            "memory_usage": {
                "prototypes": sum(p.nelement() * p.element_size() for p in self.memory.prototypes.values()),
                "examples": sum(sum(ex.embedding.nelement() * ex.embedding.element_size() for ex in exs)
                                for exs in self.memory.examples.values()),
            },
        }
        if self.adaptive_head is not None:
            stats["model_params"] = sum(p.nelement() for p in self.adaptive_head.parameters())
        return stats

    def clear_memory(self, labels: Optional[List[str]] = None):
        """classifier.py:1390-1401."""
        if labels is None:
            self.memory.clear()
        else:
            for label in labels:
                self.memory.examples.pop(label, None)
                self.memory.prototypes.pop(label, None)
            self.memory._rebuild_index()

    def merge_classifiers(self, other: "AdaptiveClassifier") -> "AdaptiveClassifier":
        """classifier.py:1403-1426."""
        if self.embedding_dim != other.embedding_dim:
            raise ValueError("Classifiers have different embedding dimensions")
        next_idx = max(self.id_to_label.keys()) + 1
        for label in other.label_to_id:
            if label not in self.label_to_id:
                self.label_to_id[label] = next_idx
                self.id_to_label[next_idx] = label
                next_idx += 1
        for label, examples in other.memory.examples.items():
            for example in examples:
                self.memory.add_example(example, label)
        if self.adaptive_head is not None:
            self._initialize_adaptive_head()
            self._train_adaptive_head()
        return self

    def _update_adaptive_head(self):
        """classifier.py:1524-1531."""
        num_classes = len(self.label_to_id)
        if self.adaptive_head is None:
            self._initialize_adaptive_head()
        elif num_classes > self.adaptive_head.model[-1].out_features:
            self.adaptive_head.update_num_classes(num_classes)
            self.adaptive_head = self.adaptive_head.to(self.device)

    # persistence (same on-disk format as classifier.py:524-628 / :630-915), see persistence.py
    def save(self, save_dir: str, include_onnx: bool = True, quantize_onnx: bool = True):
        from .persistence import save_classifier
        return save_classifier(self, save_dir)

    _save_pretrained = save

    @classmethod
    def load(cls, save_dir: str, device: Optional[str] = None, use_onnx="auto", prefer_quantized: bool = True,
             trust_remote_code: bool = False) -> "AdaptiveClassifier":
        from .persistence import load_classifier
        return load_classifier(cls, save_dir, device=device, trust_remote_code=trust_remote_code)

    _from_pretrained = load
