"""Host-side mirror of /root/reference/src/adaptive_classifier/memory.py (PrototypeMemory).

Same bookkeeping, attribute names and error behaviour; `self.index` is a FlatL2Index living in GPU HBM
(csrc/knn_exact.cu, csrc/knn_tc.cu) instead of faiss.IndexFlatL2.  Label aggregation and the
`exp(-d)` -> softmax post-processing follow memory.py:117-134 exactly (on the device).
"""
from __future__ import annotations

import functools
import logging
import threading
from collections import defaultdict
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _cabi
from .models import Example, ModelConfig

logger = logging.getLogger(__name__)


def _device() -> torch.device:
    if not torch.cuda.is_available():
        raise _cabi.AdaptiveB200Error("adaptive_classifier_b200 needs an H100 GPU; there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


class FlatL2Index:
    """Device-resident flat squared-L2 index with the faiss.IndexFlatL2 protocol the reference uses
    (memory.py:34,106,113,114,158,159,164,172,182,190,242): add / search / remove_ids / ntotal."""

    def __init__(self, d: int, capacity: int = 64):
        self.d = int(d)
        self._n = 0
        self._buf: Optional[torch.Tensor] = None
        self._cap = capacity

    @property
    def ntotal(self) -> int:
        return self._n

    def _rows(self) -> torch.Tensor:
        return self._buf[: self._n]

    def _ensure(self, extra: int):
        need = self._n + extra
        if self._buf is None or need > self._buf.shape[0]:
            cap = max(self._cap, 2 * need)
            nb = torch.empty((cap, self.d), dtype=torch.float32, device=_device())
            if self._buf is not None and self._n:
                nb[: self._n] = self._buf[: self._n]
            self._buf = nb

    def add(self, x):
        x = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x, dtype=torch.float32).reshape(-1, self.d)
        self._ensure(x.shape[0])
        self._buf[self._n : self._n + x.shape[0]] = x.to(self._buf.device)
        self._n += x.shape[0]

    def remove_ids(self, ids) -> int:
        """faiss semantics: rows after a removed one shift down."""
        ids = torch.as_tensor(ids).reshape(-1).to(torch.int64)
        ids = ids[(ids >= 0) & (ids < self._n)].unique()
        if ids.numel() == 0:
            return 0
        keep = torch.ones(self._n, dtype=torch.bool)
        keep[ids] = False
        kept = self._rows()[keep.to(self._buf.device)]
        self._n = kept.shape[0]
        self._buf[: self._n] = kept
        return int(ids.numel())

    def search_device(self, q: torch.Tensor, k: int):
        """q [nq, d] CUDA fp32 -> (D [nq,k] fp32 ascending, I [nq,k] int64; (+inf, -1) padded)."""
        return _cabi.knn_l2_topk(q, self._rows() if self._n else torch.empty((0, self.d), device=q.device), k)

    def search(self, x, k: int):
        """numpy in / numpy out like faiss (host convenience; device callers use search_device)."""
        q = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x, dtype=torch.float32).reshape(-1, self.d)
        if self._n == 0:
            nq = q.shape[0]
            return (np.full((nq, k), np.inf, dtype=np.float32), np.full((nq, k), -1, dtype=np.int64))
        d, i = self.search_device(q.to(_device()), int(k))
        return d.cpu().numpy(), i.cpu().numpy()


def _locked(fn):
    """The reference relies on the GIL for `tests/test_memory.py:226-256` (3 threads adding concurrently); here ctypes
    releases the GIL while a kernel call is enqueued, so the bookkeeping is serialised explicitly."""
    @functools.wraps(fn)
    def wrapper(self, *a, **kw):
        with self._lock:
            return fn(self, *a, **kw)
    return wrapper


class PrototypeMemory:
    """Memory system that maintains prototypes for each class (memory.py:11-245)."""

    def __init__(self, embedding_dim: int, config: Optional[ModelConfig] = None):
        self.embedding_dim = embedding_dim
        self.config = config or ModelConfig()
        self.examples = defaultdict(list)   # label -> List[Example]
        self.prototypes = {}                # label -> tensor
        self.strategic_prototypes = {}
        self.index = FlatL2Index(embedding_dim)
        self.label_to_index = {}
        self.index_to_label = {}
        self.updates_since_rebuild = 0
        self._lock = threading.RLock()

    # ------------------------------------------------------------------ add path (memory.py:41-83)
    @_locked
    def add_example(self, example: Example, label: str):
        """memory.py:41-83 (a batch of one through the device-resident store)"""
        if example.embedding is None:
            raise ValueError("Example must have an embedding")
        if example.embedding.size(-1) != self.embedding_dim:
            raise ValueError(
                f"Example embedding dimension {example.embedding.size(-1)} "
                f"does not match memory dimension {self.embedding_dim}")
        self.add_examples_batch([example], [label])

    @_locked
    def add_examples_batch(self, examples: List[Example], labels: List[str], device_rows: Optional[torch.Tensor] = None):
        """Batched equivalent of calling add_example for each pair (same final lists, prototypes and counters).

        SURVEY.md section 8(f) N2: every class keeps its retained embeddings in HBM ([cap + 1, D] slots + a logical order);
        one kernel (ac_memory_append_prune, one CTA per touched class) appends the new rows and, for a class over
        max_examples_per_class, replays the reference's per-example pruning sequentially -- mean of the cap + 1 rows, L2 distance
        to it, list reordered by that distance, farthest dropped (memory.py:196-217) -- then returns the provenance of every
        retained position, so the Example lists on the host are put in the same order.  Only the NEW rows are uploaded
        (`device_rows` [len(examples), D]: the encoder's output when the caller still has it on the device)."""
        for ex, l in zip(examples, labels):
            if ex.embedding is None:
                raise ValueError("Example must have an embedding")
            if ex.embedding.size(-1) != self.embedding_dim:
                raise ValueError(
                    f"Example embedding dimension {ex.embedding.size(-1)} "
                    f"does not match memory dimension {self.embedding_dim}")
        if not examples:
            return
        cap = int(self.config.max_examples_per_class)
        if cap > 2047:                     # the store sorts cap + 1 <= 2048 distances in shared memory
            for ex, l in zip(examples, labels):
                self._add_example_eager(ex, l)
            return
        dev = _device()
        groups: Dict[str, List[int]] = {}
        for i, l in enumerate(labels):
            groups.setdefault(l, []).append(i)
        touched = list(groups.keys())
        st = self._store(cap, dev)
        slots = [self._store_slot(st, l) for l in touched]
        new_rows = device_rows if device_rows is not None else torch.stack(
            [ex.embedding.reshape(-1).float() for ex in examples]).to(dev)
        new_index = torch.tensor([i for l in touched for i in groups[l]], dtype=torch.int32, device=dev)
        starts = [0]
        for l in touched:
            starts.append(starts[-1] + len(groups[l]))
        cls_start = torch.tensor(starts, dtype=torch.int32, device=dev)
        src, proto = _cabi.memory_append_prune(st["rows"], st["order"], st["count"], new_rows, new_index, cls_start,
                                               torch.tensor(slots, dtype=torch.int32, device=dev))
        src_h, proto_h = src.cpu().numpy(), proto.cpu()          # the call's one synchronisation
        for t, l in enumerate(touched):
            old = self.examples[l]
            n_old = len(old)
            fresh = [examples[i] for i in groups[l]]
            kept = [old[s] if s < n_old else fresh[s - n_old] for s in src_h[t].tolist() if s >= 0]
            self.examples[l] = kept
            st["mirror"][l] = [id(e) for e in kept]
            self.prototypes[l] = proto_h[t].clone()
            if l in self.label_to_index:                        # memory.py:155-159
                idx = self.label_to_index[l]
                self.index.remove_ids(torch.tensor([idx]))
                self.index.add(self.prototypes[l].unsqueeze(0))
        # same counter / rebuild behaviour as the per-example loop (memory.py:74-83)
        for _ in examples:
            if not getattr(self, "just_rebuilt", False):
                self.updates_since_rebuild += 1
            if self.updates_since_rebuild >= self.config.prototype_update_frequency:
                self._rebuild_index()
                self.just_rebuilt = True
            else:
                self.just_rebuilt = False

    # ---- device-resident class stores
    def _store(self, cap: int, dev) -> dict:
        st = self.__dict__.get("_dev_store")
        if st is None or st["cap"] != cap or st["rows"].device != dev:
            st = {"cap": cap, "rows": torch.empty((0, cap + 1, self.embedding_dim), dtype=torch.float32, device=dev),
                  "order": torch.empty((0, cap + 1), dtype=torch.int32, device=dev),
                  "count": torch.empty((0,), dtype=torch.int32, device=dev), "slot_of": {}, "mirror": {}}
            self.__dict__["_dev_store"] = st
        return st

    def _store_slot(self, st: dict, label: str) -> int:
        """class slot of `label`, created / re-uploaded when the host list is not what the store last saw (first use, clear,
        load, direct edits of memory.examples): rows in list order, identity slot order"""
        cap = st["cap"]
        slot = st["slot_of"].get(label)
        if slot is None:
            slot = len(st["slot_of"])
            st["slot_of"][label] = slot
            if slot >= st["rows"].shape[0]:
                grow = max(8, st["rows"].shape[0])
                dev = st["rows"].device
                st["rows"] = torch.cat([st["rows"], torch.empty((grow, cap + 1, self.embedding_dim), dtype=torch.float32, device=dev)])
                st["order"] = torch.cat([st["order"], torch.arange(cap + 1, dtype=torch.int32, device=dev).repeat(grow, 1)])
                st["count"] = torch.cat([st["count"], torch.zeros((grow,), dtype=torch.int32, device=dev)])
            st["mirror"][label] = None
        exs = self.examples[label] if label in self.examples else []
        if st["mirror"].get(label) != [id(e) for e in exs]:
            if len(exs) > cap:             # an over-cap list built behind the store's back: bring it under the cap first
                self._prune_examples(label)
                exs = self.examples[label]
            n = len(exs)
            if n:
                st["rows"][slot, :n] = torch.stack([e.embedding.reshape(-1).float() for e in exs]).to(st["rows"].device)
            st["order"][slot] = torch.arange(cap + 1, dtype=torch.int32, device=st["rows"].device)
            st["count"][slot] = n
            st["mirror"][label] = [id(e) for e in exs]
        return slot

    def class_rows_device(self, label: str) -> torch.Tensor:
        """[n_c, D] device rows of the class's retained examples in list order (the store's rows gathered through its order)"""
        cap = int(self.config.max_examples_per_class)
        if cap > 2047:
            return torch.stack([e.embedding.reshape(-1).float() for e in self.examples[label]]).to(_device())
        st = self._store(cap, _device())
        slot = self._store_slot(st, label)
        n = len(self.examples[label])
        return st["rows"][slot].index_select(0, st["order"][slot, :n].long())

    def _add_example_eager(self, example: Example, label: str):
        """the per-example path of memory.py:60-83 (used only when max_examples_per_class exceeds the store's 2047 rows)"""
        self.examples[label].append(example)
        if len(self.examples[label]) > self.config.max_examples_per_class:
            self._prune_examples(label)
        exs = self.examples[label]
        X = torch.stack([e.embedding.reshape(-1).float() for e in exs]).to(_device())
        mean, _ = _cabi.segment_mean(X, torch.zeros(X.shape[0], dtype=torch.int32, device=X.device), 1)
        self.prototypes[label] = mean[0].cpu()
        if label in self.label_to_index:
            self.index.remove_ids(torch.tensor([self.label_to_index[label]]))
            self.index.add(self.prototypes[label].unsqueeze(0))
        if not getattr(self, "just_rebuilt", False):
            self.updates_since_rebuild += 1
        if self.updates_since_rebuild >= self.config.prototype_update_frequency:
            self._rebuild_index()
            self.just_rebuilt = True
        else:
            self.just_rebuilt = False

    # ------------------------------------------------------------------ search (memory.py:85-136)
    def get_nearest_prototypes(self, query_embedding: torch.Tensor, k: int = 5,
                               min_similarity: Optional[float] = None) -> List[Tuple[str, float]]:
        if self.updates_since_rebuild >= self.config.prototype_update_frequency:
            self._rebuild_index()
        if self.index.ntotal == 0:
            return []
        q = query_embedding.reshape(1, -1).to(device=_device(), dtype=torch.float32)
        out = self.get_nearest_prototypes_batch(q, k)
        return out[0]

    @_locked
    def get_nearest_prototypes_batch(self, queries: torch.Tensor, k: int) -> List[List[Tuple[str, float]]]:
        """Batched form (new): queries [B, D] CUDA fp32 -> per query the list memory.py:85-136 returns."""
        if self.updates_since_rebuild >= self.config.prototype_update_frequency:
            self._rebuild_index()
        B = queries.shape[0]
        if self.index.ntotal == 0:
            return [[] for _ in range(B)]
        k = min(k, self.index.ntotal)
        d, i = self.index.search_device(queries.contiguous(), k)
        scores = _cabi.proto_scores(d, i)
        i_h = i.cpu().numpy()
        s_h = scores.cpu().numpy()
        res = []
        for b in range(B):
            row = []
            for idx, sc in zip(i_h[b], s_h[b]):
                if idx >= 0:
                    row.append((self.index_to_label[int(idx)], float(sc)))
            res.append(row)
        return res

    # ------------------------------------------------------------------ prototypes / index maintenance
    @_locked
    def _update_prototype(self, label: str):
        """memory.py:138-159: prototype = mean of the class's retained examples (device segment mean)."""
        examples = self.examples[label]
        if not examples:
            return
        rows = self.class_rows_device(label)
        mean, _ = _cabi.segment_mean(rows, torch.zeros(rows.shape[0], dtype=torch.int32, device=rows.device), 1)
        self.prototypes[label] = mean[0].cpu()
        if label in self.label_to_index:
            self.index.remove_ids(torch.tensor([self.label_to_index[label]]))
            self.index.add(self.prototypes[label].unsqueeze(0))

    @_locked
    def _rebuild_index(self):
        """memory.py:161-177: rows in sorted(label) order (one stacked upload of the C prototype rows)."""
        self.index = FlatL2Index(self.embedding_dim)
        self.label_to_index.clear()
        self.index_to_label.clear()
        sorted_labels = sorted(self.prototypes.keys())
        if sorted_labels:
            self.index.add(torch.stack([self.prototypes[l].reshape(-1).float() for l in sorted_labels]))
        for i, label in enumerate(sorted_labels):
            self.label_to_index[label] = i
            self.index_to_label[i] = label
        self.updates_since_rebuild = 0

    def _restore_from_save(self):
        """memory.py:179-194."""
        self._rebuild_index()

    @_locked
    def _prune_examples(self, label: str):
        """memory.py:196-217: keep the max_examples_per_class examples closest (L2) to the class mean."""
        examples = self.examples[label]
        if not examples:
            return
        X = torch.stack([ex.embedding.reshape(-1).float() for ex in examples]).to(_device())
        mean, _ = _cabi.segment_mean(X, torch.zeros(X.shape[0], dtype=torch.int32, device=X.device), 1)
        dist = torch.linalg.vector_norm(X - mean, dim=1).cpu().numpy()
        keep = np.argsort(dist, kind="stable")[: self.config.max_examples_per_class]
        self.examples[label] = [examples[i] for i in keep]
        assert len(self.examples[label]) <= self.config.max_examples_per_class

    # ------------------------------------------------------------------ stats / clear (memory.py:219-245)
    def get_stats(self) -> Dict[str, Any]:
        return {
            "num_classes": len(self.prototypes),
            "examples_per_class": {label: len(ex) for label, ex in self.examples.items()},
            "total_examples": sum(len(ex) for ex in self.examples.values()),
            "prototype_dimensions": self.embedding_dim,
            "updates_since_rebuild": self.updates_since_rebuild,
        }

    @_locked
    def clear(self):
        self.__dict__.pop("_dev_store", None)
        self.examples.clear()
        self.prototypes.clear()
        self.index = FlatL2Index(self.embedding_dim)
        self.label_to_index.clear()
        self.index_to_label.clear()
        self.updates_since_rebuild = 0
