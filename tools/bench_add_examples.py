#!/usr/bin/env python
"""BASELINE.json configs[3]: add_examples() continual loop -- 50k new examples, EWC-penalised head update, bert-base, one GPU.

Synthetic pre-tokenised sequences (SURVEY.md section 8(d)): 20 classes, 196 calls of 256 examples, a 21st class introduced at
call 100 so that _train_new_classes (+ Fisher / EWC) is traversed; from call ~79 on every class is over max_examples_per_class
(1000), so the distance-to-mean pruning of memory.py:196-217 runs for every added example.  Reports examples/s end to end, the
split over encoder / memory maintenance / head training, and head optimizer steps/s.  Like the reference, every call retrains
the head on the whole memory for <= 10 epochs (classifier.py:1428-1522): head training dominates by construction.

    python tools/bench_add_examples.py [--examples 50176]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(examples=50176, call=256, seq=128, quiet=False, cpu_sample=True, hbm_peak=None):
    """hbm_peak: {'hbm_gbs': ..., 'source': ...} of the GPU this runs on (bench.py peaks()); without it no HBM floor is reported"""
    import copy
    import numpy as np
    import torch
    import adaptive_classifier_b200 as acb
    from adaptive_classifier_b200 import _cabi, workload as wl

    dev = "cuda"
    model, cfg = wl.bert_base_state_dict(1234)
    enc = _cabi.Encoder.from_hf(model, max_tokens=call * seq, device=dev)
    del model

    # an AdaptiveClassifier without the HF/tokenizer constructor: the loop below drives the same methods
    clf = acb.AdaptiveClassifier.__new__(acb.AdaptiveClassifier)
    clf.config = acb.ModelConfig()
    clf.device, clf.use_onnx, clf.model_name = dev, False, "synthetic-bert-base"
    clf.encoder, clf._max_tokens, clf.embedding_dim = enc, call * seq, 768
    clf.memory = acb.PrototypeMemory(768, config=clf.config)
    clf.adaptive_head, clf.label_to_id, clf.id_to_label = None, {}, {}
    clf.train_steps, clf.training_history = 0, {}
    np.random.seed(0)

    n_calls = examples // call
    t_embed = t_mem = t_train = 0.0
    steps_total = 0
    new_class_calls = 0
    torch.cuda.synchronize()
    t0 = time.time()
    for c in range(n_calls):
        ids = wl.synthetic_ids(call, seq, seed=1000 + c)
        ncls = 21 if c >= 100 else 20
        labels = [f"class_{(c * call + i) % ncls:02d}" for i in range(call)]
        ta = time.time()
        emb_dev = clf._embed_ids_device(ids, None, None)
        emb = emb_dev.cpu()
        tb = time.time()
        has_existing = len(clf.label_to_id) > 0
        new = set(labels) - set(clf.label_to_id)
        for l in sorted(new):
            clf.label_to_id[l] = len(clf.label_to_id); clf.id_to_label[clf.label_to_id[l]] = l
        clf.memory.add_examples_batch([acb.Example(f"t{c}_{i}", l, e) for i, (l, e) in enumerate(zip(labels, emb))], labels, device_rows=emb_dev)
        for l in labels:
            clf.training_history[l] = clf.training_history.get(l, 0) + 1
        torch.cuda.synchronize()
        tc = time.time()
        if new and has_existing:
            old = copy.deepcopy(clf.adaptive_head)
            clf.adaptive_head.update_num_classes(len(clf.label_to_id))
            clf.adaptive_head = clf.adaptive_head.to(dev)
            clf._train_new_classes(old, new)
            new_class_calls += 1
        else:
            if clf.adaptive_head is None:
                clf._initialize_adaptive_head()
            clf._train_adaptive_head()
        steps_total += sum(clf.last_training_trace["steps_per_epoch"])
        clf.memory._rebuild_index()
        torch.cuda.synchronize()
        td = time.time()
        t_embed += tb - ta; t_mem += tc - tb; t_train += td - tc
    total = time.time() - t0
    stats = clf.memory.get_stats()
    last_loss = clf.last_training_trace["loss"][-1] if clf.last_training_trace["loss"] else None

    # isolated head optimizer steps/s at batch 32 through the epoch entry (one kernel launch per epoch of 625 steps)
    p = clf.adaptive_head._param_dict()
    m = {k: torch.zeros_like(v) for k, v in p.items()}
    v = {k: torch.zeros_like(t) for k, t in p.items()}
    n = 20000
    X = torch.nn.functional.normalize(torch.randn(n, 768, device=dev), dim=1)
    y = torch.randint(0, len(clf.label_to_id), (n,), device=dev)
    perm = torch.randperm(n)
    _cabi.head_train_epoch(X, y, perm, p, m, v, first_step=1, batch=32)
    torch.cuda.synchronize()
    t1 = time.time()
    _, nb = _cabi.head_train_epoch(X, y, perm, p, m, v, first_step=1 + 625, batch=32)
    torch.cuda.synchronize()
    dt = time.time() - t1
    step_us = 1e6 * dt / nb
    P_params = sum(t.numel() for t in p.values())
    out = {
        "metric": "examples/sec add_examples() continual loop (bert-base, S=128, calls of 256, 21st class at call 100: Fisher + _train_new_classes)",
        "value": n_calls * call / total, "unit": "examples/s", "examples": n_calls * call, "calls": n_calls,
        "seconds": {"encoder": round(t_embed, 3), "memory_update": round(t_mem, 3), "head_training": round(t_train, 3), "total": round(total, 3)},
        "head_optimizer_steps": steps_total, "new_class_calls": new_class_calls,
        "head_step_us_batch32": step_us, "head_steps_per_s_batch32": 1e6 / step_us,
        "head_step_roofline": {"bound": "hbm/latency", "algorithmic_bytes_per_step": 7 * 4 * P_params,
                               "floor_us_at_hbm_peak": (7 * 4 * P_params / (hbm_peak["hbm_gbs"] * 1e9) * 1e6) if hbm_peak else None,
                               "hbm_peak_source": hbm_peak["source"] if hbm_peak else None,
                               "note": "0.9 M parameters x (theta, g, m, v read; theta, m, v written); the kernel keeps theta and g in shared "
                                       "memory and m, v in L2, so the step is bound by six grid barriers + L2 operand streaming, not HBM"},
        "classes": len(clf.label_to_id), "stored_examples": stats["total_examples"],
        "examples_per_class_max": max(stats["examples_per_class"].values()), "last_step_loss": last_loss,
        "note": "every call retrains the head on the whole memory for <= 10 epochs like classifier.py:1428-1522; memory is capped at 1000 "
                "examples per class (pruning to the 1000 nearest the class mean, memory.py:196-217)"}
    if cpu_sample:
        # CPU arm of the same loop, bounded sample: the oracle restatement of _train_adaptive_head (torch CPU, same batches) on
        # the first 2560 stored embeddings for one call; examples/s = 256 / (encoder CPU time is NOT included: head loop only)
        try:
            from oracle import head_oracle as ho
            Xc = X[:2560].cpu()
            yc = y[:2560].cpu()
            pc = ho.init_head(768, len(clf.label_to_id))
            tcpu = time.time()
            losses, _, per_epoch = ho.train_loop(Xc, yc, pc, epochs=2, batch_size=32, use_scheduler=True)
            dtc = time.time() - tcpu
            out["cpu_baseline"] = {"value": len(losses) / dtc, "unit": "head optimizer steps/s", "cores": torch.get_num_threads(), "kind": "port",
                                   "sample": f"{len(losses)} optimizer steps (2 epochs over 2560 stored rows, batch 32) of the oracle restatement of "
                                             "classifier.py:1453-1520 on the host cores; the GPU figure beside it is head_steps_per_s_batch32"}
        except Exception as ex:
            out["cpu_baseline"] = {"failed": repr(ex)}
    enc.close()
    if not quiet:
        print(json.dumps(out))
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--examples", type=int, default=50176)
    ap.add_argument("--call", type=int, default=256)
    ap.add_argument("--seq", type=int, default=128)
    a = ap.parse_args()
    run(a.examples, a.call, a.seq)
