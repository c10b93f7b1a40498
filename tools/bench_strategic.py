#!/usr/bin/env python
"""Strategic mode on one GPU: best-response kernel time, predict() latency in strategic mode, one strategic training call.

    python tools/bench_strategic.py [--reps R]

1. ac_strategic_best_response on the drop-in head (768 -> 768 -> 384 -> 21, linear cost) at B = 1, 16 and 4096: CUDA-event
   time per call, FLOP from shapes (flops_per_query below), achieved FP32 rate and share of the H100 SXM data-sheet FP32 peak
   (67 TFLOP/s dense), with the bound named per B: FMA throughput where the FP32 floor is at least a quarter of the call,
   otherwise launch latency and host-side call overhead.  Before timing, the kernel's choices on the timed inputs (all rows at
   B = 1 and 16, the first 256 at B = 4096) are checked against the CPU oracle (oracle/strategic_oracle.py) wherever the
   oracle's margin exceeds 1e-4.
2. predict() latency of a seeded random-init bert-base classifier (20 classes x 10 examples) in strategic mode (linear cost)
   and in regular mode, one 16-token text, host clock around calls that end in a device synchronise.
3. Wall time of one strategic training call (ac_head_train_strategic: 20 classes x 500 stored rows = 10,000 rows, batches of
   16, 5 epochs = 3,125 steps), and the CPU oracle's strategic training on the first 4 steps, extrapolated to 3,125 steps
   (labelled as an extrapolation).
Prints one JSON line with the GPU's name and power limit; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from adaptive_classifier_b200 import _cabi, workload as wl  # noqa: E402
from adaptive_classifier_b200.classifier import dataloader_epoch_permutation  # noqa: E402
from oracle import strategic_oracle as so  # noqa: E402

D, H0, H1, C = 768, 768, 384, 21
FP32_PEAK = 67e12                     # H100 SXM data sheet, dense FP32


def flops_per_query(D, H0, H1, C, nc=50):
    """layer 0 once (2 D H0), the rank-1 update per candidate (2 H0), layers 1 and 2 per candidate, softmax ignored"""
    return 2 * D * H0 + nc * (2 * H0 + 2 * H0 * H1 + 2 * H1 * C)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit": q[1], "sm_clock_max": q[2]}
    except Exception as ex:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({ex!r})"}


def head(seed=0):
    g = torch.Generator().manual_seed(seed)
    p = {"W0": torch.randn(H0, D, generator=g) * (2.0 / D) ** 0.5, "b0": torch.zeros(H0),
         "W1": torch.randn(H1, H0, generator=g) * (2.0 / H0) ** 0.5, "b1": torch.zeros(H1),
         "W2": torch.randn(C, H1, generator=g) * (6.0 / H1) ** 0.5, "b2": torch.zeros(C)}
    return {k: v.cuda().contiguous() for k, v in p.items()}


def event_ms(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernel_section(reps):
    p = head()
    g = torch.Generator().manual_seed(1)
    alpha = (torch.randn(D, generator=g) * 0.02).cuda()
    out = {}
    fq = flops_per_query(D, H0, H1, C)
    for B in (1, 16, 4096):
        X = torch.nn.functional.normalize(torch.randn(B, D, generator=g), dim=1).cuda()
        # parity on the timed inputs: all of them at B = 1 and 16, the first 256 rows at B = 4096 (the fp64 oracle runs
        # 50 full head forwards per row on the host)
        ch, _, _ = _cabi.strategic_best_response(X, p, _cabi.AC_COST_LINEAR, alpha)
        n_chk = min(B, 256)
        ref = so.best_response(p, X[:n_chk], 0, alpha.cpu(), alpha.cpu())
        clear = ref["margin"] > 1e-4
        parity = {"checked_rows": n_chk, "clear_margin_rows": int(clear.sum()),
                  "choices_equal": bool(torch.equal(ch[:n_chk].cpu().long()[clear], ref["choice"][clear]))}
        assert parity["choices_equal"], f"kernel choices differ from the oracle at B = {B}"
        ms = event_ms(lambda: _cabi.strategic_best_response(X, p, _cabi.AC_COST_LINEAR, alpha), reps if B < 4096 else max(5, reps // 10))
        rate = B * fq / (ms * 1e-3)
        floor_ms = B * fq / FP32_PEAK * 1e3
        # the events bracket the whole Python call (ctypes, workspace lookup, output allocation, 5 launches per chunk):
        # where the FP32 floor is a small part of the time, that overhead and launch latency bound the call, not FMA throughput
        bound = "fp32 FMA" if floor_ms >= 0.25 * ms else "launch latency and host-side call overhead (fp32 floor %.2f us)" % (floor_ms * 1e3)
        out[f"b{B}"] = {"ms_per_call": round(ms, 4), "us_per_query": round(ms * 1e3 / B, 3), "flop_per_query": fq,
                        "tflops": round(rate / 1e12, 2), "share_of_fp32_peak": round(rate / FP32_PEAK, 4), "bound": bound,
                        "parity": parity}
    return out


def predict_section(reps):
    from transformers import BertTokenizerFast
    import adaptive_classifier_b200 as acb
    model, cfg = wl.bert_base_state_dict(1234)
    d = tempfile.mkdtemp(prefix="bench_strategic_")
    model.save_pretrained(d)
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + [f"w{i}" for i in range(2000)]
    BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}, do_lower_case=True).save_pretrained(d)
    texts = [" ".join(f"w{(c * 97 + e * 13 + j) % 2000}" for j in range(14)) for c in range(20) for e in range(10)]
    labels = [f"class{c}" for c in range(20) for _ in range(10)]
    res = {}
    for mode, conf in (("regular", None), ("strategic", {"enable_strategic_mode": True, "cost_function_type": "linear",
                                                         "cost_coefficients": [0.02] * 768, "strategic_training_frequency": 1000})):
        clf = acb.AdaptiveClassifier(d, device="cuda", config=conf)
        clf.add_examples(texts, labels)
        q = "w5 w17 w99 w1200 w3 w44 w8 w1999 w640 w12 w71 w300 w2 w9"
        for _ in range(5):
            clf.predict(q)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            clf.predict(q)
        torch.cuda.synchronize()
        res[f"predict_{mode}_ms"] = round((time.perf_counter() - t0) * 1e3 / reps, 3)
    return res


def training_section():
    p = head(2)
    p = {k: (v[:20] if k in ("W2", "b2") else v).contiguous() for k, v in p.items()}
    n = 10000
    g = torch.Generator().manual_seed(3)
    X = torch.nn.functional.normalize(torch.randn(n, D, generator=g), dim=1)
    y = torch.arange(n) % 20
    alpha = torch.randn(D, generator=g) * 0.02
    gen = torch.Generator().manual_seed(42)
    perms = torch.cat([dataloader_epoch_permutation(gen, n) for _ in range(5)])
    p0 = {k: v.clone() for k, v in p.items()}
    m = {k: torch.zeros_like(v) for k, v in p.items()}
    v = {k: torch.zeros_like(t) for k, t in p.items()}
    Xd, yd, ad = X.cuda(), y.cuda(), alpha.cuda()
    # warm-up on a copy, then the timed call on fresh state
    pw = {k: t.clone() for k, t in p.items()}
    _cabi.head_train_strategic(Xd[:64], yd[:64], perms[:64] % 64, pw, {k: torch.zeros_like(t) for k, t in pw.items()},
                               {k: torch.zeros_like(t) for k, t in pw.items()}, cost_kind=0, c1=ad, lr=5e-4, strategic_lambda=0.1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    stats = _cabi.head_train_strategic(Xd, yd, perms, p, m, v, cost_kind=0, c1=ad, lr=5e-4, strategic_lambda=0.1, dropout_p=0.1)
    torch.cuda.synchronize()
    gpu_s = time.perf_counter() - t0
    steps = stats.shape[0]
    t0 = time.perf_counter()
    so.strategic_training(p0, X, y, perms, 0, alpha, alpha, lr=5e-4, lam=0.1, steps=4)
    cpu_4 = time.perf_counter() - t0
    return {"rows": n, "steps": steps, "gpu_call_s": round(gpu_s, 3), "gpu_ms_per_step": round(gpu_s * 1e3 / steps, 4),
            "cpu_oracle_s_4_steps": round(cpu_4, 3), "cpu_oracle_s_extrapolated_to_all_steps": round(cpu_4 / 4 * steps, 1),
            "cpu_oracle_note": "CPU fp64+fp32 oracle port (not the reference itself), timed on 4 steps and extrapolated",
            "final_loss": float(stats[-1, 0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_strategic.py needs an H100"
    _cabi.check(_cabi.load_library().ac_device_check(), "ac_device_check")
    res = {"what": "strategic mode: best-response search, predict latency, strategic training", **gpu_info()}
    res["kernel"] = kernel_section(args.reps)
    res["predict"] = predict_section(max(20, args.reps // 4))
    res["training"] = training_section()
    res["command"] = "python tools/bench_strategic.py " + " ".join(sys.argv[1:])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
