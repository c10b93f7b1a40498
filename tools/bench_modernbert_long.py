#!/usr/bin/env python
"""ModernBERT-base encoder (ids -> unit CLS rows) at long sequence lengths.

    python tools/bench_modernbert_long.py [--steps K] [--warmup W] [--lengths 512,1024,2048,4096,8192]

Seeded random-init ModernBERT-base (workload.modernbert_base: 22 x 768, 12 heads, GeGLU 1152, RoPE, half-window 64 on two of
every three layers, max_position_embeddings 8192), ids of workload.modernbert_ids, B = 65536 / S sequences per call.  For
every S: the encoder's time and tokens/s; the attention kernels' time, algorithmic flops (sliding layers count only the keys
inside the band, (2w + 1) per query clipped to [0, S)) and TFLOP/s from the library's per-launch profiler in a separate run;
and HF ModernBertModel in torch eager with fp16 autocast (SDPA) on the same ids, which may fail or run out of memory without
taking the line down.  Before any timing, the CLS rows of two sequences at S = 2048 are checked against HF in fp32 (TF32
off) on the same GPU, bound 1.5e-3 on the row error; a mismatch aborts.  Prints one JSON line with the GPU's name and power
limit; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import bench  # noqa: E402  (timing helper; importing runs nothing)
from adaptive_classifier_b200 import _cabi, workload as wl  # noqa: E402
from bench_modernbert import gpu_info  # noqa: E402

TOKENS = 65536
PROF_GEMM_LINEAR, PROF_ATTENTION = 0, 1


def parity(enc, model, S=2048, B=2):
    ids = wl.modernbert_ids(B, S, seed=3).cuda()
    out = enc.forward_cls(ids)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            h = model(input_ids=ids.long(), attention_mask=torch.ones_like(ids, dtype=torch.long)).last_hidden_state[:, 0]
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    err = float((out - torch.nn.functional.normalize(h.float(), dim=1)).norm(dim=1).max())
    return {"S": S, "B": B, "cls_row_err_max": err, "bound": 1.5e-3, "ok": err < 1.5e-3}


def hf_fp16_ms(model, ids, steps, warmup):
    def fwd():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return model(input_ids=ids, attention_mask=torch.ones_like(ids)).last_hidden_state[:, 0, :]
    try:
        return {"ms": bench._timed_ms(torch, fwd, steps, warmup=warmup)}
    except Exception as ex:          # a baseline failure or OOM must not take the line down
        torch.cuda.empty_cache()
        return {"failed": repr(ex)[:300]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lengths", default="512,1024,2048,4096,8192")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_modernbert_long.py: no CUDA device; the CUDA path has no CPU fallback")
    _cabi.load_library()
    model, _ = wl.modernbert_base(1234)
    model = model.cuda().eval()
    enc = _cabi.Encoder.from_hf(model, max_tokens=TOKENS)
    chk = parity(enc, model)
    if not chk["ok"]:
        raise SystemExit(f"bench_modernbert_long.py: parity check against HF fp32 failed: {chk}")

    rows = []
    for S in [int(s) for s in args.lengths.split(",")]:
        B = TOKENS // S
        ids = wl.modernbert_ids(B, S, seed=7).cuda()
        ms = bench._timed_ms(torch, lambda: enc.forward_cls(ids), args.steps, warmup=args.warmup)
        _cabi.profile_enable(True)
        for _ in range(args.steps):
            enc.forward_cls(ids)
        torch.cuda.synchronize()
        _cabi.profile_enable(False)
        att, gemm = _cabi.profile_read(PROF_ATTENTION), _cabi.profile_read(PROF_GEMM_LINEAR)
        att_ms = att["ms"] / args.steps
        row = {"S": S, "B": B, "encoder_ms": ms, "tokens_per_s": B * S / (ms * 1e-3),
               "attention_ms": att_ms, "attention_flops": att["flops"] / args.steps,
               "attention_tflops": att["flops"] / max(att["ms"], 1e-9) * 1e-9,
               "gemm_ms": gemm["ms"] / args.steps, "gemm_tflops": gemm["flops"] / max(gemm["ms"], 1e-9) * 1e-9}
        hf = hf_fp16_ms(model, ids.long(), args.steps, args.warmup)
        row["hf_eager_fp16_autocast"] = hf
        if "ms" in hf:
            row["speedup_vs_hf_fp16"] = hf["ms"] / ms
        rows.append(row)
        del ids
        torch.cuda.empty_cache()

    line = {"metric": "ModernBERT-base encoder tokens/s at long sequence lengths", "unit": "tokens/s",
            "value": {str(r["S"]): r["tokens_per_s"] for r in rows}, "higher_is_better": True, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "dtype": "f16", "data": "synthetic",
            "config": {"workload": "ModernBERT-base architecture (22 x 768, 12 heads, GeGLU 1152, RoPE, half-window 64 on 2 of 3 "
                                   "layers, max_position_embeddings 8192; random init seed 1234), no padding, cls_only",
                       "tokens_per_call": TOKENS},
            "parity": chk, "rows": rows,
            "note": (f"attention flops are algorithmic (4 x keys x head_dim per query and head; sliding layers count the band "
                     f"only); attention / gemm times are the profiled run's, encoder_ms the unprofiled one; HF baseline is "
                     f"torch {torch.__version__} eager, fp16 autocast, SDPA"),
            **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
