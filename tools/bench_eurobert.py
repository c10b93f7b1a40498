#!/usr/bin/env python
"""EuroBERT-210m-shaped encoder (ids -> unit CLS rows) against HF and against the NomicBERT shape this library already runs.

    python tools/bench_eurobert.py [--steps K] [--warmup W] [--ab-reps 3]

Every call embeds 65,536 tokens (B = 65536 / S sequences, no padding, cls_only) at S = 128, 512, 2048 and 8192.
  eurobert_210m (workload.eurobert_210m: 12 x 768, SwiGLU I 3072, pre-norm with RMSNorm, RoPE) against HF EuroBertModel in
    torch eager with fp16 autocast (SDPA), and at S <= 2048 against workload.nomic_v15 through this library.  Nomic has the
    same linear work per token (4 H^2 + 3 H I multiply-adds per layer) and the same attention; the two differ in the block
    only: post-LN with LayerNorm against pre-norm with RMSNorm, so the ratio shows what the pre-norm / RMS path costs.
The two encoders alternate --ab-reps times per S in this one process and every range is reported; the GEMM and attention
times come from the library's per-launch profiler in a separate run.  Before any timing, the CLS rows are checked against HF
in fp32 (TF32 off) on the same GPU; a mismatch aborts.  An HF baseline that fails or runs out of memory is reported as such.
Prints one JSON line with the GPU's name and power limit; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from adaptive_classifier_b200 import _cabi, workload as wl  # noqa: E402
from bench_modernbert import gpu_info  # noqa: E402
from bench_rotary import TOKENS, family_rows, parity  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ab-reps", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1 or args.ab_reps < 1:
        ap.error("--steps and --ab-reps must be at least 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_eurobert.py: no CUDA device; the CUDA path has no CPU fallback")
    _cabi.load_library()

    euro, ecfg = wl.eurobert_210m(1234)
    euro = euro.cuda().eval()
    enc = _cabi.Encoder.from_hf(euro, max_tokens=TOKENS)
    # ids valid in both vocabularies (Nomic's 30528 < EuroBERT's 128256)
    ids_of = lambda B, S: wl.synthetic_ids(B, S, vocab=30528, seed=7)
    # the bound of this shape in tests/test_gpu_eurobert.py (SHAPE_BOUND): fp16 operands alone give 1.2e-3 - 1.5e-3 here
    chk = [parity(enc, euro, wl.synthetic_ids(4, 512, vocab=ecfg.vocab_size, seed=3).cuda(), 2.5e-3),
           parity(enc, euro, wl.synthetic_ids(1, 8192, vocab=ecfg.vocab_size, seed=5).cuda(), 2.5e-3)]
    if not all(c["ok"] for c in chk):
        raise SystemExit(f"bench_eurobert.py: parity check against HF fp32 failed: {chk}")
    nomic, _ = wl.nomic_v15(1234)
    nomic_enc = _cabi.Encoder.from_hf(nomic.cuda().eval(), max_tokens=TOKENS)
    del nomic
    torch.cuda.empty_cache()
    rows = family_rows(enc, euro, nomic_enc, [128, 512, 2048, 8192], ids_of, 2048, args)
    enc.close(); nomic_enc.close()
    for r in rows:          # family_rows names the comparison encoder "ref"
        if "ref" in r:
            r["nomic_v15"] = r.pop("ref")
            r["eurobert_over_nomic_time_min_max"] = r.pop("new_over_ref_time_min_max")
        r["eurobert"] = r.pop("new")

    line = {"metric": "EuroBERT-210m-shaped encoder tokens/s", "unit": "tokens/s",
            "value": {f"eurobert_{r['S']}": r["eurobert"]["tokens_per_s"] for r in rows},
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ab_reps": args.ab_reps,
            "dtype": "f16", "data": "synthetic",
            "config": {"eurobert": "workload.eurobert_210m (12 x 768, 12 heads, SwiGLU I 3072, RMSNorm, RoPE theta 250000; "
                                   "seed 1234)",
                       "nomic_v15": "workload.nomic_v15 (12 x 768, 12 heads, SwiGLU I 3072, post-LN, RoPE theta 1000; "
                                    "seed 1234) through this library, S <= 2048",
                       "tokens_per_call": TOKENS, "padding": "none", "cls_only": True},
            "parity": chk, "rows": rows,
            "note": (f"encoder times: CUDA events around {args.steps} calls, the EuroBERT and Nomic encoders alternated "
                     f"{args.ab_reps} times, min..max; gemm / attention times are a separate profiled run's; HF baseline is "
                     f"torch {torch.__version__} eager, fp16 autocast, SDPA"),
            **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
