#!/usr/bin/env python
"""NomicBERT- and jina-embeddings-v3-shaped encoders (ids -> unit CLS rows) against HF and against the encoders of the same
size this library already runs.

    python tools/bench_rotary.py [--steps K] [--warmup W] [--ab-reps 3]

Every call embeds 65,536 tokens (B = 65536 / S sequences, no padding, cls_only).
  nomic_v15 (workload.nomic_v15: 12 x 768, SwiGLU I 3072, RoPE) at S = 128, 512, 2048, against HF NomicBertModel in torch
    eager with fp16 autocast (SDPA) and against the bert-base shape (workload.bert_base_state_dict) through this library at
    S <= 512 (its position table stops there).  Linear work per token and layer: 4 H^2 + 3 H I = 9.44 M multiply-adds
    against 4 H^2 + 2 H I = 7.08 M for bert-base (1.33x); attention work is the same.
  jina_v3 (workload.jina_v3: 24 x 1024, GELU I 4096, RoPE) at S = 1024 and 8192, against HF JinaEmbeddingsV3Model with
    fp16 autocast and against workload.bge_m3 through this library (the same linear and attention work).
The library's encoders alternate --ab-reps times per S in this one process and every range is reported; the GEMM and
attention times come from the library's per-launch profiler in a separate run.  Before any timing, the CLS rows of both
new encoders are checked against HF in fp32 (TF32 off) on the same GPU; a mismatch aborts.  An HF baseline that fails or
runs out of memory is reported as such.  Prints one JSON line with the GPU's name and power limit; writes nothing.
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


def parity(enc, model, ids, bound):
    out = enc.forward_cls(ids)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            h = model(input_ids=ids.long(), attention_mask=torch.ones_like(ids, dtype=torch.long)).last_hidden_state[:, 0]
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    err = float((out - torch.nn.functional.normalize(h.float(), dim=1)).norm(dim=1).max())
    return {"B": ids.shape[0], "S": ids.shape[1], "cls_row_err_max": err, "bound": bound, "ok": err < bound}


def hf_fp16_ms(model, ids, steps, warmup):
    def fwd():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return model(input_ids=ids, attention_mask=torch.ones_like(ids)).last_hidden_state[:, 0, :]
    try:
        return {"ms": bench._timed_ms(torch, fwd, steps, warmup=warmup)}
    except Exception as ex:          # a baseline failure or OOM must not take the line down
        torch.cuda.empty_cache()
        return {"failed": repr(ex)[:300]}


def profiled(enc, ids, steps):
    enc.forward_cls(ids)
    torch.cuda.synchronize()
    _cabi.profile_enable(True)
    for _ in range(steps):
        enc.forward_cls(ids)
    torch.cuda.synchronize()
    _cabi.profile_enable(False)
    att, gemm = _cabi.profile_read(PROF_ATTENTION), _cabi.profile_read(PROF_GEMM_LINEAR)
    return {"attention_ms": att["ms"] / steps, "gemm_ms": gemm["ms"] / steps,
            "gemm_tflops": gemm["flops"] / max(gemm["ms"], 1e-9) * 1e-9}


def family_rows(new, new_model, ref, lengths, ids_of, ref_max_s, args):
    """per S: the new encoder and the reference-size encoder alternated --ab-reps times, their profiles, HF fp16"""
    rows = []
    for S in lengths:
        B = TOKENS // S
        ids = ids_of(B, S).cuda()
        encs = {"new": new} if S > ref_max_s else {"new": new, "ref": ref}
        ms = {k: [] for k in encs}
        for k, e in encs.items():
            bench._timed_ms(torch, lambda: e.forward_cls(ids), 1, warmup=args.warmup)
        for _ in range(args.ab_reps):
            for k, e in encs.items():
                ms[k].append(bench._timed_ms(torch, lambda: e.forward_cls(ids), args.steps, warmup=0))
        row = {"S": S, "B": B}
        for k in encs:
            row[k] = {"ms_min": min(ms[k]), "ms_max": max(ms[k]), "tokens_per_s": B * S / (min(ms[k]) * 1e-3),
                      **profiled(encs[k], ids, args.steps)}
        if "ref" in encs:
            row["new_over_ref_time_min_max"] = [min(ms["new"]) / max(ms["ref"]), max(ms["new"]) / min(ms["ref"])]
        hf = hf_fp16_ms(new_model, ids.long(), args.steps, args.warmup)
        row["hf_eager_fp16_autocast"] = hf
        if "ms" in hf:
            row["speedup_vs_hf_fp16"] = hf["ms"] / min(ms["new"])
        rows.append(row)
        del ids
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ab-reps", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1 or args.ab_reps < 1:
        ap.error("--steps and --ab-reps must be at least 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_rotary.py: no CUDA device; the CUDA path has no CPU fallback")
    _cabi.load_library()
    out = {}

    nomic, ncfg = wl.nomic_v15(1234)
    nomic = nomic.cuda().eval()
    enc = _cabi.Encoder.from_hf(nomic, max_tokens=TOKENS)
    chk_n = parity(enc, nomic, wl.synthetic_ids(4, 512, vocab=ncfg.vocab_size, seed=3).cuda(), 1e-3)
    bert, _ = wl.bert_base_state_dict(1234)
    bert_enc = _cabi.Encoder.from_hf(bert.cuda().eval(), max_tokens=TOKENS)
    del bert
    out["nomic"] = family_rows(enc, nomic, bert_enc, [128, 512, 2048],
                               lambda B, S: wl.synthetic_ids(B, S, vocab=ncfg.vocab_size, seed=7), 512, args)
    enc.close(); bert_enc.close()
    del nomic
    torch.cuda.empty_cache()

    jina, _ = wl.jina_v3(1234)
    jina = jina.cuda().eval()
    enc = _cabi.Encoder.from_hf(jina, max_tokens=TOKENS)
    chk_j = parity(enc, jina, wl.xlmr_ids(2, 2048, seed=3).cuda(), 1.5e-3)
    bge, _ = wl.bge_m3(1234)
    bge_enc = _cabi.Encoder.from_hf(bge.cuda().eval(), max_tokens=TOKENS)
    del bge
    torch.cuda.empty_cache()
    out["jina"] = family_rows(enc, jina, bge_enc, [1024, 8192], lambda B, S: wl.xlmr_ids(B, S, seed=7), 8192, args)
    enc.close(); bge_enc.close()
    if not (chk_n["ok"] and chk_j["ok"]):
        raise SystemExit(f"bench_rotary.py: parity check against HF fp32 failed: {chk_n} {chk_j}")

    line = {"metric": "NomicBERT / jina-embeddings-v3-shaped encoder tokens/s", "unit": "tokens/s",
            "value": {f"{fam}_{r['S']}": r["new"]["tokens_per_s"] for fam in out for r in out[fam]},
            "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ab_reps": args.ab_reps,
            "dtype": "f16", "data": "synthetic",
            "config": {"nomic": "workload.nomic_v15 (12 x 768, 12 heads, SwiGLU I 3072, RoPE theta 1000; seed 1234), "
                                "ref = workload.bert_base_state_dict through this library",
                       "jina": "workload.jina_v3 (24 x 1024, 16 heads, GELU I 4096, RoPE theta 20000; seed 1234), "
                               "ref = workload.bge_m3 through this library",
                       "tokens_per_call": TOKENS, "padding": "none", "cls_only": True},
            "parity": {"nomic": chk_n, "jina": chk_j}, "rows": out,
            "note": (f"encoder times: CUDA events around {args.steps} calls, the new and ref encoders alternated "
                     f"{args.ab_reps} times, min..max; gemm / attention times are a separate profiled run's; HF baseline is "
                     f"torch {torch.__version__} eager, fp16 autocast, SDPA"),
            **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
