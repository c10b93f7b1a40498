#!/usr/bin/env python
"""bge-m3-shaped XLM-RoBERTa encoder (ids -> unit CLS rows) at long sequence lengths, and its attention kernel alone.

    python tools/bench_xlmr_long.py [--steps K] [--warmup W] [--lengths 512,1024,2048,4096,8192] [--ab-reps 3]

Encoder: seeded random-init bge-m3 shape (workload.bge_m3: XLM-R-large, 24 x 1024, 16 heads, I 4096, 8194 positions), ids of
workload.xlmr_ids, B = 65536 / S sequences per call, cls_only.  For every S: the encoder's time and tokens/s; the attention
kernels' time, algorithmic flops and TFLOP/s and the GEMMs' time from the library's per-launch profiler in a separate run;
and HF XLMRobertaModel in torch eager with fp16 autocast (SDPA) on the same ids, which may fail or run out of memory without
taking the line down.  Before any timing, the CLS rows of two sequences at S = 2048 are checked against HF in fp32 (TF32 off)
on the same GPU, bound 1.5e-3 on the row error; a mismatch aborts.

Attention A/B at S = 1024 .. 8192, B = 65536 / S, 16 heads of 64, no mask, on the same fp16 q, k, v: attention_long_kernel
(RoBERTa handle with an 8194-row table), attention_stream_kernel (ModernBERT handle, window 0) and torch SDPA with the flash
backend.  The two library kernels are timed by the library profiler (CUDA events around the launch alone), SDPA by CUDA
events around the call; the three alternate --ab-reps times in this one process and every range is reported.
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

import bench  # noqa: E402  (timing helper; importing runs nothing)
from adaptive_classifier_b200 import _cabi, workload as wl  # noqa: E402
from bench_modernbert import gpu_info  # noqa: E402

TOKENS = 65536
HEADS, DH = 16, 64
PROF_GEMM_LINEAR, PROF_ATTENTION = 0, 1


def parity(enc, model, S=2048, B=2):
    ids = wl.xlmr_ids(B, S, seed=3).cuda()
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


def attention_handles():
    """one-layer handles that only serve Encoder.attention: RoBERTa with 8194 positions (attention_long_kernel past 512)
    and ModernBERT (attention_stream_kernel, window 0), both 16 heads of 64"""
    H, I, V = HEADS * DH, 64, 32
    g = torch.Generator().manual_seed(11)
    r = lambda *s: (0.02 * torch.randn(*s, generator=g)).cuda()
    ones, zeros = (lambda n: torch.ones(n).cuda()), (lambda n: torch.zeros(n).cuda())
    p = "encoder.layer.0."
    sd = {"embeddings.word_embeddings.weight": r(V, H), "embeddings.position_embeddings.weight": r(8194, H),
          "embeddings.token_type_embeddings.weight": r(1, H), "embeddings.LayerNorm.weight": ones(H),
          "embeddings.LayerNorm.bias": zeros(H), p + "intermediate.dense.weight": r(I, H), p + "intermediate.dense.bias": zeros(I),
          p + "output.dense.weight": r(H, I), p + "output.dense.bias": zeros(H)}
    for n in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense"):
        sd[p + n + ".weight"], sd[p + n + ".bias"] = r(H, H), zeros(H)
    for n in ("attention.output.LayerNorm", "output.LayerNorm"):
        sd[p + n + ".weight"], sd[p + n + ".bias"] = ones(H), zeros(H)
    common = dict(layers=1, hidden=H, heads=HEADS, intermediate=I, vocab=V, ln_eps=1e-5, max_tokens=TOKENS)
    long_ = _cabi.Encoder(sd, arch="roberta", max_pos=8194, pad_idx=1, **common)
    msd = {"embeddings.tok_embeddings.weight": r(V, H), "embeddings.norm.weight": ones(H), "final_norm.weight": ones(H),
           "layers.0.attn.Wqkv.weight": r(3 * H, H), "layers.0.attn.Wo.weight": r(H, H), "layers.0.mlp_norm.weight": ones(H),
           "layers.0.mlp.Wi.weight": r(2 * I, H), "layers.0.mlp.Wo.weight": r(H, I)}
    stream = _cabi.Encoder(msd, arch="modernbert", max_pos=8192, sliding_window=64, layer_sliding=[1],
                           rope_theta=(160000.0, 10000.0), **common)
    return long_, stream


def profiled_attention_ms(enc, q, k, v, steps):
    enc.attention(q, k, v)                 # warm-up (and the V^T view of this shape)
    torch.cuda.synchronize()
    _cabi.profile_enable(True)
    for _ in range(steps):
        enc.attention(q, k, v)
    torch.cuda.synchronize()
    _cabi.profile_enable(False)
    return _cabi.profile_read(PROF_ATTENTION)["ms"] / steps


def sdpa_flash_ms(q, k, v, steps):
    from torch.nn.attention import SDPBackend, sdpa_kernel
    qt, kt, vt = (t.transpose(1, 2).contiguous() for t in (q, k, v))     # [B, heads, S, 64]
    f = lambda: torch.nn.functional.scaled_dot_product_attention(qt, kt, vt)
    with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
        f()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            f()
        b.record()
        torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def attention_ab(lengths, steps, reps):
    long_, stream = attention_handles()
    rows = []
    for S in lengths:
        B = TOKENS // S
        g = torch.Generator(device="cuda").manual_seed(S)
        q, k, v = (torch.randn(B, S, HEADS, DH, generator=g, device="cuda").half() for _ in range(3))
        flops = 4.0 * B * HEADS * S * S * DH
        ms = {"attention_long_kernel": [], "attention_stream_kernel": [], "sdpa_flash": []}
        for _ in range(reps):
            ms["attention_long_kernel"].append(profiled_attention_ms(long_, q, k, v, steps))
            ms["attention_stream_kernel"].append(profiled_attention_ms(stream, q, k, v, steps))
            ms["sdpa_flash"].append(sdpa_flash_ms(q, k, v, steps))
        row = {"S": S, "B": B, "flops": flops}
        for name, t in ms.items():
            row[name] = {"ms_min": min(t), "ms_max": max(t), "tflops_min": flops / max(t) * 1e-9,
                         "tflops_max": flops / min(t) * 1e-9}
        row["long_over_stream_speedup_min"] = min(ms["attention_stream_kernel"]) / max(ms["attention_long_kernel"])
        rows.append(row)
        del q, k, v
        torch.cuda.empty_cache()
    long_.close()
    stream.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lengths", default="512,1024,2048,4096,8192")
    ap.add_argument("--ab-lengths", default="1024,2048,4096,8192")
    ap.add_argument("--ab-reps", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1 or args.ab_reps < 1:
        ap.error("--steps and --ab-reps must be at least 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_xlmr_long.py: no CUDA device; the CUDA path has no CPU fallback")
    _cabi.load_library()
    model, _ = wl.bge_m3(1234)
    model = model.cuda().eval()
    enc = _cabi.Encoder.from_hf(model, max_tokens=TOKENS)
    chk = parity(enc, model)
    if not chk["ok"]:
        raise SystemExit(f"bench_xlmr_long.py: parity check against HF fp32 failed: {chk}")

    rows = []
    for S in [int(s) for s in args.lengths.split(",")]:
        B = TOKENS // S
        ids = wl.xlmr_ids(B, S, seed=7).cuda()
        ms = bench._timed_ms(torch, lambda: enc.forward_cls(ids), args.steps, warmup=args.warmup)
        _cabi.profile_enable(True)
        for _ in range(args.steps):
            enc.forward_cls(ids)
        torch.cuda.synchronize()
        _cabi.profile_enable(False)
        att, gemm = _cabi.profile_read(PROF_ATTENTION), _cabi.profile_read(PROF_GEMM_LINEAR)
        row = {"S": S, "B": B, "encoder_ms": ms, "tokens_per_s": B * S / (ms * 1e-3),
               "attention_ms": att["ms"] / args.steps, "attention_flops": att["flops"] / args.steps,
               "attention_tflops": att["flops"] / max(att["ms"], 1e-9) * 1e-9,
               "gemm_ms": gemm["ms"] / args.steps, "gemm_tflops": gemm["flops"] / max(gemm["ms"], 1e-9) * 1e-9}
        hf = hf_fp16_ms(model, ids.long(), args.steps, args.warmup)
        row["hf_eager_fp16_autocast"] = hf
        if "ms" in hf:
            row["speedup_vs_hf_fp16"] = hf["ms"] / ms
        rows.append(row)
        del ids
        torch.cuda.empty_cache()
    enc.close()
    del model
    torch.cuda.empty_cache()
    ab = attention_ab([int(s) for s in args.ab_lengths.split(",")], args.steps, args.ab_reps)

    line = {"metric": "bge-m3-shaped XLM-R encoder tokens/s at long sequence lengths", "unit": "tokens/s",
            "value": {str(r["S"]): r["tokens_per_s"] for r in rows}, "higher_is_better": True, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "dtype": "f16", "data": "synthetic",
            "config": {"workload": "bge-m3 / snowflake-arctic-embed-l-v2.0 architecture (XLM-R-large: 24 x 1024, 16 heads, I 4096, "
                                   "vocab 250002, max_position_embeddings 8194; random init seed 1234), no padding, cls_only",
                       "tokens_per_call": TOKENS},
            "parity": chk, "rows": rows, "attention_ab": ab,
            "note": (f"attention flops are algorithmic (4 x S x head_dim per query and head; the CLS-only last layer counts "
                     f"its first 128 queries); attention / gemm times are the profiled run's, encoder_ms the unprofiled one; "
                     f"HF baseline is torch {torch.__version__} eager, fp16 autocast, SDPA; the A/B times the kernel launch "
                     f"alone (library profiler) and SDPA's call (CUDA events), {args.ab_reps} alternations, min..max"),
            **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
