#!/usr/bin/env python
"""deberta-v3-base-shaped encoder (ids -> unit CLS rows) past 512 tokens, and its attention stage alone per layer.

    python tools/bench_deberta_long.py [--steps K] [--warmup W] [--lengths 1024,2048,8192] [--ab-reps 3]

Encoder: seeded random-init deberta-v3-base shape (workload.deberta_base: 12 x 768, 12 heads, I 3072, 256 position buckets,
no absolute positions) through Encoder.from_hf, B = 65536 / S sequences per call, no padding, cls_only.  For every S: the
encoder's time and tokens/s; the attention and GEMM times from the library's per-launch profiler in a separate run; and HF
DebertaV2Model in torch eager with fp16 autocast on the same ids, at the largest batch that fits (halving from B on an
out-of-memory error, each failure recorded).  Before any timing, the CLS rows of two sequences at S = 2048 are checked
against HF in fp32 (TF32 off) on the same GPU, bound 1e-3 on the row error; a mismatch aborts.

Attention per layer at each S on the same fp16 q, k, v (B = 65536 / S, 12 heads of 64, no mask): a one-layer DeBERTa
handle (attention_stream_kernel<64, ScoreDisent>: QK^T, c2p and p2c per tile) next to a one-layer handle of plain
attention on the same streamed kernel (attention_stream_kernel<64, ScorePlain>, a ModernBERT handle with window 0, as
RoBERTa-shaped plain attention), both timed by the library profiler (CUDA events around the launch alone), alternated
--ab-reps times, min..max.  Prints one JSON line with the GPU's name and power limit; writes nothing.
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
HEADS, DH, LAYERS = 12, 64, 12
PROF_GEMM_LINEAR, PROF_ATTENTION = 0, 1


def ids_for(B, S, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (B, S), generator=g, dtype=torch.int32)
    ids[:, 0], ids[:, -1] = 1, 2
    return ids.cuda()


def parity(enc, model, vocab, S=2048, B=2):
    ids = ids_for(B, S, vocab, 3)
    out = enc.forward_cls(ids)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            h = model(input_ids=ids.long(), attention_mask=torch.ones_like(ids, dtype=torch.long)).last_hidden_state[:, 0]
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    err = float((out - torch.nn.functional.normalize(h.float(), dim=1)).norm(dim=1).max())
    return {"S": S, "B": B, "cls_row_err_max": err, "bound": 1e-3, "ok": err < 1e-3}


def hf_fp16(model, ids, steps, warmup):
    """HF eager, fp16 autocast, at the largest batch (B, B / 2, ...) that runs; ms per call at that batch"""
    failures = []
    B = ids.shape[0]
    while B >= 1:
        x = ids[:B]

        def fwd():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
                return model(input_ids=x, attention_mask=torch.ones_like(x)).last_hidden_state[:, 0, :]
        try:
            ms = bench._timed_ms(torch, fwd, steps, warmup=warmup)
            return {"B": B, "ms": ms, "tokens_per_s": B * ids.shape[1] / (ms * 1e-3), "failed_at": failures}
        except torch.OutOfMemoryError as ex:
            failures.append({"B": B, "error": repr(ex)[:160]})
        except Exception as ex:          # a baseline failure must not take the line down
            failures.append({"B": B, "error": repr(ex)[:300]})
            break
        torch.cuda.empty_cache()
        B //= 2
    torch.cuda.empty_cache()
    return {"failed_at": failures}


def attention_handles():
    """one-layer handles that only serve Encoder.attention, 12 heads of 64: DeBERTa (deberta-v3-base position settings,
    radius-8192 index) and ModernBERT with window 0 (plain attention on the same streamed kernel)"""
    from transformers import DebertaV2Config, DebertaV2Model
    H, I, V = HEADS * DH, 64, 32
    torch.manual_seed(5)
    cfg = DebertaV2Config(vocab_size=V, hidden_size=H, num_hidden_layers=1, num_attention_heads=HEADS, intermediate_size=I,
                          max_position_embeddings=512, type_vocab_size=0, relative_attention=True, position_buckets=256,
                          norm_rel_ebd="layer_norm", share_att_key=True, pos_att_type=["p2c", "c2p"],
                          position_biased_input=False, layer_norm_eps=1e-7, hidden_act="gelu", pad_token_id=0)
    m = DebertaV2Model(cfg).eval()
    sd, dims = _cabi.deberta_to_bert_state_dict(dict(m.state_dict()), cfg)
    deb = _cabi.Encoder(sd, arch="deberta", max_tokens=TOKENS, **dims)
    g = torch.Generator().manual_seed(11)
    r = lambda *s: (0.02 * torch.randn(*s, generator=g)).cuda()
    ones = lambda n: torch.ones(n).cuda()
    msd = {"embeddings.tok_embeddings.weight": r(V, H), "embeddings.norm.weight": ones(H), "final_norm.weight": ones(H),
           "layers.0.attn.Wqkv.weight": r(3 * H, H), "layers.0.attn.Wo.weight": r(H, H), "layers.0.mlp_norm.weight": ones(H),
           "layers.0.mlp.Wi.weight": r(2 * I, H), "layers.0.mlp.Wo.weight": r(H, I)}
    plain = _cabi.Encoder(msd, arch="modernbert", layers=1, hidden=H, heads=HEADS, intermediate=I, vocab=V, ln_eps=1e-5,
                          max_tokens=TOKENS, max_pos=8192, sliding_window=64, layer_sliding=[0],
                          rope_theta=(160000.0, 10000.0))
    return deb, plain


def profiled_attention_ms(enc, q, k, v, steps):
    enc.attention(q, k, v)                 # warm-up (and the V^T view of this shape)
    torch.cuda.synchronize()
    _cabi.profile_enable(True)
    for _ in range(steps):
        enc.attention(q, k, v)
    torch.cuda.synchronize()
    _cabi.profile_enable(False)
    return _cabi.profile_read(PROF_ATTENTION)["ms"] / steps


def attention_ab(lengths, steps, reps):
    deb, plain = attention_handles()
    rows = []
    for S in lengths:
        B = TOKENS // S
        g = torch.Generator(device="cuda").manual_seed(S)
        q, k, v = (torch.randn(B, S, HEADS, DH, generator=g, device="cuda").half() for _ in range(3))
        ms = {"deberta_disentangled": [], "plain_streamed": []}
        for _ in range(reps):
            ms["deberta_disentangled"].append(profiled_attention_ms(deb, q, k, v, steps))
            ms["plain_streamed"].append(profiled_attention_ms(plain, q, k, v, steps))
        row = {"S": S, "B": B}
        for name, t in ms.items():
            row[name] = {"ms_min": min(t), "ms_max": max(t)}
        row["deberta_over_plain_min"] = min(ms["deberta_disentangled"]) / max(ms["plain_streamed"])
        row["deberta_over_plain_max"] = max(ms["deberta_disentangled"]) / min(ms["plain_streamed"])
        rows.append(row)
        del q, k, v
        torch.cuda.empty_cache()
    deb.close()
    plain.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lengths", default="1024,2048,8192")
    ap.add_argument("--ab-reps", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1 or args.ab_reps < 1:
        ap.error("--steps and --ab-reps must be at least 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_deberta_long.py: no CUDA device; the CUDA path has no CPU fallback")
    _cabi.load_library()
    lengths = [int(s) for s in args.lengths.split(",")]
    model, cfg = wl.deberta_base(1234)
    model = model.cuda().eval()
    enc = _cabi.Encoder.from_hf(model, max_tokens=TOKENS)
    chk = parity(enc, model, cfg.vocab_size)
    if not chk["ok"]:
        raise SystemExit(f"bench_deberta_long.py: parity check against HF fp32 failed: {chk}")

    rows = []
    for S in lengths:
        B = TOKENS // S
        ids = ids_for(B, S, cfg.vocab_size, 7)
        ms = bench._timed_ms(torch, lambda: enc.forward_cls(ids), args.steps, warmup=args.warmup)
        _cabi.profile_enable(True)
        for _ in range(args.steps):
            enc.forward_cls(ids)
        torch.cuda.synchronize()
        _cabi.profile_enable(False)
        att, gemm = _cabi.profile_read(PROF_ATTENTION), _cabi.profile_read(PROF_GEMM_LINEAR)
        row = {"S": S, "B": B, "encoder_ms": ms, "tokens_per_s": B * S / (ms * 1e-3),
               "attention_ms": att["ms"] / args.steps, "gemm_ms": gemm["ms"] / args.steps}
        hf = hf_fp16(model, ids.long(), args.steps, args.warmup)
        row["hf_eager_fp16_autocast"] = hf
        if "tokens_per_s" in hf:
            row["speedup_vs_hf_fp16_tokens_per_s"] = row["tokens_per_s"] / hf["tokens_per_s"]
        rows.append(row)
        del ids
        torch.cuda.empty_cache()
    enc.close()
    del model
    torch.cuda.empty_cache()
    ab = attention_ab(lengths, args.steps, args.ab_reps)

    line = {"metric": "deberta-v3-base-shaped encoder tokens/s past 512 tokens", "unit": "tokens/s",
            "value": {str(r["S"]): r["tokens_per_s"] for r in rows}, "higher_is_better": True, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "dtype": "f16", "data": "synthetic",
            "config": {"workload": "deberta-v3-base architecture (12 x 768, 12 heads, I 3072, vocab 128100, 256 position "
                                   "buckets, no absolute positions; random init seed 1234), no padding, cls_only",
                       "tokens_per_call": TOKENS},
            "parity": chk, "rows": rows, "attention_per_layer": ab,
            "note": (f"attention / gemm times are the profiled run's (every layer; the CLS-only last layer computes its "
                     f"first 128 queries), encoder_ms the unprofiled one; HF baseline is torch {torch.__version__} eager, "
                     f"fp16 autocast, at the batch recorded; attention_per_layer times one layer's launch alone (library "
                     f"profiler), {args.ab_reps} alternations, min..max"),
            **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
