#!/usr/bin/env python
"""DeBERTa-v3 (deberta-v3-base shape) on the CUDA path: encoder time against HF eager and against a RoBERTa encoder of the
same shape through this library, and the attention kernel's share of the difference.

    python tools/bench_deberta.py [--steps K] [--warmup W]

- `encoder`: stage E (ids -> unit CLS rows) of workload.deberta_base (seeded random-init DebertaV2Model, 12 x 768, 12 heads
  of 64, I 3072, vocab 128100, 256 position buckets) at 65,536 tokens per call (S = 128: B = 512; S = 384: B = 170, 65,280
  tokens).  Beside it: HF DebertaV2Model in torch eager (fp32 without tf32, fp16 autocast) on the same GPU and a
  RobertaModel of identical shape (no relative terms) through this library.  Ids are uniform in [3, 128100) with [CLS] = 1
  first and [SEP] = 2 last, no padding.  The DeBERTa output is checked against the fp32 CPU oracle on 4 sequences before
  the timed region.
- `attention`: the library profiler's attention time per layer for DeBERTa and RoBERTa (same shapes): their difference is
  the cost of the c2p and p2c terms.
Prints one JSON line with the GPU's name and power limit; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (the timing helper; importing runs nothing)
from adaptive_classifier_b200 import _cabi, workload as wl  # noqa: E402
from oracle import deberta_oracle as do  # noqa: E402  (the checker, outside every timed region)
from tools.bench_minilm import gpu_info  # noqa: E402
from tools.bench_mpnet import attention_us_per_layer  # noqa: E402

TOKENS = 65536
SEQS = (128, 384)


def deberta_ids(B, S, vocab, seed=7):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (B, S), generator=g, dtype=torch.int64)
    ids[:, 0], ids[:, -1] = 1, 2
    return ids.to(torch.int32)


def roberta_same_shape(cfg):
    from transformers import RobertaConfig, RobertaModel
    torch.manual_seed(1234)
    rc = RobertaConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers,
                       num_attention_heads=cfg.num_attention_heads, intermediate_size=cfg.intermediate_size,
                       max_position_embeddings=cfg.max_position_embeddings + 2, type_vocab_size=1,
                       layer_norm_eps=cfg.layer_norm_eps, pad_token_id=1)
    return RobertaModel(rc, add_pooling_layer=False).eval()


def hf_ms(model, ids):
    ids = ids.long()
    mask = torch.ones_like(ids)

    def fwd():
        with torch.no_grad():
            return torch.nn.functional.normalize(model(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)

    def fwd16():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return model(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :]
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"hf_eager_fp32_ms": bench._timed_ms(torch, fwd, 3, warmup=1)}
    torch.backends.cuda.matmul.allow_tf32 = prev
    out["hf_eager_fp16_autocast_ms"] = bench._timed_ms(torch, fwd16, 5, warmup=2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_deberta.py: no CUDA device; the CUDA path has no CPU fallback")
    _cabi.load_library()
    dev = torch.device("cuda", 0)
    model, cfg = wl.deberta_base(1234)
    rob = roberta_same_shape(cfg)
    enc = _cabi.Encoder.from_hf(model, max_tokens=TOKENS, device=dev)
    enc_r = _cabi.Encoder.from_hf(rob, max_tokens=TOKENS, device=dev)

    encoder, attention, parity = {}, {}, {}
    sd = {k: v.detach().float() for k, v in model.state_dict().items()}
    for S in SEQS:
        B = TOKENS // S
        ids = deberta_ids(B, S, cfg.vocab_size).to(dev)
        out = enc.forward_cls(ids).cpu()
        ref = do.deberta_forward_cls(sd, ids[:4].long().cpu(), None, cfg)
        err = (out[:4] - ref).norm(dim=1).max().item()
        if not err < 1e-3:
            raise SystemExit(f"bench_deberta.py: S={S} CLS rows differ from the oracle by {err:.3g}")
        parity[f"S{S}"] = {"max_row_l2_vs_oracle": err, "rows_checked": 4}
        db_ms = bench._timed_ms(torch, lambda: enc.forward_cls(ids), args.steps, warmup=args.warmup)
        rb_ms = bench._timed_ms(torch, lambda: enc_r.forward_cls(ids), args.steps, warmup=args.warmup)
        db_att, rb_att = attention_us_per_layer(enc, ids), attention_us_per_layer(enc_r, ids)
        encoder[f"S{S}"] = {"B": B, "tokens": B * S, "this_deberta_ms": db_ms, "this_roberta_same_shape_ms": rb_ms,
                            "deberta_over_roberta": db_ms / rb_ms}
        attention[f"S{S}"] = {"deberta_us_per_layer": db_att, "roberta_us_per_layer": rb_att,
                              "c2p_p2c_overhead_us_per_layer": db_att - rb_att, "c2p_p2c_overhead_rel": db_att / rb_att - 1.0}
    enc.close()
    enc_r.close()
    del enc_r, rob
    torch.cuda.empty_cache()

    model = model.to(dev).eval()
    for S in SEQS:
        B = TOKENS // S
        try:
            hf = hf_ms(model, deberta_ids(B, S, cfg.vocab_size).to(dev))
        except Exception as ex:          # a context number must never take the measurement down
            hf = {"failed": repr(ex)}
        e = encoder[f"S{S}"]
        e.update(hf)
        if "hf_eager_fp16_autocast_ms" in hf:
            e["speedup_vs_hf_fp16_autocast"] = hf["hf_eager_fp16_autocast_ms"] / e["this_deberta_ms"]
            e["speedup_vs_hf_fp32"] = hf["hf_eager_fp32_ms"] / e["this_deberta_ms"]

    line = {"metric": "ms per 65,536-token encoder call, deberta-v3-base shape, S=128", "value": encoder["S128"]["this_deberta_ms"],
            "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "higher_is_better": False,
            "dtype": "f16", "data": "synthetic",
            "config": {"workload": "deberta-v3-base architecture (DebertaV2Model 12 x 768, 12 heads of 64, I 3072, vocab "
                                   "128100, 256 position buckets, share_att_key; random init seed 1234)",
                       "encoder_tokens_per_call": TOKENS},
            "encoder": encoder, "attention": attention, "parity": parity,
            "note": f"HF baselines: torch {torch.__version__} eager (cuBLAS / library kernels)",
            **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
