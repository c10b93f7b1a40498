#!/usr/bin/env python
"""MPNet (all-mpnet-base-v2 shape) on the CUDA path: encoder time against HF eager and against a RoBERTa encoder of the
same shape through this library, the attention kernels' share of the difference, and one predict() step.

    python tools/bench_mpnet.py [--steps K] [--warmup W]

- `encoder`: stage E (ids -> unit CLS rows) of workload.mpnet_base (seeded random-init MPNetModel, 12 x 768, 12 heads of
  64, I 3072, vocab 30527) at 65,536 tokens per call (S = 128: B = 512; S = 384, the checkpoint's max_seq_length: B = 170,
  65,280 tokens).  Beside it: HF MPNetModel in torch eager (fp32 without tf32, fp16 autocast) on the same GPU and a
  RobertaModel of identical shape (RoBERTa positions, no relative bias) through this library.  Ids are uniform in
  [1000, 30527) with <s> = 0 first and </s> = 2 last, no padding.
- `attention`: the library profiler's attention time per layer for MPNet and RoBERTa (same launches, same shapes): their
  difference is the cost of the relative position bias.
- `predict`: bench.py's step (512 x 128-token queries, 1M x 768 fp32 prototypes, 1000 classes, k = 5, E -> K -> H ->
  blend through ac_pipeline_predict_device) with the MPNet encoder; the kNN result of 16 queries is checked against the CPU
  oracle before the timed region.
Prints one JSON line with the GPU's name and power limit; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (the step's constants and timing helper; importing runs nothing)
from adaptive_classifier_b200 import _cabi, workload as wl  # noqa: E402
from adaptive_classifier_b200.models import AdaptiveHead  # noqa: E402
from oracle import knn_oracle as ko  # noqa: E402  (the checker, outside every timed region)
from tools.bench_minilm import gpu_info  # noqa: E402

TOKENS = 65536
SEQS = (128, 384)
PROF_ATTENTION = 1


def mpnet_ids(B, S, vocab, seed=7):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1000, vocab, (B, S), generator=g, dtype=torch.int64)
    ids[:, 0], ids[:, -1] = 0, 2
    return ids.to(torch.int32)


def roberta_same_shape(cfg):
    from transformers import RobertaConfig, RobertaModel
    torch.manual_seed(1234)
    rc = RobertaConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers,
                       num_attention_heads=cfg.num_attention_heads, intermediate_size=cfg.intermediate_size,
                       max_position_embeddings=cfg.max_position_embeddings, type_vocab_size=1,
                       layer_norm_eps=cfg.layer_norm_eps, pad_token_id=1)
    return RobertaModel(rc, add_pooling_layer=False).eval()


def attention_us_per_layer(enc, ids, reps=5):
    enc.forward_cls(ids)
    torch.cuda.synchronize()
    _cabi.profile_enable(True)
    for _ in range(reps):
        enc.forward_cls(ids)
    torch.cuda.synchronize()
    _cabi.profile_enable(False)
    a = _cabi.profile_read(PROF_ATTENTION)
    return 1e3 * a["ms"] / max(1, a["launches"])


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
        raise SystemExit("bench_mpnet.py: no CUDA device; the CUDA path has no CPU fallback")
    _cabi.load_library()
    dev = torch.device("cuda", 0)
    model, cfg = wl.mpnet_base(1234)
    rob = roberta_same_shape(cfg)
    D = cfg.hidden_size
    enc = _cabi.Encoder.from_hf(model, max_tokens=TOKENS, device=dev)
    enc_r = _cabi.Encoder.from_hf(rob, max_tokens=TOKENS, device=dev)

    encoder, attention = {}, {}
    for S in SEQS:
        B = TOKENS // S
        ids = mpnet_ids(B, S, cfg.vocab_size).to(dev)
        mp_ms = bench._timed_ms(torch, lambda: enc.forward_cls(ids), args.steps, warmup=args.warmup)
        rb_ms = bench._timed_ms(torch, lambda: enc_r.forward_cls(ids), args.steps, warmup=args.warmup)
        mp_att, rb_att = attention_us_per_layer(enc, ids), attention_us_per_layer(enc_r, ids)
        encoder[f"S{S}"] = {"B": B, "tokens": B * S, "this_mpnet_ms": mp_ms, "this_roberta_same_shape_ms": rb_ms,
                            "mpnet_over_roberta": mp_ms / rb_ms}
        attention[f"S{S}"] = {"mpnet_us_per_layer": mp_att, "roberta_us_per_layer": rb_att,
                              "bias_overhead_us_per_layer": mp_att - rb_att, "bias_overhead_rel": mp_att / rb_att - 1.0}
    enc_r.close()
    del enc_r, rob
    torch.cuda.empty_cache()

    # one bench.py-style predict step with the MPNet encoder
    Bq, Sq, N, C, K = bench.B_PER_GPU, bench.S, bench.N_ROWS, bench.C, bench.K_TOP
    P = wl.synthetic_rows(0, N, D, C, seed=0, device=dev)
    p_sqnorm, p_half = _cabi.row_sqnorm(P), _cabi.knn_make_shadow(P)
    row_class = (torch.arange(N, device=dev) % C).to(torch.int32)
    hp = AdaptiveHead(D, C, hidden_dims=[D, D // 2]).to(dev).eval()._param_dict()
    ids_q = mpnet_ids(Bq, Sq, cfg.vocab_size).to(dev)
    pipe = _cabi.Pipeline(enc, P, Bq, Sq, K, head=hp, row_class=row_class, p_sqnorm=p_sqnorm, p_half=p_half)
    for _ in range(max(args.warmup, 1)):
        oc, osc = pipe.predict_device(ids_q)
    torch.cuda.synchronize()
    emb, kd, ki = pipe.debug_views(Bq)
    nchk = 16
    d_ref, i_ref = ko.knn_l2(emb[:nchk].cpu().numpy(), P.cpu().numpy(), K)
    ok = bool(np.array_equal(ki[:nchk].cpu().numpy(), i_ref) and np.array_equal(kd[:nchk].cpu().numpy(), d_ref))
    if not ok:
        raise SystemExit("bench_mpnet.py: kNN parity check failed")
    step_ms = bench._timed_ms(torch, lambda: pipe.predict_device(ids_q), args.steps, warmup=0)
    del pipe, P, p_half, p_sqnorm
    torch.cuda.empty_cache()

    model = model.to(dev).eval()
    for S in SEQS:
        B = TOKENS // S
        try:
            hf = hf_ms(model, mpnet_ids(B, S, cfg.vocab_size).to(dev))
        except Exception as ex:          # a context number must never take the measurement down
            hf = {"failed": repr(ex)}
        e = encoder[f"S{S}"]
        e.update(hf)
        if "hf_eager_fp16_autocast_ms" in hf:
            e["speedup_vs_hf_fp16_autocast"] = hf["hf_eager_fp16_autocast_ms"] / e["this_mpnet_ms"]
            e["speedup_vs_hf_fp32"] = hf["hf_eager_fp32_ms"] / e["this_mpnet_ms"]

    line = {"metric": "queries/sec predict() all-mpnet-base-v2 shape 128-tok, 1M x 768 prototypes", "value": Bq / (step_ms * 1e-3),
            "unit": "queries/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": step_ms,
            "higher_is_better": True, "dtype": "f16", "data": "synthetic",
            "config": {"workload": "all-mpnet-base-v2 architecture (MPNetModel 12 x 768, 12 heads of 64, I 3072, vocab 30527, "
                                   "32 relative-attention buckets; random init seed 1234)",
                       "predict": f"S={Sq}, batch {Bq}, {N} x {D} fp32 prototypes, {C} classes, k={K}",
                       "encoder_tokens_per_call": TOKENS},
            "encoder": encoder, "attention": attention,
            "parity": {"parity_checked": True, "knn_top5_equals_oracle": ok, "queries_checked": nchk},
            "note": f"HF baselines: torch {torch.__version__} eager (cuBLAS / SDPA library kernels)",
            **gpu_info()}
    enc.close()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
