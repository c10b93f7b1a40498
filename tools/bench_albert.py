#!/usr/bin/env python
"""ALBERT and ELECTRA on the CUDA path: encoder time against a BERT of identical hidden shape through this library and
against HF eager, and the time of the two kernels these families add.

    python tools/bench_albert.py [--steps K] [--warmup W]

- `encoder`: stage E (ids -> unit CLS rows) at 65,536 tokens per call (S = 128: B = 512; S = 384: B = 170, 65,280 tokens)
  for workload.albert_base (seeded random-init AlbertModel, 12 x 768 sharing one layer, 12 heads, I 3072, E 128, vocab 30000,
  "gelu_new") and workload.electra_small (ElectraModel 12 x 256, 4 heads, I 1024, E 128, "gelu").  Beside each: a BertModel
  of the same hidden shape (E = H, erf GELU, 12 unshared layers) through this library, and the HF model itself in torch
  eager (fp32 without tf32, fp16 autocast) on the same GPU.  Ids are uniform in [1000, vocab) with [CLS] = 2 first and
  [SEP] = 3 last, no padding.  Each output is checked against the fp32 CPU oracle on 4 sequences before the timed region.
- `kernels`: from a torch.profiler run of its own (after the timed region), the average time per call of the embedding
  projection GEMM (EpiEmbProj) and of FFN1 per layer: tanh GELU (ALBERT) against erf GELU (the same-shape BERT; ELECTRA).
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
from oracle import albert_oracle as ao  # noqa: E402  (the checker, outside every timed region)
from tools.bench_deberta import hf_ms  # noqa: E402
from tools.bench_minilm import gpu_info  # noqa: E402

TOKENS = 65536
SEQS = (128, 384)
# demangled-name fragments of the kernels reported under `kernels`
KERNELS = {"emb_proj": "EpiEmbProj", "ffn1_tanh": "EpiF16<(ac::Act)4, true>", "ffn1_erf": "EpiF16<(ac::Act)1, true>"}


def ids_for(B, S, vocab, seed=7):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1000, vocab, (B, S), generator=g, dtype=torch.int64)
    ids[:, 0], ids[:, -1] = 2, 3
    return ids.to(torch.int32)


def bert_same_shape(cfg):
    from transformers import BertConfig, BertModel
    torch.manual_seed(1234)
    bc = BertConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers,
                    num_attention_heads=cfg.num_attention_heads, intermediate_size=cfg.intermediate_size,
                    max_position_embeddings=cfg.max_position_embeddings, type_vocab_size=2, hidden_act="gelu")
    return BertModel(bc, add_pooling_layer=False).eval()


def kernel_us(enc, ids, reps=5):
    """average device time per forward call of each KERNELS entry (microseconds), from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    enc.forward_cls(ids)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            enc.forward_cls(ids)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for key, frag in KERNELS.items():
            if frag in ev.key:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                out[key] = out.get(key, 0.0) + t / reps
                out[key + "_launches_per_call"] = out.get(key + "_launches_per_call", 0) + ev.count // reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_albert.py: no CUDA device; the CUDA path has no CPU fallback")
    _cabi.load_library()
    dev = torch.device("cuda", 0)
    result = {}
    for family, make in (("albert_base", wl.albert_base), ("electra_small", wl.electra_small)):
        model, cfg = make(1234)
        bert = bert_same_shape(cfg)
        enc = _cabi.Encoder.from_hf(model, max_tokens=TOKENS, device=dev)
        enc_b = _cabi.Encoder.from_hf(bert, max_tokens=TOKENS, device=dev)
        sd = {k: v.detach().float() for k, v in model.state_dict().items()}
        fam = {}
        for S in SEQS:
            B = TOKENS // S
            ids = ids_for(B, S, cfg.vocab_size).to(dev)
            out = enc.forward_cls(ids).cpu()
            ref = ao.factorized_forward_cls(sd, ids[:4].long().cpu(), None, cfg)
            err = (out[:4] - ref).norm(dim=1).max().item()
            if not err < 1e-3:
                raise SystemExit(f"bench_albert.py: {family} S={S} CLS rows differ from the oracle by {err:.3g}")
            ms = bench._timed_ms(torch, lambda: enc.forward_cls(ids), args.steps, warmup=args.warmup)
            ms_b = bench._timed_ms(torch, lambda: enc_b.forward_cls(ids), args.steps, warmup=args.warmup)
            fam[f"S{S}"] = {"B": B, "tokens": B * S, "this_ms": ms, "this_bert_same_shape_ms": ms_b, "over_bert": ms / ms_b,
                            "max_row_l2_vs_oracle": err, "rows_checked": 4}
        for S in SEQS:
            ids = ids_for(TOKENS // S, S, cfg.vocab_size).to(dev)
            fam[f"S{S}"]["kernels_us_per_call"] = kernel_us(enc, ids)
            fam[f"S{S}"]["kernels_us_per_call_bert_same_shape"] = kernel_us(enc_b, ids)
        enc.close()
        enc_b.close()
        del enc, enc_b, bert
        torch.cuda.empty_cache()
        model = model.to(dev).eval()
        for S in SEQS:
            try:
                hf = hf_ms(model, ids_for(TOKENS // S, S, cfg.vocab_size).to(dev))
            except Exception as ex:          # a context number must never take the measurement down
                hf = {"failed": repr(ex)}
            e = fam[f"S{S}"]
            e.update(hf)
            if "hf_eager_fp16_autocast_ms" in hf:
                e["speedup_vs_hf_fp16_autocast"] = hf["hf_eager_fp16_autocast_ms"] / e["this_ms"]
                e["speedup_vs_hf_fp32"] = hf["hf_eager_fp32_ms"] / e["this_ms"]
        del model
        torch.cuda.empty_cache()
        result[family] = fam

    line = {"metric": "ms per 65,536-token encoder call, albert-base-v2 shape, S=128", "value": result["albert_base"]["S128"]["this_ms"],
            "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "higher_is_better": False,
            "dtype": "f16", "data": "synthetic",
            "config": {"workloads": {"albert_base": "AlbertModel 12 x 768 sharing one layer, 12 heads, I 3072, E 128, vocab "
                                                    "30000, gelu_new; random init seed 1234",
                                     "electra_small": "ElectraModel 12 x 256, 4 heads, I 1024, E 128, vocab 30522, gelu; "
                                                      "random init seed 1234"},
                       "encoder_tokens_per_call": TOKENS},
            "encoder": result,
            "note": f"HF baselines: torch {torch.__version__} eager (cuBLAS / library kernels); kernel times from torch.profiler "
                    "in separate runs after the timed region",
            **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
