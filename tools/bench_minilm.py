#!/usr/bin/env python
"""queries/sec of the predict() step of bench.py with an all-MiniLM-L6-v2-shaped encoder instead of bert-base.

    python tools/bench_minilm.py [--steps K] [--warmup W]

Same step as bench.py's default workload (512 x 128-token queries, 1000 classes, k = 5, E -> K -> H -> blend through
ac_pipeline_predict_device) at the embedding width of the small sentence encoders: a seeded random-init BertModel of the
all-MiniLM-L6-v2 shape (6 x 384, 12 heads of 32, I 1536, vocab 30522) and 1M x 384 fp32 prototypes.  Ids are bench.py's
(uniform in [1000, 30522), [CLS] = 101 first, [SEP] = 102 last).  Before the timed region the kNN result of 16 queries of
the step is checked against the CPU oracle (`parity`).  After it, `gpu_library_baseline` times the same HF BertModel in
torch eager on the same GPU, beside this library's encoder alone.  Prints one JSON line with the GPU's name and power
limit; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (the step's constants and timing helper; importing runs nothing)
from adaptive_classifier_b200 import _cabi, workload as wl  # noqa: E402
from adaptive_classifier_b200.models import AdaptiveHead  # noqa: E402
from oracle import knn_oracle as ko  # noqa: E402  (the checker, outside every timed region)

B, S, N, C, K = bench.B_PER_GPU, bench.S, bench.N_ROWS, bench.C, bench.K_TOP
MINILM_L6 = dict(hidden_size=384, num_attention_heads=12, intermediate_size=1536, num_hidden_layers=6)
D = MINILM_L6["hidden_size"]


def encoder_gflop_per_seq(S, H=D, I=MINILM_L6["intermediate_size"], L=MINILM_L6["num_hidden_layers"]):
    """algorithmic work of one S-token sequence: QKV, output and FFN linears (2 flops per MAC) plus QK^T and PV"""
    linears = 2.0 * S * (4 * H * H + 2 * H * I)
    attention = 4.0 * S * S * H
    return L * linears * 1e-9, L * attention * 1e-9


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit": q[1], "sm_clock_max": q[2]}
    except Exception as ex:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({ex!r})"}


def hf_baseline(ids_dev, enc_ms):
    """the reference's encoder call (HF BertModel, torch eager) on the same ids, fp32 / tf32 / fp16 autocast"""
    model, _ = wl.bert_base_state_dict(1234, **MINILM_L6)
    model = model.cuda().eval()
    ids = ids_dev.long()
    mask = torch.ones_like(ids)
    out = {}

    def fwd():
        with torch.no_grad():
            return torch.nn.functional.normalize(model(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    out["hf_eager_fp32_ms"] = bench._timed_ms(torch, fwd, 3, warmup=1)
    torch.backends.cuda.matmul.allow_tf32 = True
    out["hf_eager_tf32_ms"] = bench._timed_ms(torch, fwd, 5, warmup=2)
    torch.backends.cuda.matmul.allow_tf32 = prev

    def fwd16():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return model(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :]
    out["hf_eager_fp16_autocast_ms"] = bench._timed_ms(torch, fwd16, 5, warmup=2)
    out["this_encoder_ms"] = enc_ms
    out["queries_per_s"] = {k[:-3]: ids.shape[0] / (v * 1e-3) for k, v in out.items() if k.endswith("_ms")}
    out["note"] = (f"stage E only (ids -> unit CLS rows) at B = {B} x S = {S}; cuBLAS / SDPA library kernels of torch "
                   f"{torch.__version__}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_minilm.py: no CUDA device; the CUDA path has no CPU fallback")
    _cabi.load_library()
    dev = torch.device("cuda", 0)
    model, _ = wl.bert_base_state_dict(1234, **MINILM_L6)
    enc = _cabi.Encoder.from_hf(model, max_tokens=B * S, device=dev)
    del model
    P = wl.synthetic_rows(0, N, D, C, seed=0, device=dev)
    p_sqnorm, p_half = _cabi.row_sqnorm(P), _cabi.knn_make_shadow(P)
    row_class = (torch.arange(N, device=dev) % C).to(torch.int32)
    hp = AdaptiveHead(D, C, hidden_dims=[D, D // 2]).to(dev).eval()._param_dict()
    ids_dev = wl.synthetic_ids(B, S, seed=7).to(dev)
    pipe = _cabi.Pipeline(enc, P, B, S, K, head=hp, row_class=row_class, p_sqnorm=p_sqnorm, p_half=p_half)

    for _ in range(max(args.warmup, 1)):
        oc, osc = pipe.predict_device(ids_dev)
    torch.cuda.synchronize()
    assert oc.shape == (B, K) and bool((osc[:, 0] > 0).all()) and bool((oc[:, 0] >= 0).all())
    emb, kd, ki = pipe.debug_views(B)
    nchk = 16
    d_ref, i_ref = ko.knn_l2(emb[:nchk].cpu().numpy(), P.cpu().numpy(), K)
    ok = bool(np.array_equal(ki[:nchk].cpu().numpy(), i_ref) and np.array_equal(kd[:nchk].cpu().numpy(), d_ref))
    if not ok:
        raise SystemExit("bench_minilm.py: kNN parity check failed")

    ms = bench._timed_ms(torch, lambda: pipe.predict_device(ids_dev), args.steps, warmup=0)
    enc_ms = bench._timed_ms(torch, lambda: enc.forward_cls(ids_dev), 5)
    lin, att = encoder_gflop_per_seq(S)
    line = {"metric": "queries/sec predict() all-MiniLM-L6-v2 shape 128-tok, 1M x 384 prototypes", "value": B / (ms * 1e-3),
            "unit": "queries/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms,
            "higher_is_better": True, "dtype": "f16", "data": "synthetic",
            "config": {"workload": "all-MiniLM-L6-v2 architecture (BertModel 6 x 384, 12 heads of 32, I 1536, vocab 30522; "
                                   "random init seed 1234), S=128, batch 512, 1M x 384 fp32 prototypes, 1000 classes, k=5",
                       "global_batch": B, "seq_len": S, "prototypes": N},
            "encoder": {"ms": enc_ms, "gflop_per_seq_linears": lin, "gflop_per_seq_attention": att,
                        "achieved_tflops": B * (lin + att) / (enc_ms * 1e-3) * 1e-3,
                        "note": "algorithmic flops of all 6 layers on every token; the last layer runs its output projection "
                                "and FFN on the CLS rows only, so the kernels do less than this"},
            "parity": {"parity_checked": True, "knn_top5_equals_oracle": ok, "queries_checked": nchk},
            **gpu_info()}
    del pipe, P, p_half, p_sqnorm
    torch.cuda.empty_cache()
    try:
        line["gpu_library_baseline"] = hf_baseline(ids_dev, enc_ms)
    except Exception as ex:          # a context number must never take the headline down
        line["gpu_library_baseline"] = {"failed": repr(ex)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
