"""Per-projection time of the encoder GEMMs at the flagship shape (bert-base, seed 1234, B = 512, S = 128).

Part 1: Encoder.forward_cls under torch.profiler (CUDA activities, a run of its own); every gemm_tc_kernel launch is
assigned to QKV / Wo / FFN1 / FFN2 by its position in the layer's sequence (Wo and FFN2 are the same instantiation), the
launches after the last full layer to the CLS tail.  Per projection: ms per layer, TFLOP/s, algorithmic bytes and GB/s,
the larger of the compute and memory floors at data-sheet rates and which one binds.
Part 2 (control): the same four shapes through linear_tc(epi=0, out_half=True), the lightest epilogue, timed with CUDA
events; fused - plain is the serialised epilogue cost per projection.
Prints one JSON document (GPU name, power limit and clocks included).  usage: python tools/bench_encoder_gemms.py [--reps R]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

PEAK_TFLOPS, PEAK_GBS = 989.0, 3350.0          # H100 SXM data sheet, dense fp16; HBM3
B, S, H, I = 512, 128, 768, 3072
T = B * S
# (N, K, algorithmic HBM bytes: operands + outputs + epilogue operands, one pass)
PROJ = {
    "QKV": (3 * H, H, 2 * T * H + 2 * 3 * H * H + 2 * T * 3 * H + 8 * T),
    "Wo": (H, H, 2 * T * H + 2 * H * H + 4 * T * H * 2 + 2 * T * H + 8 * T * 2),
    "FFN1": (I, H, 2 * T * H + 2 * I * H + 2 * T * I + 8 * T),
    "FFN2": (H, I, 2 * T * I + 2 * H * I + 4 * T * H * 2 + 2 * T * H + 8 * T * 2),
}
ORDER = ["QKV", "Wo", "FFN1", "FFN2"]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    from adaptive_classifier_b200 import _cabi
    from oracle import encoder_oracle as eo
    _cabi.load_library()
    sd, cfg, _ = eo.make_bert_state_dict(1234)
    L = cfg.num_hidden_layers
    enc = _cabi.Encoder(sd, arch="bert", layers=L, hidden=H, heads=12, intermediate=I, vocab=cfg.vocab_size,
                        max_pos=512, type_vocab=2, ln_eps=cfg.layer_norm_eps, max_tokens=T)
    ids = eo.synthetic_ids(B, S).to(torch.int32).cuda()
    for _ in range(3):
        enc.forward_cls(ids)
    torch.cuda.synchronize()

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            enc.forward_cls(ids)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "gemm_tc_kernel" in e.name),
                key=lambda e: e.time_range.start)
    per_fwd = len(ev) // args.reps
    us = {k: 0.0 for k in ORDER}
    tail_us = 0.0
    for j, e in enumerate(ev):
        pos = j % per_fwd
        dur = e.time_range.end - e.time_range.start
        if pos < 4 * (L - 1):
            us[ORDER[pos % 4]] += dur
        else:
            tail_us += dur
    full_layers = args.reps * (L - 1)

    # control: the same shapes with the plain fp16 epilogue
    plain = {}
    for name in ORDER:
        N, K, _ = PROJ[name]
        X = torch.randn(T, K, device="cuda").half()
        W = (torch.randn(N, K, device="cuda") * K ** -0.5).half()
        bias = torch.zeros(N, device="cuda")
        for _ in range(3):
            _cabi.linear_tc(X, W, bias, epi=0, out_half=True)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        t0.record()
        for _ in range(n):
            _cabi.linear_tc(X, W, bias, epi=0, out_half=True)
        t1.record()
        torch.cuda.synchronize()
        plain[name] = t0.elapsed_time(t1) / n
        del X, W

    rows = {}
    for name in ORDER:
        N, K, nbytes = PROJ[name]
        ms = us[name] / full_layers / 1e3
        flop = 2.0 * T * N * K
        f_c, f_m = flop / (PEAK_TFLOPS * 1e12) * 1e3, nbytes / (PEAK_GBS * 1e9) * 1e3
        rows[name] = {"ms_per_layer": ms, "tflops": flop / ms / 1e9, "alg_bytes": nbytes, "gbs": nbytes / ms / 1e6,
                      "floor_ms": max(f_c, f_m), "bound": "tensor" if f_c >= f_m else "hbm",
                      "plain_epi_ms": plain[name], "fused_minus_plain_ms": ms - plain[name]}
    out = {"gpu": gpu_info(), "shape": f"bert-base B={B} S={S} T={T}", "full_layers_timed": full_layers,
           "gemm_launches_per_forward": per_fwd, "projections": rows,
           "layer_ms": sum(r["ms_per_layer"] for r in rows.values()),
           "cls_tail_ms_per_forward": tail_us / args.reps / 1e3,
           "peak_source": "H100 SXM data sheet (989 TFLOP/s dense fp16, 3.35 TB/s); floors are not measurements"}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
