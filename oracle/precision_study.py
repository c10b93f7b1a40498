"""ORACLE-side study (test infrastructure): which tensor-core operand format keeps stage E inside the
north_star tolerance (distances / logits within 1e-3 of the fp32 CPU path)?

Emulates operand rounding of every GEMM (QKV/out/FFN projections, QK^T, PV) with fp32 accumulation:
  bf16      : one tensor-core f16-kind pass, bf16 operands
  tf32      : one tensor-core tf32 pass (hardware truncates fp32 operands to 10 mantissa bits)
  bf16x3    : split a = a_hi + a_lo (both bf16); a_hi*b_hi + a_hi*b_lo + a_lo*b_hi  (3 passes)
Reports max/mean |delta| on the unit CLS rows and the induced error on squared-L2 distances
to random unit prototypes.  Result table is pasted into DESIGN.md.
"""
import sys
import time

import torch

sys.path.insert(0, __file__.rsplit("/", 2)[0])
from oracle.encoder_oracle import (encoder_forward_cls, make_bert_state_dict, round_bf16,  # noqa: E402
                                   synthetic_ids, trunc_tf32, round_tf32)


def mm_bf16x3(a, bt):
    ah = round_bf16(a); al = round_bf16(a - ah)
    bh = round_bf16(bt); bl = round_bf16(bt - bh)
    return ah @ bh.t() + ah @ bl.t() + al @ bh.t()


def mm_bf16x2(a, bt):
    # activations split, weights bf16
    ah = round_bf16(a); al = round_bf16(a - ah)
    bh = round_bf16(bt)
    return ah @ bh.t() + al @ bh.t()


def main():
    torch.set_num_threads(8)
    B, S = 8, 128
    sd, cfg, hf = make_bert_state_dict(1234)
    ids = synthetic_ids(B, S)
    t0 = time.time()
    ref = encoder_forward_cls(sd, ids, None)
    print(f"fp32 oracle forward {time.time()-t0:.1f}s")
    with torch.no_grad():
        hf_out = hf(input_ids=ids, attention_mask=torch.ones_like(ids)).last_hidden_state[:, 0, :]
        hf_unit = torch.nn.functional.normalize(hf_out, p=2, dim=1)
    print("oracle vs HF max abs", (ref - hf_unit).abs().max().item())

    g = torch.Generator().manual_seed(0)
    P = torch.nn.functional.normalize(torch.randn(4096, 768, generator=g), dim=1)

    def dist(q):
        return ((q[:, None, :] - P[None, :, :]) ** 2).sum(-1)

    d_ref = dist(ref)
    rows = []
    variants = {
        "bf16": dict(round_fn=round_bf16),
        "tf32_trunc": dict(round_fn=trunc_tf32),
        "tf32_rne": dict(round_fn=round_tf32),
    }
    for name, kw in variants.items():
        out = encoder_forward_cls(sd, ids, None, **kw)
        e = (out - ref)
        rows.append((name, e.abs().max().item(), e.norm(dim=1).max().item(), (dist(out) - d_ref).abs().max().item()))
        print(rows[-1], flush=True)
    # split variants: only linear layers via mm; attention matmuls stay fp32 in this emulation
    for name, mm in (("bf16x3(linear only)", mm_bf16x3), ("bf16x2act(linear only)", mm_bf16x2)):
        out = encoder_forward_cls(sd, ids, None, mm=mm)
        e = (out - ref)
        rows.append((name, e.abs().max().item(), e.norm(dim=1).max().item(), (dist(out) - d_ref).abs().max().item()))
        print(rows[-1], flush=True)
    print("\n| operand format | max |dq_i| | max ||dq||_2 | max |d(dist)| |")
    for r in rows:
        print(f"| {r[0]} | {r[1]:.2e} | {r[2]:.2e} | {r[3]:.2e} |")


if __name__ == "__main__":
    main()
