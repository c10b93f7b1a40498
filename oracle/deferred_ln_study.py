"""ORACLE-side study (test infrastructure): does DEFERRING every LayerNorm into its consumers keep stage E inside the
north_star tolerance?

Today (adaptive_classifier_b200/csrc/encoder.cu) every residual sum y = sublayer(x) + x is written to HBM in fp32, read
back by a LayerNorm kernel, and written again as the fp32 residual stream plus its fp16 operand copy: 905 MB per half
layer at B = 512, S = 128.  Deferred form: the residual GEMM's epilogue writes y (fp32), fp16(y) and per-row (sum, sumsq);
LayerNorm(y) = (y - mu) r gamma + beta is never materialised:

  * the next GEMM consumes fp16(y) with weights W' = fp16(gamma * W):
        LN(y) W^T + b  =  r (y W'^T - mu c1) + c0,     c1 = rowsum(W'),  c0 = W beta + b         (rank-1 correction)
  * the next residual epilogue recomputes LN(y) from the fp32 y and the row statistics on the fly.

503 MB per half layer instead of 905 MB, and no LayerNorm launches.  This script emulates that data flow with the same
fp16 operand rounding as the kernels (fp32 accumulation, variance from sum / sum of squares in fp32) and reports the error
of the unit CLS rows and of squared-L2 distances against the fp32 oracle, next to today's fp16 data flow.
"""
import math
import sys
import time

import torch

sys.path.insert(0, __file__.rsplit("/", 2)[0])
from oracle.encoder_oracle import encoder_forward_cls, make_bert_state_dict, synthetic_ids, _gelu_erf  # noqa: E402


def r16(t):
    return t.to(torch.float16).to(torch.float32)


def stats(y, eps):
    """mu and 1/sqrt(var + eps) from fp32 sum and sum of squares (what a GEMM epilogue can accumulate)."""
    H = y.shape[-1]
    s = y.sum(-1, keepdim=True, dtype=torch.float32)
    q = (y * y).sum(-1, keepdim=True, dtype=torch.float32)
    mu = s / H
    var = (q / H - mu * mu).clamp_min(0.0)
    return mu, 1.0 / torch.sqrt(var + eps)


def deferred_forward(sd, ids, num_heads=12, eps=1e-12):
    B, S = ids.shape
    pos = torch.arange(S).unsqueeze(0).expand(B, S)
    y = (sd["embeddings.word_embeddings.weight"][ids] + sd["embeddings.token_type_embeddings.weight"][torch.zeros_like(ids)])
    y = (y + sd["embeddings.position_embeddings.weight"][pos]).reshape(B * S, -1)
    H = y.shape[-1]
    dh = H // num_heads
    g, b = sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"]   # LayerNorm pending on y
    L = 0
    while f"encoder.layer.{L}.attention.self.query.weight" in sd:
        L += 1

    def lin_deferred(y, mu, r, g, b, prefix):
        W, bias = sd[prefix + ".weight"], sd[prefix + ".bias"]
        Wp = r16(W * g[None, :])                       # fp16(gamma * W), packed once at encoder_create
        c1 = Wp.sum(1)                                 # fp32 row sums of the packed weight
        c0 = W @ b + bias                              # fp32
        acc = r16(y) @ Wp.t()                          # f16 tensor-core MMA, fp32 accumulate
        return r * (acc - mu * c1[None, :]) + c0[None, :]

    def ln_on_the_fly(y, mu, r, g, b):
        return (y - mu) * r * g + b

    for l in range(L):
        p = f"encoder.layer.{l}."
        mu, r = stats(y, eps)
        q = lin_deferred(y, mu, r, g, b, p + "attention.self.query").view(B, S, num_heads, dh).transpose(1, 2)
        k = lin_deferred(y, mu, r, g, b, p + "attention.self.key").view(B, S, num_heads, dh).transpose(1, 2)
        v = lin_deferred(y, mu, r, g, b, p + "attention.self.value").view(B, S, num_heads, dh).transpose(1, 2)
        scores = (r16(q) @ r16(k).transpose(-1, -2)) * dh ** -0.5
        probs = torch.softmax(scores, dim=-1)
        ctx = (r16(probs) @ r16(v)).transpose(1, 2).reshape(B * S, H)
        a = r16(ctx) @ r16(sd[p + "attention.output.dense.weight"]).t() + sd[p + "attention.output.dense.bias"]
        y = a + ln_on_the_fly(y, mu, r, g, b)           # residual = LN(previous y), recomputed in the epilogue
        g, b = sd[p + "attention.output.LayerNorm.weight"], sd[p + "attention.output.LayerNorm.bias"]
        mu, r = stats(y, eps)
        h = _gelu_erf(lin_deferred(y, mu, r, g, b, p + "intermediate.dense"))
        o = r16(h) @ r16(sd[p + "output.dense.weight"]).t() + sd[p + "output.dense.bias"]
        y = o + ln_on_the_fly(y, mu, r, g, b)
        g, b = sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"]
    mu, r = stats(y, eps)
    x = ln_on_the_fly(y, mu, r, g, b).view(B, S, H)
    cls = x[:, 0, :]
    return cls / cls.norm(dim=1, keepdim=True).clamp_min(1e-12)


def main():
    torch.set_num_threads(8)
    B, S = 8, 128
    sd, cfg, _ = make_bert_state_dict(1234)
    # non-trivial LayerNorm parameters and a shifted residual stream: random init has gamma = 1, beta = 0, mean ~ 0, which
    # would hide the cancellation in r (acc - mu c1)
    gen = torch.Generator().manual_seed(5)
    for k_ in list(sd.keys()):
        if k_.endswith("LayerNorm.weight"):
            sd[k_] = 1.0 + 0.3 * torch.randn(sd[k_].shape, generator=gen)
        if k_.endswith("LayerNorm.bias"):
            sd[k_] = 0.2 * torch.randn(sd[k_].shape, generator=gen)
        if k_.endswith("output.dense.bias"):
            sd[k_] = sd[k_] + 0.5            # pushes the row mean of y away from 0 (|mu| / sigma ~ 0.5)
    ids = synthetic_ids(B, S)
    t0 = time.time()
    ref = encoder_forward_cls(sd, ids, None)
    print(f"fp32 oracle forward {time.time() - t0:.1f}s")
    g = torch.Generator().manual_seed(0)
    P = torch.nn.functional.normalize(torch.randn(4096, 768, generator=g), dim=1)

    def dist(q):
        return ((q[:, None, :] - P[None, :, :]) ** 2).sum(-1)

    d_ref = dist(ref)
    rows = []
    for name, out in (("fp16 operands, LayerNorm kernels (today)", encoder_forward_cls(sd, ids, None, round_fn=r16)),
                      ("fp16 operands, deferred LayerNorm", deferred_forward(sd, ids))):
        e = out - ref
        rows.append((name, e.abs().max().item(), e.norm(dim=1).max().item(), (dist(out) - d_ref).abs().max().item()))
        print(rows[-1], flush=True)
    print("\n| data flow | max |dq_i| | max ||dq||_2 | max |d(dist)| |")
    for r in rows:
        print(f"| {r[0]} | {r[1]:.2e} | {r[2]:.2e} | {r[3]:.2e} |")


if __name__ == "__main__":
    main()
