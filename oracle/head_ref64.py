"""ORACLE (test infrastructure only): an fp64 reference of the adaptive head's training arithmetic, built from torch itself,
with derived error bounds for the fp32 kernels of csrc/head.cu and csrc/head_train.cuh.

Reference: real nn.Linear modules in float64 holding the same fp32 values the kernel sees, dropout as an injected mask,
nn.CrossEntropyLoss / nn.BCELoss (+ the EWC penalty of ewc.py:96-115 on the first C_old output rows), autograd,
clip_grad_norm_ and torch.optim.AdamW.  The same step in float32 modules is what the reference library runs.

Bounds (running error analysis, first order in the unit roundoff u = 2^-24 plus the second-order cross terms): a fixed-order
fp32 sum of K products -- with or without FMA, in any order -- lies within gamma_K * sum |a_i b_i| of the exact sum, with
gamma_K = K u / (1 - K u).  Every quantity q carries an absolute bound E_q, propagated through the network together with
its magnitude:
  product   A (E_A) times B (E_B), K terms:  gamma_K (|A| + E_A)(|B| + E_B) + E_A |B| + |A| E_B + E_A E_B
  bias add  one more term in the sum (gamma_{K+1});  mask multiply  |m| E + u |h|
  ReLU      1-Lipschitz forward; backward ReLU'(a) is a step: where |a64| <= E_a either side is a correct fp32 result, so
            the bound of da there is the whole |dh m| + its bound
  softmax   p_j (E_zj + max_k E_zk + u |z_j - max z| + 2 u (expf: 2 ulp) + gamma_C + u)     (row max and sum of C terms)
  sigmoid   s (1 - s) E_z + 4 u s                 (expf 2 ulp, one add, one division)
  BCE dz    (E_s + 8 u |s - y|) / (B C)           (seven roundings; valid away from saturation, |z| < 16)
  norm      sqrt(sum E_g^2) (triangle inequality) + (gamma_K / 2 + u)(norm + that), K terms per fixed-order chain
  AdamW     m, v: 3 and 4 roundings plus the propagated E_g, E_coef; the update, given m, v, coef: 8 u (|p| + |step|)
The reference itself (fp64, error ~1e-16 relative) is treated as exact: its own error is nine orders below every bound.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

U = 2.0 ** -24
PARAMS = ["W0", "b0", "W1", "b1", "W2", "b2"]
Tensor = torch.Tensor


def gamma(K) -> float:
    return K * U / (1.0 - K * U)


# ------------------------------------------------------------------------------------------------------- dropout hash


def _mix32(x: np.ndarray) -> np.ndarray:
    """ht_mix32 (head_train.cuh) with uint64 wraparound"""
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xFF51AFD7ED558CCD)
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xC4CEB9FE1A85EC53)
        x = x ^ (x >> np.uint64(33))
    return (x & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def ht_mask(p: float, seed: int, stream: int, idx: np.ndarray) -> np.ndarray:
    """ht_mask: element idx of mask stream `stream` -> 0 or 1 / (1 - p) (fp32)"""
    with np.errstate(over="ignore"):
        x = (np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(stream) * np.uint64(0xD1B54A32D192ED03)
             + idx.astype(np.uint64))
    r = _mix32(x)
    u = (r >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    keep = np.float32(1.0) / (np.float32(1.0) - np.float32(p))
    return np.where(u < np.float32(p), np.float32(0.0), keep).astype(np.float32)


def kernel_masks(p: float, seed: int, step: int, B: int, H0: int, H1: int) -> Tuple[Tensor, Tensor]:
    """the masks head_train_kernel draws at optimizer step `step`: stream 2 step + layer, element b * rows + r"""
    out = []
    for layer, rows in ((0, H0), (1, H1)):
        idx = np.arange(B * rows, dtype=np.uint64)
        out.append(torch.from_numpy(ht_mask(p, seed, 2 * step + layer, idx).reshape(B, rows)))
    return out[0], out[1]


# ------------------------------------------------------------------------------------------------------- reference step
def modules(p: Dict[str, Tensor], dtype=torch.float64):
    lin = []
    for i in range(3):
        W = p[f"W{i}"]
        m = nn.Linear(W.shape[1], W.shape[0], dtype=dtype)
        with torch.no_grad():
            m.weight.copy_(W.to(dtype))
            m.bias.copy_(p[f"b{i}"].to(dtype))
        lin.append(m)
    return lin


def forward(lin, X: Tensor, masks=None) -> Tensor:
    dt = lin[0].weight.dtype
    h = torch.relu(lin[0](X.to(dt)))
    if masks is not None:
        h = h * masks[0].to(dt)
    h = torch.relu(lin[1](h))
    if masks is not None:
        h = h * masks[1].to(dt)
    return lin[2](h)


def task_loss(z: Tensor, y: Tensor, loss_kind: str) -> Tensor:
    if loss_kind == "ce":
        return nn.CrossEntropyLoss()(z, y)
    return nn.BCELoss()(torch.sigmoid(z), y.to(z.dtype))


def ewc_loss(lin, ewc, B: int) -> Tensor:
    """ewc.py:96-115 on a grown head: lam / B * sum F (theta - theta*)^2 over the first C_old output rows"""
    fisher, star, lam, C_old = ewc
    dt = lin[0].weight.dtype
    tot = torch.zeros((), dtype=dt)
    for i, m in enumerate(lin):
        for t, n in ((m.weight, f"W{i}"), (m.bias, f"b{i}")):
            rows = C_old if (i == 2 and 0 < C_old < t.shape[0]) else t.shape[0]
            d = t[:rows] - star[n][:rows].to(dt)
            tot = tot + (fisher[n][:rows].to(dt) * d * d).sum()
    return lam / B * tot


def grads(p, X, y, loss_kind="ce", masks=None, ewc=None, dtype=torch.float64):
    """autograd of the task loss (+ EWC) through nn modules: (task loss, penalty, {name: grad}, z)"""
    lin = modules(p, dtype)
    z = forward(lin, X, masks)
    loss = task_loss(z, y, loss_kind)
    pen = ewc_loss(lin, ewc, X.shape[0]) if ewc is not None else torch.zeros((), dtype=dtype)
    (loss + pen).backward()
    g = {}
    for i, m in enumerate(lin):
        g[f"W{i}"], g[f"b{i}"] = m.weight.grad.detach(), m.bias.grad.detach()
    return loss.detach(), pen.detach(), g, z.detach()


def optimizer_step(p, X, y, m=None, v=None, *, step, loss_kind="ce", masks=None, ewc=None, dtype=torch.float64,
                   lr=1e-3, wd=0.01, max_norm=1.0):
    """one step of the reference loop: zero_grad, forward, loss (+ EWC), backward, clip_grad_norm_, AdamW.step.
    m, v: AdamW moments entering the step (None = fresh).  Returns (params, m, v, norm, coef, task loss, penalty)."""
    lin = modules(p, dtype)
    params = [t for l in lin for t in (l.weight, l.bias)]
    opt = torch.optim.AdamW(params, lr=lr, weight_decay=wd, betas=(0.9, 0.999), eps=1e-8)
    if m is not None:
        for t, n in zip(params, PARAMS):
            opt.state[t] = {"step": torch.tensor(float(step - 1)), "exp_avg": m[n].to(dtype).clone(),
                            "exp_avg_sq": v[n].to(dtype).clone()}
    z = forward(lin, X, masks)
    loss = task_loss(z, y, loss_kind)
    pen = ewc_loss(lin, ewc, X.shape[0]) if ewc is not None else torch.zeros((), dtype=dtype)
    (loss + pen).backward()
    norm = torch.nn.utils.clip_grad_norm_(params, max_norm=max_norm)
    coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
    opt.step()
    out = {n: t.detach() for n, t in zip(PARAMS, params)}
    mo = {n: opt.state[t]["exp_avg"] for n, t in zip(PARAMS, params)}
    vo = {n: opt.state[t]["exp_avg_sq"] for n, t in zip(PARAMS, params)}
    return out, mo, vo, norm.detach(), coef.detach(), loss.detach(), pen.detach()


# the optimizer's hyperparameters as the C ABI carries them (fp32): the kernel's bias corrections 1 - beta^t are fp64 powers of
# these values -- at t = 3, 1 - beta2^t of the fp32 0.999 differs from that of the decimal 0.999 by 1.3e-5 relative
F32 = {k: float(np.float32(v)) for k, v in (("lr", 1e-3), ("wd", 0.01), ("eps", 1e-8), ("b1", 0.9), ("b2", 0.999))}


def adamw_update(p, m, v, step, lr=F32["lr"], wd=F32["wd"], eps=F32["eps"], b1=F32["b1"], b2=F32["b2"]):
    """the AdamW parameter update of `step` given its moments (fp64): p (1 - lr wd) - lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps)"""
    bc1, bc2s = 1.0 - b1 ** step, (1.0 - b2 ** step) ** 0.5
    return p.double() * (1 - lr * wd) - lr / bc1 * m.double() / (v.double().sqrt() / bc2s + eps)


# ------------------------------------------------------------------------------------------------------- bounds
def _mm(A, EA, B, EB, K):
    """A @ B with operand bounds: gamma_K (|A| + E_A)(|B| + E_B) + E_A |B| + |A| E_B + E_A E_B"""
    aA, aB = A.abs(), B.abs()
    return gamma(K) * ((aA + EA) @ (aB + EB)) + EA @ aB + aA @ EB + EA @ EB


def analyse(p, X, y, loss_kind="ce", masks=None, *, norm_rows: Optional[int] = None, ewc=None, forward_only=False):
    """Explicit fp64 forward / backward of one step with the bound of every intermediate: {name: (value, bound)}.
    norm_rows: the batch size the mean divides by (defaults to the rows of X)."""
    P = {k: t.double() for k, t in p.items()}
    X = X.double()
    B = X.shape[0]
    nb = norm_rows or B
    D, H0, H1, C = P["W0"].shape[1], P["W0"].shape[0], P["W1"].shape[0], P["W2"].shape[0]
    mk = [masks[0].double(), masks[1].double()] if masks is not None else [torch.ones(B, H0, dtype=torch.float64),
                                                                         torch.ones(B, H1, dtype=torch.float64)]
    Z = lambda *s: torch.zeros(*s, dtype=torch.float64)  # noqa: E731
    r = {}
    # forward: a = h W^T + b (K + 1 terms), h = relu(a) * mask
    h, Eh = X, Z(B, D)
    for l, (K, rows) in enumerate(((D, H0), (H0, H1), (H1, C))):
        W, b = P[f"W{l}"], P[f"b{l}"]
        a = h @ W.t() + b
        Ea = _mm(h, Eh, W.t(), Z(W.t().shape), K + 1) + gamma(K + 1) * b.abs()
        r[f"a{l}"] = (a, Ea)
        if l < 2:
            hn = torch.relu(a) * mk[l]
            r[f"h{l}"] = (hn, mk[l].abs() * Ea + U * hn.abs())
            r[f"x{l}"] = (h, Eh)
            h, Eh = r[f"h{l}"]
    r["x2"] = (h, Eh)
    z, Ez = r["a2"]
    if loss_kind == "ce":
        mx = z.max(1, keepdim=True).values
        pr = torch.softmax(z, 1)
        Ep = pr * (Ez + Ez.max(1, keepdim=True).values + U * (z - mx).abs() + 2 * U + gamma(C) + U)
        r["softmax"] = (pr, Ep)
    s = torch.sigmoid(z)
    r["sigmoid"] = (s, s * (1 - s) * Ez + 4 * U * s)
    if forward_only:
        return r
    if loss_kind == "ce":
        onehot = torch.nn.functional.one_hot(y, C).double()
        dz = (pr - onehot) / nb
        Edz = (Ep + 2 * U * (pr - onehot).abs()) / nb
    else:
        yd = y.double()
        Es = r["sigmoid"][1]
        dz = (s - yd) / (nb * C)
        Edz = (Es + 8 * U * (s - yd).abs()) / (nb * C)
    r["dz"] = (dz, Edz)
    g = {}
    d, Ed = dz, Edz
    for l in (2, 1, 0):
        hin, Ehin = r[f"x{l}"]
        g[f"W{l}"] = (d.t() @ hin, _mm(d.t(), Ed.t(), hin, Ehin, B))
        g[f"b{l}"] = (d.sum(0), gamma(B) * d.abs().sum(0) + Ed.sum(0))
        if l == 0:
            break
        W = P[f"W{l}"]
        dh = d @ W
        Edh = _mm(d, Ed, W, Z(W.shape), W.shape[0])
        a, Ea = r[f"a{l - 1}"]
        m = mk[l - 1]
        on = (a > 0).double()
        amb = (a.abs() <= Ea).double()                     # ReLU'(a) undecided at fp32 accuracy
        dn = dh * on * m
        Edn = (on * (Edh + U * dh.abs()) + amb * (dh.abs() + Edh)) * m.abs()
        r[f"da{l - 1}"] = (dn, Edn)
        d, Ed = dn, Edn
    if ewc is not None:
        fisher, star, lam, C_old = ewc
        for n in PARAMS:
            rows = C_old if (n in ("W2", "b2") and 0 < C_old < C) else P[n].shape[0]
            dl = P[n] - star[n].double()
            add = Z(P[n].shape)
            add[:rows] = 2.0 * lam / nb * fisher[n][:rows].double() * dl[:rows]
            val, E = g[n]
            # ewc2 = 2 lam / B (2 roundings), ewc2 * F, theta - theta*, the fma: 5 u |term|, plus u |g + term|
            g[n] = (val + add, E + 5 * U * add.abs() + U * (val + add).abs())
    r["grads"] = g
    return r


def norm_bound(g: Dict[str, Tuple[Tensor, Tensor]], K: Optional[int] = None):
    """(norm, bound) of the global gradient norm: | ||g^|| - ||g|| | <= ||g^ - g|| <= sqrt(sum E_g^2) (triangle inequality),
    then the sum of squares in fixed order (gamma_K relative, K terms per chain; default: all entries) and the square root
    (gamma_K / 2 + u on the norm)"""
    ss = sum((v ** 2).sum() for v, _ in g.values())
    N = sum(v.numel() for v, _ in g.values())
    eg = float(sum((E * E).sum() for _, E in g.values()).sqrt())
    nrm = float(ss.sqrt())
    return nrm, eg + (gamma(K or N) / 2 + U) * (nrm + eg)


def moment_bounds(g, m_in, v_in, coef, Ecoef, beta1=F32["b1"], beta2=F32["b2"]):
    """AdamW moments m = b1 m + (1 - b1) c g, v = b2 v + (1 - b2) (c g)^2 and their bounds"""
    out = {}
    for n, (gv, Eg) in g.items():
        m0 = m_in[n].double() if m_in is not None else torch.zeros_like(gv)
        v0 = v_in[n].double() if v_in is not None else torch.zeros_like(gv)
        cg = coef * gv
        Ecg = coef * Eg + Ecoef * gv.abs() + U * cg.abs()
        m = beta1 * m0 + (1 - beta1) * cg
        v = beta2 * v0 + (1 - beta2) * cg * cg
        Em = (1 - beta1) * Ecg + 3 * U * (beta1 * m0.abs() + (1 - beta1) * cg.abs())
        Ev = (1 - beta2) * (2 * cg.abs() * Ecg + Ecg * Ecg) + 4 * U * (beta2 * v0 + (1 - beta2) * cg * cg)
        out[n] = (m, Em, v, Ev)
    return out


def update_bound(p_in, m, v, step, lr=F32["lr"], wd=F32["wd"], eps=F32["eps"]):
    """(fp64 update evaluated on the given m, v; its bound) -- the update alone, Adam's ill-conditioning left out"""
    new = adamw_update(p_in, m, v, step, lr, wd, eps)
    st = (new - p_in.double() * (1 - lr * wd)).abs()
    return new, 8 * U * (p_in.double().abs() + st)


def worst(got: Tensor, ref: Tensor, E: Tensor) -> float:
    """max |got - ref| / E (E = 0 demands equality)"""
    d = (got.double() - ref.double()).abs()
    return float((d / E.clamp_min(1e-300)).max()) if d.numel() else 0.0


# ------------------------------------------------------------------------------------------------------- test shapes
# (D, C, batch) of the head tests: every width of the encoder families (D -> D -> D/2 -> C), class counts from one to the
# largest that trains at D = 1024 and beyond, batches across the 32-row lane boundary and the 8-row block size.  On an H100
# they cover both homes of the AdamW moments, ring depths 2 .. 8, one and two ownership slots, grids below and at the SM count,
# and the 1024-wide batch-32 heads that only fit since the product partials share the ring.
HEAD_MATRIX = [
    (128, 1, 1), (128, 3, 7), (128, 960, 33), (128, 2, 64),
    (256, 13, 16), (256, 960, 32), (256, 130, 31), (256, 1, 64),
    (384, 12, 32), (384, 130, 33), (384, 576, 7), (384, 3, 64),
    (768, 20, 32), (768, 960, 31), (768, 2, 1), (768, 576, 16), (768, 13, 33),
    (1024, 1, 32), (1024, 576, 32), (1024, 130, 31), (1024, 13, 7), (1024, 3, 33), (1024, 2, 16), (1024, 576, 1),
]


def make_case(D, C, B, seed=0, loss_kind="ce", p_drop=0.1, step=1):
    """seeded head (init_head-like scale, nonzero biases), unit-norm rows X, targets and the kernel's dropout masks"""
    g = torch.Generator().manual_seed(1000 * D + 7 * C + B + seed)
    H0, H1 = D, D // 2
    p = {}
    for i, (rows, K) in enumerate(((H0, D), (H1, H0), (C, H1))):
        bound = (6.0 / K) ** 0.5 if i < 2 else (6.0 / (K + rows)) ** 0.5
        p[f"W{i}"] = (torch.rand(rows, K, generator=g) * 2 - 1) * bound
        p[f"b{i}"] = (torch.rand(rows, generator=g) * 2 - 1) * 0.05
    X = torch.nn.functional.normalize(torch.randn(B, D, generator=g), dim=1)
    if loss_kind == "ce":
        y = torch.randint(0, C, (B,), generator=g)
    else:
        y = (torch.rand(B, C, generator=g) < 0.3).float()
    masks = kernel_masks(p_drop, 5 + seed, step, B, H0, H1) if p_drop > 0 else None
    return p, X, y, masks


def separate_relu(p, X, masks=None, margin=4.0):
    """Moves each hidden bias by the least amount that puts every pre-activation of its column more than `margin` times
    its bound away from zero.  ReLU'(a) is a step: a pre-activation inside its rounding bound may go either way in fp32 and
    take a whole gradient row with it, so comparisons against a bound need batches without such entries.  Returns a new
    parameter dict (fp32)."""
    p = {k: t.clone() for k, t in p.items()}
    for l in (0, 1):
        r = analyse(p, X, None, masks=masks, forward_only=True)
        a, Ea = r[f"a{l}"]
        b = p[f"b{l}"].double()
        need = margin * Ea + 4 * U * a.abs() + 1e-30
        for j in torch.nonzero((a.abs() <= need).any(0)).flatten().tolist():
            col, nd = a[:, j], need[:, j]
            cands = sorted(set([0.0] + (-col + 1.01 * nd).tolist() + (-col - 1.01 * nd).tolist()), key=abs)
            for dlt in cands:
                if bool(((col + dlt).abs() > nd).all()):
                    b[j] += dlt
                    break
        p[f"b{l}"] = b.float()
    return p


def kernel_norm_terms(D: int, C: int, sms: int = 132) -> int:
    """terms in the longest fixed-order chain of head_train_kernel's gradient sum of squares: per thread its float4 groups of
    each slot (and a bias), the block tree (8 levels), the lane-strided pass over the G CTA partials and the shuffle tree"""
    items = -(-D // 8) + -(-(D // 2) // 8) + -(-C // 8)
    G = min(sms, items)
    slots = -(-items // G)
    per_slot = 4 * -(-(8 * D // 4) // 256) + 1
    return slots * per_slot + 8 + -(-G // 32) + 5
