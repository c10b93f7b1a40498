"""The fp64 reference of the head's training arithmetic (oracle/head_ref64.py) on the CPU: it equals float64 torch
(autograd, clip_grad_norm_, AdamW) and the fp32 restatement of oracle/head_oracle.py; its derived bounds hold for the fp32
modules the reference library runs; and every named wrong rule of the kernel moves a result by at least 10x its bound, so
the GPU comparisons in tests/test_gpu_head.py under those bounds would catch it."""
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import head_oracle as ho
from oracle import head_ref64 as hr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = hr.HEAD_MATRIX


def _setup(D, C, B, loss_kind="ce", seed=0):
    p, X, y, masks = hr.make_case(D, C, B, seed=seed, loss_kind=loss_kind)
    p = hr.separate_relu(p, X, masks)
    return p, X, y, masks


def _ewc(p, C, seed=3):
    g = torch.Generator().manual_seed(seed)
    fisher = {k: torch.rand(t.shape, generator=g) for k, t in p.items()}
    star = {k: t + 0.02 * (torch.rand(t.shape, generator=g) - 0.5) for k, t in p.items()}
    return fisher, star, 50.0, max(1, C // 2)


def test_reference_equals_float64_torch_and_the_fp32_oracle():
    D, C, B = 64, 5, 12
    for loss_kind in ("ce", "bce"):
        p, X, y, masks = _setup(D, C, B, loss_kind)
        ewc = _ewc(p, C)
        r = hr.analyse(p, X, y, loss_kind, masks, ewc=ewc)
        loss, pen, g, z = hr.grads(p, X, y, loss_kind, masks, ewc=ewc)
        assert float((r["a2"][0] - z).abs().max()) < 1e-12
        for n in hr.PARAMS:
            assert float((r["grads"][n][0] - g[n]).abs().max()) < 1e-12, n
        # the optimizer: AdamW from given moments == the closed form on the reference's own clipped gradient
        m = {k: 1e-3 * torch.randn(t.shape, dtype=torch.float64) for k, t in p.items()}
        v = {k: 1e-6 * torch.rand(t.shape, dtype=torch.float64) for k, t in p.items()}
        new, mo, vo, norm, coef, _, _ = hr.optimizer_step(p, X, y, m, v, step=7, loss_kind=loss_kind, masks=masks, ewc=ewc)
        nrm = float(torch.sqrt(sum((t ** 2).sum() for t in g.values())))
        assert abs(float(norm) - nrm) < 1e-12 * nrm
        c = min(1.0, 1.0 / (nrm + 1e-6))
        for n in hr.PARAMS:
            m1 = 0.9 * m[n] + 0.1 * c * g[n]
            v1 = 0.999 * v[n] + 0.001 * (c * g[n]) ** 2
            assert float((mo[n] - m1).abs().max()) < 1e-15 and float((vo[n] - v1).abs().max()) < 1e-18, n
            assert float((new[n] - hr.adamw_update(p[n], m1, v1, 7, 1e-3, 0.01, 1e-8, 0.9, 0.999)).abs().max()) < 1e-12, n
        # oracle/head_oracle.py (explicit fp32 formulas, the kernel's): inside the bound of the fp64 reference
        _, g32, _ = ho.head_grads(X, y, p, masks, loss_kind)
        rt = hr.analyse(p, X, y, loss_kind, masks)["grads"]
        for n in hr.PARAMS:
            assert hr.worst(g32[n], *rt[n]) <= 1.0, n


@pytest.mark.parametrize("D,C,B", SHAPES)
@pytest.mark.parametrize("loss_kind", ["ce", "bce"])
def test_fp32_torch_stays_inside_the_bounds(D, C, B, loss_kind):
    """the bounds are not too tight for fp32 arithmetic: the fp32 nn modules of the reference library stay inside them"""
    p, X, y, masks = _setup(D, C, B, loss_kind)
    ewc = _ewc(p, C)
    r = hr.analyse(p, X, y, loss_kind, masks, ewc=ewc)
    loss, pen, g, z = hr.grads(p, X, y, loss_kind, masks, ewc=ewc, dtype=torch.float32)
    ratios = {"z": hr.worst(z, *r["a2"])}
    for n in hr.PARAMS:
        ratios[n] = hr.worst(g[n], *r["grads"][n])
    nrm, En = hr.norm_bound(r["grads"])
    n32 = float(torch.sqrt(sum((t.double() ** 2).sum() for t in g.values())))
    ratios["norm"] = abs(n32 - nrm) / En
    lin = hr.modules(p, torch.float32)
    with torch.no_grad():
        zf = hr.forward(lin, X)
    rf = hr.analyse(p, X, y, loss_kind, None, forward_only=True)
    ratios["softmax"] = hr.worst(torch.softmax(zf, 1), *rf["softmax"]) if loss_kind == "ce" else 0.0
    ratios["sigmoid"] = hr.worst(torch.sigmoid(zf), *rf["sigmoid"])
    print(f"fp32 torch error / bound at D={D} C={C} B={B} {loss_kind}: " + ", ".join(f"{k} {v:.1e}" for k, v in ratios.items()))
    assert max(ratios.values()) <= 1.0, ratios


def _wrong_rules(D, C, B):
    """{rule: worst |wrong - right| / bound} of every named wrong rule that changes something at this shape.  BCE with 30 %
    positive labels: its gradients do not cancel over classes (a CE head with C = 1 has no gradient at all)."""
    p, X, y, masks = _setup(D, C, B, "bce")
    r = hr.analyse(p, X, y, "bce", masks)
    g = r["grads"]
    out = {}
    if B > 1:                                  # 1/B of the full batch on a partial last batch (its first B / 4 rows)
        Bt = max(1, B // 4)
        mt = (masks[0][:Bt], masks[1][:Bt])
        rt = hr.analyse(p, X[:Bt], y[:Bt], "bce", mt)["grads"]
        gw = hr.analyse(p, X[:Bt], y[:Bt], "bce", mt, norm_rows=B)["grads"]
        out["1/B of the full batch"] = max(hr.worst(gw[n][0], rt[n][0], rt[n][1]) for n in hr.PARAMS)
    if C % 8:                                  # bias gradient without the last partial 8-row block
        wrong = g["b2"][0].clone()
        wrong[8 * (C // 8):] = 0
        out["bias gradient without the last partial block"] = hr.worst(wrong, *g["b2"])
    # layer 0 drawing its mask from layer 1's stream
    m0w = torch.from_numpy(hr.ht_mask(0.1, 5, 2 * 1 + 1, np.arange(B * D, dtype=np.uint64)).reshape(B, D))
    rw = hr.analyse(p, X, y, "bce", (m0w, masks[1]))
    out["mask of the wrong layer"] = max(hr.worst(rw["a2"][0], *r["a2"]),
                                         max(hr.worst(rw["grads"][n][0], g[n][0], g[n][1]) for n in hr.PARAMS))
    ldz = (C + 3) & ~3
    if ldz > C:                                # dz padding left nonzero and reaching the input-gradient product
        dz, _ = r["dz"]
        pad = torch.full((B, ldz - C), 1.0 / B, dtype=torch.float64)
        Wpad = torch.cat([p["W2"].double(), p["W2"].double()[torch.arange(ldz - C) % C]], 0)   # rows past C: stale ones
        dh1 = torch.cat([dz, pad], 1) @ Wpad
        a1, _ = r["a1"]
        da1 = dh1 * (a1 > 0).double() * masks[1].double()
        out["dz padding nonzero"] = hr.worst(da1, *r["da1"])
    # the bias-correction table indexed by the step instead of the launch-relative t (first step 1: bc of step 2)
    K = hr.kernel_norm_terms(D, C)
    nrm, En = hr.norm_bound(g, K)
    coef = min(1.0, 1.0 / (nrm + 1e-6))
    Ecoef = coef * (En / (nrm + 1e-6) + 3 * hr.U) if nrm + 1e-6 > 1.0 - 2 * En else 0.0
    mom = hr.moment_bounds(g, None, None, coef, Ecoef)
    ratios = []
    for n in hr.PARAMS:
        m, _, v, _ = mom[n]
        right, Eu = hr.update_bound(p[n], m, v, 1)
        bc1w, bc2w = 1 - 0.9 ** 2, (1 - 0.999 ** 2) ** 0.5
        wrong = p[n].double() * (1 - 1e-5) - 1e-3 / bc1w * m / (v.sqrt() / bc2w + 1e-8)
        ratios.append(hr.worst(wrong, right, Eu))
    out["bias correction by step"] = max(ratios)
    if C >= 2:                                 # EWC on all C rows instead of the first C_old
        ewc = _ewc(p, C)
        ge = hr.analyse(p, X, y, "bce", masks, ewc=ewc)["grads"]
        gw = hr.analyse(p, X, y, "bce", masks, ewc=(ewc[0], ewc[1], ewc[2], C))["grads"]
        out["EWC on all rows"] = max(hr.worst(gw[n][0], ge[n][0], ge[n][1]) for n in ("W2", "b2"))
    # the clip coefficient without + 1e-6 differs by 1e-6 / norm: visible where the norm is small -- here BCE with
    # negative labels at z ~ -14 (s ~ 1e-6 carries a relative, not an absolute, rounding error), max_norm below the norm
    ps = {k: t.clone() for k, t in p.items()}
    ps["W2"] = ps["W2"] * 0.1
    ps["b2"] = torch.full((C,), -14.0)
    rs = hr.analyse(ps, X, torch.zeros(B, C), "bce", masks)
    ns, Ens = hr.norm_bound(rs["grads"], K)
    c_right, c_wrong = 0.5 * ns / (ns + 1e-6), 0.5 * ns / ns
    out["clip without 1e-6"] = abs(c_wrong - c_right) / (c_right * (Ens / ns + 3 * hr.U))
    # defect 2: (s - y) / (B C) at saturated logits, against fp32 torch autograd (exact but for rounding: bound 16 u |dz|)
    zs = torch.tensor([[17.0, -28.0, -40.0, 20.0]])
    ysat = torch.tensor([[0.0, 1.0, 1.0, 0.0]])
    zz = zs.clone().requires_grad_(True)
    torch.nn.BCELoss()(torch.sigmoid(zz), ysat).backward()
    old = (torch.sigmoid(zs) - ysat) / zs.numel()
    out["BCE gradient (s - y) / (B C)"] = hr.worst(old, zz.grad, 16 * hr.U * zz.grad.abs().double())
    return out


@pytest.mark.parametrize("D,C,B", SHAPES)
def test_every_named_wrong_rule_exceeds_the_bound_tenfold(D, C, B):
    out = _wrong_rules(D, C, B)
    print(f"wrong rule / bound at D={D} C={C} B={B}: " + ", ".join(f"{k} {v:.1e}" for k, v in out.items()))
    assert min(out.values()) >= 10.0, out


def test_dropout_hash_restatement_equals_the_kernel_header():
    """the numpy restatement of ht_mask against the header compiled for the CPU, bit for bit, uint64 wraparound included"""
    src = os.path.join(tempfile.mkdtemp(prefix="ht_mask_"), "m.cpp")
    with open(src, "w") as f:
        f.write('#include "cuda_shim.h"\n#define AC_CPU_SHIM 1\nstatic inline uint8_t *shim_dyn_smem() { return nullptr; }\n'
                '#include "head_train.cuh"\n#include <cstdio>\n'
                'int main() { const unsigned long long seeds[3] = {0ull, 77ull, 0xFFFFFFFFFFFFull};\n'
                '  for (auto s : seeds) for (int st = 0; st < 6; ++st) for (unsigned long long i = 0; i < 4000; i += 7)\n'
                '    printf("%.9g\\n", ac::ht::ht_mask(0.1f, s, 2000000000ull * (st % 2) + st, i * 1000003ull)); }\n')
    exe = src[:-4]
    rc = subprocess.run(["g++", "-std=c++17", "-O1", "-I/usr/local/cuda/include", "-I" + os.path.join(ROOT, "tests", "cpu_shim"),
                         "-I" + os.path.join(ROOT, "adaptive_classifier_b200", "csrc"), src,
                         os.path.join(ROOT, "tests", "cpu_shim", "cuda_shim.cpp"), "-o", exe], capture_output=True, text=True)
    assert rc.returncode == 0, rc.stderr[-2000:]
    got = np.array(subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split(), dtype=np.float32)
    want = []
    for s in (0, 77, 0xFFFFFFFFFFFF):
        for st in range(6):
            want.append(hr.ht_mask(0.1, s, 2000000000 * (st % 2) + st, np.arange(0, 4000, 7, dtype=np.uint64) * np.uint64(1000003)))
    assert np.array_equal(got, np.concatenate(want))
