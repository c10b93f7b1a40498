"""CPU restatement of strategic mode (reference strategic.py:74-123, :200-242; classifier.py:1602-1647) for the tests.

best_response() evaluates the 50-candidate utilities of every row in fp64 (and fp32) with full head forwards -- no rank-1
shortcut -- and returns the first-argmax choice together with the MARGIN between the best and the second-best fp64 utility,
so that a test can tell a real disagreement from a near-tie.  strategic_step() is one optimizer step of the reference's
strategic training with torch autograd (dropout off).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

N_CAND = 50


def candidates(x: torch.Tensor) -> torch.Tensor:
    """[B, D] fp32 -> [B, 50, D] fp32: x, then x_i += delta (fp32) for i = 0..3 x 10 deltas and i = 4 x the first 9."""
    deltas = torch.linspace(-2.0, 2.0, 10)
    B, D = x.shape
    out = x[:, None, :].repeat(1, N_CAND, 1).clone()
    c = 1
    for i in range(5):
        for j in range(10):
            if c == N_CAND:
                break
            out[:, c, i] = x[:, i] + deltas[j]
            c += 1
    return out


def head_forward(p: dict, X: torch.Tensor, dtype=torch.float64) -> torch.Tensor:
    g = {k: v.detach().to("cpu", dtype) for k, v in p.items()}
    h = torch.relu(X.to(dtype) @ g["W0"].T + g["b0"])
    h = torch.relu(h @ g["W1"].T + g["b1"])
    return h @ g["W2"].T + g["b2"]


def costs(x: torch.Tensor, cand: torch.Tensor, kind: int, c1: torch.Tensor, c2: torch.Tensor, dtype) -> torch.Tensor:
    """[B, 50] cost of every candidate.  kind 0 linear relu(c1 . (y - x)), 1 separable relu(c2 . y - c1 . x); the move
    y - x is taken from the fp32 candidate, as in the reference."""
    diff = (cand - x[:, None, :]).to(dtype)
    if kind == 0:
        return torch.relu(diff @ c1.to(dtype))
    return torch.relu(cand.to(dtype) @ c2.to(dtype) - (x.to(dtype) @ c1.to(dtype))[:, None])


def utilities(p: dict, x: torch.Tensor, kind: int, c1, c2, dtype=torch.float64) -> torch.Tensor:
    x = x.detach().to("cpu", torch.float32)
    cand = candidates(x)
    B, NC, D = cand.shape
    logits = head_forward(p, cand.reshape(B * NC, D), dtype).reshape(B, NC, -1)
    prob = torch.softmax(logits, dim=-1).max(dim=-1).values
    return prob - costs(x, cand, kind, c1.cpu(), c2.cpu(), dtype)


def best_response(p: dict, x: torch.Tensor, kind: int, c1, c2):
    """-> dict(choice [B] first argmax of the fp64 utilities, util64 [B, 50], util32 [B, 50], margin [B] best minus second
    best fp64 utility, rows [B, D] fp32 chosen candidates)."""
    u64 = utilities(p, x, kind, c1, c2, torch.float64)
    u32 = utilities(p, x, kind, c1, c2, torch.float32)
    choice = torch.argmax(u64, dim=1)            # the first maximum
    top2 = torch.topk(u64, 2, dim=1).values
    cand = candidates(x.detach().to("cpu", torch.float32))
    rows = cand[torch.arange(x.shape[0]), choice]
    return dict(choice=choice, util64=u64, util32=u32, margin=top2[:, 0] - top2[:, 1], rows=rows)


def strategic_loss(p: dict, X: torch.Tensor, y: torch.Tensor, br: torch.Tensor, lam: float) -> torch.Tensor:
    """strategic.py:218-242 for a batch whose best responses are given: CE_mean(X) + lam / B * sum of CE(br_i) over the rows
    whose first argmax differs from y_i (fp32, autograd through p)."""
    def fwd(Z):
        h = torch.relu(Z @ p["W0"].T + p["b0"])
        h = torch.relu(h @ p["W1"].T + p["b1"])
        return h @ p["W2"].T + p["b2"]
    loss = F.cross_entropy(fwd(X), y)
    out = fwd(br)
    wrong = torch.argmax(out, dim=-1) != y
    extra = F.cross_entropy(out, y, reduction="none")[wrong].sum() / X.shape[0] if bool(wrong.any()) else out.sum() * 0.0
    return loss + lam * extra


def strategic_training(p: dict, X: torch.Tensor, y: torch.Tensor, perms: torch.Tensor, kind: int, c1, c2, *, lr: float,
                       lam: float, steps: int = None):
    """The reference's _strategic_training_step with dropout off on CPU fp32: returns (losses, grad norms, final params).
    perms: [epochs * n] batch orders; steps: stop after this many steps (None = all)."""
    P = {k: v.detach().to("cpu", torch.float32).clone().requires_grad_(True) for k, v in p.items()}
    order = ["W0", "b0", "W1", "b1", "W2", "b2"]
    opt = torch.optim.AdamW([P[k] for k in order], lr=lr, weight_decay=0.01)
    X = X.detach().to("cpu", torch.float32)
    y = y.detach().to("cpu")
    n = X.shape[0]
    batch = min(16, n)
    losses, norms = [], []
    for e in range(perms.numel() // n):
        perm = perms[e * n:(e + 1) * n]
        for off in range(0, n, batch):
            if steps is not None and len(losses) == steps:
                return losses, norms, P
            idx = perm[off:off + batch]
            xb, yb = X[idx], y[idx]
            br = best_response({k: v.detach() for k, v in P.items()}, xb, kind, c1, c2)["rows"]
            opt.zero_grad()
            loss = strategic_loss(P, xb, yb, br, lam)
            loss.backward()
            norms.append(float(torch.nn.utils.clip_grad_norm_([P[k] for k in order], max_norm=1.0)))
            opt.step()
            losses.append(float(loss))
    return losses, norms, P
