"""ORACLE (test infrastructure only): CPU fp32 restatement of stage H of the hot path.

  AdaptiveHead.forward                /root/reference/src/adaptive_classifier/models.py:71-80
     (Linear(D,D) ReLU Dropout(.1) Linear(D,D/2) ReLU Dropout(.1) Linear(D/2,C), classifier.py:1238-1247)
  head post-processing                classifier.py:435-442 (softmax + topk all classes)
  one optimizer step of the loops     classifier.py:333-351 (_train_new_classes), :1489-1505 (_train_adaptive_head):
     zero_grad, forward (train mode), CrossEntropyLoss (mean), [+ EWC penalty], backward,
     clip_grad_norm_(max_norm=1.0), AdamW(lr 1e-3, betas .9/.999, eps 1e-8, wd .01).step()
  multilabel variant                  multilabel.py:387-397 (BCELoss on sigmoid outputs)
  EWC                                 ewc.py:39-94 (Fisher), :96-115 (penalty)

The arithmetic is torch's own (third-party, importable on the GPU box as well), so the step is restated
with explicit formulas AND pinned against torch autograd + torch.optim.AdamW + clip_grad_norm_ in
tests/test_oracle_cpu.py.  Dropout masks are INPUTS (RNG parity with CPU mt19937 is impossible,
SURVEY.md section 7): mask value = 0 or 1/(1-p).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

Tensor = torch.Tensor
PARAM_ORDER = ["W0", "b0", "W1", "b1", "W2", "b2"]


def head_forward(X: Tensor, p: Dict[str, Tensor], act: str = "logits",
                 masks: Optional[Tuple[Tensor, Tensor]] = None):
    """models.py:71-80.  act in {logits, softmax, sigmoid}."""
    h0 = torch.relu(X @ p["W0"].t() + p["b0"])
    if masks is not None:
        h0 = h0 * masks[0]
    h1 = torch.relu(h0 @ p["W1"].t() + p["b1"])
    if masks is not None:
        h1 = h1 * masks[1]
    z = h1 @ p["W2"].t() + p["b2"]
    if act == "softmax":
        return torch.softmax(z, dim=1)
    if act == "sigmoid":
        return torch.sigmoid(z)
    return z


def head_grads(X: Tensor, y: Tensor, p: Dict[str, Tensor], masks: Optional[Tuple[Tensor, Tensor]],
               loss_kind: str = "ce"):
    """Explicit backward of mean CE (int64 targets) or mean BCE-on-sigmoid (float targets [B,C])."""
    B = X.shape[0]
    a0 = X @ p["W0"].t() + p["b0"]
    h0 = torch.relu(a0)
    h0d = h0 * masks[0] if masks is not None else h0
    a1 = h0d @ p["W1"].t() + p["b1"]
    h1 = torch.relu(a1)
    h1d = h1 * masks[1] if masks is not None else h1
    z = h1d @ p["W2"].t() + p["b2"]
    if loss_kind == "ce":
        logp = torch.log_softmax(z, dim=1)
        loss = -logp[torch.arange(B), y].mean()
        dz = torch.softmax(z, dim=1)
        dz[torch.arange(B), y] -= 1.0
        dz = dz / B
    else:
        # nn.BCELoss(mean over B*C) on sigmoid outputs (multilabel.py:41-44, :387-397); log clamped at -100
        s = torch.sigmoid(z)
        C = z.shape[1]
        loss = -(y * torch.log(s).clamp_min(-100) + (1 - y) * torch.log(1 - s).clamp_min(-100)).mean()
        # ATen's BCE backward, then sigmoid's backward: the gradient vanishes where s rounds to 1 or s (1 - s) < 1e-12
        dz = (s - y) / ((1 - s) * s).clamp_min(1e-12) / (B * C) * (1 - s) * s
    g = {}
    g["W2"] = dz.t() @ h1d
    g["b2"] = dz.sum(0)
    dh1 = dz @ p["W2"]
    if masks is not None:
        dh1 = dh1 * masks[1]
    da1 = dh1 * (a1 > 0).float()
    g["W1"] = da1.t() @ h0d
    g["b1"] = da1.sum(0)
    dh0 = da1 @ p["W1"]
    if masks is not None:
        dh0 = dh0 * masks[0]
    da0 = dh0 * (a0 > 0).float()
    g["W0"] = da0.t() @ X
    g["b0"] = da0.sum(0)
    return loss, g, z


def ewc_penalty(p: Dict[str, Tensor], fisher: Dict[str, Tensor], star: Dict[str, Tensor],
                lam: float, batch_size: Optional[int]):
    """ewc.py:96-115: lam * sum_n sum(F_n * (theta_n - theta*_n)^2) [/ batch_size]; gradient alongside."""
    tot = torch.zeros(())
    grads = {}
    scale = lam / (batch_size if batch_size is not None else 1.0)
    for n in PARAM_ORDER:
        diff = p[n] - star[n]
        tot = tot + (fisher[n] * diff ** 2).sum()
        grads[n] = 2.0 * scale * fisher[n] * diff
    return scale * tot, grads


def clip_and_adamw(p, g, m, v, step: int, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, wd=0.01, max_norm=1.0):
    """clip_grad_norm_ (global L2, coef = max_norm/(norm+1e-6) clamped to 1) then torch.optim.AdamW
    (decoupled weight decay first, bias-corrected moments).  `step` is the 1-based step count AFTER
    this update.  Returns total grad norm before clipping."""
    total = torch.sqrt(sum((g[n].double() ** 2).sum() for n in PARAM_ORDER)).float()
    # torch: norms per tensor in fp32 then norm of norms; difference ~1 ulp, tolerance covers it
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    bc1 = 1 - b1 ** step
    bc2 = 1 - b2 ** step
    for n in PARAM_ORDER:
        gn = g[n] * coef
        p[n].mul_(1 - lr * wd)
        m[n].mul_(b1).add_(gn, alpha=1 - b1)
        v[n].mul_(b2).addcmul_(gn, gn, value=1 - b2)
        denom = (v[n].sqrt() / (bc2 ** 0.5)).add_(eps)
        p[n].addcdiv_(m[n], denom, value=-lr / bc1)
    return total


def fisher_batch(X: Tensor, sampled: Tensor, p: Dict[str, Tensor], n_batches: int,
                 fisher: Dict[str, Tensor]):
    """ewc.py:67-92 for one batch: eval mode, loss = nll(log_softmax(f(X)), sampled) (mean),
    fisher[n] += grad^2 / n_batches.  `sampled` (the multinomial draw, ewc.py:81) is an INPUT."""
    _, g, _ = head_grads(X, sampled, p, None, "ce")
    for n in PARAM_ORDER:
        fisher[n] += g[n] ** 2 / n_batches
    return g


def init_head(D: int, C: int, seed_reset: bool = True) -> Dict[str, Tensor]:
    """models.py:43-69 via classifier.py:1238-1247: hidden [D, D//2], seeded Kaiming/Xavier, zero bias."""
    import torch.nn as nn
    p = {}
    dims = [D, D, D // 2]
    for li in range(2):
        lin = nn.Linear(dims[li], dims[li + 1])
        torch.manual_seed(42)
        nn.init.kaiming_uniform_(lin.weight, mode="fan_in", nonlinearity="relu")
        p[f"W{li}"] = lin.weight.detach().clone()
        p[f"b{li}"] = torch.zeros(dims[li + 1])
    out = nn.Linear(dims[2], C)
    torch.manual_seed(42)
    nn.init.xavier_uniform_(out.weight)
    p["W2"] = out.weight.detach().clone()
    p["b2"] = torch.zeros(C)
    return p


def epoch_permutation(gen: torch.Generator, n: int) -> Tensor:
    """The order one epoch of DataLoader(TensorDataset, shuffle=True, generator=gen) visits the rows (classifier.py:315-320,
    :1453-1459): torch's _BaseDataLoaderIter draws an int64 base seed from `gen`, RandomSampler draws randperm(n), and on
    exhaustion a second randperm(n) whose empty slice is dropped.  Pinned against a real DataLoader and against the
    reference run's recorded batches (tests/golden/golden_training.npz) in tests/test_oracle_cpu.py."""
    torch.empty((), dtype=torch.int64).random_(generator=gen)
    perm = torch.randperm(n, generator=gen)
    torch.randperm(n, generator=gen)
    return perm


def train_loop(X: Tensor, Y: Tensor, p: Dict[str, Tensor], *, epochs: int, batch_size: int, use_scheduler: bool,
               loss_kind: str = "ce", batches: Optional[List[List[int]]] = None):
    """The reference's optimizer loops with dropout as identity: _train_adaptive_head (classifier.py:1453-1520: epochs 10,
    batch min(32, n), ReduceLROnPlateau(min, factor .5, patience 2, rel threshold 1e-4), early stop patience 3),
    _train_new_classes (:306-365: epochs 15, batch 32, no scheduler, EWC term == 0) and the multilabel BCE loop
    (multilabel.py:360-411: no scheduler).  `batches` (a flat list of index lists) overrides the generator-derived order.
    Updates `p` in place; returns (per-step losses, per-step grad norms, steps per epoch)."""
    n = X.shape[0]
    m = {k: torch.zeros_like(v) for k, v in p.items()}
    v = {k: torch.zeros_like(t) for k, t in p.items()}
    gen = torch.Generator().manual_seed(42)
    lr, step = 1e-3, 0
    best, bad_epochs = float("inf"), 0
    sched_best, sched_bad = float("inf"), 0
    losses, gnorms, per_epoch = [], [], []
    cursor = 0
    n_batches = (n + batch_size - 1) // batch_size
    for _epoch in range(epochs):
        if batches is None:
            perm = epoch_permutation(gen, n).tolist()
            todo = [perm[i:i + batch_size] for i in range(0, n, batch_size)]
        else:
            todo = batches[cursor:cursor + n_batches]
            cursor += n_batches
        total = 0.0
        for idx in todo:
            xb, yb = X[idx], Y[idx]
            loss, g, _ = head_grads(xb, yb, p, None, loss_kind)
            step += 1
            gn = clip_and_adamw(p, g, m, v, step, lr=lr)
            losses.append(float(loss))
            gnorms.append(float(gn))
            total += float(loss)
        per_epoch.append(len(todo))
        avg = total / len(todo)
        if use_scheduler:                   # torch ReduceLROnPlateau: is_better = a < best * (1 - 1e-4)
            if avg < sched_best * (1 - 1e-4):
                sched_best, sched_bad = avg, 0
            else:
                sched_bad += 1
            if sched_bad > 2:
                lr, sched_bad = lr * 0.5, 0
        if avg < best:
            best, bad_epochs = avg, 0
        else:
            bad_epochs += 1
            if bad_epochs >= 3:
                break
    return losses, gnorms, per_epoch
