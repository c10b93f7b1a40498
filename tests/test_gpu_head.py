"""The adaptive head's kernels (csrc/head.cu forward, csrc/head_train.cuh training) against the fp64 reference of
oracle/head_ref64.py under its derived bounds, at every encoder width (128 .. 1024), class counts from 1 to 960 and batches
across the 32-row lane and 8-row block boundaries; the launch plans these shapes take; epochs equal to the same steps one
by one, bit for bit; the kernel's own dropout masks; BCE at saturated logits; and 1024-wide classifiers end to end.
Each comparison reports its largest error as a fraction of the bound (run with -s)."""
import tempfile

import numpy as np
import pytest
import torch

from oracle import head_ref64 as hr

pytestmark = pytest.mark.gpu
U = hr.U
OLD_RED_BYTES = 8 * 64 * 8 * 4          # the product partials had their own 16 KB before they shared the ring
PLAN_LIMIT = 220 * 1024


def _dev(p):
    return {k: v.clone().cuda().contiguous() for k, v in p.items()}


def _report(section, shape, ratios):
    print(f"[{section}] {shape}: " + ", ".join(f"{k} {v:.2e}" for k, v in ratios.items()))
    assert max(ratios.values()) <= 1.0, (section, shape, ratios)


def _case(D, C, B, loss_kind="ce", seed=0, masks=True):
    p, X, y, mk = hr.make_case(D, C, B, seed=seed, loss_kind=loss_kind, p_drop=0.1 if masks else 0.0)
    return hr.separate_relu(p, X, mk), X, y, mk


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------ plans
def test_the_shape_matrix_runs_every_plan_branch(cabi):
    sms = _sms()
    seen = []
    for D, C, B in hr.HEAD_MATRIX:
        p, _, _, _ = hr.make_case(D, C, 1, p_drop=0.0)
        pl = cabi.head_train_plan(_dev(p), B)
        items = -(-D // 8) + -(-(D // 2) // 8) + -(-C // 8)
        pl["slots"] = -(-items // pl["ctas"])
        pl["shared_ring"] = pl["smem_bytes"] + OLD_RED_BYTES > PLAN_LIMIT
        seen.append(pl)
        print(f"D={D} C={C} batch={B}: {pl}")
    assert {s["moments_resident"] for s in seen} == {0, 1}
    assert any(s["stages"] == 2 for s in seen) and any(s["stages"] >= 4 for s in seen)
    assert {s["slots"] for s in seen} == {1, 2}
    assert any(s["ctas"] < sms for s in seen) and any(s["ctas"] == sms for s in seen)
    assert any(s["shared_ring"] for s in seen)


def test_heads_that_need_three_slots_are_refused_with_shape_and_bytes(cabi):
    p, _, _, _ = hr.make_case(768, 1000, 1, p_drop=0.0)
    with pytest.raises(cabi.AdaptiveB200Error) as e:
        cabi.head_train_plan(_dev(p), 32)
    msg = str(e.value)
    assert "768 -> 768 -> 384 -> 1000" in msg and "bytes" in msg, msg


# ------------------------------------------------------------------------------------------------------------ 1. forward
@pytest.mark.parametrize("D", [768, 1024])
@pytest.mark.parametrize("C", [1, 3, 65, 1000, 4096])
def test_forward_logits_softmax_sigmoid(cabi, D, C):
    for B in (1, 31, 32, 33, 64, 65, 512):
        p, X, y, _ = _case(D, C, B, masks=False)
        r = hr.analyse(p, X, None, "ce", None, forward_only=True)
        pg, Xg = _dev(p), X.cuda()
        got = {name: cabi.head_forward(Xg, pg, act).cpu() for name, act in
               (("logits", cabi.AC_ACT_LOGITS), ("softmax", cabi.AC_ACT_SOFTMAX), ("sigmoid", cabi.AC_ACT_SIGMOID))}
        _report("forward", (D, C, B), {"logits": hr.worst(got["logits"], *r["a2"]), "softmax": hr.worst(got["softmax"], *r["softmax"]),
                                       "sigmoid": hr.worst(got["sigmoid"], *r["sigmoid"])})


# ------------------------------------------------------------------------------------------------------------ 2. gradients
def _loss_bound(r, loss, loss_kind, B, C):
    """CE: per row 2 max_j E_z (the row's lse and z_y) + expf / logf / sum roundings 4 u (|lse| + 1) + gamma_C; BCE: per
    element E_s / s or E_s / (1 - s) + 2 u |log|; then the mean over rows (gamma_B)"""
    z, Ez = r["a2"]
    if loss_kind == "ce":
        lse = torch.logsumexp(z, 1)
        per = 2 * Ez.max(1).values + 4 * U * (lse.abs() + 1) + hr.gamma(C)
    else:
        s, Es = r["sigmoid"]
        per = ((Es / s + Es / (1 - s)) + 2 * U * (torch.log(s).abs() + torch.log1p(-s).abs()) + hr.gamma(C)).mean(1)
    return float(per.mean()) + hr.gamma(B + 1) * abs(loss)


@pytest.mark.parametrize("D,C,B", hr.HEAD_MATRIX)
@pytest.mark.parametrize("loss_kind", ["ce", "bce"])
def test_gradients_loss_and_fisher(cabi, D, C, B, loss_kind):
    p, X, y, _ = _case(D, C, B, loss_kind, masks=False)
    r = hr.analyse(p, X, y, loss_kind, None)
    loss64, _, _, _ = hr.grads(p, X, y, loss_kind)
    pg = _dev(p)
    g = {k: torch.zeros_like(v) for k, v in pg.items()}
    q0 = {k: torch.full_like(v, 0.25) for k, v in pg.items()}
    q = {k: v.clone() for k, v in q0.items()}
    loss = cabi.head_grad(X.cuda(), y.cuda(), pg, loss_kind=cabi.AC_LOSS_CE if loss_kind == "ce" else cabi.AC_LOSS_BCE,
                          grad_out=g, fisher=q, inv_n_batches=0.5)
    ratios = {"loss": abs(float(loss) - float(loss64)) / _loss_bound(r, float(loss64), loss_kind, B, C)}
    for n in hr.PARAMS:
        gv, E = r["grads"][n]
        ratios[n] = hr.worst(g[n].cpu(), gv, E)
        # q = 0.25 + 0.5 g^2: the square, the scale, the add (3 u) and the propagated bound of g
        Eq = 0.5 * (2 * gv.abs() * E + E * E) + 3 * U * (0.25 + 0.5 * gv * gv)
        ratios["F" + n] = hr.worst(q[n].cpu(), 0.25 + 0.5 * gv * gv, Eq)
    _report("grad", (D, C, B, loss_kind), ratios)


# ------------------------------------------------------------------------------------------------------------ 3. AdamW step
def _moments(p, seed):
    g = torch.Generator().manual_seed(seed)
    m = {k: 1e-3 * torch.randn(t.shape, generator=g) for k, t in p.items()}
    v = {k: 1e-6 * torch.rand(t.shape, generator=g) for k, t in p.items()}
    return m, v


def _check_step(cabi, section, shape, p, X, y, loss_kind, masks, step, ewc=None, inject=True, seed=0):
    """one head_train_step from nonzero moments; masks: the dropout masks of the reference, handed to the kernel (inject)
    or drawn by it from `seed`"""
    D, C, B = shape[:3]
    m0, v0 = _moments(p, 11)
    pg, mg, vg = _dev(p), _dev(m0), _dev(v0)
    ewc_g = None
    if ewc is not None:
        ewc_g = (_dev(ewc[0]), _dev(ewc[1]), ewc[2], ewc[3])
    st = cabi.head_train_step(X.cuda(), y.cuda(), pg, mg, vg, step=step,
                              loss_kind=cabi.AC_LOSS_CE if loss_kind == "ce" else cabi.AC_LOSS_BCE,
                              masks=(masks[0].cuda(), masks[1].cuda()) if inject else None, seed=seed, dropout_p=0.1,
                              ewc=ewc_g).cpu()
    r = hr.analyse(p, X, y, loss_kind, masks, ewc=ewc)
    nrm, En = hr.norm_bound(r["grads"], hr.kernel_norm_terms(D, C, _sms()))
    coef = min(1.0, 1.0 / (nrm + 1e-6))
    Ecoef = coef * (En / (nrm + 1e-6) + 3 * U) if nrm + 1e-6 > 1.0 - 2 * En else 0.0
    mom = hr.moment_bounds(r["grads"], m0, v0, coef, Ecoef)
    ratios = {"norm": hr.worst(torch.tensor([float(st[2])]), torch.tensor([nrm]), torch.tensor([En]))}
    for n in hr.PARAMS:
        m, Em, v, Ev = mom[n]
        ratios["m" + n] = hr.worst(mg[n].cpu(), m, Em)
        ratios["v" + n] = hr.worst(vg[n].cpu(), v, Ev)
        new, Eu = hr.update_bound(p[n], mg[n].cpu(), vg[n].cpu(), step)
        ratios["p" + n] = hr.worst(pg[n].cpu(), new, Eu)
    if ewc is not None:
        fisher, star, lam, C_old = ewc
        K = hr.kernel_norm_terms(D, C, _sms())
        terms = 0.0
        for n in hr.PARAMS:
            rows = C_old if n in ("W2", "b2") else p[n].shape[0]
            d = p[n][:rows].double() - star[n][:rows].double()
            terms += float((fisher[n][:rows].double() * d * d).sum())
        pen = lam / B * terms
        ratios["penalty"] = abs(float(st[1]) - pen) / ((hr.gamma(K) + 4 * U) * pen + 2 * U * pen)
    _report(section, shape, ratios)


@pytest.mark.parametrize("D,C,B", hr.HEAD_MATRIX)
def test_one_adamw_step_with_injected_masks(cabi, D, C, B):
    for loss_kind in ("ce", "bce"):
        p, X, y, masks = _case(D, C, B, loss_kind)
        _check_step(cabi, "adamw", (D, C, B, loss_kind), p, X, y, loss_kind, masks, step=3)


# ------------------------------------------------------------------------------------------------------------ 5. EWC
@pytest.mark.parametrize("D,C,B", [(128, 13, 7), (384, 130, 33), (768, 20, 32), (1024, 576, 32), (1024, 3, 16)])
def test_ewc_inside_a_training_step_on_a_grown_head(cabi, D, C, B):
    p, X, y, masks = _case(D, C, B)
    g = torch.Generator().manual_seed(3)
    fisher = {k: torch.rand(t.shape, generator=g) for k, t in p.items()}
    star = {k: t + 0.02 * (torch.rand(t.shape, generator=g) - 0.5) for k, t in p.items()}
    _check_step(cabi, "ewc", (D, C, B), p, X, y, "ce", masks, step=2, ewc=(fisher, star, 50.0, max(1, C // 2)))


# ------------------------------------------------------------------------------------------------------------ 6. dropout
@pytest.mark.parametrize("D,C,B", [(128, 3, 7), (768, 20, 32), (1024, 576, 32), (1024, 13, 33)])
def test_in_kernel_dropout_masks_are_the_restated_hash(cabi, D, C, B):
    seed, step = 1234, 5
    p, X, y, _ = hr.make_case(D, C, B, p_drop=0.0)
    masks = hr.kernel_masks(0.1, seed, step, B, D, D // 2)
    p = hr.separate_relu(p, X, masks)
    _check_step(cabi, "dropout", (D, C, B), p, X, y, "ce", masks, step=step, inject=False, seed=seed)


def test_dropout_keep_fraction_and_stream_independence():
    n = 1 << 20
    idx = np.arange(n, dtype=np.uint64)
    draws = {(st, l): hr.ht_mask(0.1, 99, 2 * st + l, idx) > 0 for st in (1, 2) for l in (0, 1)}
    sigma = (0.9 * 0.1 / n) ** 0.5
    for k, keep in draws.items():
        assert abs(keep.mean() - 0.9) < 5 * sigma, (k, keep.mean())
    keys = list(draws)
    for i in range(len(keys)):
        for j in range(i + 1, len(keys)):
            agree = (draws[keys[i]] == draws[keys[j]]).mean()       # independent streams: 0.82 +- 5 sigma
            assert abs(agree - 0.82) < 5 * (0.82 * 0.18 / n) ** 0.5, (keys[i], keys[j], agree)


# ------------------------------------------------------------------------------------------------------------ 4. epochs
@pytest.mark.parametrize("D,C,n,batch,first_step", [(1024, 576, 32 * 3 + 5, 32, 1), (1024, 13, 32 * 2 + 5, 32, 1000),
                                                    (128, 3, 300, 1, 1), (384, 130, 64 + 5, 16, 1000)])
def test_epoch_equals_the_same_steps_one_by_one_bit_for_bit(cabi, D, C, n, batch, first_step):
    g = torch.Generator().manual_seed(n)
    p, _, _, _ = hr.make_case(D, C, 1, p_drop=0.0)
    X = torch.nn.functional.normalize(torch.randn(n, D, generator=g), dim=1).cuda()
    y = torch.randint(0, C, (n,), generator=g).cuda()
    perm = torch.randperm(n, generator=g)
    pa = _dev(p)
    pb = {k: v.clone() for k, v in pa.items()}
    ma, va = ({k: torch.zeros_like(v) for k, v in pa.items()} for _ in range(2))
    mb, vb = ({k: torch.zeros_like(v) for k, v in pb.items()} for _ in range(2))
    steps = -(-n // batch)
    stats = torch.zeros((steps, 3), device="cuda")
    _, nb = cabi.head_train_epoch(X, y, perm, pa, ma, va, first_step=first_step, batch=batch, seed=77, step_stats=stats)
    assert nb == steps
    for b in range(nb):
        idx = perm[b * batch:(b + 1) * batch].cuda()
        st = cabi.head_train_step(X[idx].contiguous(), y[idx].contiguous(), pb, mb, vb, step=first_step + b, seed=77)
        assert torch.equal(st[:3].cpu(), stats[b].cpu()), b
    for k in pa:
        assert torch.equal(pa[k], pb[k]) and torch.equal(ma[k], mb[k]) and torch.equal(va[k], vb[k]), k


# ------------------------------------------------------------------------------------------------------------ 7. BCE saturated
def test_bce_gradient_at_saturated_logits_equals_torch_autograd(cabi):
    """B = 1 and W2 = 0: the logits are b2 exactly and gb2 is dz.  Logits stay 0.05 away from where fp32 rounds s to 1
    (z ~ 16.6) and where s (1 - s) crosses 1e-12 (z ~ -27.6): there expf and torch's CPU sigmoid may round apart."""
    z = torch.tensor([17.0, -17.0, 20.0, -20.0, -28.0, -40.0, -90.0, 2.0])
    C = z.numel()
    for y in (torch.ones(1, C), torch.zeros(1, C), torch.tensor([[0, 1, 0, 1, 1, 1, 1, 0]], dtype=torch.float32)):
        p, X, _, _ = hr.make_case(64, C, 1, p_drop=0.0)
        p["W2"] = torch.zeros(C, 32)
        p["b2"] = z.clone()
        zz = z.clone().unsqueeze(0).requires_grad_(True)
        torch.nn.BCELoss()(torch.sigmoid(zz), y).backward()
        pg = _dev(p)
        g = {k: torch.zeros_like(v) for k, v in pg.items()}
        cabi.head_grad(X.cuda(), y.cuda(), pg, loss_kind=cabi.AC_LOSS_BCE, grad_out=g)
        want = zz.grad[0]
        got = g["b2"].cpu()
        _report("bce-saturated", tuple(y[0].int().tolist()), {"dz": hr.worst(got, want, 16 * U * want.abs().double())})


# ------------------------------------------------------------------------------------------------------------ 8. classifiers
@pytest.fixture(scope="module")
def wide_ckpt():
    """a seeded 1-layer BERT with 1024 hidden units and a small word vocabulary"""
    from transformers import BertConfig, BertModel, BertTokenizerFast
    torch.manual_seed(0)
    words = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + [f"w{i}" for i in range(200)]
    cfg = BertConfig(vocab_size=len(words), hidden_size=1024, num_hidden_layers=1, num_attention_heads=16, intermediate_size=4096,
                     max_position_embeddings=64, type_vocab_size=2, pad_token_id=0)
    d = tempfile.mkdtemp(prefix="wide_ckpt_")
    BertModel(cfg).eval().save_pretrained(d)
    BertTokenizerFast(vocab={w: i for i, w in enumerate(words)}, do_lower_case=True).save_pretrained(d)
    return d


def _texts(n, label, seed):
    rng = np.random.default_rng(seed)
    base = 50 * label
    return [" ".join(f"w{base + int(rng.integers(0, 50))}" for _ in range(8)) for _ in range(n)]


def test_1024_wide_classifiers_train_predict_save_load(cabi, wide_ckpt):
    import adaptive_classifier_b200 as acb
    texts = sum((_texts(12, k, k) for k in range(3)), [])
    labels = sum(([f"l{k}"] * 12 for k in range(3)), [])
    for config in (None, {"enable_strategic_mode": True, "cost_coefficients": [0.1] * 1024}):
        np.random.seed(0)
        clf = acb.AdaptiveClassifier(wide_ckpt, device="cuda", config=config)
        clf.add_examples(texts, labels)                      # 36 examples: batch 32 on a 1024-wide head
        clf.add_examples(_texts(8, 3, 9), ["l3"] * 8)        # a new label: EWC Fisher pass, grown head
        pred = clf.predict(texts[0], k=2)
        assert len(pred) == 2 and all(np.isfinite(s) for _, s in pred)
        d = tempfile.mkdtemp(prefix="wide_save_")
        clf.save(d)
        clf2 = acb.AdaptiveClassifier.load(d, device="cuda")
        assert [l for l, _ in clf2.predict(texts[0], k=2)] == [l for l, _ in pred]
    ml = acb.MultiLabelAdaptiveClassifier(wide_ckpt, device="cuda", min_predictions=1)
    ml.add_examples(texts, [[l, "x"] if i % 3 == 0 else [l] for i, l in enumerate(labels)])
    ml.add_examples(_texts(6, 3, 9), [["l3"]] * 6)
    out = ml.predict_multilabel(texts[0])
    assert len(out) >= 1 and all(0.0 <= s <= 1.0 for _, s in out)
    d = tempfile.mkdtemp(prefix="wide_ml_")
    ml.save(d)
    ml2 = acb.MultiLabelAdaptiveClassifier.load(d, device="cuda")
    assert len(ml2.predict_multilabel(texts[0])) >= 1
