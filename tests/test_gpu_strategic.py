"""GPU tests of strategic mode: the best-response kernel (csrc/strategic.cu) and the strategic training call against the CPU
oracle (oracle/strategic_oracle.py), and the classifier's strategic API end to end on the tiny golden BERT checkpoint."""
import json
import logging
import os
import tempfile

import numpy as np
import pytest
import torch

import golden_npz
from oracle import strategic_oracle as so

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24


def _head(D, H0, H1, C, seed=0, dev="cuda"):
    g = torch.Generator().manual_seed(seed)
    p = {"W0": torch.randn(H0, D, generator=g) * (2.0 / D) ** 0.5, "b0": torch.randn(H0, generator=g) * 0.1,
         "W1": torch.randn(H1, H0, generator=g) * (2.0 / H0) ** 0.5, "b1": torch.randn(H1, generator=g) * 0.1,
         "W2": torch.randn(C, H1, generator=g) * (6.0 / H1) ** 0.5, "b2": torch.randn(C, generator=g) * 0.1}
    return {k: v.to(dev).contiguous() for k, v in p.items()}


def _tau(p, x, kind, c1, c2):
    """Per query, a bound on the fp32 error of any candidate's utility.  Each head layer is a K-term fp32 dot: its error is
    at most K u sum |w| |a| (u = 2^-24), and those errors add through the layers; the bound uses the fp64 absolute-value forward
    |W2| (|W1| (|W0| |y| + |b0|) + |b1|) + |b2| with K = D + H0 + H1 + 8 for the three dots, the rank-1 update and the softmax.
    A logit error e moves max softmax by at most e / 2 per logit of a two-sided change: 2 e bounds it.  The separable cost adds
    the error of two D-term dots; the linear cost is exact."""
    g = {k: v.detach().cpu().double().abs() for k, v in p.items()}
    cand = so.candidates(x.detach().cpu().float()).double().abs()
    B, NC, D = cand.shape
    h = cand.reshape(B * NC, D) @ g["W0"].T + g["b0"]
    h = h @ g["W1"].T + g["b1"]
    z = h @ g["W2"].T + g["b2"]
    K = D + g["W0"].shape[0] + g["W1"].shape[0] + 8
    e = (2 * K * U32 * z.max(dim=1).values).reshape(B, NC)
    if kind == 1:
        e = e + 2 * D * U32 * (cand @ c2.detach().cpu().double().abs() + (x.detach().cpu().double().abs() @ c1.detach().cpu().double().abs())[:, None])
    return e.max(dim=1).values


def _check_against_oracle(cabi, p, x, kind, c1, c2):
    choice, util, Y = cabi.strategic_best_response(x, p, kind, c1, c2)
    ref = so.best_response(p, x, kind, c1, c2)
    tau = _tau(p, x, kind, c1, c2)
    ch = choice.cpu().long()
    u64 = ref["util64"]
    B = x.shape[0]
    clear = ref["margin"] > 2 * tau
    assert torch.equal(ch[clear], ref["choice"][clear])
    # near-ties: the kernel's pick is within the error bound of the oracle's maximum
    got = u64[torch.arange(B), ch]
    assert bool(((u64.max(dim=1).values - got) <= 2 * tau).all())
    assert bool(((util.cpu().double() - got).abs() <= tau).all())
    # the chosen row is x with x_i + delta, bit for bit
    cand = so.candidates(x.cpu().float())
    assert torch.equal(Y.cpu(), cand[torch.arange(B), ch])
    return ch, ref


@pytest.mark.parametrize("shape,B,C,kind", [
    ((32, 32, 16), 1, 1, 0), ((32, 32, 16), 16, 2, 1), ((32, 32, 16), 513, 21, 0), ((32, 32, 16), 16, 1000, 1),
    ((768, 768, 384), 1, 21, 1), ((768, 768, 384), 16, 21, 0), ((768, 768, 384), 513, 2, 1), ((768, 768, 384), 16, 1000, 0),
])
def test_best_response_matches_the_oracle(cabi, shape, B, C, kind):
    D, H0, H1 = shape
    p = _head(D, H0, H1, C, seed=B + C)
    g = torch.Generator().manual_seed(7)
    x = torch.nn.functional.normalize(torch.randn(B, D, generator=g), dim=1).cuda()
    c1 = (torch.randn(D, generator=g) * 0.05).cuda()
    c1[::7] = 0.0                                          # zeros and negatives among the coefficients
    c2 = c1 if kind == 0 else c1 + (torch.randn(D, generator=g) * 0.01).cuda()
    ch, ref = _check_against_oracle(cabi, p, x, kind, c1, c2)
    if C > 1:
        assert bool((ch != 0).any())                       # the inputs exercise moves, not only candidate 0


def test_exact_ties_choose_candidate_zero(cabi):
    p = _head(32, 32, 16, 5, seed=3)
    p["W0"][:, :5] = 0.0                                   # no candidate changes the head's output
    x = torch.nn.functional.normalize(torch.randn(9, 32), dim=1).cuda()
    alpha = torch.zeros(32, device="cuda")
    for kind in (0, 1):
        choice, util, Y = cabi.strategic_best_response(x, p, kind, alpha, alpha)
        assert choice.tolist() == [0] * 9
        assert torch.equal(Y, x)


def test_a_single_cheap_coordinate_wins(cabi):
    D = 8
    p = {k: torch.zeros(s, device="cuda") for k, s in (("W0", (4, D)), ("b0", (4,)), ("W1", (4, 4)), ("b1", (4,)),
                                                      ("W2", (2, 4)), ("b2", (2,)))}
    p["W0"][0, 2], p["W0"][1, 2] = 1.0, -1.0               # h0 = (relu(x2), relu(-x2))
    p["W1"][0, 0], p["W1"][1, 1] = 1.0, 1.0
    p["W2"][0, 0], p["W2"][1, 1] = 5.0, 5.0                # max softmax = sigmoid(5 |x2|): grows with |x2|
    alpha = torch.full((D,), 10.0, device="cuda")
    alpha[2] = 0.0                                         # moving x2 is free
    x = torch.zeros(3, D, device="cuda")
    x[:, 2] = torch.tensor([0.1, -0.1, 0.0])
    choice, util, Y = cabi.strategic_best_response(x, p, 0, alpha, alpha)
    # x2 = 0.1: +2 gives |2.1| (candidate 1 + 10*2 + 9); x2 = -0.1: -2 gives |-2.1| (candidate 21); x2 = 0: -2 comes first
    assert choice.tolist() == [30, 21, 21]
    assert float(Y[0, 2]) == float(torch.tensor(0.1) + torch.tensor(2.0))


def test_dropout_zero_is_eval_mode_and_dropout_is_deterministic(cabi):
    p = _head(32, 32, 16, 7, seed=5)
    x = torch.nn.functional.normalize(torch.randn(40, 32), dim=1).cuda()
    alpha = torch.full((32,), 0.01, device="cuda")
    ref = cabi.strategic_best_response(x, p, 0, alpha, alpha)
    p0 = cabi.strategic_best_response(x, p, 0, alpha, alpha, dropout_p=0.0, seed=11, step=3)
    assert torch.equal(ref[0], p0[0]) and torch.equal(ref[1], p0[1])
    a = cabi.strategic_best_response(x, p, 0, alpha, alpha, dropout_p=0.5, seed=11, step=3)
    b = cabi.strategic_best_response(x, p, 0, alpha, alpha, dropout_p=0.5, seed=11, step=3)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    c = cabi.strategic_best_response(x, p, 0, alpha, alpha, dropout_p=0.5, seed=12, step=3)
    assert not torch.equal(a[1], c[1])


def test_bad_shapes_are_refused(cabi):
    x = torch.zeros(2, 4, device="cuda")
    p = _head(4, 4, 4, 2)
    with pytest.raises(cabi.AdaptiveB200Error, match="D >= 5"):
        cabi.strategic_best_response(x, p, 0, torch.zeros(4, device="cuda"))
    p = _head(10, 8, 8, 2)
    with pytest.raises(cabi.AdaptiveB200Error, match="multiples of 4"):
        cabi.strategic_best_response(torch.zeros(2, 10, device="cuda"), p, 0, torch.zeros(10, device="cuda"))


@pytest.mark.parametrize("kind,n,C,lam", [(0, 40, 5, 0.1), (1, 21, 3, 0.5), (0, 7, 2, 1.0)])
def test_strategic_training_matches_the_oracle(cabi, kind, n, C, lam):
    D, H0, H1 = 32, 32, 16
    p = _head(D, H0, H1, C, seed=n)
    g = torch.Generator().manual_seed(n)
    X = torch.nn.functional.normalize(torch.randn(n, D, generator=g), dim=1) * 1.3
    y = torch.randint(0, C, (n,), generator=g)
    c1 = torch.randn(D, generator=g) * 0.02
    c2 = c1 if kind == 0 else c1 * 0.5
    gen = torch.Generator().manual_seed(42)
    from adaptive_classifier_b200.classifier import dataloader_epoch_permutation
    perms = torch.cat([dataloader_epoch_permutation(gen, n) for _ in range(5)])
    losses, norms, P = so.strategic_training(p, X, y, perms, kind, c1, c2, lr=5e-4, lam=lam)
    m = {k: torch.zeros_like(v) for k, v in p.items()}
    v = {k: torch.zeros_like(t) for k, t in p.items()}
    stats = cabi.head_train_strategic(X.cuda(), y.cuda(), perms, p, m, v, cost_kind=kind, c1=c1.cuda(),
                                      c2=c2.cuda(), lr=5e-4, strategic_lambda=lam, dropout_p=0.0).cpu()
    assert stats.shape[0] == len(losses)
    np.testing.assert_allclose(stats[:, 0].numpy(), np.array(losses), atol=1e-5)
    np.testing.assert_allclose(stats[:, 2].numpy(), np.array(norms), rtol=1e-4, atol=1e-6)
    for k in p:
        np.testing.assert_allclose(p[k].cpu().numpy(), P[k].detach().numpy(), atol=1e-4)


# ------------------------------------------------------------------------------------------ classifier end to end
@pytest.fixture(scope="module")
def golden():
    return golden_npz.load("golden_classifier")


@pytest.fixture(scope="module")
def ckpt_dir(golden):
    from transformers import BertConfig, BertModel, BertTokenizerFast
    d = tempfile.mkdtemp(prefix="golden_ckpt_")
    cfg = BertConfig(**{k: v for k, v in json.loads(str(golden["bert_config"])).items()
                        if k in ("vocab_size", "hidden_size", "num_hidden_layers", "num_attention_heads",
                                 "intermediate_size", "max_position_embeddings", "type_vocab_size", "pad_token_id")})
    m = BertModel(cfg)
    m.load_state_dict({k[5:]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith("bert_") and k != "bert_config"})
    m.save_pretrained(d)
    BertTokenizerFast(vocab={w: i for i, w in enumerate(golden["vocab"].tolist())}, do_lower_case=True).save_pretrained(d)
    return d


def _make(cabi, ckpt_dir, golden, config, dropout=0.0, record=None):
    """make_golden_strategic's sequence: 24 texts (regular branch), the rest (new class: incremental branch), texts[30:36]
    (regular branch again).  record: list receiving (train_steps, X, Y) of every strategic training call"""
    import adaptive_classifier_b200 as acb
    torch.manual_seed(0)
    clf = acb.AdaptiveClassifier(ckpt_dir, device="cuda", config=config)
    clf._dropout_p = dropout
    if record is not None:
        orig = clf._strategic_training_step

        def step(X, Y):
            record.append((clf.train_steps, X.detach().cpu().clone(), Y.detach().cpu().clone()))
            return orig(X, Y)
        clf._strategic_training_step = step
    texts, labels = golden["texts"].tolist(), golden["labels"].tolist()
    np.random.seed(0)
    clf.add_examples(texts[:24], labels[:24])
    clf.add_examples(texts[24:], labels[24:])
    clf.add_examples(texts[30:36], labels[30:36])
    return clf


def _gold(name):
    return np.load(os.path.join(os.path.dirname(__file__), "golden", f"golden_strategic_{name}.npz"))


def _load_head(clf, g, prefix):
    clf.adaptive_head.load_state_dict({k[len(prefix):]: torch.from_numpy(g[k]) for k in g.files if k.startswith(prefix)})


def _same(a, b, atol=1e-5):
    assert [l for l, _ in a] == [l for l, _ in b]
    np.testing.assert_allclose([s for _, s in a], [s for _, s in b], atol=atol)


def _gold_preds(g, method, names, prefix=""):
    L, S = g[f"{prefix}{method}_labels"], g[f"{prefix}{method}_scores"]
    return [[(names[l], float(s)) for l, s in zip(Lr, Sr) if l >= 0] for Lr, Sr in zip(L, S)]


@pytest.fixture(scope="module", params=["linear", "separable"])
def run(request, cabi, ckpt_dir, golden):
    g = _gold(request.param)
    rec = []
    clf = _make(cabi, ckpt_dir, golden, json.loads(str(g["config"])), record=rec)
    return request.param, g, clf, rec


def test_strategic_training_runs_where_the_reference_runs_it_on_its_data(run):
    """the frequency gate (after the regular branch only), memory-order data, embeddings as stored"""
    _, g, clf, rec = run
    assert clf.strategic_mode
    assert len(rec) == int(g["n_train_calls"])
    for i, (steps, X, Y) in enumerate(rec):
        assert steps == int(g[f"train{i}_train_steps"])
        assert torch.equal(Y, torch.from_numpy(g[f"train{i}_Y"]))
        # the rows come out of the encoder (TF32 / fp16 projections): the bound of test_embeddings_match_reference
        assert np.abs(X.numpy() - g[f"train{i}_X"]).max() < 3e-4


def test_strategic_training_step_matches_the_reference(run, cabi):
    """_strategic_training_step from the reference's head state and data: per-step losses within 1e-5, pre-clip grad norms,
    final weights within 1e-4 (lr = learning_rate / 2, batches of min(16, N), 5 epochs of the manual_seed(42) DataLoader)"""
    import adaptive_classifier_b200 as acb
    _, g, clf, _ = run
    for i in range(int(g["n_train_calls"])):
        C = g[f"train{i}_before_model.6.weight"].shape[0]
        D = clf.embedding_dim
        clf.adaptive_head = acb.AdaptiveHead(D, C, hidden_dims=[D, D // 2]).cuda()
        _load_head(clf, g, f"train{i}_before_")
        clf._strategic_training_step(torch.from_numpy(g[f"train{i}_X"]).cuda(), torch.from_numpy(g[f"train{i}_Y"]).cuda())
        st = clf.last_strategic_trace.cpu().numpy()
        np.testing.assert_allclose(st[:, 0], g[f"train{i}_loss"], atol=1e-5)
        np.testing.assert_allclose(st[:, 2], g[f"train{i}_gnorm"], rtol=1e-4, atol=1e-6)
        after = clf.adaptive_head.state_dict()
        for k in after:
            np.testing.assert_allclose(after[k].cpu().numpy(), g[f"train{i}_after_{k}"], atol=1e-4)


def test_predictions_match_the_reference(run):
    """predict (dual blend), predict_strategic, predict_robust from text with the reference's final head: same labels in the
    same order; scores within 1e-3, the bound of test_predict_matches_reference_with_the_reference_trained_head -- the
    embeddings carry the encoder's TF32 / fp16 error (up to 3e-4), which the scores inherit"""
    _, g, clf, _ = run
    _load_head(clf, g, "head_")
    names = g["label_names"].tolist()
    assert [clf.id_to_label[i] for i in range(len(names))] == names
    for method in ("predict", "predict_strategic", "predict_robust"):
        want = _gold_preds(g, method, names)
        for t, w in zip(g["test_texts"].tolist(), want):
            _same(getattr(clf, method)(t, k=3), w, atol=1e-3)


def test_best_responses_match_the_reference(run, cabi):
    """the prediction-time compute_best_response calls of the reference (final head): the kernel picks the same candidate"""
    _, g, clf, _ = run
    _load_head(clf, g, "head_")
    n_sampled = len(range(0, int(g["n_br_train"]), 7))
    x = torch.from_numpy(g["br_x"][n_sampled:]).cuda()
    cost = clf.strategic_cost_function
    choice, _, _ = cost.compute_best_response(x, clf.adaptive_head._param_dict())
    assert choice.cpu().tolist() == g["br_choice"][n_sampled:].tolist()


def test_evaluate_strategic_robustness_matches_the_reference(run):
    _, g, clf, _ = run
    _load_head(clf, g, "head_")
    torch.manual_seed(5)
    res = clf.evaluate_strategic_robustness(g["test_texts"].tolist(),
                                            ["sports", "finance", "cooking", "finance", "sports", "cooking"])
    want = json.loads(str(g["robustness"]))
    assert res.keys() == want.keys()
    for k in want:
        assert res[k] == pytest.approx(want[k], abs=1e-6)
    with pytest.raises(KeyError):
        clf.evaluate_strategic_robustness(g["test_texts"].tolist()[:2], ["sports", "finance"], gaming_levels=[0.5])


@pytest.fixture(scope="module")
def strategic_clf(run):
    return run[2]


@pytest.mark.parametrize("which", ["dict", "none"])
def test_readme_configs_give_the_reference_regular_predictions(cabi, ckpt_dir, golden, caplog, which):
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_strategic_readme.npz"))
    config = json.loads(str(g[f"{which}_config"]))
    with caplog.at_level(logging.WARNING):
        clf = _make(cabi, ckpt_dir, golden, config)
    assert clf.strategic_mode is bool(g[f"{which}_strategic_mode"]) is False
    assert clf.config.enable_strategic_mode == bool(g[f"{which}_enable_after_init"])
    assert ("feature_names required" if which == "dict" else "no cost coefficients") in caplog.text
    _load_head(clf, g, f"{which}_head_")
    names = g[f"{which}_label_names"].tolist()
    for method in ("predict", "predict_strategic", "predict_robust"):
        for t, w in zip(g[f"{which}_test_texts"].tolist(), _gold_preds(g, method, names, f"{which}_")):
            _same(getattr(clf, method)(t, k=3), w, atol=1e-3)       # encoder error, as above


def test_unknown_cost_type_disables_strategic_mode(cabi, ckpt_dir):
    import adaptive_classifier_b200 as acb
    u = acb.AdaptiveClassifier(ckpt_dir, device="cuda", config={"enable_strategic_mode": True, "cost_function_type": "cubic",
                                                               "cost_coefficients": [1.0]})
    assert not u.strategic_mode and u.config.enable_strategic_mode is False


def test_bad_coefficients_fall_back_to_regular(cabi, strategic_clf, golden, caplog):
    from adaptive_classifier_b200.strategic import LinearCostFunction
    clf = strategic_clf
    keep = clf.strategic_cost_function
    t = golden["texts"].tolist()[0]
    try:
        for bad in (LinearCostFunction([1.0] * 3), LinearCostFunction(torch.ones(clf.embedding_dim, dtype=torch.int64)),
                    LinearCostFunction(torch.ones(clf.embedding_dim, dtype=torch.float64))):
            clf.strategic_cost_function = bad
            with caplog.at_level(logging.WARNING):
                assert clf.predict_strategic(t) == clf._predict_regular(t)
                assert clf.predict_robust(t) == clf._predict_regular(t)
            assert "Falling back to regular prediction" in caplog.text
    finally:
        clf.strategic_cost_function = keep


def test_save_load_keeps_strategic_mode(cabi, strategic_clf, golden):
    import adaptive_classifier_b200 as acb
    d = tempfile.mkdtemp(prefix="strategic_save_")
    strategic_clf.save(d)
    clf2 = acb.AdaptiveClassifier.load(d, device="cuda")
    assert clf2.strategic_mode
    assert list(clf2.config.cost_coefficients) == list(strategic_clf.config.cost_coefficients)
    for t in golden["texts"].tolist()[:4]:
        _same(clf2.predict_strategic(t), strategic_clf.predict_strategic(t))


def test_predict_batch_ignores_strategic_mode(cabi, ckpt_dir, golden):
    D = json.loads(str(golden["bert_config"]))["hidden_size"]
    s = _make(cabi, ckpt_dir, golden, {"enable_strategic_mode": True, "cost_coefficients": [0.1] * D,
                                       "strategic_training_frequency": 1000})
    r = _make(cabi, ckpt_dir, golden, None)
    texts = golden["texts"].tolist()[:10]
    assert s.strategic_mode
    assert s.predict_batch(texts) == r.predict_batch(texts)


@pytest.mark.parametrize("B,C,lam,p", [(8, 5, 0.3, 0.5), (3, 2, 1.0, 0.1), (16, 21, 0.1, 0.0), (1, 3, 2.0, 0.3)])
def test_strategic_loss_kind_under_dropout_masks(cabi, B, C, lam, p):
    """one AC_LOSS_CE_STRATEGIC step with injected dropout masks against a natural-order autograd restatement: the
    mispredict check of a best-response row sees the same masks as its loss (the reference's single model(br) call)"""
    D, H0, H1 = 32, 32, 16
    P = _head(D, H0, H1, C, seed=B * 7 + C)
    g = torch.Generator().manual_seed(B + C)
    X = torch.randn(2 * B, D, generator=g)
    y = torch.randint(0, C, (B,), generator=g)
    keep = 1.0 / (1.0 - p) if p > 0 else 1.0
    m0 = (torch.rand(2 * B, H0, generator=g) >= p).float() * keep
    m1 = (torch.rand(2 * B, H1, generator=g) >= p).float() * keep
    R = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in P.items()}
    h = torch.relu(X @ R["W0"].T + R["b0"]) * m0
    h = torch.relu(h @ R["W1"].T + R["b1"]) * m1
    z = h @ R["W2"].T + R["b2"]
    loss = torch.nn.functional.cross_entropy(z[:B], y)
    wrong = z[B:].argmax(-1) != y
    if bool(wrong.any()):
        loss = loss + lam * torch.nn.functional.cross_entropy(z[B:][wrong], y[wrong], reduction="sum") / B
    opt = torch.optim.AdamW([R[k] for k in ("W0", "b0", "W1", "b1", "W2", "b2")], lr=1e-3, weight_decay=0.01)
    loss.backward()
    gn = float(torch.nn.utils.clip_grad_norm_([R[k] for k in ("W0", "b0", "W1", "b1", "W2", "b2")], 1.0))
    opt.step()
    m = {k: torch.zeros_like(v) for k, v in P.items()}
    v = {k: torch.zeros_like(t) for k, t in P.items()}
    st = cabi.head_train_step(X.cuda(), torch.cat([y, y]).cuda(), P, m, v, step=1, loss_kind=cabi.AC_LOSS_CE_STRATEGIC,
                              dropout_p=p, masks=(m0.cuda(), m1.cuda()) if p > 0 else None, n_regular=B,
                              strategic_lambda=lam).cpu()
    assert float(st[0]) == pytest.approx(float(loss), abs=1e-5)
    assert float(st[2]) == pytest.approx(gn, rel=1e-4)
    for k in P:
        np.testing.assert_allclose(P[k].cpu().numpy(), R[k].detach().numpy(), atol=1e-4)
