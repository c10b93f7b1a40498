"""CPU tests of strategic mode's host side: the candidate table, the cost functions and their factory, and the CPU oracle
(oracle/strategic_oracle.py) the GPU tests compare against."""
import logging

import pytest
import torch

from adaptive_classifier_b200 import strategic as st
from oracle import strategic_oracle as so


def test_candidate_table_matches_the_reference_loop_and_draws_no_rng():
    torch.manual_seed(3)
    x = torch.randn(12)
    state = torch.random.get_rng_state()
    table = st.candidate_table(x)
    assert torch.equal(torch.random.get_rng_state(), state)
    # the reference's _generate_candidates (strategic.py:104-123), restated
    ref = [x]
    for i in range(len(x)):
        for delta in torch.linspace(-2.0, 2.0, 10):
            if delta == 0:
                continue
            c = x.clone()
            c[i] += delta
            ref.append(c)
    ref = torch.stack(ref[:50])
    assert table.shape == (50, 12)
    assert torch.equal(table, ref)
    assert torch.equal(so.candidates(x[None])[0], ref)
    with pytest.raises(ValueError):
        st.candidate_table(torch.zeros(4))


def test_factory_semantics():
    f = st.CostFunctionFactory.create_cost_function("linear", [0.5, 1.0])
    assert isinstance(f, st.LinearCostFunction) and f.cost_kind == 0
    f = st.CostFunctionFactory.create_cost_function("separable", [0.5, 1.0])
    assert type(f) is st.SeparableCostFunction and f.cost_kind == 1 and torch.equal(f.c1, f.c2)
    with pytest.raises(ValueError, match="feature_names required"):
        st.CostFunctionFactory.create_cost_function("separable", {"a": 1.0})
    with pytest.raises(ValueError, match="feature_names required"):
        st.CostFunctionFactory.create_cost_function("linear", {"a": 1.0})
    with pytest.raises(ValueError, match="Unknown cost function type"):
        st.CostFunctionFactory.create_cost_function("quadratic", [1.0])
    f = st.CostFunctionFactory.create_cost_function("linear", {"a": 2.0}, feature_names=["a", "b"])
    assert f.alpha.tolist() == [2.0, 0.0]


def test_compute_cost_matches_the_reference_formulas():
    x, y = torch.tensor([1.0, 2.0, 3.0]), torch.tensor([1.5, 2.0, 2.0])
    lin = st.LinearCostFunction([1.0, 1.0, 2.0])
    assert float(lin.compute_cost(x, y)) == 0.0                       # 0.5 - 2 < 0
    assert float(lin.compute_cost(y, x)) == pytest.approx(1.5)
    sep = st.SeparableCostFunction([1.0, 0.0, 0.0], [0.0, 0.0, 1.0])
    assert float(sep.compute_cost(x, y)) == pytest.approx(1.0)        # 2 - 1


def test_device_coefficients_refuse_what_torch_dot_refuses():
    f = st.LinearCostFunction([1.0] * 3)
    with pytest.raises(ValueError, match="do not match"):
        f.device_coefficients(8, "cpu")
    for dt in (torch.int64, torch.float64, torch.float16):           # torch.dot against fp32 embeddings raises for all three
        f = st.LinearCostFunction(torch.ones(8, dtype=dt))
        with pytest.raises(ValueError, match="differ from"):
            f.device_coefficients(8, "cpu")
    f = st.LinearCostFunction([0.5] * 8)
    assert f.device_coefficients(8, "cpu")[0] is f.device_coefficients(8, "cpu")[0]     # copied once
    f.alpha.mul_(2)                                                  # an in-place change is seen
    assert f.device_coefficients(8, "cpu")[0].tolist() == [1.0] * 8
    c1, c2 = st.SeparableCostFunction([1.0] * 8, [2.0] * 8).device_coefficients(8, "cpu")
    assert c1.dtype == torch.float32 and c2.tolist() == [2.0] * 8


def _head(D, H0, H1, C, seed=0):
    g = torch.Generator().manual_seed(seed)
    return {"W0": torch.randn(H0, D, generator=g) * (2.0 / D) ** 0.5, "b0": torch.randn(H0, generator=g) * 0.1,
            "W1": torch.randn(H1, H0, generator=g) * (2.0 / H0) ** 0.5, "b1": torch.randn(H1, generator=g) * 0.1,
            "W2": torch.randn(C, H1, generator=g) * (2.0 / H1) ** 0.5, "b2": torch.randn(C, generator=g) * 0.1}


def test_oracle_follows_the_reference_search_loop():
    """the oracle's choice is the reference's loop (strict > from -inf over per-candidate fp32 forwards) wherever the margin
    is clear of fp32 noise"""
    p = _head(16, 16, 8, 3)
    x = torch.nn.functional.normalize(torch.randn(6, 16, generator=torch.Generator().manual_seed(1)), dim=1)
    alpha = torch.linspace(-0.2, 0.3, 16)
    for kind in (0, 1):
        cf = st.LinearCostFunction(alpha) if kind == 0 else st.SeparableCostFunction(alpha, alpha)
        res = so.best_response(p, x, kind, alpha, alpha)
        for b in range(x.shape[0]):
            best, choice = float("-inf"), 0
            for c, cand in enumerate(st.candidate_table(x[b])):
                prob = torch.softmax(so.head_forward(p, cand[None], torch.float32)[0], dim=-1).max()
                u = prob - cf.compute_cost(x[b], cand)
                if u > best:
                    best, choice = u, c
            assert float(res["util32"][b, choice]) == pytest.approx(float(best), abs=1e-5)
            if res["margin"][b] > 1e-4:
                assert int(res["choice"][b]) == choice


def test_oracle_strategic_loss_penalises_only_mispredicted_best_responses():
    p = {k: v.requires_grad_(True) for k, v in _head(8, 8, 4, 3).items()}
    X = torch.randn(4, 8, generator=torch.Generator().manual_seed(2))
    y = torch.tensor([0, 1, 2, 0])
    base = torch.nn.functional.cross_entropy(so.head_forward(p, X, torch.float32), y)
    out = so.head_forward(p, X, torch.float32)
    wrong = out.argmax(-1) != y
    want = base + 0.1 * torch.nn.functional.cross_entropy(out, y, reduction="none")[wrong].sum() / 4
    assert float(so.strategic_loss(p, X, y, X, 0.1)) == pytest.approx(float(want), rel=1e-6)


# ------------------------------------------------------------------------------------------ against the reference's run
def _gold(name):
    import os
    import numpy as np
    return np.load(os.path.join(os.path.dirname(__file__), "golden", f"golden_strategic_{name}.npz"))


def _params(g, prefix):
    names = {"model.0.weight": "W0", "model.0.bias": "b0", "model.3.weight": "W1", "model.3.bias": "b1",
             "model.6.weight": "W2", "model.6.bias": "b2"}
    return {v: torch.from_numpy(g[prefix + k]) for k, v in names.items()}


@pytest.mark.parametrize("name,kind", [("linear", 0), ("separable", 1)])
def test_oracle_reproduces_the_reference_best_responses(name, kind):
    """the prediction-time compute_best_response calls of the reference run (final head): same choices; every recorded
    margin is far above fp32 noise"""
    g = _gold(name)
    assert float(g["br_margin"].min()) > 1e-4
    n_sampled = len(range(0, int(g["n_br_train"]), 7))
    x = torch.from_numpy(g["br_x"][n_sampled:])
    alpha = st.CostFunctionFactory.create_cost_function(name, __import__("json").loads(str(g["config"]))["cost_coefficients"]).c1
    res = so.best_response(_params(g, "head_"), x, kind, alpha, alpha)
    assert res["choice"].tolist() == g["br_choice"][n_sampled:].tolist()


@pytest.mark.parametrize("name,kind", [("linear", 0), ("separable", 1)])
def test_oracle_reproduces_the_reference_strategic_training(name, kind):
    """the autograd oracle from the reference's head state and data, DataLoader orders of one manual_seed(42) generator:
    per-step strategic losses within 1e-5, final weights within 1e-4"""
    import json
    import numpy as np
    from adaptive_classifier_b200.classifier import dataloader_epoch_permutation
    g = _gold(name)
    alpha = torch.tensor(json.loads(str(g["config"]))["cost_coefficients"], dtype=torch.float32)
    for i in range(int(g["n_train_calls"])):
        X, y = torch.from_numpy(g[f"train{i}_X"]), torch.from_numpy(g[f"train{i}_Y"])
        gen = torch.Generator().manual_seed(42)
        perms = torch.cat([dataloader_epoch_permutation(gen, X.shape[0]) for _ in range(5)])
        losses, norms, P = so.strategic_training(_params(g, f"train{i}_before_"), X, y, perms, kind, alpha, alpha,
                                                 lr=0.001 * 0.5, lam=0.1)
        np.testing.assert_allclose(losses, g[f"train{i}_loss"], atol=1e-5)
        np.testing.assert_allclose(norms, g[f"train{i}_gnorm"], rtol=1e-4)
        after = _params(g, f"train{i}_after_")
        for k in after:
            np.testing.assert_allclose(P[k].detach().numpy(), after[k].numpy(), atol=1e-4)
