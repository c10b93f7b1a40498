"""Golden vectors of the reference's strategic mode (test infrastructure; runs ONLY in the dev container, like
oracle/make_golden.py).

    python oracle/make_golden_strategic.py     # writes tests/golden/golden_strategic_{linear,separable,readme}.npz

Runs the UNMODIFIED reference classifier (make_golden's tiny seeded BERT checkpoint, the same texts and seeds as the
bert row of make_golden_encoders.py) with nn.Dropout patched to identity -- as gen_training does: CPU dropout masks
cannot be reproduced on a GPU -- for list coefficients of both cost types with strategic_training_frequency = 1, and records:
  * every strategic training call: its inputs, the head state before and after, the per-step strategic losses
    (StrategicOptimizer.strategic_loss wrapped) and pre-clip grad norms, and the train_steps at which it ran;
  * every compute_best_response call: x, the chosen candidate index and the margin between the best and second-best fp32
    utility of the reference's own search loop (asserted far above fp32 noise, so the fixture cannot flip on last bits);
  * predict / predict_strategic / predict_robust (k = 3) of the test texts and evaluate_strategic_robustness under
    torch.manual_seed(5);
  * the README configs (dict coefficients, no coefficients): regular predictions and the head they were made with.
The checkpoint itself is golden_classifier's (same recipe, same seed); it is not stored again.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)

MIN_MARGIN = 1e-4          # fp32 utilities of a 128 -> 128 -> 64 -> C head carry ~1e-6 of rounding


def texts_and_labels(words):
    """the sentences of make_golden_encoders.short at seed 7 (same generator, same draws)"""
    rng = np.random.default_rng(7)
    class_words = {"sports": words[0:40], "finance": words[40:80], "cooking": words[80:120]}

    def sentence(label, n):
        own = rng.choice(class_words[label], size=n, replace=True)
        noise = rng.choice(words[120:], size=max(1, n // 4), replace=True)
        toks = list(own) + list(noise)
        rng.shuffle(toks)
        return " ".join(toks)

    texts, labels = [], []
    for label in ["sports", "finance", "cooking"]:
        for _ in range(12):
            texts.append(sentence(label, int(rng.integers(4, 14))))
            labels.append(label)
    test_texts = [sentence(l, 9) for l in ["sports", "finance", "cooking", "finance", "sports", "cooking"]]
    return texts, labels, test_texts


def coefficients(D):
    return [0.05 * ((i % 5) - 2) for i in range(D)]     # zeros and negatives among them


def run(tmp, words, config):
    import torch.nn as nn
    from adaptive_classifier import AdaptiveClassifier
    from adaptive_classifier import strategic as rs
    texts, labels, test_texts = texts_and_labels(words)
    rec = {"train": [], "br": []}
    saved = []

    def patch(obj, name, make):
        saved.append((obj, name, getattr(obj, name)))
        setattr(obj, name, make(getattr(obj, name)))

    def mk_br(orig):
        def br(self_, x, f):
            y = orig(self_, x, f)
            cands = self_._generate_candidates(x)
            utils = []
            for c in cands:                     # the reference's own utilities (strategic.py:88-100), replayed
                with torch.no_grad():
                    fc = f(c.unsqueeze(0)).squeeze()
                    if len(fc.shape) > 0:
                        fc = torch.max(fc)
                utils.append(float(fc - self_.compute_cost(x, c)))
            u = np.array(utils, dtype=np.float64)
            choice = int(np.argmax(u))
            assert torch.equal(cands[choice], y), "replayed search disagrees with the reference's"
            top2 = np.sort(u)[-2:]
            rec["br"].append((x.detach().clone().numpy(), choice, float(top2[1] - top2[0])))
            return y
        return br
    patch(rs.SeparableCostFunction, "compute_best_response", mk_br)

    def mk_loss(orig):
        def loss(self_, model, emb, lab, lam=0.1):
            r = orig(self_, model, emb, lab, lam)
            rec["train"][-1]["loss"].append(float(r.detach()))
            return r
        return loss
    patch(rs.StrategicOptimizer, "strategic_loss", mk_loss)

    def mk_clip(orig):
        def clip(params, max_norm, *a, **k):
            r = orig(params, max_norm, *a, **k)
            if rec["train"] and rec["train"][-1].get("open"):
                rec["train"][-1]["gnorm"].append(float(r))
            return r
        return clip
    patch(torch.nn.utils, "clip_grad_norm_", mk_clip)
    patch(nn.Dropout, "forward", lambda orig: (lambda self_, x: x))

    def mk_step(orig):
        def step(self_, X, Y):
            st = {k: v.detach().clone().numpy() for k, v in self_.adaptive_head.state_dict().items()}
            rec["train"].append({"X": X.detach().clone().numpy(), "Y": Y.detach().clone().numpy(), "before": st, "loss": [],
                                 "gnorm": [], "train_steps": self_.train_steps, "open": True})
            r = orig(self_, X, Y)
            rec["train"][-1]["open"] = False
            rec["train"][-1]["after"] = {k: v.detach().clone().numpy() for k, v in self_.adaptive_head.state_dict().items()}
            return r
        return step
    from adaptive_classifier import classifier as rc
    patch(rc.AdaptiveClassifier, "_strategic_training_step", mk_step)
    try:
        torch.manual_seed(0)
        np.random.seed(0)
        clf = AdaptiveClassifier(tmp, device="cpu", use_onnx=False, config=config)
        clf.add_examples(texts[:24], labels[:24])          # regular branch -> strategic step (C = 2)
        clf.add_examples(texts[24:], labels[24:])          # new class -> incremental branch, no strategic step
        clf.add_examples(texts[30:36], labels[30:36])      # no new class -> regular branch -> strategic step (C = 3)
        n_br_train = len(rec["br"])
        label_names = [clf.id_to_label[i] for i in range(len(clf.id_to_label))]
        preds = {m: [getattr(clf, m)(t, k=3) for t in test_texts] for m in ("predict", "predict_strategic", "predict_robust")}
        rob = None
        if clf.strategic_mode:
            torch.manual_seed(5)
            rob = clf.evaluate_strategic_robustness(test_texts, ["sports", "finance", "cooking", "finance", "sports", "cooking"])
        head = {k: v.detach().clone().numpy() for k, v in clf.adaptive_head.state_dict().items()}
        mode = clf.strategic_mode
        enabled = clf.config.enable_strategic_mode
    finally:
        for obj, name, orig in reversed(saved):
            setattr(obj, name, orig)
    margins = [m for _, _, m in rec["br"]]
    if margins:
        assert min(margins) > MIN_MARGIN, f"a recorded best response is a near-tie (margin {min(margins):.3g})"
    out = {"config": json.dumps(config), "strategic_mode": mode, "enable_after_init": enabled, "label_names": np.array(label_names),
           "test_texts": np.array(test_texts), "n_train_calls": len(rec["train"]), "n_br_train": n_br_train}
    for m, P in preds.items():
        L = np.full((len(P), 3), -1, dtype=np.int64)
        S = np.zeros((len(P), 3), dtype=np.float64)
        for i, p in enumerate(P):
            for j, (l, s) in enumerate(p):
                L[i, j], S[i, j] = label_names.index(l), s
        out[f"{m}_labels"], out[f"{m}_scores"] = L, S
    if rob is not None:
        out["robustness"] = json.dumps(rob)
    for k, v in head.items():
        out["head_" + k] = v
    for i, t in enumerate(rec["train"]):
        out[f"train{i}_X"], out[f"train{i}_Y"], out[f"train{i}_train_steps"] = t["X"], t["Y"], t["train_steps"]
        out[f"train{i}_loss"], out[f"train{i}_gnorm"] = np.array(t["loss"]), np.array(t["gnorm"])
        for k, v in t["before"].items():
            out[f"train{i}_before_{k}"] = v
        for k, v in t["after"].items():
            out[f"train{i}_after_{k}"] = v
    if rec["br"]:
        out["br_x"] = np.stack([x for x, _, _ in rec["br"]])
        out["br_choice"] = np.array([c for _, c, _ in rec["br"]])
        out["br_margin"] = np.array(margins)
    return out


if __name__ == "__main__":
    tmp, words, vocab, model, cfg = mg._tiny_checkpoint()
    D = cfg.hidden_size
    configs = {
        "linear": {"enable_strategic_mode": True, "cost_function_type": "linear", "cost_coefficients": coefficients(D),
                   "strategic_training_frequency": 1},
        "separable": {"enable_strategic_mode": True, "cost_function_type": "separable", "cost_coefficients": coefficients(D),
                      "strategic_training_frequency": 1},
    }
    for name, config in configs.items():
        out = run(tmp, words, config)
        # keep the file small: the best responses of the training loops are checked through the losses; keep the
        # prediction-time ones (the last 6 + 3 x 6 of predict / predict_strategic / evaluate) and a sample of the rest
        keep = np.r_[np.arange(0, out["n_br_train"], 7), np.arange(out["n_br_train"], len(out["br_choice"]))]
        for k in ("br_x", "br_choice", "br_margin"):
            out[k] = out[k][keep]
        np.savez_compressed(os.path.join(mg.OUT, f"golden_strategic_{name}.npz"), **out)
    readme = {}
    for name, config in (("dict", {"enable_strategic_mode": True, "cost_coefficients": {"sentiment_words": 0.5}}),
                         ("none", {"enable_strategic_mode": True})):
        out = run(tmp, words, config)
        for k, v in out.items():
            readme[f"{name}_{k}"] = v
    np.savez_compressed(os.path.join(mg.OUT, "golden_strategic_readme.npz"), **readme)
    for f in sorted(os.listdir(mg.OUT)):
        if f.startswith("golden_strategic"):
            print(f, os.path.getsize(os.path.join(mg.OUT, f)))
