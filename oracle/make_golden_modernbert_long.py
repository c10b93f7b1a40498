"""Golden vectors of the reference's classifier on a ModernBERT checkpoint with long inputs (test infrastructure; runs ONLY in
the dev container, like oracle/make_golden.py).

    python oracle/make_golden_modernbert_long.py   # writes tests/golden/golden_classifier_modernbert_long.npz

make_golden.gen_classifier's recipe -- the UNMODIFIED reference's add_examples / _get_embeddings / predict / predict_batch --
on the tiny seeded ModernBERT checkpoint of make_golden_modernbert.py, saved with max_position_embeddings = 8192, and with
config = {"max_length": MAX_LENGTH}.  The texts have mixed lengths: some over 512 tokens, some over MAX_LENGTH (the
tokenizer truncates them), some short (padded).  ModernBERT has no position parameters, so the weights are those of
golden_classifier_modernbert_bert{0,1}.npz (asserted here) and are not stored twice; tests load them from there.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)
from make_golden_modernbert import tiny_modernbert_checkpoint  # noqa: E402

NAME = "golden_classifier_modernbert_long"
MAX_LENGTH = 1024
SEED = 15                                         # texts (chosen for clear top-k margins in the predictions)
TRAIN_WORDS = [5, 40, 300, 600, 1100, 1600]        # words per training text of each class (+ [CLS], [SEP])
TEST_WORDS = [700, 12, 1500, 520, 90, 1030]


def main():
    from adaptive_classifier import AdaptiveClassifier
    tmp, words, vocab, model, cfg = tiny_modernbert_checkpoint()
    model.config.max_position_embeddings = 8192
    model.save_pretrained(tmp)
    cfg = model.config
    prev = dict(np.load(os.path.join(mg.OUT, "golden_classifier_modernbert_bert0.npz")))
    prev.update(np.load(os.path.join(mg.OUT, "golden_classifier_modernbert_bert1.npz")))
    sd = model.state_dict()
    assert sorted(prev) == sorted("bert_" + k for k in sd)
    assert all(np.array_equal(prev["bert_" + k], v.numpy()) for k, v in sd.items()), "checkpoint differs from the golden one"

    rng = np.random.default_rng(SEED)
    class_words = {"sports": words[0:40], "finance": words[40:80], "cooking": words[80:120]}

    def sentence(label, n):
        own = rng.choice(class_words[label], size=n - max(1, n // 5), replace=True)
        noise = rng.choice(words[120:], size=max(1, n // 5), replace=True)
        toks = list(own) + list(noise)
        rng.shuffle(toks)
        return " ".join(toks)

    texts, labels = [], []
    for label in ["sports", "finance", "cooking"]:
        for n in TRAIN_WORDS:
            texts.append(sentence(label, n))
            labels.append(label)
    test_texts = [sentence(l, n) for l, n in zip(["sports", "finance", "cooking", "finance", "sports", "cooking"], TEST_WORDS)]

    torch.manual_seed(0)
    np.random.seed(0)
    clf = AdaptiveClassifier(tmp, device="cpu", use_onnx=False, config={"max_length": MAX_LENGTH})
    clf.add_examples(texts[:12], labels[:12])           # sports + finance -> _train_adaptive_head
    clf.add_examples(texts[12:], labels[12:])           # new class cooking -> _train_new_classes (+EWC)
    emb_train = torch.stack(clf._get_embeddings(texts)).numpy()
    emb_test = torch.stack(clf._get_embeddings(test_texts)).numpy()
    enc = clf.tokenizer(texts + test_texts, max_length=MAX_LENGTH, truncation=True, padding=True, return_tensors="pt")
    lens = enc["attention_mask"].sum(1)
    assert enc["input_ids"].shape[1] == MAX_LENGTH and int((lens > 512).sum()) >= 6 and int((lens < 64).sum()) >= 3
    label_names = [clf.id_to_label[i] for i in range(len(clf.id_to_label))]
    pred = [clf.predict(t, k=3) for t in test_texts]
    pred_k1 = [clf.predict(t, k=1) for t in test_texts]
    pred_b = clf.predict_batch(test_texts, k=2)

    def pack(preds, k):
        L = np.full((len(preds), k), -1, dtype=np.int64)
        S = np.zeros((len(preds), k), dtype=np.float64)
        for i, p in enumerate(preds):
            for j, (l, s) in enumerate(p):
                L[i, j] = label_names.index(l)
                S[i, j] = s
        return L, S

    pl, ps = pack(pred, 3)
    p1l, p1s = pack(pred_k1, 1)
    pbl, pbs = pack(pred_b, 2)
    head_sd = {("head_" + k): v.detach().numpy() for k, v in clf.adaptive_head.state_dict().items()}
    protos = np.stack([clf.memory.prototypes[l].numpy() for l in sorted(clf.memory.prototypes)])
    out = os.path.join(mg.OUT, f"{NAME}.npz")
    np.savez_compressed(
        out, vocab=np.array(vocab), texts=np.array(texts), labels=np.array(labels), test_texts=np.array(test_texts),
        label_names=np.array(label_names), input_ids=enc["input_ids"].numpy().astype(np.int32),
        attention_mask=enc["attention_mask"].numpy().astype(np.int32), max_length=MAX_LENGTH,
        emb_train=emb_train, emb_test=emb_test, prototypes=protos, proto_labels=np.array(sorted(clf.memory.prototypes)),
        train_steps=clf.train_steps, pred_labels=pl, pred_scores=ps, pred_k1_labels=p1l, pred_k1_scores=p1s,
        predb_labels=pbl, predb_scores=pbs, bert_config=json.dumps(cfg.to_dict()), **head_sd)
    print(os.path.basename(out), os.path.getsize(out), "labels", label_names, "pred[0]", pred[0])


if __name__ == "__main__":
    main()
