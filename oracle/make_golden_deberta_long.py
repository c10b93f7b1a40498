"""Golden vectors of the reference's classifier on a DeBERTa-v3 checkpoint with inputs past 512 tokens (test
infrastructure; runs ONLY in the dev container, like oracle/make_golden.py).

    python oracle/make_golden_deberta_long.py   # writes tests/golden/golden_classifier_deberta_long.npz

make_golden.gen_classifier's recipe -- the UNMODIFIED reference's add_examples / _get_embeddings / predict / predict_batch --
with config = {"max_length": MAX_LENGTH} on make_golden_deberta.tiny_deberta_checkpoint (hidden 128, 2 heads of 64, 3
layers, 256 position buckets, no position table: HF runs it at any length).  The texts have mixed lengths, as in
make_golden_xlmr_long.py: some over 512 tokens, some over MAX_LENGTH (the tokenizer truncates them), some short (padded).

The checkpoint is the one golden_classifier_deberta_bert0 / _bert1 already hold (this script checks that bit for bit), so
only the recorded outputs are written; the tests load the weights from those files.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)
import make_golden_deberta as mgd  # noqa: E402

NAME = "golden_classifier_deberta_long"
MAX_LENGTH = 1024
SEED = 16                                         # texts
TRAIN_WORDS = [5, 40, 300, 600, 1100, 1600]        # words per training text of each class (+ [CLS], [SEP])
TEST_WORDS = [700, 12, 1500, 520, 90, 1030]


def main():
    from adaptive_classifier import AdaptiveClassifier
    tmp, words, vocab, model, cfg = mgd.tiny_deberta_checkpoint()
    stored = {}
    for suffix in ("_bert0", "_bert1"):
        with np.load(os.path.join(mg.OUT, f"golden_classifier_deberta{suffix}.npz")) as z:
            stored.update({k[5:]: z[k] for k in z.files})
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    assert set(sd) == set(stored) and all(np.array_equal(sd[k], stored[k]) for k in sd), \
        "tiny_deberta_checkpoint no longer equals the checkpoint stored in golden_classifier_deberta_bert*.npz"

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
    assert int((enc["input_ids"] == 3).sum()) == 0, "a word fell back to [UNK]"
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
    f = os.path.join(mg.OUT, f"{NAME}.npz")
    np.savez_compressed(f, vocab=np.array(vocab), texts=np.array(texts), labels=np.array(labels),
                        test_texts=np.array(test_texts), label_names=np.array(label_names),
                        input_ids=enc["input_ids"].numpy().astype(np.int32),
                        attention_mask=enc["attention_mask"].numpy().astype(np.int32), max_length=MAX_LENGTH,
                        emb_train=emb_train, emb_test=emb_test, prototypes=protos,
                        proto_labels=np.array(sorted(clf.memory.prototypes)), train_steps=clf.train_steps,
                        training_history=json.dumps(clf.training_history), pred_labels=pl, pred_scores=ps,
                        pred_k1_labels=p1l, pred_k1_scores=p1s, predb_labels=pbl, predb_scores=pbs,
                        bert_config=json.dumps(cfg.to_dict()), **head_sd)
    print(os.path.basename(f), os.path.getsize(f))
    print("labels", label_names, "pred[0]", pred[0], "lengths", lens.tolist())


if __name__ == "__main__":
    main()
