"""Golden vectors of the reference's classifier on an XLM-RoBERTa checkpoint with an 8194-row position table and long
inputs (test infrastructure; runs ONLY in the dev container, like oracle/make_golden.py).

    python oracle/make_golden_xlmr_long.py   # writes tests/golden/golden_classifier_xlmr_long{,_bert0,_bert1}.npz

make_golden.gen_classifier's recipe -- the UNMODIFIED reference's add_examples / _get_embeddings / predict / predict_batch --
with config = {"max_length": MAX_LENGTH} on a tiny seeded XLMRobertaModel (hidden 128, 2 heads of 64, 2 layers) saved with
max_position_embeddings = 8194, the table of bge-m3 and snowflake-arctic-embed-l-v2.0, and an XLMRobertaTokenizer built
from an in-memory unigram vocabulary (one piece per word).  The texts have mixed lengths: some over 512 tokens, some over
MAX_LENGTH (the tokenizer truncates them), some short (padded).

Size: every weight is rounded through bfloat16 and position rows past MAX_LENGTH + 2 (never reached at this max_length)
are zero, so the checkpoint compresses to well under 1 MB per file; the weights go to _bert0 / _bert1 (layer 1) as in
make_golden.save_split.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)

NAME = "golden_classifier_xlmr_long"
MAX_LENGTH = 1024
MAX_POS = 8194
SEED = 15                                         # texts
TRAIN_WORDS = [5, 40, 300, 600, 1100, 1600]        # words per training text of each class (+ <s>, </s>)
TEST_WORDS = [700, 12, 1500, 520, 90, 1030]


def tiny_xlmr_checkpoint(hidden=128):
    """seeded 2-layer XLM-R with an 8194-row position table + a unigram vocabulary of 195 words"""
    from transformers import XLMRobertaConfig, XLMRobertaModel, XLMRobertaTokenizer
    words = [f"w{i}" for i in range(195)]
    pieces = [("<s>", 0.0), ("<pad>", 0.0), ("</s>", 0.0), ("<unk>", 0.0)]
    pieces += [("▁" + w, -1.0 - 0.01 * i) for i, w in enumerate(words)] + [("<mask>", 0.0)]
    cfg = XLMRobertaConfig(vocab_size=len(pieces), hidden_size=hidden, num_hidden_layers=2, num_attention_heads=2,
                           intermediate_size=hidden, max_position_embeddings=MAX_POS, type_vocab_size=1,
                           layer_norm_eps=1e-5, pad_token_id=1, bos_token_id=0, eos_token_id=2)
    torch.manual_seed(1234)
    model = XLMRobertaModel(cfg, add_pooling_layer=False)
    g = torch.Generator().manual_seed(99)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "LayerNorm" in n or n.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "weight" in n and p.dim() == 2:
                p.mul_(4.0 if "word_embeddings" in n else 3.0)
            p.copy_(p.bfloat16().float())
        # the constant part of the CLS row's input (<s> row, its position pad_idx + 1, the token type) is zeroed, so that
        # the sentences embed apart (make_golden._tiny_checkpoint)
        model.embeddings.word_embeddings.weight[0].zero_()
        model.embeddings.position_embeddings.weight[2].zero_()
        model.embeddings.position_embeddings.weight[MAX_LENGTH + 2:].zero_()
        model.embeddings.token_type_embeddings.weight.zero_()
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    tok = XLMRobertaTokenizer(vocab=pieces)
    tok.save_pretrained(tmp)
    return tmp, words, pieces, model, cfg


def main():
    from adaptive_classifier import AdaptiveClassifier
    tmp, words, pieces, model, cfg = tiny_xlmr_checkpoint()

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
    assert int((enc["input_ids"] == 3).sum()) == 0, "a word fell back to <unk>"
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
    model_sd = {("bert_" + k): v.detach().numpy() for k, v in model.state_dict().items()}
    protos = np.stack([clf.memory.prototypes[l].numpy() for l in sorted(clf.memory.prototypes)])
    mg.save_split(NAME, dict(
        vocab_pieces=np.array([p for p, _ in pieces]), vocab_scores=np.array([s for _, s in pieces]),
        texts=np.array(texts), labels=np.array(labels), test_texts=np.array(test_texts),
        label_names=np.array(label_names), input_ids=enc["input_ids"].numpy().astype(np.int32),
        attention_mask=enc["attention_mask"].numpy().astype(np.int32), max_length=MAX_LENGTH,
        emb_train=emb_train, emb_test=emb_test, prototypes=protos, proto_labels=np.array(sorted(clf.memory.prototypes)),
        train_steps=clf.train_steps, pred_labels=pl, pred_scores=ps, pred_k1_labels=p1l, pred_k1_scores=p1s,
        predb_labels=pbl, predb_scores=pbs, bert_config=json.dumps(cfg.to_dict()), **head_sd, **model_sd))
    for suffix in ("", "_bert0", "_bert1"):
        f = os.path.join(mg.OUT, f"{NAME}{suffix}.npz")
        print(os.path.basename(f), os.path.getsize(f))
    print("labels", label_names, "pred[0]", pred[0])


if __name__ == "__main__":
    main()
