"""Golden vectors of the reference's classifier on an ALBERT and an ELECTRA checkpoint (test infrastructure; runs ONLY in the
dev container, like oracle/make_golden.py).

    python oracle/make_golden_albert.py        # writes tests/golden/golden_classifier_albert*.npz, golden_classifier_electra*.npz

Runs make_golden.gen_classifier's recipe -- the UNMODIFIED reference's add_examples / _get_embeddings / predict /
predict_batch on the same texts and seeds -- with two tiny seeded checkpoints in place of the BERT one:
    albert    embedding_size 128 != hidden 256, 4 heads of 64, I 256, 3 effective layers sharing one group (as every
              published ALBERT does), "gelu_new"; AlbertTokenizer over an in-memory unigram vocabulary
    electra   the electra-small shape (embedding_size 128, hidden 256, 4 heads), 1 layer, I 256, "gelu"; ElectraTokenizer
              with the vocabulary passed as a dict (no file, no download)
The checkpoint's tensors are spread over the _bert0 / _bert1 parts and the outputs file so that every file stays under
1 MB; tests/golden_npz.py loads the parts back as one mapping.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)

WORDS = [f"w{i}" for i in range(195)]


def _perturb(model, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "LayerNorm" in n or "layer_norm" in n or n.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "weight" in n and p.dim() == 2:
                # the init std 0.02 leaves every CLS row nearly identical; larger weights keep the classes apart
                p.mul_(4.0 if "word_embeddings" in n else 3.0)


def tiny_albert_checkpoint(hidden=256):
    from transformers import AlbertConfig, AlbertModel, AlbertTokenizer
    specials = ["<pad>", "<unk>", "[CLS]", "[SEP]", "[MASK]"]
    tok = AlbertTokenizer(vocab=[(s, 0.0) for s in specials] + [("▁" + w, -1.0 - 0.01 * i) for i, w in enumerate(WORDS)])
    vocab = specials + WORDS
    cfg = AlbertConfig(vocab_size=len(vocab), embedding_size=128, hidden_size=hidden, num_hidden_layers=3,
                       num_hidden_groups=1, inner_group_num=1, num_attention_heads=hidden // 64, intermediate_size=256,
                       max_position_embeddings=128, type_vocab_size=2, hidden_act="gelu_new", pad_token_id=0)
    torch.manual_seed(4321)
    model = AlbertModel(cfg)
    _perturb(model, 97)
    with torch.no_grad():
        model.embeddings.word_embeddings.weight[2].zero_()        # the [CLS] row, as in the BERT recipe
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    tok.save_pretrained(tmp)
    return tmp, WORDS, vocab, model, cfg


def tiny_electra_checkpoint(hidden=256):
    from transformers import ElectraConfig, ElectraModel, ElectraTokenizer
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS
    tok = ElectraTokenizer(vocab={w: i for i, w in enumerate(vocab)})
    cfg = ElectraConfig(vocab_size=len(vocab), embedding_size=128, hidden_size=hidden, num_hidden_layers=1,
                        num_attention_heads=hidden // 64, intermediate_size=256, max_position_embeddings=128,
                        type_vocab_size=2, hidden_act="gelu", pad_token_id=0)
    torch.manual_seed(4322)
    model = ElectraModel(cfg)
    _perturb(model, 98)
    with torch.no_grad():
        model.embeddings.word_embeddings.weight[2].zero_()
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    tok.save_pretrained(tmp)
    return tmp, WORDS, vocab, model, cfg


def saver(name):
    def save_parts(_name, arrays, limit=900_000):
        parts = {"": {}, "_bert0": {}, "_bert1": {}}
        size = {k: 0 for k in parts}
        for k, v in arrays.items():
            if not k.startswith("bert_") or k == "bert_config":
                parts[""][k] = v
                size[""] += np.asarray(v).nbytes
        for k in sorted((k for k in arrays if k.startswith("bert_") and k != "bert_config"),
                        key=lambda k: -np.asarray(arrays[k]).nbytes):
            dst = min(parts, key=lambda p: size[p])
            parts[dst][k] = arrays[k]
            size[dst] += np.asarray(arrays[k]).nbytes
        assert max(size.values()) < limit, size
        for suffix, p in parts.items():
            np.savez_compressed(os.path.join(mg.OUT, f"{name}{suffix}.npz"), **p)
    return save_parts


if __name__ == "__main__":
    for name, ckpt in (("golden_classifier_albert", tiny_albert_checkpoint),
                       ("golden_classifier_electra", tiny_electra_checkpoint)):
        mg._tiny_checkpoint = ckpt
        mg.save_split = saver(name)
        mg.gen_classifier()
        for suffix in ("", "_bert0", "_bert1"):
            f = os.path.join(mg.OUT, f"{name}{suffix}.npz")
            print(os.path.basename(f), os.path.getsize(f))
