"""Golden vectors of the reference's classifier on a DeBERTa-v3 checkpoint, the architecture of microsoft/deberta-v3-* and
mdeberta-v3-base (test infrastructure; runs ONLY in the dev container, like oracle/make_golden.py).

    python oracle/make_golden_deberta.py        # writes tests/golden/golden_classifier_deberta*.npz

Runs make_golden.gen_classifier's recipe -- the UNMODIFIED reference's add_examples / _get_embeddings / predict /
predict_batch on the same texts and seeds -- with a tiny seeded DebertaV2Model of the v3 kind (hidden 128, 2 heads of 64,
3 layers, 256 position buckets, share_att_key, norm_rel_ebd = layer_norm, no position or token-type table) and a
DebertaV2Tokenizer built from an in-memory unigram vocabulary in place of the BERT ones.  The weights go to _bert0
(embeddings, the relative embeddings, layer 0) and _bert1 (layers 1-2) so that every file stays under 1 MB;
tests/golden_npz.py loads the three parts back as one mapping.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)

NAME = "golden_classifier_deberta"


def deberta_tokenizer(words):
    """DebertaV2Tokenizer over [PAD] [CLS] [SEP] [UNK] [MASK] + one unigram piece per word (no download)"""
    from transformers import DebertaV2Tokenizer
    specials = ["[PAD]", "[CLS]", "[SEP]", "[UNK]", "[MASK]"]
    vocab = [(s, 0.0) for s in specials] + [("▁" + w, -1.0 - 0.01 * i) for i, w in enumerate(words)]
    return DebertaV2Tokenizer(vocab=vocab), specials + words


def tiny_deberta_checkpoint(hidden=128):
    """seeded 3-layer DeBERTa-v3 with head_dim 64 + synthetic vocab, scaled like make_golden._tiny_checkpoint"""
    from transformers import DebertaV2Config, DebertaV2Model
    words = [f"w{i}" for i in range(195)]
    tok, vocab = deberta_tokenizer(words)
    cfg = DebertaV2Config(vocab_size=len(vocab), hidden_size=hidden, num_hidden_layers=3, num_attention_heads=hidden // 64,
                          intermediate_size=hidden, max_position_embeddings=512, type_vocab_size=0,
                          relative_attention=True, position_buckets=256, norm_rel_ebd="layer_norm", share_att_key=True,
                          pos_att_type=["p2c", "c2p"], position_biased_input=False, layer_norm_eps=1e-7, pad_token_id=0)
    torch.manual_seed(4321)
    model = DebertaV2Model(cfg)
    g = torch.Generator().manual_seed(97)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "LayerNorm" in n or n.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif n == "encoder.rel_embeddings.weight":
                p.copy_(torch.randn(p.shape, generator=g))
            elif "weight" in n and p.dim() == 2:
                # the init std 0.02 leaves every CLS row nearly identical; larger weights keep the classes apart
                p.mul_(4.0 if "word_embeddings" in n else 3.0)
        model.embeddings.word_embeddings.weight[1].zero_()        # the [CLS] row, as in the BERT recipe
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    tok.save_pretrained(tmp)
    return tmp, words, vocab, model, cfg


def save_parts(_name, arrays):
    parts = {"": {}, "_bert0": {}, "_bert1": {}}
    for k, v in arrays.items():
        if not k.startswith("bert_") or k == "bert_config":
            parts[""][k] = v
        else:
            parts["_bert1" if k.startswith(("bert_encoder.layer.1.", "bert_encoder.layer.2.")) else "_bert0"][k] = v
    for suffix, p in parts.items():
        np.savez_compressed(os.path.join(mg.OUT, f"{NAME}{suffix}.npz"), **p)


if __name__ == "__main__":
    mg._tiny_checkpoint = tiny_deberta_checkpoint
    mg.save_split = save_parts
    mg.gen_classifier()
    for suffix in ("", "_bert0", "_bert1"):
        f = os.path.join(mg.OUT, f"{NAME}{suffix}.npz")
        print(os.path.basename(f), os.path.getsize(f))
