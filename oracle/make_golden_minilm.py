"""Golden vectors of the reference's classifier on a head_dim-32 BERT checkpoint, the shape of all-MiniLM-L6-v2, BGE-small
and E5-small (test infrastructure; runs ONLY in the dev container, like oracle/make_golden.py).

    python oracle/make_golden_minilm.py        # writes tests/golden/golden_classifier_minilm*.npz

Runs make_golden.gen_classifier's recipe -- the UNMODIFIED reference's add_examples / _get_embeddings / predict /
predict_batch on the same texts and seeds -- with a tiny seeded BertModel of 4 heads of 32 (hidden 128, 3 layers) in place
of the 2-head one.  The weights go to _bert0 (embeddings, layer 0) and _bert1 (layers 1-2) so that every file stays under
1 MB; tests/golden_npz.py loads the three parts back as one mapping.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)

NAME = "golden_classifier_minilm"


def tiny_minilm_checkpoint(hidden=128):
    """seeded 3-layer BERT with head_dim 32 + synthetic vocab, scaled like make_golden._tiny_checkpoint"""
    from transformers import BertConfig, BertModel, BertTokenizerFast
    words = [f"w{i}" for i in range(195)]
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
    cfg = BertConfig(vocab_size=len(vocab), hidden_size=hidden, num_hidden_layers=3, num_attention_heads=hidden // 32,
                     intermediate_size=hidden, max_position_embeddings=64, type_vocab_size=2, pad_token_id=0)
    torch.manual_seed(4321)
    model = BertModel(cfg)
    g = torch.Generator().manual_seed(98)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "LayerNorm" in n or n.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "weight" in n and p.dim() == 2:
                # the init std 0.02 leaves every CLS row nearly identical; larger weights keep the classes apart
                p.mul_(4.0 if "word_embeddings" in n else 3.0)
        model.embeddings.word_embeddings.weight[2].zero_()
        model.embeddings.position_embeddings.weight[0].zero_()
        model.embeddings.token_type_embeddings.weight.zero_()
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}, do_lower_case=True).save_pretrained(tmp)
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
    mg._tiny_checkpoint = tiny_minilm_checkpoint
    mg.save_split = save_parts
    mg.gen_classifier()
    for suffix in ("", "_bert0", "_bert1"):
        f = os.path.join(mg.OUT, f"{NAME}{suffix}.npz")
        print(os.path.basename(f), os.path.getsize(f))
