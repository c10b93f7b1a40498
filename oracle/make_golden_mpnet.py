"""Golden vectors of the reference's classifier on an MPNet checkpoint, the architecture of all-mpnet-base-v2,
multi-qa-mpnet-base-* and paraphrase-mpnet-base-v2 (test infrastructure; runs ONLY in the dev container, like
oracle/make_golden.py).

    python oracle/make_golden_mpnet.py        # writes tests/golden/golden_classifier_mpnet*.npz

Runs make_golden.gen_classifier's recipe -- the UNMODIFIED reference's add_examples / _get_embeddings / predict /
predict_batch on the same texts and seeds -- with a tiny seeded MPNetModel (hidden 128, 2 heads of 64, 3 layers,
max_position_embeddings 514) and an MPNetTokenizer in place of the BERT ones.  The relative-attention-bias table is scaled
to O(1) so that the bias visibly moves the embeddings.  The weights go to _bert0 (embeddings, layer 0, the bias table) and
_bert1 (layers 1-2) so that every file stays under 1 MB; tests/golden_npz.py loads the three parts back as one mapping.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)

NAME = "golden_classifier_mpnet"


def tiny_mpnet_checkpoint(hidden=128):
    """seeded 3-layer MPNet with head_dim 64 + synthetic vocab, scaled like make_golden._tiny_checkpoint"""
    from transformers import MPNetConfig, MPNetModel, MPNetTokenizer
    words = [f"w{i}" for i in range(195)]
    vocab = ["<s>", "<pad>", "</s>", "[UNK]", "<mask>"] + words
    cfg = MPNetConfig(vocab_size=len(vocab), hidden_size=hidden, num_hidden_layers=3, num_attention_heads=hidden // 64,
                      intermediate_size=hidden, max_position_embeddings=514, layer_norm_eps=1e-5)
    torch.manual_seed(4321)
    model = MPNetModel(cfg)
    g = torch.Generator().manual_seed(97)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "LayerNorm" in n or n.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif n == "encoder.relative_attention_bias.weight":
                p.copy_(torch.randn(p.shape, generator=g))           # O(1): the bias reorders the attention weights
            elif "weight" in n and p.dim() == 2:
                # the init std 0.02 leaves every CLS row nearly identical; larger weights keep the classes apart
                p.mul_(4.0 if "word_embeddings" in n else 3.0)
        # the constant part of the CLS row's input (<s> word row, its position row 2) is zeroed, as in the BERT recipe
        model.embeddings.word_embeddings.weight[0].zero_()
        model.embeddings.position_embeddings.weight[2].zero_()
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    MPNetTokenizer(vocab={w: i for i, w in enumerate(vocab)}).save_pretrained(tmp)
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
    mg._tiny_checkpoint = tiny_mpnet_checkpoint
    mg.save_split = save_parts
    mg.gen_classifier()
    for suffix in ("", "_bert0", "_bert1"):
        f = os.path.join(mg.OUT, f"{NAME}{suffix}.npz")
        print(os.path.basename(f), os.path.getsize(f))
