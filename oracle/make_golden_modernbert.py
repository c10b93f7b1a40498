"""Golden vectors of the reference's classifier on a ModernBERT checkpoint (test infrastructure; runs ONLY in the dev
container, like oracle/make_golden.py).

    python oracle/make_golden_modernbert.py        # writes tests/golden/golden_classifier_modernbert*.npz

Runs make_golden.gen_classifier's recipe -- the UNMODIFIED reference's add_examples / _get_embeddings / predict /
predict_batch on the same texts and seeds -- with a tiny seeded ModernBERT checkpoint in place of the BERT one.  The
weights go to _bert0 (embeddings, layers 0-1, final_norm) and _bert1 (layers 2-3) so that every file stays under 1 MB;
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

NAME = "golden_classifier_modernbert"


def tiny_modernbert_checkpoint(hidden=128):
    """seeded 4-layer ModernBERT (both layer types twice, half-window 8 < the golden sentences' length) + synthetic vocab"""
    from transformers import BertTokenizerFast, ModernBertConfig, ModernBertModel
    words = [f"w{i}" for i in range(195)]
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
    cfg = ModernBertConfig(vocab_size=len(vocab), hidden_size=hidden, num_hidden_layers=4, num_attention_heads=2,
                           intermediate_size=64, local_attention=16, max_position_embeddings=512, pad_token_id=0,
                           cls_token_id=2, sep_token_id=3, bos_token_id=2, eos_token_id=3)
    torch.manual_seed(1234)
    model = ModernBertModel(cfg)
    g = torch.Generator().manual_seed(99)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "norm" in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            else:
                # the init std 0.02 leaves every CLS row nearly identical; larger weights keep the classes apart
                p.mul_(4.0 if "tok_embeddings" in n else 2.0)
        model.embeddings.tok_embeddings.weight[2].zero_()
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    tok = BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}, do_lower_case=True)
    tok.model_input_names = ["input_ids", "attention_mask"]     # ModernBERT takes no token_type_ids
    tok.save_pretrained(tmp)
    return tmp, words, vocab, model, cfg


def save_parts(_name, arrays):
    parts = {"": {}, "_bert0": {}, "_bert1": {}}
    for k, v in arrays.items():
        if not k.startswith("bert_") or k == "bert_config":
            parts[""][k] = v
        else:
            parts["_bert1" if k.startswith(("bert_layers.2.", "bert_layers.3.")) else "_bert0"][k] = v
    for suffix, p in parts.items():
        np.savez_compressed(os.path.join(mg.OUT, f"{NAME}{suffix}.npz"), **p)


if __name__ == "__main__":
    mg._tiny_checkpoint = tiny_modernbert_checkpoint
    mg.save_split = save_parts
    mg.gen_classifier()
    for suffix in ("", "_bert0", "_bert1"):
        f = os.path.join(mg.OUT, f"{NAME}{suffix}.npz")
        print(os.path.basename(f), os.path.getsize(f))
