"""Golden vectors of the reference's classifier on a EuroBERT checkpoint (test infrastructure; runs ONLY in the dev container,
like oracle/make_golden.py).

    python oracle/make_golden_eurobert.py   # writes tests/golden/golden_classifier_eurobert{,_long}{,_bert0.._bert3}.npz

The UNMODIFIED reference loads the checkpoint through AutoModel / AutoTokenizer (the native transformers EuroBertModel, no
remote code) from a local directory holding a tiny seeded EuroBertModel (hidden 256, 4 heads of 64, 2 kv heads, 2 layers,
SwiGLU I 512, RoPE theta 250000, 8192 positions) and a PreTrainedTokenizerFast that, as the real EuroBERT tokenizer does,
wraps every text in <|begin_of_text|> ... <|end_of_text|>, pads with <|end_of_text|> and returns input_ids and attention_mask
only (EuroBertModel.forward takes no token_type_ids).
    eurobert        make_golden.gen_classifier's recipe (same texts, seeds and calls)
    eurobert_long   make_golden_xlmr_long.main's recipe with max_length 1024 (texts past 512 tokens)
Every value is rounded through bfloat16 and the norm weights are moved off 1.  Both runs use the same seeded checkpoint; its
tensors are stored once, spread over golden_classifier_eurobert_bert0 .. _bert3.npz so that every file stays under 1 MB
(tests/golden_npz.py::load reads them back for either run, with weights_from for the long one).
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)
import make_golden_xlmr_long as mgx  # noqa: E402

from oracle.eurobert_oracle import SPECIALS, eurobert_tokenizer  # noqa: E402

N_PARTS = 4


def eurobert_config(n_vocab):
    from transformers import EuroBertConfig
    return EuroBertConfig(vocab_size=n_vocab, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                          num_key_value_heads=2, intermediate_size=512, max_position_embeddings=8192,
                          rope_parameters={"rope_type": "default", "rope_theta": 250000.0}, bos_token_id=0, eos_token_id=1,
                          pad_token_id=1, mask_token_id=2)


def tiny_eurobert_checkpoint():
    from transformers import EuroBertModel
    words = [f"w{i}" for i in range(195)]
    cfg = eurobert_config(len(SPECIALS) + len(words))
    torch.manual_seed(1234)
    model = EuroBertModel(cfg)
    g = torch.Generator().manual_seed(99)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "norm" in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 2:
                p.mul_(4.0 if "embed_tokens" in n else 3.0)
            p.copy_(p.bfloat16().float())
        # the constant part of the CLS row's input (the <|begin_of_text|> row) is zeroed, as in make_golden
        model.embed_tokens.weight[0].zero_()
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    eurobert_tokenizer(words).save_pretrained(tmp)
    return tmp, words, SPECIALS + words, model, cfg


def mg_model_state():
    return tiny_eurobert_checkpoint()[3].state_dict()


def save_parts(name, arrays, weights=True):
    """outputs in <name>.npz, the checkpoint (bert_*) greedily balanced over <name>_bert0 .. _bert{N_PARTS - 1}.npz
    (weights=False: not written)"""
    parts = [{} for _ in range(N_PARTS)]
    size = [0] * N_PARTS
    out = {}
    for k, v in arrays.items():
        if not k.startswith("bert_") or k == "bert_config":
            out[k] = v
    for k in sorted((k for k in arrays if k.startswith("bert_") and k != "bert_config"),
                    key=lambda k: -np.asarray(arrays[k]).nbytes):
        i = size.index(min(size))
        parts[i][k] = arrays[k]
        size[i] += np.asarray(arrays[k]).nbytes
    np.savez_compressed(os.path.join(mg.OUT, f"{name}.npz"), **out)
    if not weights:
        return
    for i, p in enumerate(parts):
        np.savez_compressed(os.path.join(mg.OUT, f"{name}_bert{i}.npz"), **p)


def main():
    mg._tiny_checkpoint = tiny_eurobert_checkpoint
    mg.save_split = lambda _name, arrays: save_parts("golden_classifier_eurobert", arrays)   # gen_classifier's own name
    mg.gen_classifier()
    base = {k: v.clone() for k, v in mg_model_state().items()}
    mg.save_split = lambda name, arrays: save_parts(name, arrays, weights=False)

    def long_checkpoint():          # make_golden_xlmr_long records (piece, score) pairs
        tmp, words, vocab, model, cfg = tiny_eurobert_checkpoint()
        assert all(torch.equal(v, base[k]) for k, v in model.state_dict().items())    # the weights stored with the first run
        return tmp, words, [(p, 0.0) for p in vocab], model, cfg
    mgx.tiny_xlmr_checkpoint = long_checkpoint
    mgx.NAME = "golden_classifier_eurobert_long"
    try:
        mgx.main()
    except FileNotFoundError as e:   # its closing size report lists the weight parts this run does not write
        assert "golden_classifier_eurobert_long_bert0.npz" in str(e), e
    for name, parts in (("golden_classifier_eurobert", N_PARTS), ("golden_classifier_eurobert_long", 0)):
        for suffix in [""] + [f"_bert{i}" for i in range(parts)]:
            f = os.path.join(mg.OUT, f"{name}{suffix}.npz")
            print(os.path.basename(f), os.path.getsize(f))
            assert os.path.getsize(f) < 1_000_000


if __name__ == "__main__":
    main()
