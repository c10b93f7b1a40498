"""Golden vectors of the reference's classifier on a NomicBERT and a jina-embeddings-v3 checkpoint (test infrastructure; runs
ONLY in the dev container, like oracle/make_golden.py).

    python oracle/make_golden_rotary.py   # writes tests/golden/golden_classifier_{nomic,jina3}{,_bert0,_bert1}.npz

The UNMODIFIED reference loads both through AutoModel.from_pretrained (the native transformers modules, no remote code):
    nomic   make_golden.gen_classifier's recipe (same texts, seeds and calls) on a tiny seeded NomicBertModel (hidden 128,
            2 heads of 64, 2 layers, SwiGLU I 256, RoPE theta 1000, 2048 positions) with a BertTokenizerFast built from a
            dict vocabulary
    jina3   make_golden_xlmr_long.main's recipe with max_length 1024 (texts past 512 tokens, so add_examples runs the long
            attention kernel on the GPU side) on a tiny seeded JinaEmbeddingsV3Model (hidden 128, 2 heads, 2 layers, GELU I
            256 with biases, RoPE theta 20000, 8194 positions) with the in-memory unigram XLMRobertaTokenizer of that recipe
The checkpoint's tensors are spread over the _bert0 / _bert1 parts and the outputs file so that every file stays under 1 MB.
"""
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)
import make_golden_albert as mga  # noqa: E402
import make_golden_xlmr_long as mgx  # noqa: E402


def _perturb(model, seed):
    """make_golden's recipe: LayerNorms and biases moved, weights scaled up (word embeddings x4), every value rounded
    through bfloat16 so the checkpoint compresses"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "layernorm" in n.lower() or n.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "weight" in n and p.dim() == 2:
                p.mul_(4.0 if "word_embeddings" in n else 3.0)
            p.copy_(p.bfloat16().float())


def tiny_nomic_checkpoint(hidden=128):
    from transformers import BertTokenizerFast, NomicBertConfig, NomicBertModel
    words = [f"w{i}" for i in range(195)]
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
    cfg = NomicBertConfig(vocab_size=len(vocab), hidden_size=hidden, num_hidden_layers=2, num_attention_heads=hidden // 64,
                          intermediate_size=2 * hidden, max_position_embeddings=2048, type_vocab_size=2, pad_token_id=0)
    torch.manual_seed(1234)
    model = NomicBertModel(cfg)
    _perturb(model, 99)
    with torch.no_grad():
        # the constant part of the CLS row's input ([CLS] word row, token types) is zeroed, as in make_golden
        model.embeddings.word_embeddings.weight[2].zero_()
        model.embeddings.token_type_embeddings.weight.zero_()
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}, do_lower_case=True).save_pretrained(tmp)
    return tmp, words, vocab, model, cfg


def tiny_jina_checkpoint(hidden=128):
    from transformers import JinaEmbeddingsV3Config, JinaEmbeddingsV3Model, XLMRobertaTokenizer
    words = [f"w{i}" for i in range(195)]
    pieces = [("<s>", 0.0), ("<pad>", 0.0), ("</s>", 0.0), ("<unk>", 0.0)]
    pieces += [("▁" + w, -1.0 - 0.01 * i) for i, w in enumerate(words)] + [("<mask>", 0.0)]
    cfg = JinaEmbeddingsV3Config(vocab_size=len(pieces), hidden_size=hidden, num_hidden_layers=2,
                                 num_attention_heads=hidden // 64, intermediate_size=2 * hidden, max_position_embeddings=8194,
                                 type_vocab_size=1, layer_norm_eps=1e-5, pad_token_id=1, bos_token_id=0, eos_token_id=2,
                                 hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    torch.manual_seed(1234)
    model = JinaEmbeddingsV3Model(cfg)          # with the pooler, as AutoModel builds it (the reference never uses it)
    _perturb(model, 99)
    with torch.no_grad():
        model.embeddings.word_embeddings.weight[0].zero_()       # <s>
        model.embeddings.token_type_embeddings.weight.zero_()
    tmp = tempfile.mkdtemp(prefix="golden_ckpt_")
    model.save_pretrained(tmp)
    XLMRobertaTokenizer(vocab=pieces).save_pretrained(tmp)
    return tmp, words, pieces, model, cfg


def main():
    mg._tiny_checkpoint = tiny_nomic_checkpoint
    mg.save_split = mga.saver("golden_classifier_nomic")
    mg.gen_classifier()
    mgx.tiny_xlmr_checkpoint = tiny_jina_checkpoint
    mgx.NAME = "golden_classifier_jina3"
    # the 1024-token id and mask arrays exceed the saver's uncompressed budget; the files are checked compressed below
    mg.save_split = lambda name, arrays: mga.saver(name)(name, arrays, limit=1_200_000)
    mgx.main()
    for name in ("golden_classifier_nomic", "golden_classifier_jina3"):
        for suffix in ("", "_bert0", "_bert1"):
            f = os.path.join(mg.OUT, f"{name}{suffix}.npz")
            print(os.path.basename(f), os.path.getsize(f))
            assert os.path.getsize(f) < 1_000_000


if __name__ == "__main__":
    main()
