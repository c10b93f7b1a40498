"""Golden classifier runs of the reference on tiny seeded encoder checkpoints (test infrastructure; runs ONLY in the dev
container, like oracle/make_golden.py).

    python oracle/make_golden_encoders.py [row ...] [--out DIR]    # every row into tests/golden by default

FAMILIES has one row per run; row <name> writes golden_classifier_<name>*.npz (row bert: golden_classifier*.npz).  A row
gives the checkpoint builder, the recipe with its text seed, and how the checkpoint's tensors are stored: split over the
_bert<i> parts (make_golden.by_prefix / greedy), or not at all for a long run on the checkpoint of its short run
(weights_from: asserted equal to the tensors that run stored in tests/golden, which the tests load for both runs).
tests/golden_npz.py loads the parts back as one mapping.

Both recipes run the UNMODIFIED reference's add_examples (two classes, then a new class: _train_adaptive_head, then
_train_new_classes with EWC), _get_embeddings, predict (k = 3, k = 1) and predict_batch (k = 2) on seeded texts:
  short  36 texts of 4-13 class words and a quarter as many noise words, add_examples on 24 then 12, max_length 512; also
         the reference-trained head's top-1 on the training texts
  long   18 texts of 5-1600 words, a fifth of them noise, add_examples on 12 then 6, max_length 1024: some texts over 512
         tokens, some over 1024 (the tokenizer truncates them), some short (padded); ids and mask stored as int32
"""
import argparse
import dataclasses
import functools
import json
import os
import sys
from typing import Callable, Optional

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (sets up the reference / faiss-shim import paths)

sys.path.insert(0, os.path.join(mg.ROOT, "tests"))
import golden_npz  # noqa: E402

from oracle.eurobert_oracle import SPECIALS as EUROBERT_SPECIALS, eurobert_tokenizer  # noqa: E402

WORDS = [f"w{i}" for i in range(195)]       # words[0:120]: 40 per class; words[120:]: noise
CLASSES = ["sports", "finance", "cooking"]
TEST_CLASSES = ["sports", "finance", "cooking", "finance", "sports", "cooking"]
LONG_LENGTH = 1024
TRAIN_WORDS = [5, 40, 300, 600, 1100, 1600]        # long recipe: words per training text of each class (+ 2 specials)
TEST_WORDS = [700, 12, 1500, 520, 90, 1030]


# ------------------------------------------------------------------------------------------------ checkpoint builders
def _unigram(specials):
    """(piece, score) vocabulary of a unigram tokenizer: the specials, then one piece per word"""
    return [(s, 0.0) for s in specials] + [("▁" + w, -1.0 - 0.01 * i) for i, w in enumerate(WORDS)]


def _round_bf16(model):
    """every value rounded through bfloat16, so that the checkpoint compresses to under 1 MB per file"""
    with torch.no_grad():
        for p in model.parameters():
            p.copy_(p.bfloat16().float())


def minilm():
    """3-layer BERT with 4 heads of 32 (hidden 128), the head_dim of all-MiniLM-L6-v2, BGE-small and E5-small"""
    from transformers import BertConfig, BertModel, BertTokenizerFast
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS
    cfg = BertConfig(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=3, num_attention_heads=4,
                     intermediate_size=128, max_position_embeddings=64, type_vocab_size=2, pad_token_id=0)
    torch.manual_seed(4321)
    model = BertModel(cfg)
    mg.perturb(model, 98)
    with torch.no_grad():       # the constant part of the CLS row's input, as in make_golden._tiny_checkpoint
        model.embeddings.word_embeddings.weight[2].zero_()
        model.embeddings.position_embeddings.weight[0].zero_()
        model.embeddings.token_type_embeddings.weight.zero_()
    return mg.saved(model, BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}, do_lower_case=True), WORDS, vocab)


def mpnet():
    """3-layer MPNet (hidden 128, 2 heads of 64, 514 positions), the architecture of all-mpnet-base-v2; the
    relative-attention-bias table is drawn O(1) so that the bias visibly moves the embeddings"""
    from transformers import MPNetConfig, MPNetModel, MPNetTokenizer
    vocab = ["<s>", "<pad>", "</s>", "[UNK]", "<mask>"] + WORDS
    cfg = MPNetConfig(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=3, num_attention_heads=2,
                      intermediate_size=128, max_position_embeddings=514, layer_norm_eps=1e-5)
    torch.manual_seed(4321)
    model = MPNetModel(cfg)
    g = torch.Generator().manual_seed(97)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n == "encoder.relative_attention_bias.weight":
                p.copy_(torch.randn(p.shape, generator=g))
            else:
                mg.perturb_param(n, p, g)
        model.embeddings.word_embeddings.weight[0].zero_()         # <s> and its position row 2
        model.embeddings.position_embeddings.weight[2].zero_()
    return mg.saved(model, MPNetTokenizer(vocab={w: i for i, w in enumerate(vocab)}), WORDS, vocab)


def deberta():
    """3-layer DeBERTa-v3 (hidden 128, 2 heads of 64, 256 position buckets, share_att_key, norm_rel_ebd = layer_norm, no
    position or token-type table), the architecture of deberta-v3-* and mdeberta-v3-base; the relative embeddings are
    drawn O(1)"""
    from transformers import DebertaV2Config, DebertaV2Model, DebertaV2Tokenizer
    specials = ["[PAD]", "[CLS]", "[SEP]", "[UNK]", "[MASK]"]
    vocab = specials + WORDS
    cfg = DebertaV2Config(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=3, num_attention_heads=2,
                          intermediate_size=128, max_position_embeddings=512, type_vocab_size=0,
                          relative_attention=True, position_buckets=256, norm_rel_ebd="layer_norm", share_att_key=True,
                          pos_att_type=["p2c", "c2p"], position_biased_input=False, layer_norm_eps=1e-7, pad_token_id=0)
    torch.manual_seed(4321)
    model = DebertaV2Model(cfg)
    g = torch.Generator().manual_seed(97)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n == "encoder.rel_embeddings.weight":
                p.copy_(torch.randn(p.shape, generator=g))
            else:
                mg.perturb_param(n, p, g)
        model.embeddings.word_embeddings.weight[1].zero_()        # [CLS]
    return mg.saved(model, DebertaV2Tokenizer(vocab=_unigram(specials)), WORDS, vocab)


def modernbert(max_position_embeddings=512):
    """4-layer ModernBERT (hidden 128, 2 heads, both layer types twice, half-window 8 < the short recipe's sentences)"""
    from transformers import BertTokenizerFast, ModernBertConfig, ModernBertModel
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS
    cfg = ModernBertConfig(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=4, num_attention_heads=2,
                           intermediate_size=64, local_attention=16, max_position_embeddings=max_position_embeddings,
                           pad_token_id=0, cls_token_id=2, sep_token_id=3, bos_token_id=2, eos_token_id=3)
    torch.manual_seed(1234)
    model = ModernBertModel(cfg)
    g = torch.Generator().manual_seed(99)
    with torch.no_grad():
        for n, p in model.named_parameters():       # no biases; every weight but the norms is x2, not x3
            if "norm" in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            else:
                p.mul_(4.0 if "tok_embeddings" in n else 2.0)
        model.embeddings.tok_embeddings.weight[2].zero_()
    tok = BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}, do_lower_case=True)
    tok.model_input_names = ["input_ids", "attention_mask"]     # ModernBERT takes no token_type_ids
    return mg.saved(model, tok, WORDS, vocab)


def albert():
    """ALBERT with embedding_size 128 != hidden 256, 4 heads of 64, I 256, 3 effective layers sharing one group (as every
    published ALBERT does), "gelu_new"; AlbertTokenizer over a unigram vocabulary"""
    from transformers import AlbertConfig, AlbertModel, AlbertTokenizer
    specials = ["<pad>", "<unk>", "[CLS]", "[SEP]", "[MASK]"]
    vocab = specials + WORDS
    cfg = AlbertConfig(vocab_size=len(vocab), embedding_size=128, hidden_size=256, num_hidden_layers=3,
                       num_hidden_groups=1, inner_group_num=1, num_attention_heads=4, intermediate_size=256,
                       max_position_embeddings=128, type_vocab_size=2, hidden_act="gelu_new", pad_token_id=0)
    torch.manual_seed(4321)
    model = AlbertModel(cfg)
    mg.perturb(model, 97)
    with torch.no_grad():
        model.embeddings.word_embeddings.weight[2].zero_()        # [CLS]
    return mg.saved(model, AlbertTokenizer(vocab=_unigram(specials)), WORDS, vocab)


def electra():
    """the electra-small shape (embedding_size 128, hidden 256, 4 heads), 1 layer, I 256, erf GELU"""
    from transformers import ElectraConfig, ElectraModel, ElectraTokenizer
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS
    cfg = ElectraConfig(vocab_size=len(vocab), embedding_size=128, hidden_size=256, num_hidden_layers=1,
                        num_attention_heads=4, intermediate_size=256, max_position_embeddings=128,
                        type_vocab_size=2, hidden_act="gelu", pad_token_id=0)
    torch.manual_seed(4322)
    model = ElectraModel(cfg)
    mg.perturb(model, 98)
    with torch.no_grad():
        model.embeddings.word_embeddings.weight[2].zero_()
    return mg.saved(model, ElectraTokenizer(vocab={w: i for i, w in enumerate(vocab)}), WORDS, vocab)


def nomic():
    """NomicBERT (hidden 128, 2 heads of 64, 2 layers, SwiGLU I 256, RoPE theta 1000, 2048 positions)"""
    from transformers import BertTokenizerFast, NomicBertConfig, NomicBertModel
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS
    cfg = NomicBertConfig(vocab_size=len(vocab), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                          intermediate_size=256, max_position_embeddings=2048, type_vocab_size=2, pad_token_id=0)
    torch.manual_seed(1234)
    model = NomicBertModel(cfg)
    mg.perturb(model, 99)
    _round_bf16(model)
    with torch.no_grad():
        model.embeddings.word_embeddings.weight[2].zero_()
        model.embeddings.token_type_embeddings.weight.zero_()
    return mg.saved(model, BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}, do_lower_case=True), WORDS, vocab)


def _xlmr_pieces():
    return _unigram(["<s>", "<pad>", "</s>", "<unk>"]) + [("<mask>", 0.0)]


def jina3():
    """jina-embeddings-v3 (hidden 128, 2 heads, 2 layers, GELU I 256 with biases, RoPE theta 20000, 8194 positions) with
    the pooler, as AutoModel builds it (the reference never uses it)"""
    from transformers import JinaEmbeddingsV3Config, JinaEmbeddingsV3Model, XLMRobertaTokenizer
    pieces = _xlmr_pieces()
    cfg = JinaEmbeddingsV3Config(vocab_size=len(pieces), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                                 intermediate_size=256, max_position_embeddings=8194, type_vocab_size=1,
                                 layer_norm_eps=1e-5, pad_token_id=1, bos_token_id=0, eos_token_id=2,
                                 hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    torch.manual_seed(1234)
    model = JinaEmbeddingsV3Model(cfg)
    mg.perturb(model, 99)
    _round_bf16(model)
    with torch.no_grad():
        model.embeddings.word_embeddings.weight[0].zero_()       # <s>
        model.embeddings.token_type_embeddings.weight.zero_()
    return mg.saved(model, XLMRobertaTokenizer(vocab=pieces), WORDS, pieces)


def xlmr_long():
    """XLM-R (hidden 128, 2 heads of 64, 2 layers, no pooler) with the 8194-row position table of bge-m3 and
    snowflake-arctic-embed-l-v2.0; the rows past LONG_LENGTH + 2, never reached, are zero so that the table compresses"""
    from transformers import XLMRobertaConfig, XLMRobertaModel, XLMRobertaTokenizer
    pieces = _xlmr_pieces()
    cfg = XLMRobertaConfig(vocab_size=len(pieces), hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                           intermediate_size=128, max_position_embeddings=8194, type_vocab_size=1,
                           layer_norm_eps=1e-5, pad_token_id=1, bos_token_id=0, eos_token_id=2)
    torch.manual_seed(1234)
    model = XLMRobertaModel(cfg, add_pooling_layer=False)
    mg.perturb(model, 99)
    _round_bf16(model)
    with torch.no_grad():
        model.embeddings.word_embeddings.weight[0].zero_()         # <s>, its position pad_idx + 1, the token type
        model.embeddings.position_embeddings.weight[2].zero_()
        model.embeddings.position_embeddings.weight[LONG_LENGTH + 2:].zero_()
        model.embeddings.token_type_embeddings.weight.zero_()
    return mg.saved(model, XLMRobertaTokenizer(vocab=pieces), WORDS, pieces)


def eurobert():
    """EuroBERT (hidden 256, 4 heads of 64, 2 kv heads, 2 layers, SwiGLU I 512, RoPE theta 250000, 8192 positions) and
    oracle/eurobert_oracle.eurobert_tokenizer, which as the real one wraps every text in <|begin_of_text|> ...
    <|end_of_text|>, pads with <|end_of_text|> and returns no token_type_ids"""
    from transformers import EuroBertConfig, EuroBertModel
    vocab = EUROBERT_SPECIALS + WORDS
    cfg = EuroBertConfig(vocab_size=len(vocab), hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                         num_key_value_heads=2, intermediate_size=512, max_position_embeddings=8192,
                         rope_parameters={"rope_type": "default", "rope_theta": 250000.0}, bos_token_id=0,
                         eos_token_id=1, pad_token_id=1, mask_token_id=2)
    torch.manual_seed(1234)
    model = EuroBertModel(cfg)
    mg.perturb(model, 99)
    _round_bf16(model)
    with torch.no_grad():
        model.embed_tokens.weight[0].zero_()        # <|begin_of_text|>
    return mg.saved(model, eurobert_tokenizer(WORDS), WORDS, vocab)


def eurobert_pieces():
    """eurobert() with its vocabulary as (piece, 0.0) pairs, the form golden_classifier_eurobert_long has it in"""
    checkpoint = eurobert()
    return checkpoint._replace(vocab=[(p, 0.0) for p in checkpoint.vocab])


# ------------------------------------------------------------------------------------------------ recipes
def _sentence(rng, words, label, n_own, n_noise):
    first = 40 * CLASSES.index(label)
    own = rng.choice(words[first:first + 40], size=n_own, replace=True)
    noise = rng.choice(words[120:], size=n_noise, replace=True)
    toks = list(own) + list(noise)
    rng.shuffle(toks)
    return " ".join(toks)


def _record(checkpoint, texts, labels, test_texts, split, config):
    """the reference's run on the saved checkpoint: outputs to store, and the trained classifier"""
    from adaptive_classifier import AdaptiveClassifier
    torch.manual_seed(0)
    np.random.seed(0)
    clf = AdaptiveClassifier(checkpoint.dir, device="cpu", use_onnx=False, config=config)
    clf.add_examples(texts[:split], labels[:split])     # sports + finance -> _train_adaptive_head
    clf.add_examples(texts[split:], labels[split:])     # new class cooking -> _train_new_classes (+EWC)
    emb_train = torch.stack(clf._get_embeddings(texts)).numpy()
    emb_test = torch.stack(clf._get_embeddings(test_texts)).numpy()
    enc = clf.tokenizer(texts + test_texts, max_length=clf.config.max_length, truncation=True, padding=True,
                        return_tensors="pt")
    label_names = [clf.id_to_label[i] for i in range(len(clf.id_to_label))]

    def pack(preds, k):
        L = np.full((len(preds), k), -1, dtype=np.int64)
        S = np.zeros((len(preds), k), dtype=np.float64)
        for i, p in enumerate(preds):
            for j, (l, s) in enumerate(p):
                L[i, j] = label_names.index(l)
                S[i, j] = s
        return L, S

    pl, ps = pack([clf.predict(t, k=3) for t in test_texts], 3)
    p1l, p1s = pack([clf.predict(t, k=1) for t in test_texts], 1)
    pbl, pbs = pack(clf.predict_batch(test_texts, k=2), 2)
    vocab = checkpoint.vocab
    if isinstance(vocab[0], str):
        out = dict(vocab=np.array(vocab))
    else:
        out = dict(vocab_pieces=np.array([p for p, _ in vocab]), vocab_scores=np.array([s for _, s in vocab]))
    out.update(
        texts=np.array(texts), labels=np.array(labels), test_texts=np.array(test_texts),
        label_names=np.array(label_names), input_ids=enc["input_ids"].numpy(), attention_mask=enc["attention_mask"].numpy(),
        emb_train=emb_train, emb_test=emb_test,
        prototypes=np.stack([clf.memory.prototypes[l].numpy() for l in sorted(clf.memory.prototypes)]),
        proto_labels=np.array(sorted(clf.memory.prototypes)), training_history=json.dumps(clf.training_history),
        train_steps=clf.train_steps, pred_labels=pl, pred_scores=ps, pred_k1_labels=p1l, pred_k1_scores=p1s,
        predb_labels=pbl, predb_scores=pbs, bert_config=json.dumps(checkpoint.config.to_dict()),
        **{"head_" + k: v.detach().numpy() for k, v in clf.adaptive_head.state_dict().items()})
    return out, clf


def short(checkpoint, seed):
    rng = np.random.default_rng(seed)

    def sentence(label, n):
        return _sentence(rng, checkpoint.words, label, n, max(1, n // 4))

    texts, labels = [], []
    for label in CLASSES:
        for _ in range(12):
            texts.append(sentence(label, int(rng.integers(4, 14))))
            labels.append(label)
    test_texts = [sentence(label, 9) for label in TEST_CLASSES]
    out, clf = _record(checkpoint, texts, labels, test_texts, split=24, config=None)
    names = out["label_names"].tolist()
    out["train_top1"] = np.array([names.index(p[0][0]) for p in clf.predict_batch(texts, k=1)])
    return out


def long(checkpoint, seed):
    rng = np.random.default_rng(seed)

    def sentence(label, n):
        return _sentence(rng, checkpoint.words, label, n - max(1, n // 5), max(1, n // 5))

    texts, labels = [], []
    for label in CLASSES:
        for n in TRAIN_WORDS:
            texts.append(sentence(label, n))
            labels.append(label)
    test_texts = [sentence(label, n) for label, n in zip(TEST_CLASSES, TEST_WORDS)]
    out, clf = _record(checkpoint, texts, labels, test_texts, split=12, config={"max_length": LONG_LENGTH})
    ids, mask = out["input_ids"], out["attention_mask"]
    lens = mask.sum(1)
    assert ids.shape[1] == LONG_LENGTH and (lens > 512).sum() >= 6 and (lens < 64).sum() >= 3, lens
    assert not (ids == clf.tokenizer.unk_token_id).any(), "a word fell back to the unknown token"
    out.update(input_ids=ids.astype(np.int32), attention_mask=mask.astype(np.int32), max_length=LONG_LENGTH)
    return out


# ------------------------------------------------------------------------------------------------ the table
@dataclasses.dataclass
class Row:
    name: str
    checkpoint: Callable                    # () -> make_golden.Checkpoint
    recipe: Callable                        # short or long
    seed: int                               # of the texts
    parts: Optional[Callable] = None        # how make_golden.save stores the checkpoint's tensors ...
    weights_from: Optional[str] = None      # ... or the row whose tensors in tests/golden equal this row's checkpoint

    @property
    def fixture(self):
        return "golden_classifier" + ("" if self.name == "bert" else "_" + self.name)


_LAYERS_1_2 = mg.by_prefix("bert_encoder.layer.1.", "bert_encoder.layer.2.")

FAMILIES = [
    Row("bert", mg._tiny_checkpoint, short, 7, mg.by_prefix("bert_encoder.layer.1.")),
    Row("minilm", minilm, short, 7, _LAYERS_1_2),
    Row("mpnet", mpnet, short, 7, _LAYERS_1_2),
    Row("deberta", deberta, short, 7, _LAYERS_1_2),
    Row("deberta_long", deberta, long, 16, weights_from="deberta"),
    Row("modernbert", modernbert, short, 7, mg.by_prefix("bert_layers.2.", "bert_layers.3.")),
    Row("modernbert_long", functools.partial(modernbert, max_position_embeddings=8192), long, 15,
        weights_from="modernbert"),
    Row("albert", albert, short, 7, mg.greedy(2, with_outputs=True)),
    Row("electra", electra, short, 7, mg.greedy(2, with_outputs=True)),
    Row("nomic", nomic, short, 7, mg.greedy(2, with_outputs=True)),
    Row("jina3", jina3, long, 15, mg.greedy(2, with_outputs=True)),
    Row("xlmr_long", xlmr_long, long, 15, mg.by_prefix("bert_encoder.layer.1.")),
    Row("eurobert", eurobert, short, 7, mg.greedy(4)),
    Row("eurobert_long", eurobert_pieces, long, 15, weights_from="eurobert"),
]
ROWS = {row.name: row for row in FAMILIES}


def generate(names, out):
    """runs the named rows, in FAMILIES order (a row with weights_from after the row it reads)"""
    for row in FAMILIES:
        if row.name not in names:
            continue
        checkpoint = row.checkpoint()
        weights = {"bert_" + k: v.detach().numpy() for k, v in checkpoint.model.state_dict().items()}
        if row.weights_from is not None:
            stored = golden_npz.load(ROWS[row.weights_from].fixture)
            stored = {k: stored[k] for k in stored.files if k.startswith("bert_") and k != "bert_config"}
            assert weights.keys() == stored.keys() and all(np.array_equal(weights[k], stored[k]) for k in weights), \
                f"the {row.name} checkpoint differs from the one stored with {ROWS[row.weights_from].fixture}"
            weights = {}
        mg.save(out, row.fixture, {**row.recipe(checkpoint, row.seed), **weights}, row.parts)


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("rows", nargs="*", choices=list(ROWS), help="rows to run (default: all)")
    ap.add_argument("--out", default=mg.OUT, help="output directory (default: tests/golden)")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    generate(args.rows or list(ROWS), args.out)
