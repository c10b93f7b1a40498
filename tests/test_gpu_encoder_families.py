"""GPU tests every encoder family shares, driven by FAMILIES: one row per golden classifier run of the reference
(tests/golden/golden_classifier_<name>.npz, made by the same row of oracle/make_golden_encoders.py from the unmodified
reference).

  * the drop-in classifier on the tiny seeded checkpoint and tokenizer the reference ran on: tokenized ids, embeddings,
    label ids, training history, prototypes; then predict (k = 3, k = 1) and predict_batch (k = 2) with the
    reference-trained head, before and after a save / load round trip
  * the CUDA-graph replay of the pipeline step against the eager step, and the replayed embedding against the family's
    fp32 oracle where the row gives one
  * AdaptiveClassifier on a fabricated local checkpoint directory: add_examples, embeddings against the oracle, predict,
    predict_batch and a save / load round trip

Each family's encoder-level tests stay in its tests/test_gpu_<family>.py."""
import dataclasses
import json
from typing import Callable, Optional

import numpy as np
import pytest
import torch

import golden_npz
from oracle import albert_oracle as ao
from oracle import deberta_oracle as do
from oracle import encoder_oracle as eo
from oracle import eurobert_oracle as euo
from oracle import mpnet_oracle as mo
from test_albert_cpu import albert_ids, albert_model, electra_model
from test_deberta_cpu import deberta_ids, deberta_model, deberta_tokenizer_words
from test_eurobert_cpu import tiny_model as eurobert_model
from test_gpu_eurobert import SHAPE_BOUND
from test_gpu_minilm import MINILM
from test_gpu_modernbert import _ids as modernbert_ids, _model as modernbert_model
from test_gpu_parity import _encoder, _head, _synthetic_index
from test_gpu_xlmr_long import _ids as xlmr_ids, _tiny_xlmr
from test_mpnet_cpu import mpnet_model
from test_rotary_cpu import tiny_model as rotary_model

pytestmark = pytest.mark.gpu

WIDE = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=1000)
LONG = dict(max_length=1024, b200_max_tokens=4096)      # a 4096-token workspace splits the 1024-token batches
SCHEDULE = [3, 3, 3, 3, 8, 8, 8, 1, 1]                 # pipeline batch sizes: partial, full, single, at Bmax 8


def _sd(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


# ------------------------------------------------------------------------------------------------ tokenizers
def _wordpiece(golden, type_ids=True):
    from transformers import BertTokenizerFast
    tok = BertTokenizerFast(vocab={w: i for i, w in enumerate(golden["vocab"].tolist())}, do_lower_case=True)
    if not type_ids:                                     # ModernBERT takes no token_type_ids
        tok.model_input_names = ["input_ids", "attention_mask"]
    return tok


def _albert_unigram(golden):
    from transformers import AlbertTokenizer
    vocab = golden["vocab"].tolist()
    return AlbertTokenizer(vocab=[(s, 0.0) for s in vocab[:5]] + [("▁" + w, -1.0 - 0.01 * i) for i, w in enumerate(vocab[5:])])


def _electra(golden):
    from transformers import ElectraTokenizer
    return ElectraTokenizer(vocab={w: i for i, w in enumerate(golden["vocab"].tolist())})


def _mpnet(golden):
    from transformers import MPNetTokenizer
    return MPNetTokenizer(vocab={w: i for i, w in enumerate(golden["vocab"].tolist())})


def _deberta_words(golden):
    return deberta_tokenizer_words(golden["vocab"].tolist()[5:])


def _xlmr_pieces(golden):
    from transformers import XLMRobertaTokenizer
    return XLMRobertaTokenizer(vocab=[(p, float(s)) for p, s in zip(golden["vocab_pieces"].tolist(),
                                                                    golden["vocab_scores"].tolist())])


def _eurobert(golden):
    vocab = golden["vocab"].tolist() if "vocab" in golden else golden["vocab_pieces"].tolist()
    assert vocab[:len(euo.SPECIALS)] == euo.SPECIALS
    return euo.eurobert_tokenizer(vocab[len(euo.SPECIALS):])


def _no_pooler(config):
    from transformers import AutoModel
    return AutoModel.from_config(config, add_pooling_layer=False)


# ------------------------------------------------------------------------------------------------ local checkpoints
def _minilm_local(words):
    from transformers import BertConfig, BertModel, BertTokenizerFast
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
    torch.manual_seed(77)
    m = BertModel(BertConfig(vocab_size=len(vocab), num_hidden_layers=6, max_position_embeddings=64, **MINILM)).eval()
    with torch.no_grad():
        m.embeddings.word_embeddings.weight.mul_(4.0)
        m.embeddings.word_embeddings.weight[2].zero_()
        m.embeddings.position_embeddings.weight[0].zero_()
        m.embeddings.token_type_embeddings.weight.zero_()
    return m, BertTokenizerFast(vocab={w: i for i, w in enumerate(vocab)}, do_lower_case=True)


def _mpnet_local(words):
    from transformers import MPNetTokenizer
    vocab = ["<s>", "<pad>", "</s>", "[UNK]", "<mask>"] + words
    m = mpnet_model(seed=77, num_hidden_layers=4, **{**WIDE, "vocab_size": len(vocab)})
    with torch.no_grad():
        m.embeddings.word_embeddings.weight.mul_(4.0)
        m.embeddings.word_embeddings.weight[0].zero_()
    return m, MPNetTokenizer(vocab={w: i for i, w in enumerate(vocab)})


def _deberta_local(words):
    tok = deberta_tokenizer_words(words)
    m = deberta_model(seed=77, num_hidden_layers=4, proj_scale=2.0, **{**WIDE, "vocab_size": 5 + len(words)})
    with torch.no_grad():
        m.embeddings.word_embeddings.weight.mul_(4.0)
        m.embeddings.word_embeddings.weight[1].zero_()
    return m, tok


def _albert_local(words):
    from transformers import AlbertTokenizer
    specials = ["<pad>", "<unk>", "[CLS]", "[SEP]", "[MASK]"]
    tok = AlbertTokenizer(vocab=[(s, 0.0) for s in specials] + [("▁" + w, -1.0 - 0.01 * i) for i, w in enumerate(words)])
    m = albert_model(seed=77, num_hidden_layers=12, scale=1.0, **{**WIDE, "vocab_size": 5 + len(words)})
    with torch.no_grad():
        m.embeddings.word_embeddings.weight.mul_(4.0)
        m.embeddings.word_embeddings.weight[2].zero_()
    return m, tok


def _electra_local(words):
    from transformers import ElectraTokenizer
    tok = ElectraTokenizer(vocab={w: i for i, w in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words)})
    m = electra_model(seed=78, num_hidden_layers=12, intermediate_size=1024, scale=1.0, vocab_size=5 + len(words))
    with torch.no_grad():
        m.embeddings.word_embeddings.weight.mul_(4.0)
        m.embeddings.word_embeddings.weight[2].zero_()
    return m, tok


def _factorized_oracle(m, enc):
    return ao.factorized_forward_cls(_sd(m), enc["input_ids"], enc["attention_mask"], m.config,
                                     token_type_ids=enc.get("token_type_ids"))


# ------------------------------------------------------------------------------------------------ the table
@dataclasses.dataclass
class Pipe:
    """a CUDA-graph pipeline over a seeded encoder: model() builds it, ids(B, S, seed) makes a batch, oracle(model, ids)
    gives the unit CLS rows the replayed embedding is held to (None: no oracle check)"""
    model: Callable
    ids: Callable
    S: list
    oracle: Optional[Callable] = None
    encoder: Callable = lambda cabi, m, max_tokens: cabi.Encoder.from_hf(m, max_tokens=max_tokens)


@dataclasses.dataclass
class Local:
    """checkpoint(words) -> (HF model, tokenizer) to save as a local directory; oracle(model, tokenizer output) -> unit
    CLS rows"""
    checkpoint: Callable
    oracle: Callable


@dataclasses.dataclass
class Family:
    golden: str
    tokenizer: Callable
    weights_from: Optional[str] = None      # a long run shares the checkpoint of its short run
    model: Optional[Callable] = None        # config -> HF model; AutoModel.from_config by default
    config: dict = dataclasses.field(default_factory=dict)     # AdaptiveClassifier config
    split: int = 24                         # add_examples(texts[:split]) then add_examples(texts[split:])
    abs_bound: Optional[float] = 3e-4       # embeddings and prototypes: max abs error ...
    row_bound: float = 1e-3                 # ... and max row error norm against the reference
    pipe: Optional[Pipe] = None
    local: Optional[Local] = None

    @property
    def name(self):
        return self.golden[len("golden_classifier_"):]


def _rand_ids(B, S, seed):
    return torch.randint(5, 300, (B, S), generator=torch.Generator().manual_seed(seed))


_DEBERTA_PIPE = dict(model=lambda: deberta_model(num_hidden_layers=3, **WIDE),
                     ids=lambda B, S, seed: deberta_ids(B, S, False, vocab=1000, seed=seed)[0],
                     oracle=lambda m, ids: do.deberta_forward_cls(_sd(m), ids, None, m.config))
_MODERNBERT = dict(hidden_size=768, num_attention_heads=12, intermediate_size=1152, num_hidden_layers=3, vocab_size=1000)

FAMILIES = [
    Family("golden_classifier_minilm", _wordpiece,
           pipe=Pipe(model=lambda: eo.make_bert_state_dict(1234, num_hidden_layers=3, **MINILM)[:2],
                     ids=lambda B, S, seed: eo.synthetic_ids(B, S, seed=seed), S=[64],
                     oracle=lambda m, ids: eo.encoder_forward_cls(m[0], ids, None, num_heads=12),
                     encoder=lambda cabi, m, max_tokens: _encoder(cabi, *m, max_tokens=max_tokens)),
           local=Local(_minilm_local, lambda m, enc: eo.encoder_forward_cls(
               _sd(m), enc["input_ids"], enc["attention_mask"], num_heads=12, ln_eps=m.config.layer_norm_eps))),
    Family("golden_classifier_mpnet", _mpnet,
           pipe=Pipe(model=lambda: mpnet_model(num_hidden_layers=3, **WIDE),
                     ids=lambda B, S, seed: eo.synthetic_ids(B, S, vocab=1000, seed=seed, arch="roberta"), S=[64],
                     oracle=lambda m, ids: mo.mpnet_forward_cls(_sd(m), ids, None, num_heads=12, ln_eps=1e-5)),
           local=Local(_mpnet_local, lambda m, enc: mo.mpnet_forward_cls(
               _sd(m), enc["input_ids"], enc["attention_mask"], num_heads=12, ln_eps=1e-5))),
    Family("golden_classifier_deberta", _deberta_words, pipe=Pipe(**_DEBERTA_PIPE, S=[64]),
           local=Local(_deberta_local, lambda m, enc: do.deberta_forward_cls(
               _sd(m), enc["input_ids"], enc["attention_mask"], m.config))),
    Family("golden_classifier_deberta_long", _deberta_words, weights_from="golden_classifier_deberta",
           config=dict(max_length=1024), split=12, pipe=Pipe(**_DEBERTA_PIPE, S=[1024])),
    Family("golden_classifier_albert", _albert_unigram,
           pipe=Pipe(model=lambda: albert_model(num_hidden_layers=3, scale=1.0, **WIDE),
                     ids=lambda B, S, seed: albert_ids(B, S, False, vocab=1000, seed=seed)[0], S=[64],
                     oracle=lambda m, ids: ao.factorized_forward_cls(_sd(m), ids, None, m.config)),
           local=Local(_albert_local, _factorized_oracle)),
    Family("golden_classifier_electra", _electra, local=Local(_electra_local, _factorized_oracle)),
    Family("golden_classifier_modernbert", lambda g: _wordpiece(g, type_ids=False),
           pipe=Pipe(model=lambda: modernbert_model(3, **_MODERNBERT),
                     ids=lambda B, S, seed: modernbert_ids(B, S, 1000, seed, False)[0], S=[160])),
    Family("golden_classifier_modernbert_long", lambda g: _wordpiece(g, type_ids=False),
           weights_from="golden_classifier_modernbert", config=LONG, split=12,
           pipe=Pipe(model=lambda: modernbert_model(3, local_attention=128, max_position_embeddings=8192, **_MODERNBERT),
                     ids=lambda B, S, seed: modernbert_ids(B, S, 1000, seed, False)[0], S=[1024])),
    Family("golden_classifier_nomic", _wordpiece,
           pipe=Pipe(model=lambda: rotary_model("nomic", seed=3, layers=3), ids=_rand_ids, S=[128])),
    Family("golden_classifier_jina3", _xlmr_pieces, config=LONG, split=12,
           pipe=Pipe(model=lambda: rotary_model("jina", seed=3, layers=3), ids=_rand_ids, S=[1024])),
    Family("golden_classifier_eurobert", _eurobert, abs_bound=None, row_bound=SHAPE_BOUND,
           pipe=Pipe(model=lambda: eurobert_model(seed=3, layers=3, kv=2), ids=_rand_ids, S=[128])),
    Family("golden_classifier_eurobert_long", _eurobert, weights_from="golden_classifier_eurobert", config=LONG, split=12,
           abs_bound=None, row_bound=SHAPE_BOUND,
           pipe=Pipe(model=lambda: eurobert_model(seed=3, layers=3, kv=2), ids=_rand_ids, S=[1024])),
    Family("golden_classifier_xlmr_long", _xlmr_pieces, model=_no_pooler, config=LONG, split=12,
           pipe=Pipe(model=lambda: _tiny_xlmr(3, layers=3), ids=lambda B, S, seed: xlmr_ids(B, S, 300, seed, False)[0],
                     S=[1024])),
]


# ------------------------------------------------------------------------------------------------ golden classifier
def golden_checkpoint(golden_name, d):
    """saves the tiny seeded checkpoint and the tokenizer of a golden run to directory d; returns the run"""
    from transformers import AutoConfig, AutoModel
    family = next(f for f in FAMILIES if f.golden == golden_name)
    golden = golden_npz.load(family.golden, weights_from=family.weights_from)
    cfgd = json.loads(str(golden["bert_config"]))
    config = AutoConfig.for_model(cfgd["model_type"], **{k: v for k, v in cfgd.items()
                                                         if k not in ("model_type", "transformers_version", "architectures")})
    m = (family.model or AutoModel.from_config)(config)
    m.load_state_dict({k[5:]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith("bert_") and k != "bert_config"})
    m.save_pretrained(d)
    family.tokenizer(golden).save_pretrained(d)
    return golden


@pytest.fixture(scope="module", params=FAMILIES, ids=lambda f: f.name)
def golden_run(cabi, request, tmp_path_factory):
    """AdaptiveClassifier on the local checkpoint directory the reference ran on (AutoModel / AutoTokenizer)"""
    import adaptive_classifier_b200 as acb
    family = request.param
    d = str(tmp_path_factory.mktemp(family.name))
    golden = golden_checkpoint(family.golden, d)
    texts, labels = golden["texts"].tolist(), golden["labels"].tolist()
    np.random.seed(0)
    clf = acb.AdaptiveClassifier(d, device="cuda", config=dict(family.config))
    clf.add_examples(texts[:family.split], labels[:family.split])
    clf.add_examples(texts[family.split:], labels[family.split:])
    return family, golden, clf


def _close(out, ref, family):
    e = out - ref
    if family.abs_bound is not None:
        assert np.abs(e).max() < family.abs_bound, np.abs(e).max()
    assert np.linalg.norm(e, axis=1).max() < family.row_bound, np.linalg.norm(e, axis=1).max()


def test_golden_embeddings_labels_and_prototypes_match_reference(golden_run):
    family, golden, trained = golden_run
    texts, tests_ = golden["texts"].tolist(), golden["test_texts"].tolist()
    ids, _, tt = trained._tokenize(texts + tests_)
    assert torch.equal(ids.long(), torch.from_numpy(golden["input_ids"]).long())     # truncation and padding as the reference
    assert (tt is None) == ("token_type_ids" not in trained.tokenizer.model_input_names)
    if "max_length" in golden:
        assert ids.shape[1] > 512
    for part, key in ((texts, "emb_train"), (tests_, "emb_test")):
        emb = torch.stack(trained._get_embeddings(part)).numpy()
        assert emb.shape == golden[key].shape
        _close(emb, golden[key], family)
    names = golden["label_names"].tolist()
    assert [trained.id_to_label[i] for i in range(len(names))] == names
    if "training_history" in golden:
        assert trained.training_history == json.loads(str(golden["training_history"]))
    assert golden["proto_labels"].tolist() == sorted(trained.memory.prototypes)
    protos = np.stack([trained.memory.prototypes[l].numpy() for l in sorted(trained.memory.prototypes)])
    _close(protos, golden["prototypes"], family)


def _cmp(preds, L, S, names):
    for p, l_row, s_row in zip(preds, L, S):
        exp = [(names[i], s) for i, s in zip(l_row.tolist(), s_row.tolist()) if i >= 0]
        assert [l for l, _ in p] == [l for l, _ in exp], (p, exp)
        assert np.allclose([s for _, s in p], [s for _, s in exp], atol=1e-3), (p, exp)


def _same(preds, preds2):
    for p, p2 in zip(preds, preds2):
        assert [l for l, _ in p2] == [l for l, _ in p] and np.allclose([s for _, s in p2], [s for _, s in p], atol=1e-5)


def test_golden_predictions_match_reference_and_survive_save_load(golden_run, tmp_path):
    """predict / predict_batch with the reference-trained head; after a save / load round trip the same answers"""
    import adaptive_classifier_b200 as acb
    _, golden, trained = golden_run
    names = golden["label_names"].tolist()
    own_head = {k: v.detach().clone() for k, v in trained.adaptive_head.state_dict().items()}
    trained.adaptive_head.load_state_dict({k[5:]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith("head_")})
    tests_ = golden["test_texts"].tolist()
    try:
        top3 = [trained.predict(t, k=3) for t in tests_]
        _cmp(top3, golden["pred_labels"], golden["pred_scores"], names)
        _cmp([trained.predict(t, k=1) for t in tests_], golden["pred_k1_labels"], golden["pred_k1_scores"], names)
        batch = trained.predict_batch(tests_, k=2)
        _cmp(batch, golden["predb_labels"], golden["predb_scores"], names)
        out = str(tmp_path / "saved")
        trained.save(out)
        clf2 = acb.AdaptiveClassifier.load(out, device="cuda")
        assert clf2.label_to_id == trained.label_to_id and clf2.config.max_length == trained.config.max_length
        top3_2, batch_2 = [clf2.predict(t, k=3) for t in tests_], clf2.predict_batch(tests_, k=2)
        _cmp(top3_2, golden["pred_labels"], golden["pred_scores"], names)
        _cmp(batch_2, golden["predb_labels"], golden["predb_scores"], names)
        _same(top3, top3_2)
        _same(batch, batch_2)
    finally:
        trained.adaptive_head.load_state_dict(own_head)


# ------------------------------------------------------------------------------------------------ pipeline
@pytest.mark.parametrize("family,S", [pytest.param(f, S, id=f"{f.name}-{S}") for f in FAMILIES if f.pipe for S in f.pipe.S])
def test_pipeline_host_step_replayed_as_a_cuda_graph_equals_the_eager_step(cabi, family, S):
    """3-layer encoder, prototypes and head as wide as the encoder: the captured host step replays like the device step"""
    p = family.pipe
    m = p.model()
    Bmax, N, C, k = 8, 3000, 20, 5
    enc = p.encoder(cabi, m, Bmax * S)
    P, _ = _synthetic_index(N, enc.hidden, C)
    _, pg = _head(enc.hidden, C)
    row_class = (torch.arange(N) % C).to(torch.int32).cuda()
    pl = cabi.Pipeline(enc, P.cuda(), Bmax, S, k, head=pg, row_class=row_class)
    for rep, B in enumerate(SCHEDULE):
        ids = p.ids(B, S, 100 + rep).to(torch.int32)
        oc_h, osc_h = pl.predict_host(ids.pin_memory())
        oc_h, osc_h = oc_h.clone(), osc_h.clone()
        oc, osc = pl.predict_device(ids.cuda())
        torch.cuda.synchronize()
        assert torch.equal(oc.cpu(), oc_h) and torch.equal(osc.cpu(), osc_h), (rep, B)
    if p.oracle is not None:
        emb, _, _ = pl.debug_views(1)                   # the last step's single sequence
        ref = p.oracle(m, p.ids(1, S, 100 + len(SCHEDULE) - 1))
        assert (emb.cpu() - ref).norm(dim=1).max() < 1e-3
    pl.close(); enc.close()


# ------------------------------------------------------------------------------------------------ local checkpoint
@pytest.mark.parametrize("family", [pytest.param(f, id=f.name) for f in FAMILIES if f.local])
def test_adaptive_classifier_on_a_local_checkpoint(cabi, tmp_path, family):
    """AdaptiveClassifier on a fabricated local checkpoint directory (loaded through AutoModel / AutoTokenizer):
    add_examples, predict, predict_batch and a save / load round trip; the embeddings equal the fp32 oracle's"""
    import adaptive_classifier_b200 as acb
    words = [f"w{i}" for i in range(195)]
    m, tok = family.local.checkpoint(words)
    H = m.config.hidden_size
    d = str(tmp_path / family.name)
    m.save_pretrained(d)
    tok.save_pretrained(d)
    rng = np.random.default_rng(3)
    classes = {"a": words[0:60], "b": words[60:120], "c": words[120:180]}
    texts, labels = [], []
    for lab, ws in classes.items():
        for _ in range(8):
            texts.append(" ".join(rng.choice(ws, size=int(rng.integers(5, 12)))))
            labels.append(lab)
    np.random.seed(0)
    clf = acb.AdaptiveClassifier(d, device="cuda")
    assert clf.embedding_dim == H
    clf.add_examples(texts[:16], labels[:16])
    clf.add_examples(texts[16:], labels[16:])
    emb = torch.stack(clf._get_embeddings(texts[:6]))
    enc = clf.tokenizer(texts[:6], max_length=512, truncation=True, padding=True, return_tensors="pt")
    assert (emb - family.local.oracle(m, enc)).norm(dim=1).max() < 1e-3
    queries = [" ".join(rng.choice(ws, size=9)) for ws in classes.values()]
    single = [clf.predict(q, k=3) for q in queries]
    batch = clf.predict_batch(queries, k=3)
    assert len(batch) == len(queries)
    for p in single + batch:
        assert 1 <= len(p) <= 3 and {l for l, _ in p} <= {"a", "b", "c"} and abs(sum(s for _, s in p) - 1.0) < 1e-5
    out = str(tmp_path / "saved")
    clf.save(out)
    clf2 = acb.AdaptiveClassifier.load(out, device="cuda")
    assert clf2.embedding_dim == H and clf2.label_to_id == clf.label_to_id
    _same(single + batch, [clf2.predict(q, k=3) for q in queries] + clf2.predict_batch(queries, k=3))
