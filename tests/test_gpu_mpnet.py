"""GPU tests of the MPNet encoders (all-mpnet-base-v2, multi-qa-mpnet-base-*, paraphrase-mpnet-base-v2: the post-LN BERT
block with RoBERTa positions and a relative position bias on every layer's attention scores) against the fp32 oracle of
oracle/mpnet_oracle.py (pinned to HF MPNetModel by tests/test_mpnet_cpu.py), HF itself on the CPU, and the reference's own
classifier outputs on the golden MPNet checkpoint; then the CUDA-graph pipeline step and the drop-in classifier."""
import json

import numpy as np
import pytest
import torch

import golden_npz
from oracle import encoder_oracle as eo
from oracle import mpnet_oracle as mo
from test_gpu_minilm import _check_cls
from test_gpu_parity import _head, _synthetic_index
from test_mpnet_cpu import mpnet_ids, mpnet_model

pytestmark = pytest.mark.gpu

WIDE = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=1000)


def _mpnet_encoder(cabi, m, max_tokens, cls_only=True):
    sd, dims = cabi.mpnet_to_bert_state_dict(dict(m.state_dict()), m.config)
    return cabi.Encoder(sd, arch="mpnet", max_tokens=max_tokens, cls_only=cls_only, **dims)


def _hf_sd(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


# ------------------------------------------------------------------------------------------------ encoder
@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("B,S,pad", [(3, 16, False), (5, 77, True), (4, 128, False), (3, 129, False), (3, 200, True),
                                     (2, 384, False), (1, 512, False)])
def test_mpnet_encoder_matches_oracle(cabi, B, S, pad, cls_only):
    """2 x 768, 12 heads of 64, O(1) bias table and perturbed LayerNorms; S <= 128 runs attention_kernel<64, ScoreRelBias>,
    longer sequences attention_stream_kernel<64, ScoreRelBias>.  cls_only off also compares the whole last hidden state
    (bounds of test_gpu_parity.py::test_encoder_with_nontrivial_layernorms_matches_oracle and ::test_encoder_long_sequences)"""
    m = mpnet_model(num_hidden_layers=2, **WIDE)
    ids, mask = mpnet_ids(B, S, pad, vocab=WIDE["vocab_size"])
    ref, ref_hidden = mo.mpnet_forward_cls(_hf_sd(m), ids, mask, num_heads=12, ln_eps=1e-5, return_hidden=True)
    enc = _mpnet_encoder(cabi, m, B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    e = out - ref
    assert e.abs().max() < 3e-4 and e.norm(dim=1).max() < 1e-3, (e.abs().max(), e.norm(dim=1).max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5
    if not cls_only:
        hidden = enc.last_hidden(B, S).cpu()
        keep = mask.bool()
        assert (hidden.view(B, S, -1)[keep] - ref_hidden[keep]).abs().max() < 5e-3
    enc.close()


def test_mpnet_base_at_the_benched_batch_matches_oracle_on_sampled_rows(cabi):
    """the all-mpnet-base-v2 shape (workload.mpnet_base, bias table scaled to O(1)) at B = 512 x S = 128: 8 sampled sequences
    against the fp32 CPU oracle"""
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.mpnet_base(1234)
    with torch.no_grad():
        m.encoder.relative_attention_bias.weight.mul_(50.0)
    B, S = 512, 128
    ids = eo.synthetic_ids(B, S, vocab=cfg.vocab_size, arch="roberta")
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda()).cpu()
    sel = torch.tensor([0, 1, 63, 127, 128, 300, 510, 511])
    ref = mo.mpnet_forward_cls(_hf_sd(m), ids[sel], None, num_heads=12, ln_eps=cfg.layer_norm_eps)
    e = out[sel] - ref
    assert e.norm(dim=1).max() < 1e-3 and e.abs().max() < 2e-4, (e.norm(dim=1).max(), e.abs().max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5 and bool(torch.isfinite(out).all())
    enc.close()


def test_mpnet_through_from_hf_matches_hf(cabi):
    """a seeded MPNetModel through Encoder.from_hf, against HF on the CPU"""
    m = mpnet_model(seed=11, num_hidden_layers=3, **WIDE)
    ids, mask = mpnet_ids(4, 150, True, vocab=WIDE["vocab_size"])
    with torch.no_grad():
        ref = torch.nn.functional.normalize(m(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=4 * 150)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check_cls(out, ref)
    enc.close()


# ------------------------------------------------------------------------------------------------ golden classifier
@pytest.fixture(scope="module")
def golden():
    return golden_npz.load("golden_classifier_mpnet")


@pytest.fixture(scope="module")
def trained(cabi, golden, tmp_path_factory):
    """the tiny seeded 2-head x 64 MPNet checkpoint + vocab the reference ran on, driven through the drop-in classifier"""
    from transformers import MPNetConfig, MPNetModel, MPNetTokenizer
    import adaptive_classifier_b200 as acb
    d = str(tmp_path_factory.mktemp("golden_mpnet"))
    cfg = MPNetConfig(**{k: v for k, v in json.loads(str(golden["bert_config"])).items()
                         if k in ("vocab_size", "hidden_size", "num_hidden_layers", "num_attention_heads", "intermediate_size",
                                  "max_position_embeddings", "layer_norm_eps")})
    m = MPNetModel(cfg)
    m.load_state_dict({k[5:]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith("bert_") and k != "bert_config"})
    m.save_pretrained(d)
    MPNetTokenizer(vocab={w: i for i, w in enumerate(golden["vocab"].tolist())}).save_pretrained(d)
    texts, labels = golden["texts"].tolist(), golden["labels"].tolist()
    np.random.seed(0)
    clf = acb.AdaptiveClassifier(d, device="cuda")
    clf.add_examples(texts[:24], labels[:24])
    clf.add_examples(texts[24:], labels[24:])
    return clf


def test_mpnet_classifier_embeddings_and_prototypes_match_reference(trained, golden):
    emb = torch.stack(trained._get_embeddings(golden["texts"].tolist())).numpy()
    ref = golden["emb_train"]
    assert emb.shape == ref.shape
    assert np.abs(emb - ref).max() < 3e-4 and np.linalg.norm(emb - ref, axis=1).max() < 1e-3
    names = golden["label_names"].tolist()
    assert [trained.id_to_label[i] for i in range(len(names))] == names
    assert trained.training_history == json.loads(str(golden["training_history"]))
    protos = np.stack([trained.memory.prototypes[l].numpy() for l in sorted(trained.memory.prototypes)])
    assert golden["proto_labels"].tolist() == sorted(trained.memory.prototypes)
    assert np.abs(protos - golden["prototypes"]).max() < 3e-4


def test_mpnet_classifier_predictions_match_reference_with_the_reference_trained_head(trained, golden, tmp_path):
    """predict / predict_batch with the reference-trained head, then the same answers after a save / load round trip"""
    import adaptive_classifier_b200 as acb
    names = golden["label_names"].tolist()
    own_head = {k: v.detach().clone() for k, v in trained.adaptive_head.state_dict().items()}
    trained.adaptive_head.load_state_dict({k[5:]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith("head_")})
    tests_ = golden["test_texts"].tolist()

    def cmp(preds, L, S):
        for p, l_row, s_row in zip(preds, L, S):
            exp = [(names[i], s) for i, s in zip(l_row.tolist(), s_row.tolist()) if i >= 0]
            assert [l for l, _ in p] == [l for l, _ in exp], (p, exp)
            assert np.allclose([s for _, s in p], [s for _, s in exp], atol=1e-3), (p, exp)

    try:
        cmp([trained.predict(t, k=3) for t in tests_], golden["pred_labels"], golden["pred_scores"])
        cmp([trained.predict(t, k=1) for t in tests_], golden["pred_k1_labels"], golden["pred_k1_scores"])
        cmp(trained.predict_batch(tests_, k=2), golden["predb_labels"], golden["predb_scores"])
        out = str(tmp_path / "saved")
        trained.save(out)
        clf2 = acb.AdaptiveClassifier.load(out, device="cuda")
        assert clf2.label_to_id == trained.label_to_id
        cmp([clf2.predict(t, k=3) for t in tests_], golden["pred_labels"], golden["pred_scores"])
        cmp(clf2.predict_batch(tests_, k=2), golden["predb_labels"], golden["predb_scores"])
    finally:
        trained.adaptive_head.load_state_dict(own_head)


# ------------------------------------------------------------------------------------------------ downstream
def test_pipeline_host_step_replayed_as_a_cuda_graph_equals_the_eager_step_mpnet(cabi):
    """a 3-layer MPNet encoder, 768-wide prototypes and head: the captured host step replays like the device step"""
    m = mpnet_model(num_hidden_layers=3, **WIDE)
    Bmax, S, N, D, C, k = 8, 64, 3000, 768, 20, 5
    P, _ = _synthetic_index(N, D, C)
    enc = _mpnet_encoder(cabi, m, Bmax * S)
    _, pg = _head(D, C)
    row_class = (torch.arange(N) % C).to(torch.int32).cuda()
    pl = cabi.Pipeline(enc, P.cuda(), Bmax, S, k, head=pg, row_class=row_class)
    for rep, B in enumerate([3, 3, 3, 3, 8, 8, 8, 1, 1]):
        ids = eo.synthetic_ids(B, S, vocab=WIDE["vocab_size"], seed=100 + rep, arch="roberta").to(torch.int32)
        oc_h, osc_h = pl.predict_host(ids.pin_memory())
        oc_h, osc_h = oc_h.clone(), osc_h.clone()
        oc, osc = pl.predict_device(ids.cuda())
        torch.cuda.synchronize()
        assert torch.equal(oc.cpu(), oc_h) and torch.equal(osc.cpu(), osc_h), (rep, B)
    emb, _, _ = pl.debug_views(1)
    ids = eo.synthetic_ids(1, S, vocab=WIDE["vocab_size"], seed=108, arch="roberta")
    ref = mo.mpnet_forward_cls(_hf_sd(m), ids, None, num_heads=12, ln_eps=1e-5)
    assert (emb.cpu() - ref).norm(dim=1).max() < 1e-3
    pl.close(); enc.close()


def test_adaptive_classifier_on_a_local_mpnet_checkpoint(cabi, tmp_path):
    """AdaptiveClassifier on a fabricated local MPNet checkpoint directory (MPNetModel + MPNetTokenizer, loaded through
    AutoModel / AutoTokenizer): add_examples, predict, predict_batch and a save / load round trip; the embeddings equal the
    fp32 oracle's"""
    from transformers import MPNetTokenizer
    import adaptive_classifier_b200 as acb
    words = [f"w{i}" for i in range(195)]
    vocab = ["<s>", "<pad>", "</s>", "[UNK]", "<mask>"] + words
    m = mpnet_model(seed=77, num_hidden_layers=4, hidden_size=768, num_attention_heads=12, intermediate_size=3072,
                    vocab_size=len(vocab))
    with torch.no_grad():
        m.embeddings.word_embeddings.weight.mul_(4.0)
        m.embeddings.word_embeddings.weight[0].zero_()
    d = str(tmp_path / "mpnet")
    m.save_pretrained(d)
    MPNetTokenizer(vocab={w: i for i, w in enumerate(vocab)}).save_pretrained(d)
    rng = np.random.default_rng(3)
    classes = {"a": words[0:60], "b": words[60:120], "c": words[120:180]}
    texts, labels = [], []
    for lab, ws in classes.items():
        for _ in range(8):
            texts.append(" ".join(rng.choice(ws, size=int(rng.integers(5, 12)))))
            labels.append(lab)
    np.random.seed(0)
    clf = acb.AdaptiveClassifier(d, device="cuda")
    assert clf.embedding_dim == 768
    clf.add_examples(texts[:16], labels[:16])
    clf.add_examples(texts[16:], labels[16:])
    emb = torch.stack(clf._get_embeddings(texts[:6]))
    enc = clf.tokenizer(texts[:6], max_length=512, truncation=True, padding=True, return_tensors="pt")
    ref = mo.mpnet_forward_cls(_hf_sd(m), enc["input_ids"], enc["attention_mask"], num_heads=12, ln_eps=1e-5)
    assert (emb - ref).norm(dim=1).max() < 1e-3
    queries = [" ".join(rng.choice(ws, size=9)) for ws in classes.values()]
    single = [clf.predict(q, k=3) for q in queries]
    batch = clf.predict_batch(queries, k=3)
    assert len(batch) == len(queries)
    for p in single + batch:
        assert 1 <= len(p) <= 3 and {l for l, _ in p} <= {"a", "b", "c"} and abs(sum(s for _, s in p) - 1.0) < 1e-5
    out = str(tmp_path / "saved")
    clf.save(out)
    clf2 = acb.AdaptiveClassifier.load(out, device="cuda")
    assert clf2.embedding_dim == 768 and clf2.label_to_id == clf.label_to_id
    for p, p2 in zip(single + batch, [clf2.predict(q, k=3) for q in queries] + clf2.predict_batch(queries, k=3)):
        assert [l for l, _ in p2] == [l for l, _ in p] and np.allclose([s for _, s in p2], [s for _, s in p], atol=1e-5)
