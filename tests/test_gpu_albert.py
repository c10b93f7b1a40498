"""GPU tests of the ALBERT (albert-base / large v1 / v2) and ELECTRA (discriminators) encoders: factorized embeddings with
the E -> H projection, ALBERT's shared layers packed once, and the tanh-approximated GELU of "gelu_new".  Against the fp32
oracle of oracle/albert_oracle.py (pinned to HF by tests/test_albert_cpu.py), HF itself on the CPU, an fp64 reference of the
activation alone, and the reference's own classifier outputs on the golden ALBERT / ELECTRA checkpoints; then the CUDA-graph
pipeline step and the drop-in classifier on local checkpoints.

Encoder bounds are those of test_gpu_deberta.py: max abs < 3e-4 and max row norm < 1e-3 on the unit CLS rows.  The
768-wide test models keep HF's initial weight scale (LayerNorms and biases perturbed): with every weight matrix tripled, as
the 256-wide CPU oracle tests do, the fp16 operand rounding alone moves the CLS rows of 4 to 12 layers by 1.1e-3 to 1.9e-3
(row norm; max abs <= 2e-4), in ELECTRA's unshared erf layers as much as in ALBERT's shared tanh ones."""
import json

import numpy as np
import pytest
import torch

import golden_npz
from oracle import albert_oracle as ao
from test_albert_cpu import albert_ids, albert_model, electra_model, fp16_grid, gelu_tanh64, tanh_gelu_bound
from test_gpu_minilm import _check_cls
from test_gpu_parity import _head, _synthetic_index

pytestmark = pytest.mark.gpu

BASE = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=1000)


def _sd(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


def _encoder(cabi, m, max_tokens, cls_only=True, clone_layers=False):
    fn = cabi.albert_to_bert_state_dict if m.config.model_type == "albert" else cabi.electra_to_bert_state_dict
    sd, dims = fn(dict(m.state_dict()), m.config)
    if clone_layers:   # every layer its own copy: defeats the sharing
        sd = {k: (v.clone() if k.startswith("encoder.layer.") else v) for k, v in sd.items()}
    return cabi.Encoder(sd, arch="bert", max_tokens=max_tokens, cls_only=cls_only, **dims)


def _check(out, ref):
    e = out - ref
    assert e.abs().max() < 3e-4 and e.norm(dim=1).max() < 1e-3, (e.abs().max(), e.norm(dim=1).max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5


# ------------------------------------------------------------------------------------------------ activation alone
def test_tanh_gelu_epilogue_on_every_fp16_value(cabi):
    """ac_linear_tc epi 3 on exact pre-activations: A = identity rows (K = 64), so output (m, n) is act(W[n, m] + 0) for one
    fp16 weight; W holds every fp16 value in [-10, 10].  Bound: tests/test_albert_cpu.py::tanh_gelu_bound"""
    x = fp16_grid()
    K = 64
    N = (x.numel() + K - 1) // K
    N = (N + 7) // 8 * 8
    W = torch.zeros(N * K, dtype=torch.float16)
    W[: x.numel()] = x
    W = W.view(N, K)
    X = torch.eye(K, dtype=torch.float16)
    Y = cabi.linear_tc(X.cuda(), W.cuda(), torch.zeros(N, device="cuda"), epi=3, out_half=True).cpu()
    out = Y.t().reshape(-1)[: x.numel()].double()
    ref = gelu_tanh64(x)
    frac = ((out - ref).abs() / tanh_gelu_bound(ref))
    worst = int(frac.argmax())
    # outputs below the fp16 normal range round absolutely (the 2^-25 term dominates their bound); over the normal ones the
    # fraction measures the relative terms, fp16 rounding plus the fp32 evaluation allowance
    normal = ref.abs() >= 2.0 ** -14
    fn = frac.masked_fill(~normal, 0.0)
    wn = int(fn.argmax())
    print(f"tanh GELU epilogue: {x.numel()} fp16 values, worst error / bound = {frac.max().item():.3f} at x = "
          f"{x[worst].item():.6g}; over the {int(normal.sum())} normal fp16 outputs {fn.max().item():.3f} at x = "
          f"{x[wn].item():.6g}")
    assert bool(torch.isfinite(out).all()) and frac.max().item() <= 1.0


# ------------------------------------------------------------------------------------------------ encoders
@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("B,S", [(3, 16), (5, 77), (4, 128), (3, 129), (3, 300), (2, 512)])
def test_albert_base_shape_matches_oracle(cabi, B, S, cls_only):
    """albert-base shape (768, 12 heads, I 3072, E 128, "gelu_new"), 4 shared layers, padded; full hidden state too"""
    m = albert_model(num_hidden_layers=4, scale=1.0, **BASE)
    ids, mask = albert_ids(B, S, True, vocab=BASE["vocab_size"])
    ref, ref_hidden = ao.factorized_forward_cls(_sd(m), ids, mask, m.config, return_hidden=True)
    enc = _encoder(cabi, m, B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ref)
    if not cls_only:
        # the hidden rows are LayerNorm outputs of norm ~sqrt(768) = 28 (elements O(1)), not unit rows: the CLS rows' 3e-4
        # bound per element of a unit row corresponds to ~8e-3 here.  5e-3 keeps that relative precision with margin.
        hidden = enc.last_hidden(B, S).cpu().view(B, S, -1)
        keep = mask.bool()
        assert (hidden[keep] - ref_hidden[keep]).abs().max() < 5e-3
    enc.close()


def test_projection_with_embedding_size_zero_means_hidden(cabi):
    """embedding_size = 0 means hidden also when a projection is given (an ALBERT with E = H): the handle computes the same
    bits as one built with embedding_size = H, and matches the oracle"""
    m = albert_model(num_hidden_layers=2, embedding_size=768, scale=1.0, **BASE)
    sd, dims = cabi.albert_to_bert_state_dict(dict(m.state_dict()), m.config)
    assert dims["embedding_size"] == 768 and "embeddings_project.weight" in sd
    ids, mask = albert_ids(3, 100, True, vocab=BASE["vocab_size"])
    outs = []
    for E in (768, 0):
        enc = cabi.Encoder(sd, arch="bert", max_tokens=3 * 100, **{**dims, "embedding_size": E})
        outs.append(enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu())
        enc.close()
    assert torch.equal(outs[0], outs[1])
    _check(outs[1], ao.factorized_forward_cls(_sd(m), ids, mask, m.config))


@pytest.mark.parametrize("over", [dict(num_hidden_layers=4, num_hidden_groups=2, inner_group_num=2),
                                  dict(num_hidden_layers=3, embedding_size=768), dict(num_hidden_layers=2, hidden_act="gelu"),
                                  dict(num_hidden_layers=1)])
def test_albert_variants_match_oracle(cabi, over):
    """groups x inner layers, E = H (the projection still runs), v1's erf GELU, and one layer (the CLS tail reads the
    projection's output directly)"""
    m = albert_model(scale=1.0, **{**BASE, **over})
    ids, mask = albert_ids(4, 150, True, vocab=BASE["vocab_size"])
    enc = _encoder(cabi, m, 4 * 150)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ao.factorized_forward_cls(_sd(m), ids, mask, m.config))
    enc.close()


def test_albert_base_at_the_benched_batch_matches_oracle_on_sampled_rows(cabi):
    """the seeded workload.albert_base (12 shared layers) at B = 512 x S = 128: 8 sampled sequences against the oracle"""
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.albert_base(1234)
    B, S = 512, 128
    ids, _ = albert_ids(B, S, False, vocab=cfg.vocab_size, seed=3)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda()).cpu()
    sel = torch.tensor([0, 1, 63, 127, 128, 300, 510, 511])
    _check(out[sel], ao.factorized_forward_cls(_sd(m), ids[sel], None, cfg))
    assert bool(torch.isfinite(out).all())
    enc.close()


def test_albert_large_shape_matches_oracle(cabi):
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.albert_large(1234)
    ids, mask = albert_ids(3, 200, True, vocab=cfg.vocab_size, seed=4)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * 200)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ao.factorized_forward_cls(_sd(m), ids, mask, cfg))
    enc.close()


@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("B,S", [(3, 16), (5, 77), (3, 129), (3, 300), (2, 512)])
def test_electra_small_shape_matches_oracle(cabi, B, S, cls_only):
    """electra-small shape: hidden 256 (new to this library), 4 heads, E 128, I 1024, 4 layers"""
    m = electra_model(num_hidden_layers=4, intermediate_size=1024, vocab_size=1000)
    ids, mask = albert_ids(B, S, True, vocab=1000)
    enc = _encoder(cabi, m, B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ao.factorized_forward_cls(_sd(m), ids, mask, m.config))
    enc.close()


@pytest.mark.parametrize("family", ["electra_base", "bert_gelu_new"])
def test_from_hf_matches_hf(cabi, family):
    """an electra-base-shaped ElectraModel (E = H: no projection) and a BertModel with hidden_act "gelu_new", through
    Encoder.from_hf against HF on the CPU"""
    if family == "electra_base":
        m = electra_model(seed=11, num_hidden_layers=12, embedding_size=768, scale=1.0, **BASE)
    else:
        from transformers import BertConfig, BertModel
        torch.manual_seed(12)
        m = BertModel(BertConfig(num_hidden_layers=4, hidden_act="gelu_new", vocab_size=1000), add_pooling_layer=False).eval()
    ids, mask = albert_ids(4, 150, True, vocab=1000)
    with torch.no_grad():
        ref = torch.nn.functional.normalize(m(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=4 * 150)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check_cls(out, ref)
    enc.close()


# ------------------------------------------------------------------------------------------------ sharing
def _handle_bytes(make):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    enc = make()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return enc, free0 - torch.cuda.mem_get_info()[0]


def test_shared_layers_are_packed_once_and_compute_the_same_bits(cabi):
    """a 12-layer shared albert-base handle takes less device memory over a 1-layer handle (same max_tokens) than one layer's
    packed weights; its output is bitwise that of a handle built from cloned per-layer tensors"""
    from adaptive_classifier_b200 import workload as wl
    m12, _ = wl.albert_base(1234)
    m1 = albert_model(num_hidden_layers=1, scale=1.0, **{**BASE, "vocab_size": 30000})
    T = 8 * 128
    enc1, b1 = _handle_bytes(lambda: _encoder(cabi, m1, T))
    enc12, b12 = _handle_bytes(lambda: _encoder(cabi, m12, T))
    layer_bytes = (4 * 768 * 768 + 2 * 768 * 3072) * 2
    print(f"albert-base handles: 1 layer {b1 / 2**20:.1f} MiB, 12 shared layers {b12 / 2**20:.1f} MiB, one layer's packed "
          f"weights {layer_bytes / 2**20:.1f} MiB")
    assert b12 - b1 < layer_bytes, (b1, b12)
    enc1.close()
    encc, bc = _handle_bytes(lambda: _encoder(cabi, m12, T, clone_layers=True))
    assert bc - b12 > 10 * layer_bytes, (bc, b12)     # the unshared packing really is larger
    ids, mask = albert_ids(8, 128, True, vocab=30000, seed=9)
    a = enc12.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    b = encc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    assert torch.equal(a, b)
    enc12.close(); encc.close()


# ------------------------------------------------------------------------------------------------ golden classifier
def _golden_tokenizer(golden):
    vocab = golden["vocab"].tolist()
    cfgd = json.loads(str(golden["bert_config"]))
    if cfgd["model_type"] == "albert":
        from transformers import AlbertTokenizer
        return AlbertTokenizer(vocab=[(s, 0.0) for s in vocab[:5]] + [("▁" + w, -1.0 - 0.01 * i)
                                                                     for i, w in enumerate(vocab[5:])])
    from transformers import ElectraTokenizer
    return ElectraTokenizer(vocab={w: i for i, w in enumerate(vocab)})


@pytest.fixture(scope="module", params=["golden_classifier_albert", "golden_classifier_electra"])
def golden_run(cabi, request, tmp_path_factory):
    """the tiny seeded checkpoint + tokenizer the reference ran on, through the drop-in classifier"""
    from transformers import AlbertConfig, AlbertModel, ElectraConfig, ElectraModel
    import adaptive_classifier_b200 as acb
    golden = golden_npz.load(request.param)
    d = str(tmp_path_factory.mktemp(request.param))
    cfgd = json.loads(str(golden["bert_config"]))
    C, M = {"albert": (AlbertConfig, AlbertModel), "electra": (ElectraConfig, ElectraModel)}[cfgd["model_type"]]
    m = M(C(**{k: v for k, v in cfgd.items() if k not in ("model_type", "transformers_version", "architectures")}))
    m.load_state_dict({k[5:]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith("bert_") and k != "bert_config"})
    m.save_pretrained(d)
    _golden_tokenizer(golden).save_pretrained(d)
    texts, labels = golden["texts"].tolist(), golden["labels"].tolist()
    np.random.seed(0)
    clf = acb.AdaptiveClassifier(d, device="cuda")
    clf.add_examples(texts[:24], labels[:24])
    clf.add_examples(texts[24:], labels[24:])
    return clf, golden


def test_classifier_embeddings_and_prototypes_match_reference(golden_run):
    trained, golden = golden_run
    emb = torch.stack(trained._get_embeddings(golden["texts"].tolist())).numpy()
    ref = golden["emb_train"]
    assert emb.shape == ref.shape
    assert np.abs(emb - ref).max() < 3e-4 and np.linalg.norm(emb - ref, axis=1).max() < 1e-3
    names = golden["label_names"].tolist()
    assert [trained.id_to_label[i] for i in range(len(names))] == names
    assert trained.training_history == json.loads(str(golden["training_history"]))
    protos = np.stack([trained.memory.prototypes[l].numpy() for l in sorted(trained.memory.prototypes)])
    assert np.abs(protos - golden["prototypes"]).max() < 3e-4


def test_classifier_predictions_match_reference_with_the_reference_trained_head(golden_run, tmp_path):
    """predict / predict_batch with the reference-trained head, then the same answers after a save / load round trip"""
    import adaptive_classifier_b200 as acb
    trained, golden = golden_run
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
        cmp(trained.predict_batch(tests_, k=2), golden["predb_labels"], golden["predb_scores"])
        out = str(tmp_path / "saved")
        trained.save(out)
        clf2 = acb.AdaptiveClassifier.load(out, device="cuda")
        assert clf2.label_to_id == trained.label_to_id
        cmp([clf2.predict(t, k=3) for t in tests_], golden["pred_labels"], golden["pred_scores"])
    finally:
        trained.adaptive_head.load_state_dict(own_head)


# ------------------------------------------------------------------------------------------------ downstream
def test_pipeline_host_step_replayed_as_a_cuda_graph_equals_the_eager_step_albert(cabi):
    """a 3-layer shared albert-base-shaped encoder (projection, tanh GELU), 768-wide prototypes and head"""
    m = albert_model(num_hidden_layers=3, scale=1.0, **BASE)
    Bmax, S, N, D, C, k = 8, 64, 3000, 768, 20, 5
    P, _ = _synthetic_index(N, D, C)
    enc = _encoder(cabi, m, Bmax * S)
    _, pg = _head(D, C)
    row_class = (torch.arange(N) % C).to(torch.int32).cuda()
    pl = cabi.Pipeline(enc, P.cuda(), Bmax, S, k, head=pg, row_class=row_class)
    for rep, B in enumerate([3, 3, 3, 3, 8, 8, 8, 1, 1]):
        ids, _ = albert_ids(B, S, False, vocab=BASE["vocab_size"], seed=100 + rep)
        ids = ids.to(torch.int32)
        oc_h, osc_h = pl.predict_host(ids.pin_memory())
        oc_h, osc_h = oc_h.clone(), osc_h.clone()
        oc, osc = pl.predict_device(ids.cuda())
        torch.cuda.synchronize()
        assert torch.equal(oc.cpu(), oc_h) and torch.equal(osc.cpu(), osc_h), (rep, B)
    emb, _, _ = pl.debug_views(1)
    ids, _ = albert_ids(1, S, False, vocab=BASE["vocab_size"], seed=108)
    assert (emb.cpu() - ao.factorized_forward_cls(_sd(m), ids, None, m.config)).norm(dim=1).max() < 1e-3
    pl.close(); enc.close()


@pytest.mark.parametrize("family", ["albert", "electra"])
def test_adaptive_classifier_on_a_local_checkpoint(cabi, tmp_path, family):
    """AdaptiveClassifier on a fabricated local albert-base-v2-shaped / electra-small-shaped checkpoint directory (loaded
    through AutoModel / AutoTokenizer): add_examples, predict, predict_batch and a save / load round trip; the embeddings
    equal the fp32 oracle's"""
    import adaptive_classifier_b200 as acb
    from transformers import AlbertTokenizer, ElectraTokenizer
    words = [f"w{i}" for i in range(195)]
    if family == "albert":
        specials = ["<pad>", "<unk>", "[CLS]", "[SEP]", "[MASK]"]
        tok = AlbertTokenizer(vocab=[(s, 0.0) for s in specials] + [("▁" + w, -1.0 - 0.01 * i) for i, w in enumerate(words)])
        m = albert_model(seed=77, num_hidden_layers=12, scale=1.0, **{**BASE, "vocab_size": 5 + len(words)})
        H = 768
    else:
        tok = ElectraTokenizer(vocab={w: i for i, w in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words)})
        m = electra_model(seed=78, num_hidden_layers=12, intermediate_size=1024, scale=1.0, vocab_size=5 + len(words))
        H = 256
    with torch.no_grad():
        m.embeddings.word_embeddings.weight.mul_(4.0)
        m.embeddings.word_embeddings.weight[2].zero_()
    d = str(tmp_path / family)
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
    ref = ao.factorized_forward_cls(_sd(m), enc["input_ids"], enc["attention_mask"], m.config,
                                    token_type_ids=enc.get("token_type_ids"))
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
    assert clf2.embedding_dim == H and clf2.label_to_id == clf.label_to_id
    for p, p2 in zip(single + batch, [clf2.predict(q, k=3) for q in queries] + clf2.predict_batch(queries, k=3)):
        assert [l for l, _ in p2] == [l for l, _ in p] and np.allclose([s for _, s in p2], [s for _, s in p], atol=1e-5)

