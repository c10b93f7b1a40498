"""GPU tests of ModernBERT at 512 < S <= 8192 (the streamed one-pass attention kernel and max_pos-row RoPE tables) against
the query-block fp32 oracle of oracle/modernbert_long_oracle.py (pinned to HF ModernBertModel by
tests/test_modernbert_long_cpu.py), run on the GPU in fp32 with TF32 off; the reference's classifier outputs with
max_length 1024; the unchanged S <= 512 results; and the CUDA-graph replay of the pipeline step at S = 1024."""
import json

import numpy as np
import pytest
import torch

import golden_npz
from oracle.modernbert_long_oracle import modernbert_forward_cls_blocked
from test_gpu_modernbert import _check, _ids, _model
from test_gpu_parity import _head, _synthetic_index

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_oracle():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _oracle(m, ids, mask):
    from adaptive_classifier_b200._cabi import modernbert_settings
    c = m.config
    s = modernbert_settings(c)
    sd = {k: v.detach().float().cuda() for k, v in m.state_dict().items()}
    with torch.no_grad():
        unit, hid = modernbert_forward_cls_blocked(sd, ids.cuda(), mask.cuda(), num_heads=c.num_attention_heads,
                                                   layer_sliding=[bool(v) for v in s["layer_sliding"]],
                                                   sliding_window=s["sliding_window"], rope_theta=s["rope_theta"],
                                                   norm_eps=c.norm_eps, return_hidden=True)
    return unit.cpu(), hid.cpu()


def _run(cabi, m, ids, mask, cls_only):
    B, S = ids.shape
    ref, ref_hidden = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ref)
    if not cls_only:
        hid = enc.last_hidden(B, S).cpu().view(B, S, -1)
        keep = mask.bool()
        assert (hid[keep] - ref_hidden[keep]).abs().max() < 2e-2 * ref_hidden[keep].abs().max()
    enc.close()


@pytest.mark.parametrize("S,B,pad", [(513, 2, True), (640, 1, False), (1000, 3, True), (2048, 2, True), (8192, 1, False),
                                     (8192, 2, True)])
@pytest.mark.parametrize("local_attention", [16, 128])
@pytest.mark.parametrize("cls_only", [True, False])
def test_modernbert_long_tiny_matches_oracle(cabi, S, B, pad, local_attention, cls_only):
    """hidden 128 / 2 heads, 4 layers (full, sliding, sliding, full), half-window 8 or 64, non-unit norm gammas; padded
    sequences end at 128 n +- 1 and at other lengths (_ids)"""
    m = _model(7, local_attention=local_attention, max_position_embeddings=8192)
    ids, mask = _ids(B, S, 300, S + B, pad)
    if pad and B >= 2:
        mask[1, 128 * (S // 256) + 1:] = 0
        ids[1, 128 * (S // 256) + 1:] = 0
    _run(cabi, m, ids, mask, cls_only)


@pytest.mark.parametrize("local_attention", [16, 128])
@pytest.mark.parametrize("cls_only", [True, False])
def test_modernbert_long_mask_with_a_hole(cabi, local_attention, cls_only):
    """keys 130-400 of sequence 0 masked: query rows near the hole see key blocks with no valid key first"""
    m = _model(5, local_attention=local_attention, max_position_embeddings=8192)
    ids, mask = _ids(2, 1000, 300, 17, True)
    mask[0, 130:401] = 0
    ids[0, 130:401] = 0
    _run(cabi, m, ids, mask, cls_only)


@pytest.mark.parametrize("B,S,pad", [(1, 8192, False), (2, 2048, True)])
def test_modernbert_long_base_shape(cabi, B, S, pad):
    """ModernBERT-base (22 x 768, 12 heads, I 1152, half-window 64 on 2 of 3 layers), vocab 50368, seeded init"""
    over = dict(vocab_size=50368, max_position_embeddings=8192, pad_token_id=50283, local_attention=128, hidden_size=768,
                num_hidden_layers=22, num_attention_heads=12, intermediate_size=1152)
    m = _model(1234, gamma_noise=0.1, **over)
    g = torch.Generator().manual_seed(S)
    ids = torch.randint(1000, 50000, (B, S), generator=g)
    ids[:, 0] = 50281
    mask = torch.ones(B, S, dtype=torch.int64)
    if pad:
        mask[1, 1300:] = 0
        ids[mask == 0] = 50283
    ref, _ = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ref)
    enc.close()


@pytest.mark.parametrize("S", [300, 512])
@pytest.mark.parametrize("cls_only", [True, False])
def test_8192_row_tables_leave_short_sequences_unchanged(cabi, S, cls_only):
    """the same weights with max_position_embeddings 512 and 8192: the encoders give the same bits at S <= 512"""
    short, long_ = _model(9, max_position_embeddings=512), _model(9, max_position_embeddings=8192)
    assert all(torch.equal(a, b) for a, b in zip(short.state_dict().values(), long_.state_dict().values()))
    ids, mask = _ids(3, S, 300, S, True)
    ids, mask = ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()
    outs = []
    for m in (short, long_):
        enc = cabi.Encoder.from_hf(m, max_tokens=3 * S, cls_only=cls_only)
        outs.append((enc.forward_cls(ids, mask).cpu(), None if cls_only else enc.last_hidden(3, S).cpu()))
        enc.close()
    assert torch.equal(outs[0][0], outs[1][0])
    if not cls_only:
        assert torch.equal(outs[0][1], outs[1][1])


def test_bert_past_512_and_modernbert_past_max_pos_are_refused(cabi):
    from transformers import BertConfig, BertModel
    torch.manual_seed(0)
    bert = BertModel(BertConfig(vocab_size=300, hidden_size=128, num_hidden_layers=1, num_attention_heads=2,
                                intermediate_size=256, max_position_embeddings=1024)).eval()
    enc = cabi.Encoder.from_hf(bert, max_tokens=2048)
    ids = torch.full((1, 513), 7, dtype=torch.int32, device="cuda")
    with pytest.raises(cabi.AdaptiveB200Error, match=r"S=513 > 512 is not supported \(the reference truncates at max_length"):
        enc.forward_cls(ids)
    enc.close()
    m = _model(3, max_position_embeddings=1024)
    enc = cabi.Encoder.from_hf(m, max_tokens=4096)
    enc.forward_cls(torch.full((1, 1024), 7, dtype=torch.int32, device="cuda"))
    with pytest.raises(cabi.AdaptiveB200Error, match="max_pos=1024"):
        enc.forward_cls(torch.full((1, 1025), 7, dtype=torch.int32, device="cuda"))
    enc.close()


@pytest.fixture(scope="module")
def golden():
    return golden_npz.load("golden_classifier_modernbert_long")


@pytest.fixture(scope="module")
def ckpt(golden, tmp_path_factory):
    """the tiny seeded ModernBERT checkpoint (weights of golden_classifier_modernbert, max_position_embeddings 8192)"""
    from transformers import BertTokenizerFast, ModernBertConfig, ModernBertModel
    d = str(tmp_path_factory.mktemp("golden_modernbert_long"))
    w = golden_npz.load("golden_classifier_modernbert")
    m = ModernBertModel(ModernBertConfig(**json.loads(str(golden["bert_config"]))))
    m.load_state_dict({k[5:]: torch.from_numpy(w[k]) for k in w.files if k.startswith("bert_") and k != "bert_config"})
    m.save_pretrained(d)
    tok = BertTokenizerFast(vocab={w: i for i, w in enumerate(golden["vocab"].tolist())}, do_lower_case=True)
    tok.model_input_names = ["input_ids", "attention_mask"]
    tok.save_pretrained(d)
    return d


@pytest.fixture(scope="module")
def trained(cabi, golden, ckpt):
    """driven through the drop-in classifier with max_length 1024; a 4096-token workspace makes _embed_ids_device split the
    1024-token batches into chunks of 4 sequences"""
    import adaptive_classifier_b200 as acb
    texts, labels = golden["texts"].tolist(), golden["labels"].tolist()
    np.random.seed(0)
    clf = acb.AdaptiveClassifier(ckpt, device="cuda", config={"max_length": int(golden["max_length"]), "b200_max_tokens": 4096})
    clf.add_examples(texts[:12], labels[:12])
    clf.add_examples(texts[12:], labels[12:])
    return clf


def test_long_classifier_embeddings_and_prototypes_match_reference(trained, golden):
    ids, _, _ = trained._tokenize(golden["texts"].tolist() + golden["test_texts"].tolist())
    assert torch.equal(ids, torch.from_numpy(golden["input_ids"]))        # truncation at 1024 and padding as the reference
    emb = torch.stack(trained._get_embeddings(golden["texts"].tolist())).numpy()
    ref = golden["emb_train"]
    assert emb.shape == ref.shape
    assert np.abs(emb - ref).max() < 3e-4 and np.linalg.norm(emb - ref, axis=1).max() < 1e-3
    emb_t = torch.stack(trained._get_embeddings(golden["test_texts"].tolist())).numpy()
    assert np.abs(emb_t - golden["emb_test"]).max() < 3e-4
    names = golden["label_names"].tolist()
    assert [trained.id_to_label[i] for i in range(len(names))] == names
    protos = np.stack([trained.memory.prototypes[l].numpy() for l in sorted(trained.memory.prototypes)])
    assert golden["proto_labels"].tolist() == sorted(trained.memory.prototypes)
    assert np.abs(protos - golden["prototypes"]).max() < 3e-4


def _cmp(preds, L, S, names):
    for p, l_row, s_row in zip(preds, L, S):
        exp = [(names[i], s) for i, s in zip(l_row.tolist(), s_row.tolist()) if i >= 0]
        assert [l for l, _ in p] == [l for l, _ in exp], (p, exp)
        assert np.allclose([s for _, s in p], [s for _, s in exp], atol=1e-3), (p, exp)


def test_long_classifier_predictions_match_reference_and_survive_save_load(trained, golden, tmp_path):
    import adaptive_classifier_b200 as acb
    names = golden["label_names"].tolist()
    own_head = {k: v.detach().clone() for k, v in trained.adaptive_head.state_dict().items()}
    trained.adaptive_head.load_state_dict({k[5:]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith("head_")})
    tests_ = golden["test_texts"].tolist()
    try:
        _cmp([trained.predict(t, k=3) for t in tests_], golden["pred_labels"], golden["pred_scores"], names)
        _cmp([trained.predict(t, k=1) for t in tests_], golden["pred_k1_labels"], golden["pred_k1_scores"], names)
        _cmp(trained.predict_batch(tests_, k=2), golden["predb_labels"], golden["predb_scores"], names)
        before = [trained.predict(t, k=3) for t in tests_]
        out = str(tmp_path / "saved")
        trained.save(out)
        clf2 = acb.AdaptiveClassifier.load(out, device="cuda")
        assert clf2.config.max_length == 1024
        after = [clf2.predict(t, k=3) for t in tests_]
        for p, p2 in zip(before, after):
            assert [l for l, _ in p2] == [l for l, _ in p] and np.allclose([s for _, s in p2], [s for _, s in p], atol=1e-5)
    finally:
        trained.adaptive_head.load_state_dict(own_head)


def test_pipeline_host_step_replayed_as_a_cuda_graph_equals_the_eager_step_at_1024(cabi):
    """the streamed attention kernel captures and replays like the S <= 512 ones"""
    m = _model(3, hidden_size=768, num_attention_heads=12, intermediate_size=1152, num_hidden_layers=3, vocab_size=1000,
               local_attention=128, max_position_embeddings=8192)
    Bmax, S, N, D, C, k = 8, 1024, 3000, 768, 20, 5
    P, _ = _synthetic_index(N, D, C)
    enc = cabi.Encoder.from_hf(m, max_tokens=Bmax * S)
    _, pg = _head(D, C)
    row_class = (torch.arange(N) % C).to(torch.int32).cuda()
    pl = cabi.Pipeline(enc, P.cuda(), Bmax, S, k, head=pg, row_class=row_class)
    for rep, B in enumerate([3, 3, 3, 3, 8, 8, 8]):
        ids = _ids(B, S, 1000, 100 + rep, False)[0].to(torch.int32)
        oc_h, osc_h = pl.predict_host(ids.pin_memory())
        oc_h, osc_h = oc_h.clone(), osc_h.clone()
        oc, osc = pl.predict_device(ids.cuda())
        torch.cuda.synchronize()
        assert torch.equal(oc.cpu(), oc_h) and torch.equal(osc.cpu(), osc_h), (rep, B)
    pl.close(); enc.close()
