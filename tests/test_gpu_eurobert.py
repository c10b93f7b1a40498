"""GPU tests of the EuroBERT encoder (AC_ARCH_EUROBERT: pre-norm block with RMSNorm, RoPE, SwiGLU):
Bounds: with fp16 GEMM operands (the encoder's precision) this block family loses more than the BERT family does.
Emulating the operand roundings on the CPU (fp16 residual copy, fp16 gamma-scaled weights, fp16 q / k / v, P and context)
gives unit-row errors up to 3e-3 on these tiny models and 1.2e-3 - 1.5e-3 on the seeded eurobert_210m shape, against fp32;
no single rounding dominates.  So the unit-row error norm and the squared distances to 1024 random unit rows are held to
TINY_BOUND (tiny models) and SHAPE_BOUND (eurobert_210m, the goldens) instead of test_gpu_rotary.py's 1e-3.
  * tiny models against oracle/eurobert_oracle.py (pinned to HF by tests/test_eurobert_cpu.py), run on the GPU in fp32 with
    TF32 off: S <= 512 with cls_only on and off and the full hidden state, S up to 8192 with both paddings and a mask hole,
    with and without grouped-query attention, a single layer, and a residual stream with rows up to ~1e4
  * the eurobert_210m shape at B = 512 x 128 (sampled rows), 1 x 8192 and 2 x 2048
  * from_hf against HF, the S > max_pos refusal, and AdaptiveClassifier with max_length 8192 on the golden runs' local
    checkpoint directory
The reference's classifier outputs (goldens of oracle/make_golden_encoders.py eurobert eurobert_long) and the CUDA-graph
replay of the pipeline step are tests/test_gpu_encoder_families.py's."""
import numpy as np
import pytest
import torch

from oracle import eurobert_oracle as eo
from test_eurobert_cpu import GPU_UNIT_BOUND as TINY_BOUND, padded_batch, tiny_model

pytestmark = pytest.mark.gpu
SHAPE_BOUND = 2.5e-3


def _check(out, ref, tol=TINY_BOUND):
    """test_gpu_rotary.py::_check's two measures: unit-row error norm and squared distances to 1024 random unit rows"""
    e = out - ref
    assert e.norm(dim=1).max() < tol, e.norm(dim=1).max()
    P = torch.nn.functional.normalize(torch.randn(1024, out.shape[1], generator=torch.Generator().manual_seed(0)), dim=1)
    dd = (((out[:, None, :] - P[None]) ** 2).sum(-1) - ((ref[:, None, :] - P[None]) ** 2).sum(-1)).abs().max()
    assert dd < tol, dd


@pytest.fixture(autouse=True)
def fp32_oracle():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _oracle(m, ids, mask):
    sd = {k: v.detach().float().cuda() for k, v in m.state_dict().items()}
    with torch.no_grad():
        unit, hid = eo.eurobert_forward_for(m.config, sd, ids.cuda(), mask.cuda(), return_hidden=True)
    return unit.cpu(), hid.cpu()


def _run(enc, ids, mask):
    return enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()


def _check_hidden(enc, ref_hidden, mask):
    B, S = mask.shape
    hid = enc.last_hidden(B, S).cpu().view(B, S, -1)
    keep = mask.bool()
    assert (hid[keep] - ref_hidden[keep]).abs().max() < 2e-2 * ref_hidden[keep].abs().max()


# ------------------------------------------------------------------------------------------------ tiny encoders
@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("S", [16, 77, 128, 129, 300, 512])
def test_tiny_matches_oracle_up_to_512(cabi, S, cls_only):
    m = tiny_model(layers=3, kv=2)
    ids, mask, _ = padded_batch(S, S + 1)
    ref, ref_hidden = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * S, cls_only=cls_only)
    _check(_run(enc, ids, mask), ref)
    if not cls_only:
        _check_hidden(enc, ref_hidden, mask)
    enc.close()


@pytest.mark.parametrize("kv", [4, 1])
@pytest.mark.parametrize("S", [513, 1100, 2048, 4097, 8192])
def test_tiny_matches_oracle_past_512(cabi, S, kv):
    """past 512 tokens the attention runs attention_long_kernel; both paddings, with and without GQA"""
    m = tiny_model(layers=2, kv=kv)
    ids, mask, _ = padded_batch(S, S + 2)
    ref, ref_hidden = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * S, cls_only=S != 2048)
    _check(_run(enc, ids, mask), ref)
    if S == 2048:
        _check_hidden(enc, ref_hidden, mask)
    enc.close()


def test_tiny_mask_with_a_hole(cabi):
    """keys 130-900 of sequence 0 masked (whole key blocks without a valid key); positions still run 0..S-1"""
    m = tiny_model(seed=5, kv=2)
    ids, mask, _ = padded_batch(2000, 17)
    mask[0, 130:901] = 0
    ids[0, 130:901] = 1
    ref, _ = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * 2000)
    _check(_run(enc, ids, mask), ref)
    enc.close()


@pytest.mark.parametrize("cls_only", [True, False])
def test_single_layer(cabi, cls_only):
    """layer 0 is also the last: the raw embeddings' RMS statistics feed the QKV right before the CLS-only tail"""
    m = tiny_model(layers=1, kv=1, seed=9)
    ids, mask, _ = padded_batch(200, 3)
    ref, ref_hidden = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * 200, cls_only=cls_only)
    _check(_run(enc, ids, mask), ref)
    if not cls_only:
        _check_hidden(enc, ref_hidden, mask)
    enc.close()


@pytest.mark.parametrize("cls_only", [True, False])
def test_large_residual_rows(cabi, cls_only):
    """Llama-style massive activations: the <|begin_of_text|> row (id 0, row 0 of every sequence) carries |y| up to ~1e4
    through the residual stream; the RMS statistics are taken from the fp32 sums"""
    m = tiny_model(layers=3, kv=2, seed=13)
    with torch.no_grad():
        m.embed_tokens.weight[0] = 1e4 * torch.nn.functional.normalize(
            torch.randn(256, generator=torch.Generator().manual_seed(1)), dim=0) * torch.linspace(0.2, 6.0, 256)
    ids, mask, _ = padded_batch(300, 21)
    ids[0, 0] = ids[1, 0] = 0
    assert m.embed_tokens.weight[0].abs().max() > 3e3
    ref, _ = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * 300, cls_only=cls_only)
    _check(_run(enc, ids, mask), ref)
    enc.close()


def test_from_hf_matches_hf(cabi):
    m = tiny_model(seed=11, layers=3, kv=2).cuda()
    ids, mask, _ = padded_batch(300, 4)
    with torch.no_grad():
        hf = m(input_ids=ids.cuda(), attention_mask=mask.cuda()).last_hidden_state
    ref = torch.nn.functional.normalize(hf[:, 0], dim=1).cpu()
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * 300)
    _check(_run(enc, ids, mask), ref)
    enc.close()


def test_past_max_pos_is_refused(cabi):
    m = tiny_model(layers=1, max_pos=2048)
    enc = cabi.Encoder.from_hf(m, max_tokens=2 * 2049)
    enc.forward_cls(torch.full((1, 2048), 7, dtype=torch.int32, device="cuda"))
    with pytest.raises(cabi.AdaptiveB200Error, match=r"S=2049 exceeds this EuroBERT encoder's max_pos=2048 "
                                                     r"\(min\(max_position_embeddings, 8192\)\)"):
        enc.forward_cls(torch.full((1, 2049), 7, dtype=torch.int32, device="cuda"))
    enc.close()
    m = tiny_model(layers=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=8193)
    with pytest.raises(cabi.AdaptiveB200Error, match=r"S=8193 exceeds .*max_pos=8192"):
        enc.forward_cls(torch.full((1, 8193), 7, dtype=torch.int32, device="cuda"))
    enc.close()


# ------------------------------------------------------------------------------------------------ published shape
def test_eurobert_210m_at_the_benched_batch_matches_oracle_on_sampled_rows(cabi):
    """the seeded workload.eurobert_210m (12 x 768, SwiGLU, theta 250000) at B = 512 x S = 128: 8 sampled sequences"""
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.eurobert_210m()
    B, S = 512, 128
    ids = wl.synthetic_ids(B, S, vocab=cfg.vocab_size, seed=3).long()
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda()).cpu()
    enc.close()
    sel = torch.tensor([0, 1, 63, 127, 128, 300, 510, 511])
    ref, _ = _oracle(m, ids[sel], torch.ones(len(sel), S, dtype=torch.int64))
    _check(out[sel], ref, SHAPE_BOUND)
    assert bool(torch.isfinite(out).all())


@pytest.mark.parametrize("B,S,pad", [(1, 8192, False), (2, 2048, True)])
def test_eurobert_210m_long_matches_oracle(cabi, B, S, pad):
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.eurobert_210m()
    ids = wl.synthetic_ids(B, S, vocab=cfg.vocab_size, seed=S).long()
    mask = torch.ones(B, S, dtype=torch.int64)
    if pad:
        mask[1, 1300:] = 0
        ids[1, mask[1] == 0] = cfg.pad_token_id
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = _run(enc, ids, mask)
    enc.close()
    ref, _ = _oracle(m, ids, mask)
    _check(out, ref, SHAPE_BOUND)


# ------------------------------------------------------------------------------------------------ max_length 8192
@pytest.fixture(scope="module", params=["golden_classifier_eurobert", "golden_classifier_eurobert_long"])
def golden_run(cabi, request, tmp_path_factory):
    """the local checkpoint directory a golden run of the reference used (AutoModel / AutoTokenizer), and the run"""
    from test_gpu_encoder_families import golden_checkpoint
    d = str(tmp_path_factory.mktemp(request.param))
    return golden_checkpoint(request.param, d), d


def test_classifier_with_max_length_8192_embeds_trains_predicts_saves_and_loads(golden_run, tmp_path):
    """AdaptiveClassifier(<local EuroBERT checkpoint>, config={"max_length": 8192}) on texts of up to ~6000 tokens"""
    import adaptive_classifier_b200 as acb
    golden, d = golden_run
    words = golden["vocab"].tolist()[4:] if "vocab" in golden else golden["vocab_pieces"].tolist()[4:]
    rng = np.random.default_rng(3)
    classes = {"a": words[0:60], "b": words[60:120]}
    texts, labels = [], []
    for i, n in enumerate([6000, 40, 3000, 700, 9000, 12]):
        lab = "ab"[i % 2]
        texts.append(" ".join(rng.choice(classes[lab], size=n)))
        labels.append(lab)
    clf = acb.AdaptiveClassifier(d, device="cuda", config={"max_length": 8192, "b200_max_tokens": 16384})
    ids, mask, _ = clf._tokenize(texts)
    assert ids.shape[1] == 8192 and int(mask.sum(1).max()) == 8192
    clf.add_examples(texts, labels)
    emb = torch.stack(clf._get_embeddings(texts))
    assert bool(torch.isfinite(emb).all()) and (emb.norm(dim=1) - 1).abs().max() < 1e-4
    before = [clf.predict(t, k=2) for t in texts]
    assert sum(p[0][0] == l for p, l in zip(before, labels)) >= 4
    out = str(tmp_path / "saved8192")
    clf.save(out)
    clf2 = acb.AdaptiveClassifier.load(out, device="cuda")
    after = [clf2.predict(t, k=2) for t in texts]
    for p, p2 in zip(before, after):
        assert [l for l, _ in p2] == [l for l, _ in p] and np.allclose([s for _, s in p2], [s for _, s in p], atol=1e-5)
