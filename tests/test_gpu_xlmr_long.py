"""GPU tests of long XLM-RoBERTa encoders (bge-m3, snowflake-arctic-embed-l-v2.0: RoBERTa arch, 8194-row position table) at
512 < S <= 8192.

  * attention_long_kernel alone (Encoder.attention on a RoBERTa handle with a long table) against the fp64 reference and
    error bound of test_gpu_attention.py, on the inputs that file builds: peaked scores, a moving running maximum, one
    dominant key per key block, every seam, every mask, loud neighbours; the same q, k, v through a ModernBERT handle
    (attention_stream_kernel, window 0) under the same bound
  * the whole encoder against oracle/encoder_oracle.py (arch "roberta", pinned to HF XLMRobertaModel by
    tests/test_xlmr_long_cpu.py), run on the GPU in fp32 with TF32 off
  * S <= 512 unchanged by the long table and the refusals
The reference's classifier outputs with max_length 1024 (tests/golden/golden_classifier_xlmr_long.npz) and the CUDA-graph
replay of the pipeline step at S = 1024 are tests/test_gpu_encoder_families.py's."""
import pytest
import torch

from oracle import encoder_oracle as eo
from test_gpu_attention import (MASKS, attention_ref, make_mask, random_qkv, ramp_qkv, spike_qkv)

pytestmark = pytest.mark.gpu

HEADS, DH = 4, 64
LONG_POS = 8194          # XLM-R: positions 2 .. 8193 for 8192 tokens


def _roberta_sd(H, I, V, max_pos, layers=1, seed=11):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: (0.02 * torch.randn(*s, generator=g)).cuda()
    sd = {"embeddings.word_embeddings.weight": r(V, H), "embeddings.position_embeddings.weight": r(max_pos, H),
          "embeddings.token_type_embeddings.weight": r(1, H), "embeddings.LayerNorm.weight": torch.ones(H).cuda(),
          "embeddings.LayerNorm.bias": torch.zeros(H).cuda()}
    for l in range(layers):
        p = f"encoder.layer.{l}."
        sd[p + "intermediate.dense.weight"], sd[p + "intermediate.dense.bias"] = r(I, H), torch.zeros(I).cuda()
        sd[p + "output.dense.weight"], sd[p + "output.dense.bias"] = r(H, I), torch.zeros(H).cuda()
        for n in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = r(H, H), torch.zeros(H).cuda()
        for n in ("attention.output.LayerNorm", "output.LayerNorm"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = torch.ones(H).cuda(), torch.zeros(H).cuda()
    return sd


def _xlmr_attention_encoder(cabi, max_pos=LONG_POS, heads=HEADS, dh=DH, max_tokens=16384):
    H = heads * dh
    return cabi.Encoder(_roberta_sd(H, 64, 32, max_pos), arch="roberta", layers=1, hidden=H, heads=heads, intermediate=64,
                        vocab=32, max_pos=max_pos, pad_idx=1, ln_eps=1e-5, max_tokens=max_tokens)


@pytest.fixture(scope="module")
def long_enc(cabi):
    e = _xlmr_attention_encoder(cabi)
    yield e
    e.close()


@pytest.fixture(scope="module")
def modern_enc(cabi):
    from test_gpu_attention import make_encoder
    e = make_encoder(cabi, "modern")          # 2 heads of 64
    yield e
    e.close()


WORST = {}


def check(family, enc, q, k, v, mask=None, **kw):
    dev = lambda t: None if t is None else t.cuda()
    out = enc.attention(dev(q), dev(k), dev(v), dev(mask), pad_fill=1000.0, **kw)
    ref, tol = attention_ref(q.cuda(), k.cuda(), v.cuda(), mask)
    assert torch.isfinite(out).all(), f"{family}: non-finite context"
    rows = slice(None) if not kw.get("cls_rows") else slice(0, 128)
    ratio = (out[:, rows].double() - ref[:, rows]).abs() / tol[:, rows]
    worst = ratio.max().item()
    WORST[family] = max(WORST.get(family, 0.0), worst)
    if worst > 1.0:
        b, s, h, d = [int(i) for i in (ratio == ratio.max()).nonzero()[0]]
        pytest.fail(f"{family} S={q.shape[1]}: |out - ref| = {worst:.2f} x bound at (b={b}, q={s}, h={h}, d={d})")
    return out


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlong attention, largest error / bound per family: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))


# ------------------------------------------------------------------------------------------------ attention alone
@pytest.mark.parametrize("logit_std", [0.3, 8.0, 200.0])
@pytest.mark.parametrize("S", [1000, 4096])
def test_peaked_scores(long_enc, S, logit_std):
    B = 3 if S <= 1000 else 2
    q, k, v = random_qkv(B, S, HEADS, DH, logit_std, seed=S)
    check("peaked", long_enc, q, k, v, make_mask("right", B, S))


@pytest.mark.parametrize("pattern", ["rising", "falling", "middle"])
def test_running_maximum_moves_at_8192(long_enc, pattern):
    q, k, v = ramp_qkv(1, 8192, HEADS, DH, pattern, 20.0, seed=8192 + len(pattern))
    check("max_moves", long_enc, q, k, v)


def test_one_dominant_key_in_each_key_block(long_enc):
    S = 1000
    for blk in range((S + 127) // 128):
        key = min(128 * blk + 77, S - 1)
        q, k, v = spike_qkv(2, S, HEADS, DH, key, seed=blk)
        check("spike", long_enc, q, k, v)


@pytest.mark.parametrize("S", [513, 639, 640, 641, 1023, 1024, 1025, 2049, 8191, 8192])
def test_sequence_length_seams(long_enc, S):
    B = max(1, min(3, 16384 // S))
    q, k, v = random_qkv(B, S, HEADS, DH, 3.0, seed=2000 + S)
    check("seams", long_enc, q, k, v, make_mask("right", B, S))


@pytest.mark.parametrize("name", MASKS)
def test_masks(long_enc, name):
    S = 1100
    q, k, v = random_qkv(3, S, HEADS, DH, 3.0, seed=S + len(name))
    out = check("masks", long_enc, q, k, v, make_mask(name, 3, S))
    if name == "empty":
        assert (out[2] == 0).all()


@pytest.mark.parametrize("loud", [0, 1])
def test_heads_and_sequences_do_not_leak(long_enc, loud):
    B, S = 4, 700
    q, k, v = random_qkv(B, S, HEADS, DH, 1.0, seed=S + loud)
    for t, f in ((q, 10 ** 0.5), (k, 10 ** 0.5), (v, 10.0)):
        t[:, :, loud::2] *= f
        t[loud::2] *= f
    check("leak", long_enc, q, k, v, make_mask("right", B, S))


def test_cls_rows_equal_the_full_launch_bitwise(long_enc):
    q, k, v = random_qkv(3, 1500, HEADS, DH, 8.0, seed=5)
    mask = make_mask("right", 3, 1500)
    full = check("cls", long_enc, q, k, v, mask)
    first = check("cls", long_enc, q, k, v, mask, cls_rows=True)
    assert torch.equal(first[:, :128], full[:, :128])


def test_handle_reuse_is_bitwise_stable(cabi, long_enc):
    cases = [(2, 4000), (3, 777), (2, 4000), (1, 8192), (5, 777)]
    for i, (B, S) in enumerate(cases):
        q, k, v = random_qkv(B, S, HEADS, DH, 8.0, seed=S + B)
        mask = make_mask("right", B, S).cuda()
        fresh = _xlmr_attention_encoder(cabi)
        want = fresh.attention(q.cuda(), k.cuda(), v.cuda(), mask, pad_fill=1000.0)
        fresh.close()
        got = long_enc.attention(q.cuda(), k.cuda(), v.cuda(), mask, pad_fill=1000.0)
        assert torch.equal(got, want), f"call {i}: B={B} S={S}"


@pytest.mark.parametrize("S", [1000, 4096, 8192])
def test_streamed_kernel_on_the_same_inputs_is_inside_the_same_bound(long_enc, modern_enc, S):
    """attention_stream_kernel (ModernBERT handle, window 0) and attention_long_kernel on the same q, k, v: both inside the
    fp64 bound; no bitwise claim (the long kernel sums the row in a different order)"""
    B, heads = (2 if S <= 4096 else 1), 2
    q, k, v = random_qkv(B, S, heads, DH, 8.0, seed=S + 99)
    mask = make_mask("right", B, S)
    check("vs_stream", modern_enc, q, k, v, mask)
    q4, k4, v4 = (t.repeat(1, 1, HEADS // heads, 1) for t in (q, k, v))
    check("vs_stream", long_enc, q4, k4, v4, mask)


# ------------------------------------------------------------------------------------------------ whole encoder
@pytest.fixture(autouse=False)
def fp32_oracle():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _tiny_xlmr(seed=7, layers=3):
    """HF XLMRobertaModel, hidden 128 / 2 heads of 64, 8194 positions, non-unit LayerNorm gammas"""
    from transformers import XLMRobertaConfig, XLMRobertaModel
    torch.manual_seed(seed)
    cfg = XLMRobertaConfig(vocab_size=300, hidden_size=128, num_hidden_layers=layers, num_attention_heads=2,
                           intermediate_size=256, max_position_embeddings=LONG_POS, type_vocab_size=1, layer_norm_eps=1e-5,
                           pad_token_id=1)
    m = XLMRobertaModel(cfg, add_pooling_layer=False).eval()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "LayerNorm.weight" in n:
                p.copy_(1.0 + 0.3 * torch.randn(p.shape, generator=g))
            elif "LayerNorm.bias" in n:
                p.copy_(0.2 * torch.randn(p.shape, generator=g))
    return m


def _oracle(m, ids, mask):
    sd = {k: v.detach().float().cuda() for k, v in m.state_dict().items()}
    with torch.no_grad():
        unit, hid = eo.encoder_forward_cls(sd, ids.cuda(), mask.cuda(), arch="roberta", num_heads=m.config.num_attention_heads,
                                           ln_eps=m.config.layer_norm_eps, pad_idx=1, return_hidden=True)
    return unit.cpu(), hid.cpu()


def _ids(B, S, vocab, seed, pad):
    """<s> first, </s> last; with pad, sequence b > 0 is right-padded to 128 n +- 1 or an odd length"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(5, vocab, (B, S), generator=g)
    ids[:, 0] = 0
    mask = torch.ones(B, S, dtype=torch.int64)
    for b in range(1, B if pad else 1):
        n = [S - 127, 128 * max(1, S // 256) + 1, S - 129, S // 3][b % 4]
        mask[b, n:] = 0
    for b in range(B):
        n = int(mask[b].sum())
        ids[b, n - 1] = 2
        ids[b, n:] = 1
    return ids, mask


def _check(out, ref, unit_tol=1e-3):
    e = out - ref
    assert e.norm(dim=1).max() < unit_tol, e.norm(dim=1).max()
    P = torch.nn.functional.normalize(torch.randn(1024, out.shape[1], generator=torch.Generator().manual_seed(0)), dim=1)
    dd = (((out[:, None, :] - P[None]) ** 2).sum(-1) - ((ref[:, None, :] - P[None]) ** 2).sum(-1)).abs().max()
    assert dd < 1e-3, dd


@pytest.mark.parametrize("S,B,pad", [(513, 3, True), (640, 1, False), (1000, 3, True), (2048, 2, True), (4097, 2, True),
                                     (8192, 1, False), (8192, 2, True)])
@pytest.mark.parametrize("cls_only", [True, False])
def test_tiny_xlmr_matches_oracle(cabi, fp32_oracle, S, B, pad, cls_only):
    m = _tiny_xlmr()
    ids, mask = _ids(B, S, 300, S + B, pad)
    ref, ref_hidden = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ref)
    if not cls_only:
        hid = enc.last_hidden(B, S).cpu().view(B, S, -1)
        keep = mask.bool()
        assert (hid[keep] - ref_hidden[keep]).abs().max() < 2e-2 * ref_hidden[keep].abs().max()
    enc.close()


@pytest.mark.parametrize("cls_only", [True, False])
def test_tiny_xlmr_mask_with_a_hole(cabi, fp32_oracle, cls_only):
    """keys 130-900 of sequence 0 masked (whole key blocks without a valid key); pad ids there, so positions skip them"""
    m = _tiny_xlmr(5)
    ids, mask = _ids(2, 2000, 300, 17, True)
    mask[0, 130:901] = 0
    ids[0, 130:901] = 1
    ref, _ = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=4000, cls_only=cls_only)
    _check(enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu(), ref)
    enc.close()


@pytest.mark.parametrize("B,S,pad", [(1, 8192, False), (2, 2048, True)])
def test_bge_m3_shape_matches_oracle(cabi, fp32_oracle, B, S, pad):
    """bge-m3 / arctic-embed-l-v2.0 shape (24 x 1024, 16 heads, 8194 positions, vocab 250002), seeded init, under the
    RoBERTa-large bounds of test_gpu_parity.py"""
    from adaptive_classifier_b200 import workload as wl
    m, _ = wl.bge_m3()
    ids = wl.xlmr_ids(B, S, seed=S).long()
    mask = torch.ones(B, S, dtype=torch.int64)
    if pad:
        mask[1, 1300:] = 0
        ids[1, 1299] = 2
        ids[mask == 0] = 1
    ref, _ = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    enc.close()
    _check(out, ref, unit_tol=1.5e-3)


@pytest.mark.parametrize("S", [300, 512])
@pytest.mark.parametrize("cls_only", [True, False])
def test_8194_row_table_leaves_short_sequences_unchanged(cabi, S, cls_only):
    """the same weights with the first 514 position rows and with all 8194: the same bits at S <= 512"""
    long_ = _tiny_xlmr(9)
    from transformers import XLMRobertaConfig, XLMRobertaModel
    cfg = XLMRobertaConfig(**{**long_.config.to_dict(), "max_position_embeddings": 514})
    short = XLMRobertaModel(cfg, add_pooling_layer=False).eval()
    sd = long_.state_dict()
    sd["embeddings.position_embeddings.weight"] = sd["embeddings.position_embeddings.weight"][:514]
    short.load_state_dict({k: v for k, v in sd.items() if k in short.state_dict()})
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


def test_past_the_table_and_head_dim_32_are_refused(cabi):
    m = _tiny_xlmr(3, layers=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=2 * 8193)
    enc.forward_cls(torch.full((1, 8192), 7, dtype=torch.int32, device="cuda"))
    with pytest.raises(cabi.AdaptiveB200Error, match=r"S=8193 exceeds 8192.*max_position_embeddings=8194"):
        enc.forward_cls(torch.full((1, 8193), 7, dtype=torch.int32, device="cuda"))
    enc.close()
    enc = _xlmr_attention_encoder(cabi, max_pos=1000)      # positions 2 .. 999: S <= 998
    q, k, v = random_qkv(1, 998, HEADS, DH, 1.0, seed=0)
    enc.attention(q.cuda(), k.cuda(), v.cuda())
    q, k, v = random_qkv(1, 999, HEADS, DH, 1.0, seed=0)
    with pytest.raises(cabi.AdaptiveB200Error, match=r"S=999 exceeds 998.*max_position_embeddings=1000"):
        enc.attention(q.cuda(), k.cuda(), v.cuda())
    enc.close()
    enc = _xlmr_attention_encoder(cabi, heads=8, dh=32)
    q, k, v = random_qkv(1, 600, 8, 32, 1.0, seed=0)
    with pytest.raises(cabi.AdaptiveB200Error, match=r"S=600 > 512 needs head_dim 64"):
        enc.attention(q.cuda(), k.cuda(), v.cuda())
    enc.close()
