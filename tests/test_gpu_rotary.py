"""GPU tests of the rotary encoders (NomicBERT, jina-embeddings-v3: AC_ARCH_ROTARY, post-LN block with RoPE on q and k):
  * the SwiGLU epilogue alone (ac_linear_tc epi 4) on every fp16 value in [-20, 20] against fp64 silu
  * tiny Nomic / jina models against oracle/rotary_oracle.py (pinned to HF by tests/test_rotary_cpu.py), run on the GPU in
    fp32 with TF32 off: S <= 512 with cls_only on and off and the full hidden state, S up to 2048 (Nomic) / 8192 (jina)
    with both paddings and a mask hole
  * the nomic_v15 shape at B = 512 x 128 and the jina_v3 shape at 1 x 8192 and 2 x 2048
  * from_hf against HF and the S > max_pos refusal
The reference's classifier outputs (goldens of oracle/make_golden_encoders.py nomic jina3) and the CUDA-graph replay of
the pipeline step are tests/test_gpu_encoder_families.py's."""
import pytest
import torch

from oracle import rotary_oracle as ro
from test_albert_cpu import fp16_grid
from test_rotary_cpu import padded_batch, silu64, silu_bound, tiny_model

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def fp32_oracle():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _oracle(m, ids, mask, tt=None, cfg=None):
    sd = {k: v.detach().float().cuda() for k, v in m.state_dict().items()}
    with torch.no_grad():
        unit, hid = ro.rotary_forward_for(cfg or m.config, sd, ids.cuda(), mask.cuda(), None if tt is None else tt.cuda(),
                                          return_hidden=True)
    return unit.cpu(), hid.cpu()


def _run(enc, ids, mask, tt=None):
    return enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda(),
                           None if tt is None else tt.to(torch.int32).cuda()).cpu()


def _check(out, ref, unit_tol=1e-3):
    """the bounds of test_gpu_xlmr_long.py: unit-row error norm and squared distances to 1024 random unit rows"""
    e = out - ref
    assert e.norm(dim=1).max() < unit_tol, e.norm(dim=1).max()
    P = torch.nn.functional.normalize(torch.randn(1024, out.shape[1], generator=torch.Generator().manual_seed(0)), dim=1)
    dd = (((out[:, None, :] - P[None]) ** 2).sum(-1) - ((ref[:, None, :] - P[None]) ** 2).sum(-1)).abs().max()
    assert dd < 1e-3, dd


def _check_albert(out, ref):
    """the bounds of test_gpu_albert.py::_check"""
    e = out - ref
    assert e.abs().max() < 3e-4 and e.norm(dim=1).max() < 1e-3, (e.abs().max(), e.norm(dim=1).max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5


# ------------------------------------------------------------------------------------------------ SwiGLU epilogue
def test_swiglu_epilogue_on_every_fp16_value(cabi):
    """ac_linear_tc epi 4 on exact pre-activations: A = identity rows (K = 64), weight rows interleaved in 32-row groups
    (64 g + j activated, 64 g + 32 + j multipliers = 1), so output (m, 32 g + j) is silu(W[64 g + j, m]) for one fp16
    weight; the activated rows hold every fp16 value in [-20, 20], then large magnitudes.  Bound:
    tests/test_rotary_cpu.py::silu_bound"""
    x = fp16_grid(-20.0, 20.0)
    big = torch.tensor([-65504.0, -1000.0, -100.0, -89.0, -88.0, -87.0, 88.0, 100.0, 1000.0, 65504.0], dtype=torch.float16)
    vals = torch.cat([x, big])
    G = (vals.numel() + 2047) // 2048
    W = torch.ones(G, 64, 64, dtype=torch.float16)
    act = torch.zeros(G * 2048, dtype=torch.float16)
    act[: vals.numel()] = vals
    W[:, :32, :] = act.view(G, 32, 64)
    Y = cabi.linear_tc(torch.eye(64, dtype=torch.float16).cuda(), W.view(64 * G, 64).cuda(), torch.zeros(64 * G).cuda(),
                       epi=4, out_half=True).cpu()
    assert Y.shape == (64, 32 * G)
    out = Y.view(64, G, 32).permute(1, 2, 0).reshape(-1)[: vals.numel()].double()
    n = x.numel()
    ref = silu64(x)
    frac = (out[:n] - ref).abs() / silu_bound(ref)
    worst = int(frac.argmax())
    normal = ref.abs() >= 2.0 ** -14
    fn = frac.masked_fill(~normal, 0.0)
    print(f"SwiGLU epilogue: {n} fp16 values, worst error / bound = {frac.max().item():.3f} at x = {x[worst].item():.6g}; "
          f"over the {int(normal.sum())} normal fp16 outputs {fn.max().item():.3f} at x = {x[int(fn.argmax())].item():.6g}")
    assert bool(torch.isfinite(out).all()) and frac.max().item() <= 1.0
    # large magnitudes: a signed zero or a tiny value below -88.7, y itself far above 0; never NaN
    ob, xb = out[n:], big.double()
    assert (ob[xb < -88] <= 0).all() and (ob[xb < -88].abs() <= 2.0 ** -14).all(), ob
    assert torch.equal(ob[xb > 87], xb[xb > 87]), ob


# ------------------------------------------------------------------------------------------------ tiny encoders
@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("S", [16, 77, 128, 129, 300, 512])
@pytest.mark.parametrize("family", ["nomic", "jina"])
def test_tiny_matches_oracle_up_to_512(cabi, family, S, cls_only):
    m = tiny_model(family, layers=3)
    ids, mask, tt = padded_batch(S, S + 1, types=True)
    ref, ref_hidden = _oracle(m, ids, mask, tt)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * S, cls_only=cls_only)
    _check(_run(enc, ids, mask, tt), ref)
    if not cls_only:
        hid = enc.last_hidden(3, S).cpu().view(3, S, -1)
        keep = mask.bool()
        assert (hid[keep] - ref_hidden[keep]).abs().max() < 2e-2 * ref_hidden[keep].abs().max()
    enc.close()


@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("family,S", [("nomic", 513), ("nomic", 1100), ("nomic", 2048), ("jina", 513), ("jina", 2048),
                                      ("jina", 4097), ("jina", 8192)])
def test_tiny_matches_oracle_past_512(cabi, family, S, cls_only):
    """past 512 tokens the attention runs attention_long_kernel; both paddings"""
    m = tiny_model(family, layers=2)
    ids, mask, tt = padded_batch(S, S + 2)
    ref, ref_hidden = _oracle(m, ids, mask, tt)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * S, cls_only=cls_only)
    _check(_run(enc, ids, mask, tt), ref)
    if not cls_only:
        hid = enc.last_hidden(3, S).cpu().view(3, S, -1)
        keep = mask.bool()
        assert (hid[keep] - ref_hidden[keep]).abs().max() < 2e-2 * ref_hidden[keep].abs().max()
    enc.close()


@pytest.mark.parametrize("family", ["nomic", "jina"])
def test_tiny_mask_with_a_hole(cabi, family):
    """keys 130-900 of sequence 0 masked (whole key blocks without a valid key); positions still run 0..S-1"""
    m = tiny_model(family, seed=5)
    ids, mask, tt = padded_batch(2000, 17)
    mask[0, 130:901] = 0
    ids[0, 130:901] = 1
    ref, _ = _oracle(m, ids, mask, tt)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * 2000)
    _check(_run(enc, ids, mask, tt), ref)
    enc.close()


@pytest.mark.parametrize("family", ["nomic", "jina"])
def test_from_hf_matches_hf(cabi, family):
    m = tiny_model(family, seed=11, layers=3).cuda()
    ids, mask, tt = padded_batch(300, 4, types=True)
    with torch.no_grad():
        hf = m(input_ids=ids.cuda(), attention_mask=mask.cuda(), token_type_ids=tt.cuda()).last_hidden_state
    ref = torch.nn.functional.normalize(hf[:, 0], dim=1).cpu()
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * 300)
    _check(_run(enc, ids, mask, tt), ref)
    enc.close()


def test_past_max_pos_is_refused(cabi):
    m = tiny_model("nomic", layers=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=2 * 2049)
    enc.forward_cls(torch.full((1, 2048), 7, dtype=torch.int32, device="cuda"))
    with pytest.raises(cabi.AdaptiveB200Error, match=r"S=2049 exceeds this rotary encoder's max_pos=2048 "
                                                     r"\(min\(max_position_embeddings, 8192\)\)"):
        enc.forward_cls(torch.full((1, 2049), 7, dtype=torch.int32, device="cuda"))
    enc.close()
    m = tiny_model("jina", layers=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=8193)
    with pytest.raises(cabi.AdaptiveB200Error, match=r"S=8193 exceeds .*max_pos=8192"):
        enc.forward_cls(torch.full((1, 8193), 7, dtype=torch.int32, device="cuda"))
    enc.close()


# ------------------------------------------------------------------------------------------------ published shapes
def test_nomic_v15_at_the_benched_batch_matches_oracle_on_sampled_rows(cabi):
    """the seeded workload.nomic_v15 (12 x 768, SwiGLU) at B = 512 x S = 128: 8 sampled sequences against the oracle"""
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.nomic_v15()
    B, S = 512, 128
    ids = wl.synthetic_ids(B, S, vocab=cfg.vocab_size, seed=3).long()
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda()).cpu()
    enc.close()
    sel = torch.tensor([0, 1, 63, 127, 128, 300, 510, 511])
    ref, _ = _oracle(m, ids[sel], torch.ones(len(sel), S, dtype=torch.int64))
    _check_albert(out[sel], ref)
    assert bool(torch.isfinite(out).all())


@pytest.mark.parametrize("B,S,pad", [(1, 8192, False), (2, 2048, True)])
def test_jina_v3_shape_matches_oracle(cabi, B, S, pad):
    """jina-embeddings-v3 shape (24 x 1024, 16 heads, vocab 250002), seeded init, under the bge-m3 bounds of
    test_gpu_xlmr_long.py"""
    from adaptive_classifier_b200 import workload as wl
    m, _ = wl.jina_v3()
    ids = wl.xlmr_ids(B, S, seed=S).long()
    mask = torch.ones(B, S, dtype=torch.int64)
    if pad:
        mask[1, 1300:] = 0
        ids[1, 1299] = 2
        ids[mask == 0] = 1
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = _run(enc, ids, mask)
    enc.close()
    ref, _ = _oracle(m, ids, mask)
    _check(out, ref, unit_tol=1.5e-3)
