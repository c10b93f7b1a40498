"""GPU tests of DeBERTa-v3 encoders past 512 tokens (handles built with rel_radius AC_MODERNBERT_MAX_S: relative operand
boxes of block offsets -D .. D, larger offsets clamped to +-D): the attention stage alone against the fp64 reference and
per-element bound of test_gpu_deberta.py, bit equality with radius-512 handles at S <= 512, whole encoders against the
fp32 oracle up to 8192 tokens and the refusals.  The reference's golden classifier at max_length 1024 and the CUDA-graph
pipeline step at S = 1024 are tests/test_gpu_encoder_families.py's."""
import math

import pytest
import torch

from oracle import deberta_oracle as do
from test_deberta_cpu import deberta_ids, deberta_model
from test_gpu_deberta import WIDE, _mask, _qkv

pytestmark = pytest.mark.gpu

LONG = 8192
CONFIGS = {"b256": {}, "b16": dict(position_buckets=16), "nob64": dict(position_buckets=-1, max_relative_positions=64)}


def _dims(cabi, m, radius_long=True):
    sd, dims = cabi.deberta_to_bert_state_dict(dict(m.state_dict()), m.config)
    if not radius_long:
        dims.pop("rel_index_long")
    return sd, dims


def _oracle(m, ids, mask, return_hidden=False):
    """the fp32 oracle on the GPU (the CPU would need tens of GB at 8192 tokens); fp32 matmuls, no TF32"""
    sd = {k: v.detach().float().cuda() for k, v in m.state_dict().items()}
    with torch.device("cuda"):
        out = do.deberta_forward_cls(sd, ids.cuda(), None if mask is None else mask.cuda(), m.config,
                                     return_hidden=return_hidden)
    return tuple(t.cpu() for t in out) if return_hidden else out.cpu()


# ------------------------------------------------------------------------------------------------ attention stage alone
def _attention_handle(cabi, heads, over, pos_std, seed, radius_long=True, max_tokens=2 * LONG):
    """one-layer handle with seeded N(0, pos_std) layer-0 position tables; returns it, the fp16 tables as the kernel sees
    them and the index table it was given (with its radius)"""
    m = deberta_model(num_hidden_layers=1, hidden_size=64 * heads, num_attention_heads=heads, intermediate_size=128,
                      vocab_size=100, **over)
    sd, dims = _dims(cabi, m, radius_long)
    g = torch.Generator().manual_seed(seed)
    span, H = dims["pos_span"], 64 * heads
    dims["pos_key"] = pos_std * torch.randn(1, 2 * span, H, generator=g)
    dims["pos_query"] = pos_std * torch.randn(1, 2 * span, H, generator=g)
    idx = dims["rel_index_long"] if radius_long else dims["rel_index"]
    enc = cabi.Encoder(sd, arch="deberta", max_tokens=max_tokens, **dims)
    return enc, dims["pos_key"][0].half(), dims["pos_query"][0].half(), idx.long(), (idx.numel() + 1) // 2


def _attention_ref(q, k, v, pk, pq, rel_index, radius, mask, cls_rows=False):
    """test_gpu_deberta._deberta_attention_ref at any S, in fp64 on the GPU over 512-query chunks: (context, bound)"""
    B, S, heads, dh = q.shape
    dev = "cuda"
    qd, kd = q.double().to(dev).transpose(1, 2), k.double().to(dev).transpose(1, 2)     # [B, heads, S, dh]
    PK = pk.double().to(dev).view(-1, heads, dh).transpose(0, 1)                       # [heads, 2 span, dh]
    PQ = pq.double().to(dev).view(-1, heads, dh).transpose(0, 1)
    vv = v.double().to(dev).permute(0, 2, 1, 3)
    ri = rel_index.to(dev)
    keep = torch.ones(B, S, dtype=torch.bool, device=dev) if mask is None else (mask.to(dev) != 0)
    att = keep[:, None, None, :]
    scale = 1.0 / math.sqrt(3 * dh)
    pos = torch.arange(S, device=dev)
    nq = min(S, 128) if cls_rows else S
    outs, tols = [], []
    for i0 in range(0, nq, 512):
        i1 = min(nq, i0 + 512)
        c = ri[radius - 1 + pos[i0:i1, None] - pos[None, :]].expand(B, heads, i1 - i0, S)      # c(i - j) at [.., i, j]

        def terms(qq, kk, pkk, pqq):
            c2p = torch.gather(qq[:, :, i0:i1] @ pkk.transpose(-1, -2), -1, c)
            kp = kk @ pqq.transpose(-1, -2)                                                     # [B, heads, S (j), 2 span]
            p2c = torch.gather(kp, -1, c.transpose(-1, -2)).transpose(-1, -2)                  # k_j . PosQ[c(i - j)]
            return (qq[:, :, i0:i1] @ kk.transpose(-1, -2) + c2p + p2c) * scale

        s = terms(qd, kd, PK, PQ)
        E = terms(qd.abs(), kd.abs(), PK.abs(), PQ.abs())
        x = s.masked_fill(~att, -math.inf)
        mx = x.amax(-1, keepdim=True)
        p = torch.exp(x - torch.where(torch.isinf(mx), torch.zeros_like(mx), mx))
        w = p / p.sum(-1, keepdim=True).clamp_min(1e-300)
        out, wabs, reach = w @ vv, w @ vv.abs(), att.expand(B, 1, i1 - i0, S).double() @ vv.abs()
        emax = E.masked_fill(~att, 0).amax(-1, keepdim=True)
        tol = (2.0 ** -10 + 2.0 ** -16 * emax) * wabs + 2.0 ** -11 * out.abs() + 2.0 ** -25 * reach + 2.0 ** -24
        outs.append(out.permute(0, 2, 1, 3).cpu())
        tols.append(tol.permute(0, 2, 1, 3).cpu())
        del s, E, x, p, w
    return torch.cat(outs, 1), torch.cat(tols, 1)


def _check_stage(enc, q, k, v, pk, pq, idx, radius, mask, cls_rows=False):
    out = enc.attention(q.cuda(), k.cuda(), v.cuda(), None if mask is None else mask.cuda(), cls_rows=cls_rows,
                        pad_fill=1000.0).cpu()
    ref, tol = _attention_ref(q, k, v, pk, pq, idx, radius, mask, cls_rows)
    rows = ref.shape[1]
    err = (out[:, :rows].double() - ref).abs()
    frac = (err / tol).max().item()
    assert bool(torch.isfinite(out[:, :rows]).all()) and frac <= 1.0, (frac, err.max().item())
    return frac


SEAMS_LONG = [513, 639, 640, 641, 767, 768, 769, 896, 897, 1024, 2048, 4096, 8191, 8192]


@pytest.mark.parametrize("S", SEAMS_LONG)
def test_long_attention_at_every_seam(cabi, S):
    """256 buckets, right padding, scores of std ~ 8: both sides of the block seams where offsets reach and pass D = 5"""
    heads, B = (2, 1) if S > 2048 else (4, 2)
    enc, pk, pq, idx, R = _attention_handle(cabi, heads, {}, 2.0, seed=S)
    q, k, v = _qkv(B, S, heads, 2.0, seed=S + 5)
    _check_stage(enc, q, k, v, pk, pq, idx, R, deberta_ids(B, S, True)[1] if B > 1 else None)
    enc.close()


@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("case", ["scores0.3", "peaked", "q0", "k0"])
@pytest.mark.parametrize("mask_kind", ["none", "right", "left", "holes"])
@pytest.mark.parametrize("S", [769, 2048])
def test_long_attention_matches_fp64(cabi, S, mask_kind, case, cfg):
    """q = 0: P depends on the p2c term alone; k = 0: on the c2p term alone; peaked: score std ~ 30"""
    heads, B = 4, 3
    std = {"scores0.3": 0.55, "peaked": 5.0, "q0": 2.5, "k0": 2.5}[case]
    pos_std = {"scores0.3": 0.55, "peaked": 5.0, "q0": 4.0, "k0": 4.0}[case]
    enc, pk, pq, idx, R = _attention_handle(cabi, heads, CONFIGS[cfg], pos_std, seed=S)
    q, k, v = _qkv(B, S, heads, std, seed=S + 1, zero_q=case == "q0", zero_k=case == "k0")
    _check_stage(enc, q, k, v, pk, pq, idx, R, _mask(B, S, mask_kind, seed=S + 2))
    enc.close()


@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("S", [1024, 8192])
def test_long_attention_cls_rows(cabi, S, cfg):
    """the first query block alone (CLS-only tail) sees every key block: offsets 0 .. -(S / 128 - 1)"""
    heads, B = 2, 2
    enc, pk, pq, idx, R = _attention_handle(cabi, heads, CONFIGS[cfg], 2.0, seed=S + 9)
    q, k, v = _qkv(B, S, heads, 2.0, seed=S + 3)
    _check_stage(enc, q, k, v, pk, pq, idx, R, deberta_ids(B, S, True, left=True)[1], cls_rows=True)
    enc.close()


# ------------------------------------------------------------------------------------------------ bitwise at S <= 512
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_radius_8192_handles_equal_radius_512_handles_bit_for_bit(cabi, cfg):
    """the stage alone (every mask kind, cls_rows) and forward_cls (CLS rows and the full hidden state) at S <= 512"""
    heads = 4
    a = _attention_handle(cabi, heads, CONFIGS[cfg], 2.0, seed=3, radius_long=False, max_tokens=3 * 512)
    b = _attention_handle(cabi, heads, CONFIGS[cfg], 2.0, seed=3, radius_long=True, max_tokens=3 * 512)
    assert a[4] == 512 and b[4] == LONG
    for S in (16, 77, 129, 300, 384, 385, 512):
        q, k, v = _qkv(3, S, heads, 2.8, seed=S)
        for kind in ("none", "right", "left", "holes"):
            mask = _mask(3, S, kind, seed=S + 1)
            mask = None if mask is None else mask.cuda()
            for cls_rows in (False, True):
                oa = a[0].attention(q.cuda(), k.cuda(), v.cuda(), mask, cls_rows=cls_rows)
                ob = b[0].attention(q.cuda(), k.cuda(), v.cuda(), mask, cls_rows=cls_rows)
                rows = min(S, 128) if cls_rows else S
                assert torch.equal(oa[:, :rows], ob[:, :rows]), (S, kind, cls_rows)
    a[0].close(); b[0].close()
    m = deberta_model(num_hidden_layers=2, **CONFIGS[cfg], **WIDE)
    for cls_only in (True, False):
        encs = []
        for long_ in (False, True):
            sd, dims = _dims(cabi, m, long_)
            encs.append(cabi.Encoder(sd, arch="deberta", max_tokens=3 * 512, cls_only=cls_only, **dims))
        for S in (16, 77, 300, 512):
            ids, mask = deberta_ids(3, S, True, vocab=WIDE["vocab_size"])
            ids, mask = ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()
            outs = [e.forward_cls(ids, mask) for e in encs]
            assert torch.equal(outs[0], outs[1]), (S, cls_only)
            if not cls_only:
                assert torch.equal(encs[0].last_hidden(3, S), encs[1].last_hidden(3, S)), S
        for e in encs:
            e.close()


# ------------------------------------------------------------------------------------------------ whole encoders
@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("B,S", [(3, 600), (2, 1100), (2, 2048), (1, 8192)])
def test_long_deberta_encoder_matches_oracle(cabi, B, S, cls_only, cfg):
    """2 x 256 (4 heads of 64; 2 x 128 at 8192), O(1) position terms, right padding; the valid rows of the hidden state
    too, under test_gpu_deberta.py's bounds at 512"""
    width = dict(hidden_size=128, num_attention_heads=2, intermediate_size=256) if S > 2048 else {}
    m = deberta_model(num_hidden_layers=2, **width, **CONFIGS[cfg])
    ids, mask = deberta_ids(B, S, True)
    ref, ref_hidden = _oracle(m, ids, mask, return_hidden=True)
    sd, dims = _dims(cabi, m)
    enc = cabi.Encoder(sd, arch="deberta", max_tokens=B * S, cls_only=cls_only, **dims)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    e = out - ref
    assert e.abs().max() < 3e-4 and e.norm(dim=1).max() < 1e-3, (e.abs().max(), e.norm(dim=1).max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5
    if not cls_only:
        hidden = enc.last_hidden(B, S).cpu().view(B, S, -1)
        keep = mask.bool()
        eh = hidden[keep] - ref_hidden[keep]
        assert eh.abs().max() < 5e-3, eh.abs().max()
    enc.close()


@pytest.mark.parametrize("B,S", [(1, 8192), (4, 2048)])
def test_deberta_base_long_matches_oracle(cabi, B, S):
    """the deberta-v3-base shape (workload.deberta_base) through Encoder.from_hf, every CLS row against the oracle"""
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.deberta_base(1234)
    ids, mask = deberta_ids(B, S, B > 1, vocab=cfg.vocab_size, seed=3)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    ref = _oracle(m, ids, mask)
    e = out - ref
    assert e.norm(dim=1).max() < 1e-3 and e.abs().max() < 2e-4, (e.norm(dim=1).max(), e.abs().max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5 and bool(torch.isfinite(out).all())
    enc.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(cabi):
    m = deberta_model(num_hidden_layers=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=LONG + 1)
    ids = torch.ones(1, LONG + 1, dtype=torch.int32, device="cuda")
    with pytest.raises(cabi.AdaptiveB200Error, match=f"S={LONG + 1} exceeds {LONG}"):
        enc.forward_cls(ids)
    enc.close()
    # absolute positions: the 512 limit and its message stay
    m = deberta_model(num_hidden_layers=1, position_biased_input=True)
    enc = cabi.Encoder.from_hf(m, max_tokens=1024)
    with pytest.raises(cabi.AdaptiveB200Error, match="S=513 > 512 is not supported"):
        enc.forward_cls(torch.ones(1, 513, dtype=torch.int32, device="cuda"))
    enc.close()
    # a long radius on a nonzero position table
    sd, dims = cabi.deberta_to_bert_state_dict(dict(m.state_dict()), m.config)
    dims["rel_index_long"] = cabi.deberta_rel_index(256, 512, LONG)[0]
    with pytest.raises(cabi.AdaptiveB200Error, match="all-zero pos_emb"):
        cabi.Encoder(sd, arch="deberta", max_tokens=1024, **dims)
