"""GPU tests of the DeBERTa-v3 encoders (deberta-v3-xsmall / small / base / large, mdeberta-v3-base: the post-LN BERT block
with disentangled c2p + p2c attention) against the fp32 oracle of oracle/deberta_oracle.py (pinned to HF DebertaV2Model by
tests/test_deberta_cpu.py), HF itself on the CPU and an fp64 reference of the attention stage alone.  The golden classifier
run, the CUDA-graph pipeline step and the drop-in classifier on a local checkpoint are tests/test_gpu_encoder_families.py's.

Attention-stage bound, per output element (test_gpu_attention.py's, plus one term for the score arithmetic):

    |out - ref| <= 2^-10 (w . |v|) + 2^-11 |ref| + 2^-25 sum_attended |v| + 2^-24 + 2^-16 max_j E(i, j) (w . |v|)
    E(i, j) = (|q_i| . |k_j| + |q_i| . |PosK[c]| + |k_j| . |PosQ[c]|) / sqrt(3 dh)

  the kernel sums the three 64-term fp32 dot products in fp32 (relative error < 70 x 2^-24 < 2^-17 of E); a logit error e
  moves every weight by a factor within exp(+-2e), so the context by at most 2 e (w . |v|) + ... : 2^-16 E (w . |v|).
"""
import json
import math

import pytest
import torch

from oracle import deberta_oracle as do
from test_deberta_cpu import deberta_ids, deberta_model
from test_gpu_attention import attended_ref
from test_gpu_minilm import _check_cls

pytestmark = pytest.mark.gpu

WIDE = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=1000)
MAX_S = 512


def _hf_sd(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


def _deberta_encoder(cabi, m, max_tokens, cls_only=True):
    sd, dims = cabi.deberta_to_bert_state_dict(dict(m.state_dict()), m.config)
    return cabi.Encoder(sd, arch="deberta", max_tokens=max_tokens, cls_only=cls_only, **dims)


# ------------------------------------------------------------------------------------------------ encoder
@pytest.mark.parametrize("buckets", [256, 16])
@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("B,S,pad", [(3, 16, True), (5, 77, True), (4, 128, True), (3, 129, True), (3, 300, True),
                                     (2, 512, True)])
def test_deberta_encoder_matches_oracle(cabi, B, S, pad, cls_only, buckets):
    """2 x 768, 12 heads of 64, O(1) position terms and perturbed LayerNorms; valid rows of the full hidden state too"""
    m = deberta_model(num_hidden_layers=2, position_buckets=buckets, **WIDE)
    ids, mask = deberta_ids(B, S, pad, vocab=WIDE["vocab_size"])
    ref, ref_hidden = do.deberta_forward_cls(_hf_sd(m), ids, mask, m.config, return_hidden=True)
    enc = _deberta_encoder(cabi, m, B * S, cls_only=cls_only)
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


def test_deberta_base_at_the_benched_batch_matches_oracle_on_sampled_rows(cabi):
    """the deberta-v3-base shape (workload.deberta_base) at B = 512 x S = 128: 8 sampled sequences against the oracle"""
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.deberta_base(1234)
    B, S = 512, 128
    ids, _ = deberta_ids(B, S, False, vocab=cfg.vocab_size, seed=3)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda()).cpu()
    sel = torch.tensor([0, 1, 63, 127, 128, 300, 510, 511])
    ref = do.deberta_forward_cls(_hf_sd(m), ids[sel], None, cfg)
    e = out[sel] - ref
    assert e.norm(dim=1).max() < 1e-3 and e.abs().max() < 2e-4, (e.norm(dim=1).max(), e.abs().max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5 and bool(torch.isfinite(out).all())
    enc.close()


@pytest.mark.parametrize("over", [{}, dict(share_att_key=False, position_biased_input=True, type_vocab_size=2)])
def test_deberta_through_from_hf_matches_hf(cabi, over):
    """a seeded DebertaV2Model through Encoder.from_hf, against HF on the CPU"""
    m = deberta_model(seed=11, num_hidden_layers=3, proj_scale=2.0, **WIDE, **over)
    ids, mask = deberta_ids(4, 150, True, vocab=WIDE["vocab_size"])
    with torch.no_grad():
        ref = torch.nn.functional.normalize(m(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=4 * 150)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check_cls(out, ref)
    enc.close()


# ------------------------------------------------------------------------------------------------ attention stage alone
def _attention_handle(cabi, heads, buckets, pos_std, seed):
    """a one-layer DeBERTa handle whose layer-0 position tables are seeded N(0, pos_std) [1, 2 span, H]; returns the handle,
    the fp16-rounded tables as the kernel sees them, and rel_index"""
    m = deberta_model(num_hidden_layers=1, hidden_size=64 * heads, num_attention_heads=heads, intermediate_size=128,
                      vocab_size=100, position_buckets=buckets)
    sd, dims = cabi.deberta_to_bert_state_dict(dict(m.state_dict()), m.config)
    g = torch.Generator().manual_seed(seed)
    span, H = dims["pos_span"], 64 * heads
    dims["pos_key"] = pos_std * torch.randn(1, 2 * span, H, generator=g)
    dims["pos_query"] = pos_std * torch.randn(1, 2 * span, H, generator=g)
    enc = cabi.Encoder(sd, arch="deberta", max_tokens=8 * MAX_S, **dims)
    return enc, dims["pos_key"][0].half(), dims["pos_query"][0].half(), dims["rel_index"].long()


def _deberta_attention_ref(q, k, v, pk, pq, rel_index, mask):
    """(context, bound) [B, S, heads, dh] fp64: softmax over the attended keys of (q.k + q.PosK[c(i-j)] + k.PosQ[c(i-j)])
    / sqrt(3 dh); rows without an attended key are 0"""
    B, S, heads, dh = q.shape
    pos = torch.arange(S)
    c = rel_index[MAX_S - 1 + pos[:, None] - pos[None, :]].expand(B, heads, S, S)   # c(i - j) at [.., i, j]
    qd, kd = q.double().transpose(1, 2), k.double().transpose(1, 2)            # [B, heads, S, dh]
    PK = pk.double().view(-1, heads, dh).transpose(0, 1)                       # [heads, 2 span, dh]
    PQ = pq.double().view(-1, heads, dh).transpose(0, 1)
    scale = 1.0 / math.sqrt(3 * dh)

    def terms(qq, kk, pkk, pqq):
        c2p = torch.gather(qq @ pkk.transpose(-1, -2), -1, c)                  # q_i . PosK[c(i - j)]
        p2c = torch.gather(kk @ pqq.transpose(-1, -2), -1, c.transpose(-1, -2)).transpose(-1, -2)   # k_j . PosQ[c(i - j)]
        return (qq @ kk.transpose(-1, -2) + c2p + p2c) * scale

    s = terms(qd, kd, PK, PQ)
    E = terms(qd.abs(), kd.abs(), PK.abs(), PQ.abs())
    att = attended_ref(B, S, mask)
    x = s.masked_fill(~att, -math.inf)
    mx = x.amax(-1, keepdim=True)
    p = torch.exp(x - torch.where(torch.isinf(mx), torch.zeros_like(mx), mx))
    w = p / p.sum(-1, keepdim=True).clamp_min(1e-300)
    vv = v.double().permute(0, 2, 1, 3)
    out, wabs, reach = w @ vv, w @ vv.abs(), att.double() @ vv.abs()
    emax = E.masked_fill(~att, 0).amax(-1, keepdim=True)
    tol = (2.0 ** -10 + 2.0 ** -16 * emax) * wabs + 2.0 ** -11 * out.abs() + 2.0 ** -25 * reach + 2.0 ** -24
    return out.permute(0, 2, 1, 3), tol.permute(0, 2, 1, 3)


def _qkv(B, S, heads, std, seed, zero_q=False, zero_k=False):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, S, heads, 64, generator=g) for _ in range(3))
    q = torch.zeros_like(q) if zero_q else std * q
    k = torch.zeros_like(k) if zero_k else std * k
    return q.half(), k.half(), v.half()


def _mask(B, S, kind, seed):
    if kind == "none":
        return None
    if kind == "right":
        return deberta_ids(B, S, True)[1]
    if kind == "left":
        return deberta_ids(B, S, True, left=True)[1]
    g = torch.Generator().manual_seed(seed)                                   # holes, one sequence with a single key
    m = (torch.rand(B, S, generator=g) > 0.3).to(torch.int32)
    m[0] = 0
    m[0, S // 2] = 1
    return m


SEAMS = [1, 2, 8, 64, 127, 128, 129, 255, 256, 257, 383, 384, 385, 511, 512]
FRACTIONS = {}


@pytest.mark.parametrize("buckets", [256, 16])
@pytest.mark.parametrize("case", ["scores0.3", "scores8", "peaked", "q0", "k0"])
@pytest.mark.parametrize("mask_kind", ["none", "right", "left", "holes"])
@pytest.mark.parametrize("S", [16, 77, 129, 300, 512])
def test_deberta_attention_stage_matches_fp64(cabi, S, mask_kind, case, buckets):
    """q = 0: P depends on the p2c term alone; k = 0: on the c2p term alone (plus masks); peaked: score std ~ 30"""
    heads, B = 4, 3
    std = {"scores0.3": 0.55, "scores8": 2.8, "peaked": 5.0, "q0": 2.5, "k0": 2.5}[case]
    pos_std = {"scores0.3": 0.55, "scores8": 2.8, "peaked": 5.0, "q0": 4.0, "k0": 4.0}[case]
    enc, pk, pq, ri = _attention_handle(cabi, heads, buckets, pos_std, seed=S)
    q, k, v = _qkv(B, S, heads, std, seed=S + 1, zero_q=case == "q0", zero_k=case == "k0")
    mask = _mask(B, S, mask_kind, seed=S + 2)
    out = enc.attention(q.cuda(), k.cuda(), v.cuda(), None if mask is None else mask.cuda(), pad_fill=1000.0).cpu()
    ref, tol = _deberta_attention_ref(q, k, v, pk, pq, ri, mask)
    err = (out.double() - ref).abs()
    frac = (err / tol).max().item()
    FRACTIONS[case] = max(FRACTIONS.get(case, 0.0), frac)
    assert bool(torch.isfinite(out).all()) and frac <= 1.0, (frac, err.max().item())
    enc.close()


@pytest.mark.parametrize("S", SEAMS)
def test_deberta_attention_at_every_block_seam(cabi, S):
    """sequence lengths on both sides of every 128-key / 128-query seam up to 512, with right padding"""
    heads, B = 4, 2
    enc, pk, pq, ri = _attention_handle(cabi, heads, 256, 2.0, seed=S)
    q, k, v = _qkv(B, S, heads, 2.0, seed=S + 5)
    mask = deberta_ids(B, S, True)[1] if S > 2 else None
    out = enc.attention(q.cuda(), k.cuda(), v.cuda(), None if mask is None else mask.cuda(), pad_fill=1000.0).cpu()
    ref, tol = _deberta_attention_ref(q, k, v, pk, pq, ri, mask)
    frac = ((out.double() - ref).abs() / tol).max().item()
    FRACTIONS["seams"] = max(FRACTIONS.get("seams", 0.0), frac)
    assert frac <= 1.0, frac
    enc.close()


def test_deberta_attention_report_fractions():
    """prints the largest error seen per family as a fraction of the bound (recorded in DESIGN.md)"""
    print("deberta attention error / bound:", json.dumps({k: round(v, 3) for k, v in sorted(FRACTIONS.items())}))
