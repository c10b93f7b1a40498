"""CPU tests of DeBERTa-v3 past 512 tokens: the fp32 oracle against HF DebertaV2Model at long S, the radius-8192 index
table against HF's relative positions, the saturation rule that bounds the handle's relative operand boxes at every S,
the reference's golden embeddings at max_length 1024, and which configs Encoder.from_hf gives the long table to."""
import json

import numpy as np
import pytest
import torch

import golden_npz
from oracle import deberta_oracle as do
from test_deberta_cpu import _sd, deberta_ids, deberta_model

# (position_buckets, max_relative_positions) -> D of the published settings and the others the tests cover
CONFIGS = {(256, 512): 5, (16, 512): 5, (-1, 512): 5, (-1, 64): 2}
HF_CONFIGS = [dict(), dict(position_buckets=16), dict(position_buckets=-1, max_relative_positions=64)]


def box_radius(idx: torch.Tensor, radius: int) -> int:
    """restatement of encoder.cu deberta_box_radius: the least d <= (radius - 1) / 128 with c(r) constant for
    r >= 128 d - 127 and for r <= 127 - 128 d (entry radius - 1 + r of idx is c(r))"""
    c = idx.long()
    cap = (radius - 1) // 128
    for d in range(cap):
        hi = c[radius - 1 + 128 * d - 127:]
        lo = c[: radius - 1 + 127 - 128 * d + 1]
        if bool((hi == c[-1]).all()) and bool((lo == c[0]).all()):
            return d
    return cap


def box_indices(idx: torch.Tensor, radius: int, n: int, d: int) -> torch.Tensor:
    """[2 terms, 255] index rows pos_gather_kernel reads for box d of n (rows 0..254; row 255 is zero)"""
    delta = 128 * (d - n // 2)
    t = torch.arange(255)
    rows = []
    for r in (delta + t - 127, delta + 127 - t):
        rows.append(idx.long()[radius - 1 + r.clamp(1 - radius, radius - 1)])
    return torch.stack(rows)


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("over", HF_CONFIGS, ids=["b256", "b16", "nob64"])
@pytest.mark.parametrize("left", [False, True], ids=["right", "left"])
@pytest.mark.parametrize("B,S", [(3, 600), (2, 1100), (2, 2048)])
def test_deberta_oracle_matches_hf_past_512(B, S, left, over):
    m = deberta_model(**over)
    ids, mask = deberta_ids(B, S, True, left=left)
    with torch.no_grad():
        hidden = m(input_ids=ids, attention_mask=mask).last_hidden_state
    ref = torch.nn.functional.normalize(hidden[:, 0, :], dim=1)
    out, out_hidden = do.deberta_forward_cls(_sd(m), ids, mask, m.config, return_hidden=True)
    keep = mask.bool()
    assert (out - ref)[keep[:, 0]].abs().max() < 1e-6
    assert (out_hidden[keep] - hidden[keep]).abs().max() < 1e-6 * max(1.0, hidden.abs().max().item())


# ------------------------------------------------------------------------------------------------ index table
@pytest.mark.parametrize("buckets,max_rel", list(CONFIGS))
def test_long_rel_index_equals_hf_build_relative_position_at_2048(buckets, max_rel):
    """entry 8191 + (i - j) of the radius-8192 table is HF's c2p index, and the p2c index it gathers, on every pair of
    S = 2048; the first 1023 entries around the centre are the radius-512 table"""
    from transformers.models.deberta_v2.modeling_deberta_v2 import build_relative_position
    from adaptive_classifier_b200._cabi import AC_ENCODER_MAX_S, AC_MODERNBERT_MAX_S, deberta_rel_index
    R, S = AC_MODERNBERT_MAX_S, 2048
    table, span = deberta_rel_index(buckets, max_rel, R)
    assert table.shape == (2 * R - 1,) and table.dtype == torch.int32
    x = torch.zeros(1, S, 8)
    rp = build_relative_position(x, x, bucket_size=buckets, max_position=max_rel)[0]
    i = torch.arange(S)[:, None]
    j = torch.arange(S)[None, :]
    assert torch.equal(table[R - 1 + i - j].long(), torch.clamp(rp + span, 0, 2 * span - 1))
    assert torch.equal(table[R - 1 + i - j].long(), torch.clamp(-rp.t() + span, 0, 2 * span - 1))
    short, _ = deberta_rel_index(buckets, max_rel)
    M = AC_ENCODER_MAX_S
    assert torch.equal(table[R - M: R + M - 1], short)


@pytest.mark.parametrize("buckets,max_rel", [(256, 512), (-1, 512)])
def test_long_rel_index_equals_hf_on_the_full_range(buckets, max_rel):
    """the published settings over every r in (-8192, 8192), through HF's own make_log_bucket_position"""
    from transformers.models.deberta_v2.modeling_deberta_v2 import make_log_bucket_position
    from adaptive_classifier_b200._cabi import AC_MODERNBERT_MAX_S, deberta_rel_index
    R = AC_MODERNBERT_MAX_S
    table, span = deberta_rel_index(buckets, max_rel, R)
    r = torch.arange(-(R - 1), R, dtype=torch.long)
    rp = make_log_bucket_position(r, buckets, max_rel) if buckets > 0 else r
    assert torch.equal(table.long(), torch.clamp(rp + span, 0, 2 * span - 1))


# ------------------------------------------------------------------------------------------------ saturation rule
@pytest.mark.parametrize("cfg", list(CONFIGS), ids=lambda c: f"{c[0]}_{c[1]}")
def test_box_radius_of_each_config_and_constant_beyond_it(cfg):
    from adaptive_classifier_b200._cabi import AC_MODERNBERT_MAX_S, deberta_rel_index
    R = AC_MODERNBERT_MAX_S
    table, span = deberta_rel_index(*cfg, R)
    D = box_radius(table, R)
    assert D == CONFIGS[cfg]
    c = table.long()
    r = torch.arange(-(R - 1), R)
    assert bool((c[r >= 128 * D - 127] == 2 * span - 1).all()) and bool((c[r <= 127 - 128 * D] == 0).all())
    # D is the least such radius: the box at -(D - 1) or the one at D - 1 still holds more than one row
    n = 2 * D + 1
    inner = [box_indices(table, R, n, n // 2 + s * (D - 1)) for s in (-1, 1)]
    assert any(len(torch.unique(b)) > 1 for b in inner)
    # every offset past D reads exactly the rows of the box at +-D
    for off in range(D + 1, (R - 1) // 128 + 1):
        for s in (-1, 1):
            far = box_indices(table, R, 2 * off + 1, off + s * off)
            assert torch.equal(far, box_indices(table, R, n, n // 2 + s * D)), (off, s)


@pytest.mark.parametrize("cfg", list(CONFIGS), ids=lambda c: f"{c[0]}_{c[1]}")
def test_every_offset_up_to_512_reads_the_same_rows_from_both_radii(cfg):
    """the boxes of block offsets -3 .. 3 (S <= 512) built from the radius-8192 table with its D equal the ones of the
    radius-512 table with its own D, so a long-radius handle computes bit for bit what a radius-512 one does"""
    from adaptive_classifier_b200._cabi import AC_ENCODER_MAX_S, AC_MODERNBERT_MAX_S, deberta_rel_index
    tl, _ = deberta_rel_index(*cfg, AC_MODERNBERT_MAX_S)
    ts, _ = deberta_rel_index(*cfg)
    Dl, Ds = box_radius(tl, AC_MODERNBERT_MAX_S), box_radius(ts, AC_ENCODER_MAX_S)
    assert Ds <= 3
    for off in range(-3, 4):
        a = box_indices(tl, AC_MODERNBERT_MAX_S, 2 * Dl + 1, max(-Dl, min(Dl, off)) + Dl)
        b = box_indices(ts, AC_ENCODER_MAX_S, 2 * Ds + 1, max(-Ds, min(Ds, off)) + Ds)
        exact = box_indices(ts, AC_ENCODER_MAX_S, 7, off + 3)
        assert torch.equal(a, b) and torch.equal(b, exact), off


def test_box_memory_of_the_base_and_large_shapes():
    """layers x (2 D + 1) x heads x 64 KiB: 7 boxes per (layer, head, term) at radius 512, 11 at 8192"""
    from adaptive_classifier_b200._cabi import AC_ENCODER_MAX_S, AC_MODERNBERT_MAX_S, deberta_rel_index
    n = {R: 2 * box_radius(deberta_rel_index(256, 512, R)[0], R) + 1 for R in (AC_ENCODER_MAX_S, AC_MODERNBERT_MAX_S)}
    assert n == {AC_ENCODER_MAX_S: 7, AC_MODERNBERT_MAX_S: 11}
    mib = lambda layers, heads, R: layers * n[R] * heads * 2 * 256 * 64 * 2 / 1e6
    assert round(mib(12, 12, AC_ENCODER_MAX_S)) == 66 and round(mib(12, 12, AC_MODERNBERT_MAX_S)) == 104
    assert round(mib(24, 16, AC_ENCODER_MAX_S)) == 176 and round(mib(24, 16, AC_MODERNBERT_MAX_S)) == 277


# ------------------------------------------------------------------------------------------------ golden
def test_deberta_oracle_reproduces_reference_embeddings_at_max_length_1024():
    from transformers import DebertaV2Config
    g = golden_npz.load("golden_classifier_deberta_long", weights_from="golden_classifier_deberta")
    cfgd = json.loads(str(g["bert_config"]))
    assert cfgd == json.loads(str(golden_npz.load("golden_classifier_deberta")["bert_config"]))
    c = DebertaV2Config(**{k: v for k, v in cfgd.items() if k not in ("model_type", "transformers_version", "architectures")})
    sd = {k[5:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(g["input_ids"])
    mask = torch.from_numpy(g["attention_mask"])
    lens = mask.sum(1)
    assert ids.shape[1] == 1024 and int((lens > 512).sum()) >= 6 and int((lens < 64).sum()) >= 3
    out = do.deberta_forward_cls(sd, ids, mask, c)
    ref = np.concatenate([g["emb_train"], g["emb_test"]])
    assert out.shape == ref.shape
    assert np.abs(out.numpy() - ref).max() < 1e-5


# ------------------------------------------------------------------------------------------------ from_hf / refusals
@pytest.mark.parametrize("over,long", [({}, True), (dict(position_buckets=16), True),
                                       (dict(position_buckets=-1, max_relative_positions=64), True),
                                       (dict(position_biased_input=True), False),
                                       (dict(position_biased_input=True, type_vocab_size=2), False)])
def test_only_relative_only_configs_get_the_long_table(over, long):
    from adaptive_classifier_b200._cabi import AC_MODERNBERT_MAX_S, deberta_rel_index, deberta_to_bert_state_dict
    m = deberta_model(num_hidden_layers=1, **over)
    _, dims = deberta_to_bert_state_dict(dict(m.state_dict()), m.config)
    assert dims["rel_index"].shape == (1023,) and dims["max_pos"] == 512
    assert ("rel_index_long" in dims) == long
    if long:
        b = over.get("position_buckets", 256)
        mr = over.get("max_relative_positions", 512)
        assert torch.equal(dims["rel_index_long"], deberta_rel_index(b, mr, AC_MODERNBERT_MAX_S)[0])


def _create(cabi, arch, rel_radius):
    """ac_encoder_create on a config its argument checks refuse before any device call: returns (rc, message)"""
    import ctypes
    L = cabi.load_library()
    cfg = cabi.EncoderConfig(arch, 2, 256, 4, 512, 400, 512, 2, 0, 1e-12, cabi.AC_PREC_F16, 1024, 1)
    dummy = ctypes.c_void_p(0x1000)
    cfg.rel_bias = cfg.pos_key = cfg.pos_query = cfg.rel_index = dummy
    cfg.pos_span = 256
    cfg.rel_radius = rel_radius
    h = ctypes.c_void_p()
    rc = L.ac_encoder_create(ctypes.byref(cfg), ctypes.byref(cabi.EncoderWeights()), ctypes.byref(h))
    return rc, L.ac_last_error().decode()


@pytest.mark.parametrize("arch,rel_radius", [(4, -1), (4, 512), (4, 8193), (4, 100), (0, 8192), (1, 1024), (3, 8192)])
def test_encoder_create_refuses_bad_rel_radius(cabi, arch, rel_radius):
    rc, msg = _create(cabi, arch, rel_radius)
    assert rc == -1, (rc, msg)                                       # AC_E_INVALID
    assert f"rel_radius={rel_radius}" in msg, msg
