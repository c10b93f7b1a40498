"""CPU tests of the ModernBERT encoder support: the fp32 oracle (oracle/modernbert_oracle.py) pinned
against the installed HF ModernBertModel, the RoPE tables handed to the library, the reference's golden embeddings, and
the settings Encoder.from_hf refuses before any device call."""
import numpy as np
import pytest
import torch

import golden_npz
from oracle.modernbert_oracle import make_modernbert, modernbert_forward_cls


def _tiny(seed=3, layers=4, local_attention=8, **over):
    kw = dict(vocab_size=300, hidden_size=128, num_hidden_layers=layers, num_attention_heads=2, intermediate_size=192,
              local_attention=local_attention, max_position_embeddings=512, pad_token_id=0)
    sd, cfg, m = make_modernbert(seed, **{**kw, **over})
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "norm" in n:                                   # non-unit gamma (the init is all ones)
                p.add_(0.3 * torch.randn(p.shape, generator=g))
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    return sd, cfg, m


def _oracle_kwargs(cfg):
    from adaptive_classifier_b200._cabi import modernbert_settings
    s = modernbert_settings(cfg)
    return dict(num_heads=cfg.num_attention_heads, layer_sliding=[bool(v) for v in s["layer_sliding"]],
                sliding_window=s["sliding_window"], rope_theta=s["rope_theta"], norm_eps=cfg.norm_eps)


@pytest.mark.parametrize("S", [16, 77, 150, 300])
def test_modernbert_oracle_matches_hf(S):
    sd, cfg, m = _tiny()
    assert cfg.sliding_window == 4 and 2 * cfg.sliding_window + 1 < S     # the band cuts every sequence
    assert set(cfg.layer_types[:3]) == {"full_attention", "sliding_attention"}
    g = torch.Generator().manual_seed(S)
    B = 3
    ids = torch.randint(1, 300, (B, S), generator=g)
    mask = torch.ones(B, S, dtype=torch.int64)
    mask[1, S * 2 // 3:] = 0                                   # padded rows
    mask[2, S - 3:] = 0
    ids[mask == 0] = 0
    with torch.no_grad():
        ref = m(input_ids=ids, attention_mask=mask).last_hidden_state
        unit, hidden = modernbert_forward_cls(sd, ids, mask, return_hidden=True, **_oracle_kwargs(cfg))
    ref_unit = ref[:, 0] / ref[:, 0].norm(dim=1, keepdim=True)
    assert (unit - ref_unit).abs().max() < 1e-5
    valid = mask.bool()
    assert (hidden[valid] - ref[valid]).abs().max() < 1e-5


def test_modernbert_oracle_band_edge_is_inclusive():
    """|i - j| <= sliding_window (masking_utils.sliding_window_bidirectional_overlay) holds, not < sliding_window + 1 - 1"""
    sd, cfg, m = _tiny(layers=2)
    ids = torch.randint(1, 300, (1, 40), generator=torch.Generator().manual_seed(1))
    kw = _oracle_kwargs(cfg)
    with torch.no_grad():
        ref = m(input_ids=ids).last_hidden_state
        ok = modernbert_forward_cls(sd, ids, None, return_hidden=True, **kw)[1]
        narrow = modernbert_forward_cls(sd, ids, None, return_hidden=True, **{**kw, "sliding_window": kw["sliding_window"] - 1})[1]
        wide = modernbert_forward_cls(sd, ids, None, return_hidden=True, **{**kw, "sliding_window": kw["sliding_window"] + 1})[1]
    assert (ok - ref).abs().max() < 1e-5
    assert (narrow - ref).abs().max() > 1e-3 and (wide - ref).abs().max() > 1e-3


def test_rope_tables_equal_hf_rotary_embedding():
    from transformers.models.modernbert.modeling_modernbert import ModernBertRotaryEmbedding
    from adaptive_classifier_b200._cabi import AC_ENCODER_MAX_S, modernbert_rope_table, modernbert_settings
    _, cfg, _ = _tiny()
    rot = ModernBertRotaryEmbedding(cfg)
    pos = torch.arange(AC_ENCODER_MAX_S)[None]
    theta = dict(zip(("full_attention", "sliding_attention"), modernbert_settings(cfg)["rope_theta"]))
    assert theta == {"full_attention": 160000.0, "sliding_attention": 10000.0}
    for lt, th in theta.items():
        cos, sin = rot(torch.zeros(1, dtype=torch.float32), pos, lt)
        t = modernbert_rope_table(th)
        assert t.shape == (AC_ENCODER_MAX_S, 64) and t.dtype == torch.float32
        assert torch.equal(t[:, :32], cos[0, :, :32]) and torch.equal(t[:, :32], cos[0, :, 32:])
        assert torch.equal(t[:, 32:], sin[0, :, :32]) and torch.equal(t[:, 32:], sin[0, :, 32:])


@pytest.mark.parametrize("over, what", [
    (dict(hidden_activation="silu"), "hidden_activation"),
    (dict(norm_bias=True), "norm_bias"),
    (dict(attention_bias=True), "attention_bias"),
    (dict(mlp_bias=True), "mlp_bias"),
    (dict(rope_parameters={"full_attention": {"rope_type": "linear", "rope_theta": 160000.0, "factor": 2.0},
                           "sliding_attention": {"rope_type": "default", "rope_theta": 10000.0}}), "rope_type"),
    (dict(num_attention_heads=4), "head_dim"),
])
def test_from_hf_rejects_unsupported_modernbert_settings(over, what):
    from adaptive_classifier_b200._cabi import AdaptiveB200Error, Encoder
    _, cfg, m = _tiny(layers=3, **over)
    with pytest.raises(AdaptiveB200Error, match=what):
        Encoder.from_hf(m, device="cpu")


def test_modernbert_oracle_reproduces_reference_embeddings():
    """the fp32 oracle on the golden checkpoint gives the unmodified reference's own _get_embeddings output"""
    gold = golden_npz.load("golden_classifier_modernbert")
    from transformers import ModernBertConfig
    import json
    cfg = ModernBertConfig(**json.loads(str(gold["bert_config"])))
    sd = {k[5:]: torch.from_numpy(gold[k]) for k in gold.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(gold["input_ids"]).long()
    mask = torch.from_numpy(gold["attention_mask"]).long()
    n = len(gold["texts"])
    with torch.no_grad():
        unit = modernbert_forward_cls(sd, ids, mask, **_oracle_kwargs(cfg)).numpy()
    ref = np.concatenate([gold["emb_train"], gold["emb_test"]])
    assert unit.shape == ref.shape and n == gold["emb_train"].shape[0]
    assert np.abs(unit - ref).max() < 1e-5
