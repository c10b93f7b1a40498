"""CPU tests of ModernBERT at sequence lengths past 512: the query-block oracle (oracle/modernbert_long_oracle.py) pinned to
the unchanged oracle and to HF ModernBertModel (eager) at S up to 2048, the max_pos-row RoPE tables handed to the library,
the max_position_embeddings limit, and the reference's long-input golden embeddings."""
import json

import numpy as np
import pytest
import torch

import golden_npz
from oracle.modernbert_long_oracle import modernbert_forward_cls_blocked
from oracle.modernbert_oracle import make_modernbert, modernbert_forward_cls


def _tiny(seed=3, layers=4, local_attention=16, max_position_embeddings=8192, **over):
    kw = dict(vocab_size=300, hidden_size=128, num_hidden_layers=layers, num_attention_heads=2, intermediate_size=192,
              local_attention=local_attention, max_position_embeddings=max_position_embeddings, pad_token_id=0)
    sd, cfg, m = make_modernbert(seed, **{**kw, **over})
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "norm" in n:                                   # non-unit gamma (the init is all ones)
                p.add_(0.3 * torch.randn(p.shape, generator=g))
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    return sd, cfg, m


def _kwargs(cfg):
    from adaptive_classifier_b200._cabi import modernbert_settings
    s = modernbert_settings(cfg)
    return dict(num_heads=cfg.num_attention_heads, layer_sliding=[bool(v) for v in s["layer_sliding"]],
                sliding_window=s["sliding_window"], rope_theta=s["rope_theta"], norm_eps=cfg.norm_eps)


def _batch(B, S, lens, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(5, 300, (B, S), generator=g)
    ids[:, 0] = 2
    mask = torch.ones(B, S, dtype=torch.int64)
    for b, n in enumerate(lens):
        mask[b, n:] = 0
    ids[mask == 0] = 0
    return ids, mask


@pytest.mark.parametrize("S", [77, 300])
def test_query_block_oracle_equals_the_unchanged_oracle(S):
    sd, cfg, _ = _tiny(local_attention=16, max_position_embeddings=512)
    ids, mask = _batch(3, S, [S, S * 2 // 3, S - 3], S)
    kw = _kwargs(cfg)
    with torch.no_grad():
        ref, ref_h = modernbert_forward_cls(sd, ids, mask, return_hidden=True, **kw)
        for qb in (128, 32):
            unit, hid = modernbert_forward_cls_blocked(sd, ids, mask, return_hidden=True, q_block=qb, **kw)
            valid = mask.bool()
            assert (unit - ref).abs().max() < 1e-6
            assert (hid[valid] - ref_h[valid]).abs().max() < 1e-6 * max(1.0, float(ref_h[valid].abs().max()))


@pytest.mark.parametrize("S,local_attention,lens", [
    (600, 16, [600, 513]),                   # half-window 8
    (1100, 128, [1100, 385, 641]),           # half-window 64; valid lengths 128 n +- 1
    (2048, 400, [2048, 1151]),               # half-window 200: the band spans several 128-key blocks
])
def test_query_block_oracle_matches_hf_past_512(S, local_attention, lens):
    sd, cfg, m = _tiny(local_attention=local_attention)
    assert cfg.max_position_embeddings == 8192 and 2 * cfg.sliding_window + 1 < S
    ids, mask = _batch(len(lens), S, lens, S + local_attention)
    with torch.no_grad():
        ref = m(input_ids=ids, attention_mask=mask).last_hidden_state
        unit, hidden = modernbert_forward_cls_blocked(sd, ids, mask, return_hidden=True, **_kwargs(cfg))
    ref_unit = ref[:, 0] / ref[:, 0].norm(dim=1, keepdim=True)
    assert (unit - ref_unit).abs().max() < 1e-5
    valid = mask.bool()
    assert (hidden[valid] - ref[valid]).abs().max() < 1e-5


def test_rope_tables_of_8192_rows_equal_hf_rotary_embedding():
    from transformers.models.modernbert.modeling_modernbert import ModernBertRotaryEmbedding
    from adaptive_classifier_b200._cabi import AC_MODERNBERT_MAX_S, modernbert_rope_table, modernbert_settings
    _, cfg, _ = _tiny()
    s = modernbert_settings(cfg)
    assert s["max_pos"] == AC_MODERNBERT_MAX_S == 8192
    rot = ModernBertRotaryEmbedding(cfg)
    pos = torch.arange(s["max_pos"])[None]
    for lt, th in zip(("full_attention", "sliding_attention"), s["rope_theta"]):
        cos, sin = rot(torch.zeros(1, dtype=torch.float32), pos, lt)
        t = modernbert_rope_table(th, s["max_pos"])
        assert t.shape == (8192, 64) and t.dtype == torch.float32
        assert torch.equal(t[:, :32], cos[0, :, :32]) and torch.equal(t[:, :32], cos[0, :, 32:])
        assert torch.equal(t[:, 32:], sin[0, :, :32]) and torch.equal(t[:, 32:], sin[0, :, 32:])
        # the first 512 rows are the table a 512-position encoder gets: S <= 512 runs compute the same bits
        assert torch.equal(t[:512], modernbert_rope_table(th))


def test_max_pos_follows_the_config():
    from adaptive_classifier_b200._cabi import modernbert_settings
    for mpe, want in ((128, 512), (512, 512), (1024, 1024), (8192, 8192)):
        assert modernbert_settings(_tiny(layers=3, max_position_embeddings=mpe)[1])["max_pos"] == want


def test_max_position_embeddings_over_8192_is_refused_by_name():
    from adaptive_classifier_b200._cabi import AdaptiveB200Error, Encoder
    _, cfg, m = _tiny(layers=3, max_position_embeddings=16384)
    with pytest.raises(AdaptiveB200Error, match="max_position_embeddings"):
        Encoder.from_hf(m, device="cpu")


def test_query_block_oracle_reproduces_reference_long_embeddings():
    """the oracle on the golden checkpoint gives the unmodified reference's _get_embeddings output with max_length 1024"""
    from transformers import ModernBertConfig
    gold = golden_npz.load("golden_classifier_modernbert_long", weights_from="golden_classifier_modernbert")
    cfg = ModernBertConfig(**json.loads(str(gold["bert_config"])))
    assert cfg.max_position_embeddings == 8192 and int(gold["max_length"]) == 1024
    sd = {k[5:]: torch.from_numpy(gold[k]) for k in gold.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(gold["input_ids"]).long()
    mask = torch.from_numpy(gold["attention_mask"]).long()
    lens = mask.sum(1)
    assert ids.shape[1] == 1024 and bool((lens > 512).any()) and bool((lens < 64).any())
    with torch.no_grad():
        unit = modernbert_forward_cls_blocked(sd, ids, mask, **_kwargs(cfg)).numpy()
    ref = np.concatenate([gold["emb_train"], gold["emb_test"]])
    assert unit.shape == ref.shape
    assert np.abs(unit - ref).max() < 1e-5
