"""CPU tests of the EuroBERT encoder (AC_ARCH_EUROBERT: pre-norm block with RMSNorm, RoPE, SwiGLU, grouped-query attention):
  * oracle/eurobert_oracle.py against HF EuroBertModel (eager attention), padded both ways, S from 16 to 2048, kv heads
    = heads, heads / 2 and 1, and a non-default RoPE theta
  * the RoPE table the encoder reads against EuroBertRotaryEmbedding, bit for bit, at 8192 rows
  * the mapping consumes every parameter, and its GQA expansion is HF repeat_kv bit for bit
  * the golden classifier runs of oracle/make_golden_encoders.py eurobert eurobert_long against the oracle
  * each wrong rule (LayerNorm for RMSNorm, centred RMSNorm, layer-0 norm as identity, final norm skipped, RoPE dropped,
    padding-aware positions, tiled kv heads, gate / up swapped) moves the embeddings far past the GPU bound
  * eurobert_settings, remote-code and ac_encoder_create refusals, which run before any device call"""
import ctypes
import json
import re

import numpy as np
import pytest
import torch

import golden_npz
from oracle import eurobert_oracle as eo
from test_rotary_cpu import _Tracked, padded_batch

GPU_UNIT_BOUND = 5e-3          # unit-row error norm of tests/test_gpu_eurobert.py on the tiny models (TINY_BOUND there)


def tiny_model(seed=7, layers=2, hidden=256, heads=4, kv=2, inter=512, theta=10000.0, max_pos=8192, **over):
    """HF EuroBertModel in eager attention; norm weights moved off 1, q / k scaled up so that the attention is far from
    uniform and positions matter (x4 at hidden 256 spreads the scores as x8 does at hidden 128 in test_rotary_cpu.py), the
    other projections scaled up so that every sublayer moves the residual stream"""
    from transformers import EuroBertConfig, EuroBertModel
    torch.manual_seed(seed)
    cfg = EuroBertConfig(vocab_size=300, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                         num_key_value_heads=kv, intermediate_size=inter, max_position_embeddings=max_pos,
                         rope_parameters={"rope_type": "default", "rope_theta": theta}, bos_token_id=0, eos_token_id=2,
                         pad_token_id=1, mask_token_id=3, attn_implementation="eager", **over)
    m = EuroBertModel(cfg)
    m.eval()
    assert m.config._attn_implementation == "eager"
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "norm" in n:
                p.copy_(1.0 + 0.3 * torch.randn(p.shape, generator=g))
            elif "q_proj" in n or "k_proj" in n:
                p.mul_(4.0)
            elif p.dim() == 2 and "embed_tokens" not in n:
                p.mul_(3.0)
    return m


def sd_of(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


def hf_forward(m, ids, mask):
    with torch.no_grad():
        return m(input_ids=ids, attention_mask=mask).last_hidden_state


@pytest.mark.parametrize("kv", [4, 2, 1])
@pytest.mark.parametrize("S", [16, 77, 300, 600, 2048])
def test_oracle_matches_hf(S, kv):
    m = tiny_model(kv=kv)
    ids, mask, _ = padded_batch(S, S)
    hf = hf_forward(m, ids, mask)
    unit, hid = eo.eurobert_forward_for(m.config, sd_of(m), ids, mask, return_hidden=True)
    keep = mask.bool()
    assert (hid[keep] - hf[keep]).abs().max() < 1e-6 * max(1.0, hf[keep].abs().max().item())
    # row 0 is what the classifier pools, a pad row in the left-padded sequence
    assert (unit - torch.nn.functional.normalize(hf[:, 0], dim=1)).abs().max() < 1e-6


def test_oracle_matches_hf_with_the_published_theta():
    m = tiny_model(kv=2, theta=250000.0, seed=3)
    ids, mask, _ = padded_batch(600, 8)
    hf = hf_forward(m, ids, mask)
    unit, hid = eo.eurobert_forward_for(m.config, sd_of(m), ids, mask, return_hidden=True)
    keep = mask.bool()
    assert (hid[keep] - hf[keep]).abs().max() < 1e-6 * max(1.0, hf[keep].abs().max().item())
    assert (unit - torch.nn.functional.normalize(hf[:, 0], dim=1)).abs().max() < 1e-6


@pytest.mark.parametrize("theta", [10000.0, 250000.0])
def test_rope_table_is_bit_equal_to_hf_rotary_emb(cabi, theta):
    m = tiny_model(layers=1, theta=theta)
    x = torch.zeros(1, 8192, m.config.hidden_size)
    cos, sin = m.rotary_emb(x, torch.arange(8192)[None])
    table = cabi.modernbert_rope_table(theta, 8192)
    assert torch.equal(cos[0, :, :32], cos[0, :, 32:]) and torch.equal(sin[0, :, :32], sin[0, :, 32:])
    assert torch.equal(table[:, :32], cos[0, :, :32]) and torch.equal(table[:, 32:], sin[0, :, :32])


@pytest.mark.parametrize("kv", [4, 2, 1])
def test_mapping_consumes_every_parameter_and_expands_kv_heads_as_repeat_kv(cabi, kv):
    from transformers.models.eurobert.modeling_eurobert import repeat_kv
    m = tiny_model(layers=3, kv=kv)
    sd = _Tracked(m.state_dict())
    out, dims = cabi.eurobert_to_modernbert_names(sd, m.config)
    assert set(sd) == sd.read, set(sd) - sd.read
    names = {"embeddings.tok_embeddings.weight", "final_norm.weight"}
    for l in range(3):
        names |= {f"layers.{l}.{n}.weight" for n in ("attn_norm", "mlp_norm", "attn.Wqkv", "attn.Wo", "mlp.Wi", "mlp.Wo")}
    assert set(out) == names
    H, heads = 256, 4
    for l in range(3):
        p = f"layers.{l}."
        wqkv = out[p + "attn.Wqkv.weight"]
        assert wqkv.shape == (3 * H, H)
        assert torch.equal(wqkv[:H], sd[p + "self_attn.q_proj.weight"])
        for i, n in ((1, "k_proj"), (2, "v_proj")):
            w = sd[p + f"self_attn.{n}.weight"]                                   # [kv 64, H]
            ref = repeat_kv(w.view(1, kv, 64, H), heads // kv).reshape(heads * 64, H)
            assert torch.equal(wqkv[i * H:(i + 1) * H], ref)
        assert torch.equal(out[p + "mlp.Wi.weight"], torch.cat([sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]]))
        assert out[p + "attn_norm.weight"] is sd[p + "input_layernorm.weight"]
    assert dims == dict(layers=3, hidden=H, heads=heads, intermediate=512, vocab=300, max_pos=8192, ln_eps=1e-5, pad_idx=1,
                        rope_theta=10000.0)


@pytest.mark.parametrize("mpe,expect", [(128, 512), (2048, 2048), (8192, 8192), (16384, 8192)])
def test_sequence_limit_follows_max_position_embeddings(cabi, mpe, expect):
    m = tiny_model(layers=1)
    m.config.max_position_embeddings = mpe
    assert cabi.eurobert_settings(m.config)["max_pos"] == expect


# ------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize("name", ["golden_classifier_eurobert", "golden_classifier_eurobert_long"])
def test_golden_embeddings_match_the_oracle(name):
    golden = golden_npz.load(name, weights_from="golden_classifier_eurobert")
    cfg = json.loads(str(golden["bert_config"]))
    sd = {k[5:]: torch.from_numpy(golden[k]).float() for k in golden.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(golden["input_ids"]).long()
    mask = torch.from_numpy(golden["attention_mask"]).long()
    assert "token_type_ids" not in golden and cfg["num_key_value_heads"] == 2
    unit = eo.eurobert_forward_for(cfg, sd, ids, mask)
    ref = np.concatenate([golden["emb_train"], golden["emb_test"]])
    assert unit.shape[0] == len(golden["texts"]) + len(golden["test_texts"])
    assert np.abs(unit.numpy() - ref).max() < 1e-5
    assert (ids[:, 0] == 0).all()                                       # <|begin_of_text|> pooled
    if name.endswith("_long"):
        assert ids.shape[1] == 1024 and int((mask.sum(1) > 512).sum()) >= 3


# ------------------------------------------------------------------------------------------------ wrong rules
@pytest.mark.parametrize("wrong", eo.WRONG_RULES)
def test_each_wrong_rule_moves_the_embeddings_past_the_gpu_bound(wrong):
    m = tiny_model(seed=3, kv=2)
    ids, mask, _ = padded_batch(300, 5)
    sd = sd_of(m)
    ref = eo.eurobert_forward_for(m.config, sd, ids, mask)
    bad = eo.eurobert_forward_for(m.config, sd, ids, mask, wrong=wrong)
    moved = (bad - ref).norm(dim=1).max().item()
    assert moved >= 20 * GPU_UNIT_BOUND, (wrong, moved)


# ------------------------------------------------------------------------------------------------ refusals
def _with(m, **attrs):
    for k, v in attrs.items():
        setattr(m.config, k, v)
    return m


@pytest.mark.parametrize("attrs,name", [
    (dict(rope_parameters={"rope_type": "llama3", "rope_theta": 250000.0, "factor": 8.0}), "rope_type='llama3'"),
    (dict(rope_parameters={"rope_type": "yarn", "rope_theta": 250000.0, "factor": 4.0}), "rope_type='yarn'"),
    (dict(rope_parameters={"rope_type": "dynamic", "rope_theta": 250000.0, "factor": 2.0}), "rope_type='dynamic'"),
    (dict(rope_parameters={"rope_type": "linear", "rope_theta": 250000.0, "factor": 2.0}), "rope_type='linear'"),
    (dict(attention_bias=True), "attention_bias=True"),
    (dict(mlp_bias=True), "mlp_bias=True"),
    (dict(head_dim=128), "head_dim=128"),
    (dict(num_attention_heads=8, num_key_value_heads=8, head_dim=None), "head_dim=32"),
    (dict(hidden_size=192, num_attention_heads=3, num_key_value_heads=3), "hidden_size=192"),
    (dict(hidden_size=1152, num_attention_heads=18, num_key_value_heads=18), "hidden_size=1152"),
    (dict(hidden_act="gelu"), "hidden_act='gelu'"),
    (dict(num_key_value_heads=3), "num_key_value_heads=3"),
])
def test_from_hf_refuses_unimplemented_settings_by_name(cabi, attrs, name):
    m = _with(tiny_model(layers=1), **attrs)
    with pytest.raises(cabi.AdaptiveB200Error, match=re.escape(name)):
        cabi.Encoder.from_hf(m)


def test_from_hf_refuses_remote_code_modules_by_name(cabi):
    """a module that carries model_type 'eurobert' but is not the native class (the Hub's trust_remote_code EuroBertModel
    names its parameters differently)"""
    config = tiny_model(layers=1).config

    class RemoteCodeModel(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.config = config
            self.emb = torch.nn.Embedding(300, 256)

    with pytest.raises(cabi.AdaptiveB200Error, match="trust_remote_code"):
        cabi.Encoder.from_hf(RemoteCodeModel())


def _create_refusal(cabi, arch=6, hidden=256, heads=4, max_pos=8192, rope=True, weights=True, proj=False, ffn_act=2):
    """ac_encoder_create on a config its argument checks refuse: returns (rc, message).  The checks run before any device
    call, so the dummy pointers are never read."""
    L = cabi.load_library()
    cfg = cabi.EncoderConfig(arch, 2, hidden, heads, 512, 400, max_pos, 1, 1, 1e-5, cabi.AC_PREC_F16, 1024, 1)
    dummy = ctypes.c_void_p(0x1000)
    if rope:
        cfg.rope_full = dummy
    cfg.ffn_act = ffn_act
    w = cabi.EncoderWeights()
    arr = (ctypes.c_void_p * 2)(0x1000, 0x1000)
    if weights:
        w.wqkv = w.wi = w.attn_norm_w = ctypes.cast(arr, cabi._PP)
        w.final_norm_w = dummy
    if proj:
        w.emb_proj_w = w.emb_proj_b = dummy
    h = ctypes.c_void_p()
    rc = L.ac_encoder_create(ctypes.byref(cfg), ctypes.byref(w), ctypes.byref(h))
    return rc, L.ac_last_error().decode()


@pytest.mark.parametrize("kw,name", [
    (dict(rope=False), "AC_ARCH_EUROBERT needs rope_full"),
    (dict(max_pos=8193), "max_pos=8193"),
    (dict(max_pos=511), "max_pos=511"),
    (dict(weights=False), "AC_ARCH_EUROBERT needs wqkv, wi, attn_norm_w"),
    (dict(hidden=256, heads=8), "head_dim must be 64 for AC_ARCH_EUROBERT"),
    (dict(proj=True), "emb_proj_w"),
    (dict(ffn_act=0), "AC_ARCH_EUROBERT takes ffn_act=2 (AC_FFN_SWIGLU) only (ffn_act=0)"),
    (dict(ffn_act=1), "AC_ARCH_EUROBERT takes ffn_act=2 (AC_FFN_SWIGLU) only (ffn_act=1)"),
    (dict(arch=0), "is implemented for AC_ARCH_ROTARY / AC_ARCH_EUROBERT only (arch=0)"),
])
def test_encoder_create_refuses_bad_eurobert_settings(cabi, kw, name):
    rc, msg = _create_refusal(cabi, **kw)
    assert rc == -1, (rc, msg)                                       # AC_E_INVALID
    assert name in msg, msg
