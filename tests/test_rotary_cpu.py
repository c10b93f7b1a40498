"""CPU tests of the rotary encoders (NomicBERT, jina-embeddings-v3: AC_ARCH_ROTARY):
  * oracle/rotary_oracle.py against HF NomicBertModel / JinaEmbeddingsV3Model (eager attention), padded both ways, with
    and without token_type_ids, S from 16 to 2048
  * the RoPE table the encoder reads against HF's rotary_emb, bit for bit
  * the mappings consume every parameter but the pooler, and supply zero biases where the checkpoint has none
  * the golden classifier runs of oracle/make_golden_encoders.py nomic jina3 against the oracle
  * each wrong rule (no RoPE, GPT-J pairs, padding-aware positions, RoPE on v, gate / up swapped) moves the embeddings far
    past the GPU bound
  * from_hf and ac_encoder_create refusals, which run before any device call"""
import json
import re

import numpy as np
import pytest
import torch

import golden_npz
from oracle import rotary_oracle as ro

GPU_UNIT_BOUND = 3e-4          # max |GPU - oracle| on unit CLS rows (tests/test_gpu_rotary.py, as test_gpu_albert.py)


def tiny_model(family, seed=7, layers=2, hidden=128, heads=2, inter=256, **over):
    """HF NomicBertModel / JinaEmbeddingsV3Model in eager attention; LayerNorms and biases perturbed, projections scaled up
    so that the attention is far from uniform and positions matter"""
    from transformers import JinaEmbeddingsV3Config, JinaEmbeddingsV3Model, NomicBertConfig, NomicBertModel
    torch.manual_seed(seed)
    common = dict(vocab_size=300, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                  intermediate_size=inter, type_vocab_size=2, attn_implementation="eager")
    if family == "nomic":
        m = NomicBertModel(NomicBertConfig(**{**common, "max_position_embeddings": 2048, **over}))
    else:
        m = JinaEmbeddingsV3Model(JinaEmbeddingsV3Config(**{**common, "max_position_embeddings": 8194, "layer_norm_eps": 1e-5,
                                                            "hidden_dropout_prob": 0.0, "attention_probs_dropout_prob": 0.0,
                                                            **over}), add_pooling_layer=False)
    m.eval()
    assert m.config._attn_implementation == "eager"
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "layernorm.weight" in n.lower():
                p.copy_(1.0 + 0.3 * torch.randn(p.shape, generator=g))
            elif "layernorm.bias" in n.lower() or n.endswith(".bias"):
                p.copy_(0.2 * torch.randn(p.shape, generator=g))
            elif "q_proj" in n or "k_proj" in n:
                p.mul_(8.0)
            elif p.dim() == 2 and "embeddings" not in n:
                p.mul_(3.0)
    return m


def padded_batch(S, seed, vocab=300, types=False):
    """three sequences: full length, right-padded, left-padded (pad id 1); CLS-like id 0 first and id 2 last"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(5, vocab, (3, S), generator=g)
    mask = torch.ones(3, S, dtype=torch.int64)
    n = max(2, (2 * S) // 3 + 1)
    mask[1, n:] = 0
    mask[2, :S - n] = 0
    for b in range(3):
        idx = mask[b].nonzero().flatten()
        ids[b, idx[0]], ids[b, idx[-1]] = 0, 2
    ids[mask == 0] = 1
    tt = (torch.arange(S)[None].expand(3, S) >= S // 2).long() if types else None
    return ids, mask, tt


def sd_of(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


def hf_forward(m, ids, mask, tt):
    with torch.no_grad():
        kw = {} if tt is None else {"token_type_ids": tt}
        return m(input_ids=ids, attention_mask=mask, **kw).last_hidden_state


@pytest.mark.parametrize("types", [False, True])
@pytest.mark.parametrize("S", [16, 77, 129, 300, 600, 1100, 2048])
@pytest.mark.parametrize("family", ["nomic", "jina"])
def test_oracle_matches_hf(family, S, types):
    m = tiny_model(family)
    ids, mask, tt = padded_batch(S, S, types=types)
    hf = hf_forward(m, ids, mask, tt)
    unit, hid = ro.rotary_forward_for(m.config, sd_of(m), ids, mask, tt, return_hidden=True)
    keep = mask.bool()
    assert (hid[keep] - hf[keep]).abs().max() < 1e-6 * max(1.0, hf[keep].abs().max().item())
    # row 0 is what the classifier pools, a pad row in the left-padded sequence
    assert (unit - torch.nn.functional.normalize(hf[:, 0], dim=1)).abs().max() < 1e-6


@pytest.mark.parametrize("theta", [1000.0, 20000.0])
def test_rope_table_is_bit_equal_to_hf_rotary_emb(cabi, theta):
    m = tiny_model("nomic" if theta == 1000.0 else "jina", layers=1)
    assert m.config.rope_parameters["rope_theta"] == theta
    x = torch.zeros(1, 8192, m.config.hidden_size)
    cos, sin = m.rotary_emb(x, torch.arange(8192)[None])
    table = cabi.modernbert_rope_table(theta, 8192)
    assert torch.equal(cos[0, :, :32], cos[0, :, 32:]) and torch.equal(sin[0, :, :32], sin[0, :, 32:])
    assert torch.equal(table[:, :32], cos[0, :, :32]) and torch.equal(table[:, 32:], sin[0, :, :32])


class _Tracked(dict):
    """a state_dict that records which names were read"""
    def __init__(self, *a):
        super().__init__(*a)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)

    def get(self, k, default=None):
        if k in self:
            self.read.add(k)
        return super().get(k, default)


def _bert_names(layers):
    names = [f"embeddings.{n}" for n in ("word_embeddings.weight", "token_type_embeddings.weight", "LayerNorm.weight",
                                         "LayerNorm.bias")]
    for l in range(layers):
        for n in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense",
                  "attention.output.LayerNorm", "intermediate.dense", "output.dense", "output.LayerNorm"):
            names += [f"encoder.layer.{l}.{n}.weight", f"encoder.layer.{l}.{n}.bias"]
    return set(names)


@pytest.mark.parametrize("family", ["nomic", "jina"])
def test_mappings_consume_every_parameter_but_the_pooler(cabi, family):
    from transformers import JinaEmbeddingsV3Model
    m = tiny_model(family, layers=3)
    if family == "jina":                                  # with the pooler the default construction has
        m = JinaEmbeddingsV3Model(m.config)
    sd = _Tracked(m.state_dict())
    to_bert = cabi.nomic_bert_to_bert_state_dict if family == "nomic" else cabi.jina_v3_to_bert_state_dict
    out, dims = to_bert(sd, m.config)
    unread = set(sd) - sd.read
    assert unread == {k for k in sd if k.startswith("pooler.")}, unread
    assert set(out) == _bert_names(3)
    H, I = 128, 256
    ffn1 = out["encoder.layer.1.intermediate.dense.weight"]
    if family == "nomic":
        assert torch.equal(ffn1, torch.cat([sd["layers.1.mlp.gate_proj.weight"], sd["layers.1.mlp.up_proj.weight"]]))
        for n, rows in (("attention.self.query", H), ("attention.output.dense", H), ("intermediate.dense", 2 * I),
                        ("output.dense", H)):
            b = out[f"encoder.layer.1.{n}.bias"]
            assert b.shape == (rows,) and not b.any()
        assert dims["ffn_act"] == cabi.AC_FFN_SWIGLU and dims["rope_theta"] == 1000.0 and dims["max_pos"] == 2048
    else:
        assert ffn1 is sd["layers.1.mlp.fc1.weight"]
        assert out["encoder.layer.1.attention.self.key.bias"] is sd["layers.1.self_attn.k_proj.bias"]
        assert dims["ffn_act"] == cabi.AC_FFN_GELU_ERF and dims["rope_theta"] == 20000.0 and dims["max_pos"] == 8192
    assert dims["type_vocab"] == 2 and dims["layers"] == 3


@pytest.mark.parametrize("mpe,expect", [(128, 512), (2048, 2048), (8194, 8192), (16384, 8192)])
def test_sequence_limit_follows_max_position_embeddings(cabi, mpe, expect):
    m = tiny_model("jina", layers=1)
    m.config.max_position_embeddings = mpe
    _, dims = cabi.jina_v3_to_bert_state_dict(dict(m.state_dict()), m.config)
    assert dims["max_pos"] == expect


# ------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize("name", ["golden_classifier_nomic", "golden_classifier_jina3"])
def test_golden_embeddings_match_the_oracle(name):
    golden = golden_npz.load(name)
    cfg = json.loads(str(golden["bert_config"]))
    sd = {k[5:]: torch.from_numpy(golden[k]).float() for k in golden.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(golden["input_ids"]).long()
    mask = torch.from_numpy(golden["attention_mask"]).long()
    tt = torch.from_numpy(golden["token_type_ids"]).long() if "token_type_ids" in golden else None
    unit = ro.rotary_forward_for(cfg, sd, ids, mask, tt)
    ref = np.concatenate([golden["emb_train"], golden["emb_test"]])
    assert unit.shape[0] == len(golden["texts"]) + len(golden["test_texts"])
    assert np.abs(unit.numpy() - ref).max() < 1e-5
    if cfg["model_type"] == "jina_embeddings_v3":
        assert ids.shape[1] == 1024 and int((mask.sum(1) > 512).sum()) >= 3


# ------------------------------------------------------------------------------------------------ wrong rules
@pytest.mark.parametrize("family,wrong", [(f, w) for f in ("nomic", "jina") for w in ro.WRONG_RULES
                                          if not (f == "jina" and w == "swap_gate_up")])
def test_each_wrong_rule_moves_the_embeddings_past_the_gpu_bound(family, wrong):
    m = tiny_model(family, seed=3)
    ids, mask, tt = padded_batch(300, 5)
    sd = sd_of(m)
    ref = ro.rotary_forward_for(m.config, sd, ids, mask, tt)
    bad = ro.rotary_forward_for(m.config, sd, ids, mask, tt, wrong=wrong)
    moved = (bad - ref).abs().max().item()
    assert moved >= 20 * GPU_UNIT_BOUND, (family, wrong, moved)


# ------------------------------------------------------------------------------------------------ SwiGLU activation bound
EVAL_ALLOWANCE = 2.0 ** -15    # relative fp32 evaluation error of encoder.cu silu (derived there: < 3e-6 for |y| <= 20)


def silu64(x: torch.Tensor) -> torch.Tensor:
    x = x.double()
    return x / (1.0 + torch.exp(-x))


def silu_bound(ref: torch.Tensor) -> torch.Tensor:
    """|fp16(out) - ref| <= 2^-11 |ref| (fp16 rounding) + EVAL_ALLOWANCE |ref| (fp32 evaluation) + 2^-25 (half an fp16
    subnormal ulp)"""
    a = ref.abs()
    return 2.0 ** -11 * a * (1 + EVAL_ALLOWANCE) + EVAL_ALLOWANCE * a + 2.0 ** -25


def test_other_activations_violate_the_silu_bound():
    """the bound tells silu from the GELUs an epilogue might compute instead; correctly rounded silu passes it"""
    from test_albert_cpu import fp16_grid
    x = fp16_grid(-20.0, 20.0)
    ref = silu64(x)
    ok = silu64(x).to(torch.float16).double()
    assert ((ok - ref).abs() / silu_bound(ref)).max() <= 1.0
    for f in (torch.nn.functional.gelu, lambda t: torch.nn.functional.gelu(t, approximate="tanh")):
        wrong = f(x.double()).to(torch.float16).double()
        ratio = (wrong - ref).abs() / silu_bound(ref)
        assert (ratio > 1).sum() > 1000 and ratio.max() > 50


# ------------------------------------------------------------------------------------------------ refusals
def _with(m, **attrs):
    for k, v in attrs.items():
        setattr(m.config, k, v)
    return m


@pytest.mark.parametrize("family,attrs,name", [
    ("nomic", dict(rope_parameters={"rope_type": "dynamic", "rope_theta": 1000.0, "factor": 2.0}), "rope_type='dynamic'"),
    ("jina", dict(rope_parameters={"rope_type": "yarn", "rope_theta": 20000.0, "factor": 4.0}), "rope_type='yarn'"),
    ("nomic", dict(rope_parameters={"rope_type": "linear", "rope_theta": 1000.0, "factor": 2.0}), "rope_type='linear'"),
    ("nomic", dict(head_dim=32), "head_dim=32"),
    ("jina", dict(num_attention_heads=4), "head_dim=32"),
    ("nomic", dict(hidden_size=192, num_attention_heads=3, head_dim=64), "hidden_size=192"),
    ("jina", dict(hidden_size=1152, num_attention_heads=18), "hidden_size=1152"),
    ("nomic", dict(hidden_act="gelu"), "hidden_act='gelu'"),
    ("jina", dict(hidden_act="silu"), "hidden_act='silu'"),
    ("jina", dict(hidden_act="relu"), "hidden_act='relu'"),
])
def test_from_hf_refuses_unimplemented_settings_by_name(cabi, family, attrs, name):
    m = _with(tiny_model(family, layers=1), **attrs)
    with pytest.raises(cabi.AdaptiveB200Error, match=re.escape(name)):
        cabi.Encoder.from_hf(m)


@pytest.mark.parametrize("family", ["nomic", "jina"])
def test_from_hf_refuses_remote_code_modules_by_name(cabi, family):
    """a module that carries the model_type but is not the native class (the Hub's trust_remote_code classes name their
    parameters differently)"""
    config = tiny_model(family, layers=1).config

    class RemoteCodeModel(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.config = config
            self.emb = torch.nn.Embedding(300, 128)

    with pytest.raises(cabi.AdaptiveB200Error, match="trust_remote_code"):
        cabi.Encoder.from_hf(RemoteCodeModel())


def test_silu_stays_refused_for_bert_family_configs(cabi):
    from transformers import BertConfig, BertModel
    m = BertModel(BertConfig(vocab_size=100, hidden_size=128, num_hidden_layers=1, num_attention_heads=2,
                             intermediate_size=128, hidden_act="silu"), add_pooling_layer=False)
    assert "silu" not in cabi.FFN_ACTS
    with pytest.raises(cabi.AdaptiveB200Error, match="hidden_act='silu'"):
        cabi.Encoder.from_hf(m)


def _create_refusal(cabi, arch=5, hidden=256, heads=4, max_pos=2048, rope=True, proj=False, ffn_act=2):
    """ac_encoder_create on a config its argument checks refuse: returns (rc, message).  The checks run before any device
    call, so the dummy pointers are never read."""
    import ctypes
    L = cabi.load_library()
    cfg = cabi.EncoderConfig(arch, 2, hidden, heads, 512, 400, max_pos, 2, 0, 1e-12, cabi.AC_PREC_F16, 1024, 1)
    dummy = ctypes.c_void_p(0x1000)
    cfg.rel_bias = cfg.pos_key = cfg.pos_query = cfg.rel_index = dummy   # the MPNet / DeBERTa tables are present
    cfg.pos_span = 256
    if rope:
        cfg.rope_full = dummy
    cfg.ffn_act = ffn_act
    w = cabi.EncoderWeights()
    if proj:
        w.emb_proj_w = w.emb_proj_b = dummy
    h = ctypes.c_void_p()
    rc = L.ac_encoder_create(ctypes.byref(cfg), ctypes.byref(w), ctypes.byref(h))
    return rc, L.ac_last_error().decode()


@pytest.mark.parametrize("kw,name", [
    (dict(rope=False), "rope_full"),
    (dict(max_pos=8193), "max_pos=8193"),
    (dict(max_pos=511), "max_pos=511"),
    (dict(hidden=256, heads=8), "head_dim must be 64 for AC_ARCH_ROTARY"),
    (dict(proj=True), "emb_proj_w"),
    (dict(arch=0), "ffn_act=2"),
    (dict(arch=1), "ffn_act=2"),
    (dict(arch=3), "ffn_act=2"),
    (dict(arch=4), "ffn_act=2"),
    (dict(ffn_act=3), "unknown ffn_act=3"),
])
def test_encoder_create_refuses_bad_rotary_settings(cabi, kw, name):
    rc, msg = _create_refusal(cabi, **kw)
    assert rc == -1, (rc, msg)                                       # AC_E_INVALID
    assert name in msg, msg

