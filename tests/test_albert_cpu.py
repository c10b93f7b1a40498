"""CPU tests of the ALBERT (albert-base / large v1 / v2) and ELECTRA (discriminators) encoders: the fp32 oracle of
oracle/albert_oracle.py pinned against HF AlbertModel / ElectraModel, the product's weight renaming and ALBERT's sharing map
against HF, the reference's golden embeddings of both checkpoints, the settings Encoder.from_hf refuses before any device
call, and the power of the GPU activation test to tell tanh GELU from erf GELU."""
import json
import math

import numpy as np
import pytest
import torch

import golden_npz
from oracle import albert_oracle as ao


def albert_model(seed=5, scale=3.0, **over):
    """seeded AlbertModel (embedding_size 128 < hidden 256, 4 heads) with perturbed LayerNorms and biases and the weight
    matrices scaled by `scale`"""
    from transformers import AlbertConfig, AlbertModel
    kw = dict(vocab_size=400, embedding_size=128, hidden_size=256, num_hidden_layers=3, num_hidden_groups=1,
              inner_group_num=1, num_attention_heads=4, intermediate_size=512, max_position_embeddings=512,
              type_vocab_size=2, hidden_act="gelu_new", pad_token_id=0)
    kw.update(over)
    torch.manual_seed(seed)
    return _perturb(AlbertModel(AlbertConfig(**kw), add_pooling_layer=False).eval(), seed, scale)


def electra_model(seed=6, scale=3.0, **over):
    from transformers import ElectraConfig, ElectraModel
    kw = dict(vocab_size=400, embedding_size=128, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
              intermediate_size=512, max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu", pad_token_id=0)
    kw.update(over)
    torch.manual_seed(seed)
    return _perturb(ElectraModel(ElectraConfig(**kw)).eval(), seed, scale)


def _perturb(m, seed, scale):
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "LayerNorm" in n or "layer_norm" in n or n.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 2:
                p.mul_(scale)
    return m


def albert_ids(B, S, pad, vocab=400, seed=7):
    """[CLS] = 2 first, [SEP] = 3 last, ids in [5, vocab); padding (id 0, mask 0) at the end of sequences 1.. when pad"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(5, vocab, (B, S), generator=g)
    ids[:, 0] = 2
    ids[:, -1] = 3
    mask = torch.ones_like(ids)
    if pad:
        for b in range(1, B):
            n = max(2, S - (S * b) // (B + 1))
            ids[b, n - 1] = 3
            ids[b, n:] = 0
            mask[b, n:] = 0
    return ids, mask


def _sd(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


MODELS = {
    "albert": lambda: albert_model(),
    "albert_2groups_2inner": lambda: albert_model(num_hidden_layers=4, num_hidden_groups=2, inner_group_num=2),
    "albert_e_eq_h": lambda: albert_model(embedding_size=256),
    "albert_v1_gelu": lambda: albert_model(hidden_act="gelu"),
    "electra": lambda: electra_model(),
    "electra_e_eq_h": lambda: electra_model(embedding_size=256),
}


@pytest.mark.parametrize("B,S", [(3, 16), (3, 77), (3, 129), (2, 300)])
@pytest.mark.parametrize("which", list(MODELS))
def test_oracle_matches_hf(which, B, S):
    m = MODELS[which]()
    ids, mask = albert_ids(B, S, True)
    with torch.no_grad():
        hidden = m(input_ids=ids, attention_mask=mask).last_hidden_state
    ref = torch.nn.functional.normalize(hidden[:, 0, :], dim=1)
    out, out_hidden = ao.factorized_forward_cls(_sd(m), ids, mask, m.config, return_hidden=True)
    assert (out - ref).abs().max() < 1e-6
    keep = mask.bool()
    assert (out_hidden[keep] - hidden[keep]).abs().max() < 1e-6 * max(1.0, hidden.abs().max().item())


class Seen(dict):
    def __init__(self, *a):
        super().__init__(*a)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return dict.__getitem__(self, k)


@pytest.mark.parametrize("which", list(MODELS))
def test_state_dict_mapping_consumes_every_parameter(which):
    from adaptive_classifier_b200 import _cabi
    m = MODELS[which]()
    c = m.config
    sd = Seen({k: v for k, v in m.state_dict().items() if not k.startswith("pooler.")})
    fn = _cabi.albert_to_bert_state_dict if c.model_type == "albert" else _cabi.electra_to_bert_state_dict
    out, dims = fn(sd, c)
    if c.model_type == "albert":
        assert sd.read == set(sd)
    else:   # ELECTRA's names are BERT's: the mapping passes them through
        assert set(out) == {k for k in sd if not k.endswith(("position_ids", "token_type_ids"))}
    L = dims["layers"]
    assert L == c.num_hidden_layers * getattr(c, "inner_group_num", 1)
    assert len(out) == 5 + 16 * L + (2 if "embeddings_project.weight" in out else 0)
    assert ("embeddings_project.weight" in out) == (c.model_type == "albert" or c.embedding_size != c.hidden_size)
    assert dims["embedding_size"] == (0 if c.model_type == "electra" and c.embedding_size == c.hidden_size
                                      else c.embedding_size)
    assert dims["ffn_act"] == (_cabi.AC_FFN_GELU_TANH if c.hidden_act == "gelu_new" else _cabi.AC_FFN_GELU_ERF)


@pytest.mark.parametrize("L,G,inner", [(12, 1, 1), (24, 1, 1), (4, 2, 2), (6, 3, 1), (5, 3, 1), (7, 2, 3), (3, 3, 2)])
def test_albert_sharing_map_is_hf_group_walk(L, G, inner):
    """the effective-layer -> source-tensor assignment of albert_to_bert_state_dict is the order in which HF AlbertModel runs
    its layer modules (forward hooks), and layers that share a module map to the very same tensor objects"""
    from adaptive_classifier_b200._cabi import albert_to_bert_state_dict
    m = albert_model(num_hidden_layers=L, num_hidden_groups=G, inner_group_num=inner, intermediate_size=128)
    order = []
    for g, grp in enumerate(m.encoder.albert_layer_groups):
        for j, layer in enumerate(grp.albert_layers):
            layer.register_forward_hook(lambda mod, a, o, gj=(g, j): order.append(gj))
    with torch.no_grad():
        m(input_ids=torch.tensor([[2, 7, 3]]))
    sd = m.state_dict()
    out, dims = albert_to_bert_state_dict(sd, m.config)
    assert dims["layers"] == len(order) == L * inner
    for l, (g, j) in enumerate(order):
        src = f"encoder.albert_layer_groups.{g}.albert_layers.{j}."
        assert out[f"encoder.layer.{l}.attention.self.query.weight"] is sd[src + "attention.query.weight"]
        assert out[f"encoder.layer.{l}.output.LayerNorm.bias"] is sd[src + "full_layer_layer_norm.bias"]
    ptrs = {out[f"encoder.layer.{l}.intermediate.dense.weight"].data_ptr() for l in range(L * inner)}
    assert len(ptrs) == len(set(order))


@pytest.mark.parametrize("name", ["golden_classifier_albert", "golden_classifier_electra"])
def test_oracle_reproduces_reference_embeddings(name):
    """golden_classifier_{albert,electra}*.npz: the unmodified reference's _get_embeddings on tiny seeded checkpoints"""
    from transformers import AlbertConfig, ElectraConfig
    g = golden_npz.load(name)
    cfgd = json.loads(str(g["bert_config"]))
    C = {"albert": AlbertConfig, "electra": ElectraConfig}[cfgd["model_type"]]
    c = C(**{k: v for k, v in cfgd.items() if k not in ("model_type", "transformers_version", "architectures")})
    assert c.embedding_size == 128 and c.hidden_size == 256
    sd = {k[5:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(g["input_ids"])
    mask = torch.from_numpy(g["attention_mask"])
    assert (mask == 0).any()
    out = ao.factorized_forward_cls(sd, ids, mask, c)
    ref = np.concatenate([g["emb_train"], g["emb_test"]])
    assert out.shape == ref.shape
    assert np.abs(out.numpy() - ref).max() < 1e-5


class _Stub:
    """an HF-model stand-in with only a config: the refusals must come before any weight is read or copied"""
    def __init__(self, config):
        self.config = config

    def state_dict(self):
        return {}


def _albert_cfg(**over):
    from transformers import AlbertConfig
    kw = dict(vocab_size=30000, embedding_size=128, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
              intermediate_size=3072, hidden_act="gelu_new")
    kw.update(over)
    return AlbertConfig(**kw)


def _electra_cfg(**over):
    from transformers import ElectraConfig
    kw = dict(embedding_size=128, hidden_size=256, num_attention_heads=4, intermediate_size=1024)
    kw.update(over)
    return ElectraConfig(**kw)


@pytest.mark.parametrize("cfg,name", [
    (lambda: _albert_cfg(hidden_size=4096, num_attention_heads=64, intermediate_size=16384), "hidden_size=4096"),
    (lambda: _albert_cfg(hidden_size=2048, num_attention_heads=16, intermediate_size=8192), "hidden_size=2048"),
    (lambda: _albert_cfg(num_attention_heads=6), "head_dim=128"),
    (lambda: _albert_cfg(embedding_size=96), "embedding_size=96"),
    (lambda: _albert_cfg(embedding_size=1024), "embedding_size=1024"),
    (lambda: _albert_cfg(hidden_act="relu"), "hidden_act='relu'"),
    (lambda: _albert_cfg(position_embedding_type="relative_key"), "position_embedding_type='relative_key'"),
    (lambda: _albert_cfg(num_hidden_groups=13), "num_hidden_groups=13"),
    (lambda: _electra_cfg(hidden_size=320, num_attention_heads=5), "hidden_size=320"),
    (lambda: _electra_cfg(num_attention_heads=2), "head_dim=128"),
    (lambda: _electra_cfg(embedding_size=64), "embedding_size=64"),
    (lambda: _electra_cfg(hidden_act="silu"), "hidden_act='silu'"),
    (lambda: _electra_cfg(position_embedding_type="relative_key_query"), "position_embedding_type"),
])
def test_from_hf_refuses_unimplemented_settings(cfg, name):
    from adaptive_classifier_b200._cabi import AdaptiveB200Error, Encoder
    with pytest.raises(AdaptiveB200Error, match=name.replace("[", r"\[")):
        Encoder.from_hf(_Stub(cfg()), device="cpu")


def test_from_hf_refuses_other_bert_activations():
    from transformers import BertConfig
    from adaptive_classifier_b200._cabi import AdaptiveB200Error, Encoder
    with pytest.raises(AdaptiveB200Error, match="hidden_act='relu'"):
        Encoder.from_hf(_Stub(BertConfig(hidden_act="relu")), device="cpu")


# ---- the activation test of tests/test_gpu_albert.py -----------------------------------------------------------------
EVAL_ALLOWANCE = 2.0 ** -15   # relative fp32 evaluation error of encoder.cu gelu_tanh (stated there)


def fp16_grid(lo=-10.0, hi=10.0) -> torch.Tensor:
    """every fp16 value in [lo, hi], ascending, as fp16"""
    bits = torch.arange(0, 1 << 16, dtype=torch.int32).to(torch.int16).view(torch.float16)
    v = bits[torch.isfinite(bits) & (bits.float() >= lo) & (bits.float() <= hi)]
    return torch.unique(v.float()).to(torch.float16)


def gelu_tanh64(x: torch.Tensor) -> torch.Tensor:
    x = x.double()
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def tanh_gelu_bound(ref: torch.Tensor) -> torch.Tensor:
    """|fp16(out) - ref| <= 2^-11 |ref| (fp16 rounding) + EVAL_ALLOWANCE |ref| (fp32 evaluation) + 2^-25 (half an fp16
    subnormal ulp: results below 2^-14 round absolutely)"""
    a = ref.abs()
    return 2.0 ** -11 * a * (1 + EVAL_ALLOWANCE) + EVAL_ALLOWANCE * a + 2.0 ** -25


def test_erf_gelu_violates_the_tanh_activation_bound():
    """an epilogue that kept exact-erf GELU would fail the GPU activation test, on many values and by far"""
    x = fp16_grid()
    ref = gelu_tanh64(x)
    erf = torch.nn.functional.gelu(x.double()).to(torch.float16).double()
    ratio = (erf - ref).abs() / tanh_gelu_bound(ref)
    assert (ratio > 1).sum() > 1000 and ratio.max() > 50, (int((ratio > 1).sum()), ratio.max().item())
    # and the correctly rounded tanh GELU itself passes with room
    ok = gelu_tanh64(x).to(torch.float16).double()
    assert ((ok - ref).abs() / tanh_gelu_bound(ref)).max() <= 1.0


def _create_refusal(cabi, arch=0, hidden=256, heads=4, embedding_size=0, ffn_act=0, proj=True, proj_b=True):
    """ac_encoder_create on a config its argument checks refuse: returns (rc, message).  The checks run before any device
    call, so the dummy pointers are never read."""
    import ctypes
    L = cabi.load_library()
    cfg = cabi.EncoderConfig(arch, 2, hidden, heads, 512, 400, 512, 2, 0, 1e-12, cabi.AC_PREC_F16, 1024, 1)
    dummy = ctypes.c_void_p(0x1000)
    cfg.rel_bias = cfg.pos_key = cfg.pos_query = cfg.rel_index = dummy   # the MPNet / DeBERTa tables are present
    cfg.pos_span = 256
    cfg.embedding_size, cfg.ffn_act = embedding_size, ffn_act
    w = cabi.EncoderWeights()
    if proj:
        w.emb_proj_w = dummy
    if proj_b:
        w.emb_proj_b = dummy
    h = ctypes.c_void_p()
    rc = L.ac_encoder_create(ctypes.byref(cfg), ctypes.byref(w), ctypes.byref(h))
    return rc, L.ac_last_error().decode()


@pytest.mark.parametrize("kw,name", [
    (dict(arch=3), "emb_proj_w"),                                   # MPNet
    (dict(arch=4), "emb_proj_w"),                                   # DeBERTa-v2's embed_proj runs before the LayerNorm
    (dict(embedding_size=96), "embedding_size=96"),
    (dict(embedding_size=384), "embedding_size=384"),
    (dict(embedding_size=128, proj=False, proj_b=False), "embedding_size=128"),
    (dict(embedding_size=128, proj_b=False), "emb_proj_b"),
    (dict(ffn_act=2), "ffn_act=2"),
])
def test_encoder_create_refuses_bad_projection_and_activation_settings(cabi, kw, name):
    rc, msg = _create_refusal(cabi, **kw)
    assert rc == -1, (rc, msg)                                       # AC_E_INVALID
    assert name in msg, msg
