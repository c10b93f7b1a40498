"""CPU tests of the MPNet encoders (all-mpnet-base-v2, multi-qa-mpnet-base-*, paraphrase-mpnet-base-v2): the fp32 oracle of
oracle/mpnet_oracle.py with its relative position bias pinned against HF MPNetModel, the product's bias table and weight
renaming against HF, the reference's golden embeddings of the MPNet checkpoint, and the settings Encoder.from_hf refuses
before any device call."""
import json

import numpy as np
import pytest
import torch

import golden_npz
from oracle import encoder_oracle as eo
from oracle import mpnet_oracle as mo


def mpnet_model(seed=5, bias_std=2.0, **over):
    """seeded MPNetModel with perturbed LayerNorms and an O(1) relative-attention-bias table (the init's std 0.02 would
    leave the bias nearly invisible)"""
    from transformers import MPNetConfig, MPNetModel
    kw = dict(vocab_size=400, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=512,
              max_position_embeddings=514, layer_norm_eps=1e-5)
    kw.update(over)
    torch.manual_seed(seed)
    m = MPNetModel(MPNetConfig(**kw)).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "LayerNorm" in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
        m.encoder.relative_attention_bias.weight.copy_(bias_std * torch.randn(m.encoder.relative_attention_bias.weight.shape,
                                                                              generator=g))
    return m


def mpnet_ids(B, S, pad, vocab=400, seed=7):
    """<s> first, </s> last, padding (id 1, mask 0) at the end of sequences 1.. when pad"""
    ids = eo.synthetic_ids(B, S, vocab=vocab, seed=seed, arch="roberta")
    mask = torch.ones_like(ids)
    if pad:
        for b in range(1, B):
            n = max(2, S - (S * b) // (B + 1))
            ids[b, n - 1] = 2
            ids[b, n:] = 1
            mask[b, n:] = 0
    return ids, mask


SHAPES = [(3, 16, False), (3, 77, True), (2, 300, True)]


@pytest.mark.parametrize("B,S,pad", SHAPES)
def test_mpnet_oracle_matches_hf(B, S, pad):
    """position bias after the scale and before the mask; S = 300 reaches distances past 8 (log buckets) and 128 (saturated)"""
    m = mpnet_model()
    ids, mask = mpnet_ids(B, S, pad)
    with torch.no_grad():
        hidden = m(input_ids=ids, attention_mask=mask).last_hidden_state
    ref = torch.nn.functional.normalize(hidden[:, 0, :], dim=1)
    sd = {k: v.detach().float() for k, v in m.state_dict().items()}
    out, out_hidden = mo.mpnet_forward_cls(sd, ids, mask, num_heads=4, ln_eps=1e-5, return_hidden=True)
    assert (out - ref).abs().max() < 1e-6
    assert (out_hidden - hidden).abs().max() < 1e-6 * max(1.0, hidden.abs().max().item())


@pytest.mark.parametrize("B,S,pad", SHAPES)
def test_mpnet_bias_moves_the_embeddings_far_beyond_the_gpu_tolerance(B, S, pad):
    """a kernel that dropped the bias would miss the GPU tests' 1e-3 row bound by orders of magnitude"""
    m = mpnet_model()
    ids, mask = mpnet_ids(B, S, pad)
    sd = {k: v.detach().float() for k, v in m.state_dict().items()}
    with_bias = mo.mpnet_forward_cls(sd, ids, mask, num_heads=4, ln_eps=1e-5)
    without = mo.mpnet_forward_cls(sd, ids, mask, num_heads=4, ln_eps=1e-5, bias_scale=0.0)
    assert (with_bias - without).norm(dim=1).min() > 2e-2


def test_mpnet_relative_bias_table_equals_hf_compute_position_bias():
    """entry (h, 511 + key - query) of the table is HF's bias of (h, query, key), bit for bit, on every pair of S = 512"""
    from adaptive_classifier_b200._cabi import AC_ENCODER_MAX_S, mpnet_relative_bias_table
    m = mpnet_model()
    S = AC_ENCODER_MAX_S
    with torch.no_grad():
        hf = m.encoder.compute_position_bias(torch.zeros(1, S, 256))[0]                    # [heads, S, S]
    table = mpnet_relative_bias_table(m.encoder.relative_attention_bias.weight, 4)
    assert table.shape == (4, 2 * S - 1) and table.dtype == torch.float32
    q = torch.arange(S)[:, None]
    k = torch.arange(S)[None, :]
    assert torch.equal(table[:, S - 1 + k - q], hf)
    assert torch.equal(mo.mpnet_position_bias(m.encoder.relative_attention_bias.weight.detach(), S), hf)


def test_mpnet_to_bert_state_dict_consumes_every_non_pooler_parameter():
    from adaptive_classifier_b200._cabi import mpnet_to_bert_state_dict

    class Seen(dict):
        def __init__(self, *a):
            super().__init__(*a)
            self.read = set()

        def __getitem__(self, k):
            self.read.add(k)
            return dict.__getitem__(self, k)

    m = mpnet_model(num_hidden_layers=3)
    sd = Seen(m.state_dict())
    out, dims = mpnet_to_bert_state_dict(sd, m.config)
    assert sd.read == {k for k in sd if not k.startswith("pooler.")}
    assert len(out) == 5 + 16 * 3 and torch.equal(out["embeddings.token_type_embeddings.weight"], torch.zeros(1, 256))
    assert dims["rel_bias"].shape == (4, 1023) and dims["pad_idx"] == 1 and dims["max_pos"] == 514 and dims["type_vocab"] == 1


def test_mpnet_oracle_reproduces_reference_embeddings():
    """golden_classifier_mpnet*.npz: the unmodified reference's _get_embeddings on a 2-head x 64 MPNet checkpoint"""
    g = golden_npz.load("golden_classifier_mpnet")
    cfgd = json.loads(str(g["bert_config"]))
    assert cfgd["model_type"] == "mpnet" and cfgd["hidden_size"] // cfgd["num_attention_heads"] == 64
    sd = {k[5:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(g["input_ids"])
    mask = torch.from_numpy(g["attention_mask"])
    assert (ids == 1).any()                                             # padded rows: positions follow the pad rule
    out = mo.mpnet_forward_cls(sd, ids, mask, num_heads=cfgd["num_attention_heads"], ln_eps=cfgd["layer_norm_eps"])
    ref = np.concatenate([g["emb_train"], g["emb_test"]])
    assert out.shape == ref.shape
    assert np.abs(out.numpy() - ref).max() < 1e-5


@pytest.mark.parametrize("over,name", [(dict(hidden_act="relu"), "hidden_act='relu'"),
                                       (dict(hidden_size=256, num_attention_heads=8), "head_dim=32"),
                                       (dict(relative_attention_num_buckets=64), "relative_attention_num_buckets=64")])
def test_from_hf_refuses_unimplemented_mpnet_settings(over, name):
    from adaptive_classifier_b200._cabi import AdaptiveB200Error, Encoder
    m = mpnet_model(num_hidden_layers=1, **over)
    with pytest.raises(AdaptiveB200Error, match=name):
        Encoder.from_hf(m, device="cpu")
