"""CPU tests of the head_dim-32 BERT encoders (all-MiniLM-L6/L12-v2, BGE-small, E5-small, GTE-small: 384 hidden = 12 heads
of 32): the fp32 oracle of oracle/encoder_oracle.py pinned against HF BertModel at that shape, the reference's golden
embeddings of the head_dim-32 checkpoint, and the head sizes Encoder.from_hf refuses before any device call."""
import json

import numpy as np
import pytest
import torch

import golden_npz
from oracle import encoder_oracle as eo

MINILM = dict(hidden_size=384, num_attention_heads=12, intermediate_size=1536, num_hidden_layers=6)


@pytest.mark.parametrize("B,S", [(3, 24), (4, 77)])
def test_encoder_oracle_matches_hf_at_the_minilm_shape(B, S):
    sd, cfg, hf = eo.make_bert_state_dict(1234, **MINILM)
    ids = eo.synthetic_ids(B, S)
    mask = torch.ones_like(ids)
    for b in range(1, B):
        n = S - 5 * b
        mask[b, n:] = 0
        ids[b, n:] = 0
    with torch.no_grad():
        ref = torch.nn.functional.normalize(hf(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)
    out = eo.encoder_forward_cls(sd, ids, mask, num_heads=12)
    assert (out - ref).abs().max() < 1e-6


def test_encoder_oracle_reproduces_reference_embeddings_minilm():
    """golden_classifier_minilm*.npz: the unmodified reference's _get_embeddings on a 4-head x 32 BERT checkpoint"""
    g = golden_npz.load("golden_classifier_minilm")
    cfgd = json.loads(str(g["bert_config"]))
    assert cfgd["hidden_size"] // cfgd["num_attention_heads"] == 32
    sd = {k[5:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(g["input_ids"])
    mask = torch.from_numpy(g["attention_mask"])
    out = eo.encoder_forward_cls(sd, ids, mask, num_heads=cfgd["num_attention_heads"], ln_eps=cfgd["layer_norm_eps"])
    ref = np.concatenate([g["emb_train"], g["emb_test"]])
    assert out.shape == ref.shape
    assert np.abs(out.numpy() - ref).max() < 1e-5


def _tiny(arch, hidden, heads):
    if arch == "distilbert":
        from transformers import DistilBertConfig, DistilBertModel
        return DistilBertModel(DistilBertConfig(vocab_size=100, dim=hidden, n_heads=heads, n_layers=1, hidden_dim=256,
                                                max_position_embeddings=32))
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel
    Cfg, Model = (BertConfig, BertModel) if arch == "bert" else (RobertaConfig, RobertaModel)
    return Model(Cfg(vocab_size=100, hidden_size=hidden, num_attention_heads=heads, num_hidden_layers=1,
                     intermediate_size=256, max_position_embeddings=34))


@pytest.mark.parametrize("arch", ["bert", "roberta", "distilbert"])
@pytest.mark.parametrize("hidden,heads,head_dim", [(128, 8, 16), (384, 8, 48), (256, 2, 128)])
def test_from_hf_refuses_other_head_dims(arch, hidden, heads, head_dim):
    from adaptive_classifier_b200._cabi import AdaptiveB200Error, Encoder
    m = _tiny(arch, hidden, heads)
    with pytest.raises(AdaptiveB200Error, match=f"head_dim={head_dim}"):
        Encoder.from_hf(m, device="cpu")


def test_check_head_dim_accepts_32_and_64_and_refuses_a_remainder():
    from adaptive_classifier_b200._cabi import AdaptiveB200Error, check_head_dim
    check_head_dim(384, 12)
    check_head_dim(768, 12)
    check_head_dim(1024, 16)
    with pytest.raises(AdaptiveB200Error, match="not divisible"):
        check_head_dim(384, 7)
