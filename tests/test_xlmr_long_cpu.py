"""CPU tests of the long XLM-RoBERTa path's references: oracle/encoder_oracle.py (arch "roberta") against HF XLMRobertaModel
(eager attention) with an 8194-row position table at S past 512, where RoBERTa positions run past 514; and the golden
classifier run of oracle/make_golden_encoders.py xlmr_long (the reference with max_length 1024) against that oracle."""
import json

import numpy as np
import pytest
import torch

import golden_npz
from oracle import encoder_oracle as eo


def _tiny_xlmr(seed=7):
    from transformers import XLMRobertaConfig, XLMRobertaModel
    torch.manual_seed(seed)
    cfg = XLMRobertaConfig(vocab_size=300, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                           max_position_embeddings=8194, type_vocab_size=1, layer_norm_eps=1e-5, pad_token_id=1, attn_implementation="eager")
    m = XLMRobertaModel(cfg, add_pooling_layer=False).eval()
    assert m.config._attn_implementation == "eager"
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "LayerNorm" in n:
                p.add_(0.2 * torch.randn(p.shape, generator=g))
            elif "position_embeddings" in n:
                p.mul_(5.0)                  # positions past 514 must move the result
    return m


def _padded_ids(S, seed):
    """three sequences: full length, right-padded to 128 n + 1, left-padded to 128 n - 1 (pad id 1, <s> 0, </s> 2)"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(5, 300, (3, S), generator=g)
    mask = torch.ones(3, S, dtype=torch.int64)
    n1 = 128 * (S // 128 - 1) + 1
    n2 = 128 * (S // 128 - 1) - 1
    mask[1, n1:] = 0
    mask[2, :S - n2] = 0
    for b in range(3):
        idx = mask[b].nonzero().flatten()
        ids[b, idx[0]], ids[b, idx[-1]] = 0, 2
    ids[mask == 0] = 1
    return ids, mask


@pytest.mark.parametrize("S", [600, 1100, 2048])
def test_oracle_matches_hf_xlmroberta_past_514_positions(S):
    m = _tiny_xlmr()
    ids, mask = _padded_ids(S, S)
    with torch.no_grad():
        hf = m(input_ids=ids, attention_mask=mask).last_hidden_state
    sd = {k: v.detach().float() for k, v in m.state_dict().items()}
    unit, hid = eo.encoder_forward_cls(sd, ids, mask, arch="roberta", num_heads=2, ln_eps=1e-5, pad_idx=1, return_hidden=True)
    keep = mask.bool()
    assert (hid[keep] - hf[keep]).abs().max() < 1e-5
    # the left-padded sequence's CLS row is the first valid one in HF's layout; the classifier pools row 0 either way
    hf_unit = torch.nn.functional.normalize(hf[:, 0], dim=1)
    assert (unit - hf_unit).abs().max() < 1e-6
    # positions did reach past 514: cumsum(non-pad) + 1
    assert int(((ids != 1).cumsum(1) * (ids != 1) + 1).max()) == S + 1


@pytest.fixture(scope="module")
def golden():
    return golden_npz.load("golden_classifier_xlmr_long")


def test_golden_embeddings_match_the_oracle(golden):
    cfg = json.loads(str(golden["bert_config"]))
    assert cfg["max_position_embeddings"] == 8194 and cfg["model_type"] == "xlm-roberta"
    sd = {k[5:]: torch.from_numpy(golden[k]).float() for k in golden.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(golden["input_ids"]).long()
    mask = torch.from_numpy(golden["attention_mask"]).long()
    assert ids.shape[1] == 1024 and int((mask.sum(1) > 512).sum()) >= 6
    unit = eo.encoder_forward_cls(sd, ids, mask, arch="roberta", num_heads=cfg["num_attention_heads"],
                                  ln_eps=cfg["layer_norm_eps"], pad_idx=1)
    n = len(golden["texts"])
    ref = np.concatenate([golden["emb_train"], golden["emb_test"]])
    assert np.abs(unit.numpy() - ref).max() < 1e-5
    assert unit.shape[0] == n + len(golden["test_texts"])
