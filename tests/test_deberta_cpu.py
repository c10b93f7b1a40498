"""CPU tests of the DeBERTa-v3 encoders (deberta-v3-xsmall / small / base / large, mdeberta-v3-base: the post-LN BERT block
with disentangled c2p + p2c attention): the fp32 oracle of oracle/deberta_oracle.py pinned against HF DebertaV2Model, the
product's index table, position tables and weight renaming against HF, the reference's golden embeddings of the DeBERTa
checkpoint, how far each wrong attention rule would move the embeddings, and the settings Encoder.from_hf refuses before
any device call."""
import json

import numpy as np
import pytest
import torch

import golden_npz
from oracle import deberta_oracle as do


def deberta_model(seed=5, rel_std=1.0, proj_scale=3.0, **over):
    """seeded DebertaV2Model of the v3 kind (256 log buckets, share_att_key, LayerNorm-ed relative embeddings, no position or
    type table) with perturbed LayerNorms, larger projections and O(1) relative embeddings, so that both position terms
    move the scores by O(1)"""
    from transformers import DebertaV2Config, DebertaV2Model
    kw = dict(vocab_size=400, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=512,
              max_position_embeddings=512, type_vocab_size=0, relative_attention=True, position_buckets=256,
              norm_rel_ebd="layer_norm", share_att_key=True, pos_att_type=["p2c", "c2p"], position_biased_input=False,
              layer_norm_eps=1e-7, hidden_act="gelu", pad_token_id=0)
    kw.update(over)
    torch.manual_seed(seed)
    m = DebertaV2Model(DebertaV2Config(**kw)).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "LayerNorm" in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif n == "encoder.rel_embeddings.weight":
                p.copy_(rel_std * torch.randn(p.shape, generator=g))
            elif "proj" in n and p.dim() == 2:
                p.mul_(proj_scale)
    return m


def deberta_ids(B, S, pad, vocab=400, seed=7, left=False):
    """[CLS] = 1 first, [SEP] = 2 last, ids in [3, vocab); padding (id 0, mask 0) at the end of sequences 1.. when pad (at
    the start with left)"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (B, S), generator=g)
    ids[:, 0] = 1
    ids[:, -1] = 2
    mask = torch.ones_like(ids)
    if pad:
        for b in range(1, B):
            n = max(2, S - (S * b) // (B + 1))
            if left:
                ids[b, : S - n] = 0
                mask[b, : S - n] = 0
            else:
                ids[b, n - 1] = 2
                ids[b, n:] = 0
                mask[b, n:] = 0
    return ids, mask


def deberta_tokenizer_words(words):
    """DebertaV2Tokenizer over [PAD] [CLS] [SEP] [UNK] [MASK] + one unigram piece per word, built in memory"""
    from transformers import DebertaV2Tokenizer
    vocab = [(t, 0.0) for t in ("[PAD]", "[CLS]", "[SEP]", "[UNK]", "[MASK]")]
    return DebertaV2Tokenizer(vocab=vocab + [("\u2581" + w, -1.0 - 0.01 * i) for i, w in enumerate(words)])


def _sd(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


CASES = [(3, 16, True, {}), (3, 77, True, {}), (3, 129, True, {}), (2, 300, True, {}),
         (3, 77, True, dict(position_buckets=16)), (2, 129, True, dict(position_buckets=16)),
         (3, 77, True, dict(share_att_key=False)), (2, 300, True, dict(share_att_key=False, position_buckets=16)),
         (3, 77, True, dict(position_biased_input=True)), (3, 129, True, dict(type_vocab_size=2)),
         (2, 129, True, dict(position_buckets=-1, max_relative_positions=64))]


@pytest.mark.parametrize("B,S,pad,over", CASES)
def test_deberta_oracle_matches_hf(B, S, pad, over):
    """buckets 16 reach the log range inside S <= 128; padded query rows get HF's uniform softmax, so every row compares"""
    m = deberta_model(**over)
    ids, mask = deberta_ids(B, S, pad)
    with torch.no_grad():
        hidden = m(input_ids=ids, attention_mask=mask).last_hidden_state
    ref = torch.nn.functional.normalize(hidden[:, 0, :], dim=1)
    out, out_hidden = do.deberta_forward_cls(_sd(m), ids, mask, m.config, return_hidden=True)
    assert (out - ref).abs().max() < 1e-6
    keep = mask.bool()
    assert (out_hidden[keep] - hidden[keep]).abs().max() < 1e-6 * max(1.0, hidden.abs().max().item())


@pytest.mark.parametrize("buckets,max_rel", [(256, 512), (32, 512), (16, 512), (256, -1), (-1, 512), (-1, 64)])
def test_deberta_rel_index_equals_hf_build_relative_position(buckets, max_rel):
    """entry 511 + (i - j) of the table is HF's clamp(bucket(i - j) + span, 0, 2 span - 1), bit for bit, on every pair of
    S = 512; and the p2c index HF gathers, -bucket(j - i) + span, is the same entry (the bucket is odd)"""
    from transformers.models.deberta_v2.modeling_deberta_v2 import build_relative_position
    from adaptive_classifier_b200._cabi import AC_ENCODER_MAX_S, deberta_rel_index
    S = AC_ENCODER_MAX_S
    mr = max_rel if max_rel >= 1 else 512
    table, span = deberta_rel_index(buckets, mr)
    assert table.shape == (2 * S - 1,) and table.dtype == torch.int32
    assert span == (buckets if buckets > 0 else mr)
    x = torch.zeros(1, S, 8)
    rp = build_relative_position(x, x, bucket_size=buckets, max_position=mr)[0]
    i = torch.arange(S)[:, None]
    j = torch.arange(S)[None, :]
    assert torch.equal(table[S - 1 + i - j].long(), torch.clamp(rp + span, 0, 2 * span - 1))
    assert torch.equal(table[S - 1 + i - j].long(), torch.clamp(-rp.t() + span, 0, 2 * span - 1))


@pytest.mark.parametrize("share", [True, False])
def test_deberta_to_bert_state_dict_consumes_every_parameter_and_builds_hf_position_tables(share):
    from adaptive_classifier_b200._cabi import deberta_to_bert_state_dict

    class Seen(dict):
        def __init__(self, *a):
            super().__init__(*a)
            self.read = set()

        def __getitem__(self, k):
            self.read.add(k)
            return dict.__getitem__(self, k)

    m = deberta_model(num_hidden_layers=3, share_att_key=share)
    sd = Seen(m.state_dict())
    out, dims = deberta_to_bert_state_dict(sd, m.config)
    assert sd.read == set(sd)
    assert len(out) == 5 + 16 * 3
    assert torch.equal(out["embeddings.token_type_embeddings.weight"], torch.zeros(1, 256))
    assert torch.equal(out["embeddings.position_embeddings.weight"], torch.zeros(512, 256))
    assert dims["pos_key"].shape == (3, 512, 256) and dims["pos_query"].shape == (3, 512, 256) and dims["pos_span"] == 256
    assert dims["type_vocab"] == 1 and dims["pad_idx"] == 0 and dims["max_pos"] == 512
    with torch.no_grad():
        rel = m.encoder.get_rel_embedding()
        for l, layer in enumerate(m.encoder.layer):
            att = layer.attention.self
            pk = att.key_proj(rel) if share else att.pos_key_proj(rel)
            pq = att.query_proj(rel) if share else att.pos_query_proj(rel)
            assert (dims["pos_key"][l] - pk).abs().max() < 1e-6 and (dims["pos_query"][l] - pq).abs().max() < 1e-6


MUTATIONS = [dict(c2p=False), dict(p2c=False), dict(p2c_transposed=False), dict(scale_factor=1),
             dict(p2c_index_of_r=True)]


@pytest.mark.parametrize("mut", MUTATIONS, ids=lambda d: next(iter(d)))
@pytest.mark.parametrize("B,S,over", [(3, 77, {}), (2, 300, {}), (3, 77, dict(position_buckets=16))])
def test_each_wrong_attention_rule_moves_the_embeddings_far_beyond_the_gpu_tolerance(B, S, over, mut):
    """a kernel that dropped a term, transposed p2c wrongly, scaled by sqrt(dh) or gathered p2c at the mirrored bucket would
    miss the GPU tests' 1e-3 row bound by at least 20x on every CLS row"""
    m = deberta_model(proj_scale=5.0, **over)
    ids, mask = deberta_ids(B, S, True)
    sd = _sd(m)
    good = do.deberta_forward_cls(sd, ids, mask, m.config)
    bad = do.deberta_forward_cls(sd, ids, mask, m.config, **mut)
    assert (good - bad).norm(dim=1).min() > 2e-2, (good - bad).norm(dim=1)


def test_deberta_oracle_reproduces_reference_embeddings():
    """golden_classifier_deberta*.npz: the unmodified reference's _get_embeddings on a 2-head x 64 DeBERTa-v3 checkpoint"""
    from transformers import DebertaV2Config
    g = golden_npz.load("golden_classifier_deberta")
    cfgd = json.loads(str(g["bert_config"]))
    assert cfgd["model_type"] == "deberta-v2" and cfgd["hidden_size"] // cfgd["num_attention_heads"] == 64
    c = DebertaV2Config(**{k: v for k, v in cfgd.items() if k not in ("model_type", "transformers_version", "architectures")})
    sd = {k[5:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("bert_") and k != "bert_config"}
    ids = torch.from_numpy(g["input_ids"])
    mask = torch.from_numpy(g["attention_mask"])
    assert (mask == 0).any()
    out = do.deberta_forward_cls(sd, ids, mask, c)
    ref = np.concatenate([g["emb_train"], g["emb_test"]])
    assert out.shape == ref.shape
    assert np.abs(out.numpy() - ref).max() < 1e-5


@pytest.mark.parametrize("over,name", [
    (dict(conv_kernel_size=3), "conv_kernel_size=3"),
    (dict(embedding_size=128), "embedding_size=128"),
    (dict(relative_attention=False), "relative_attention=False"),
    (dict(pos_att_type=["c2p"]), "pos_att_type"),
    (dict(pos_att_type=["p2c", "c2p", "p2p"]), "pos_att_type"),
    (dict(hidden_act="relu"), "hidden_act='relu'"),
    (dict(hidden_size=256, num_attention_heads=8), "head_dim=32"),
    (dict(attention_head_size=32), "head_dim=32"),
    (dict(max_position_embeddings=1024), "max_position_embeddings=1024")])
def test_from_hf_refuses_unimplemented_deberta_settings(over, name):
    from adaptive_classifier_b200._cabi import AdaptiveB200Error, Encoder
    m = deberta_model(num_hidden_layers=1, **over)
    with pytest.raises(AdaptiveB200Error, match=name.replace("[", r"\[")):
        Encoder.from_hf(m, device="cpu")


def test_from_hf_refuses_deberta_v1():
    from transformers import DebertaConfig, DebertaModel
    from adaptive_classifier_b200._cabi import AdaptiveB200Error, Encoder
    torch.manual_seed(0)
    m = DebertaModel(DebertaConfig(vocab_size=100, hidden_size=128, num_hidden_layers=1, num_attention_heads=2,
                                   intermediate_size=256)).eval()
    with pytest.raises(AdaptiveB200Error, match="model_type='deberta'"):
        Encoder.from_hf(m, device="cpu")
