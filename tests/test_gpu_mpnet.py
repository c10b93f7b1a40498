"""GPU tests of the MPNet encoders (all-mpnet-base-v2, multi-qa-mpnet-base-*, paraphrase-mpnet-base-v2: the post-LN BERT
block with RoBERTa positions and a relative position bias on every layer's attention scores) against the fp32 oracle of
oracle/mpnet_oracle.py (pinned to HF MPNetModel by tests/test_mpnet_cpu.py) and HF itself on the CPU.  The golden
classifier run, the CUDA-graph pipeline step and the drop-in classifier on a local checkpoint are
tests/test_gpu_encoder_families.py's."""
import pytest
import torch

from oracle import encoder_oracle as eo
from oracle import mpnet_oracle as mo
from test_gpu_minilm import _check_cls
from test_mpnet_cpu import mpnet_ids, mpnet_model

pytestmark = pytest.mark.gpu

WIDE = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=1000)


def _mpnet_encoder(cabi, m, max_tokens, cls_only=True):
    sd, dims = cabi.mpnet_to_bert_state_dict(dict(m.state_dict()), m.config)
    return cabi.Encoder(sd, arch="mpnet", max_tokens=max_tokens, cls_only=cls_only, **dims)


def _hf_sd(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


# ------------------------------------------------------------------------------------------------ encoder
@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("B,S,pad", [(3, 16, False), (5, 77, True), (4, 128, False), (3, 129, False), (3, 200, True),
                                     (2, 384, False), (1, 512, False)])
def test_mpnet_encoder_matches_oracle(cabi, B, S, pad, cls_only):
    """2 x 768, 12 heads of 64, O(1) bias table and perturbed LayerNorms; S <= 128 runs attention_kernel<64, ScoreRelBias>,
    longer sequences attention_stream_kernel<64, ScoreRelBias>.  cls_only off also compares the whole last hidden state
    (bounds of test_gpu_parity.py::test_encoder_with_nontrivial_layernorms_matches_oracle and ::test_encoder_long_sequences)"""
    m = mpnet_model(num_hidden_layers=2, **WIDE)
    ids, mask = mpnet_ids(B, S, pad, vocab=WIDE["vocab_size"])
    ref, ref_hidden = mo.mpnet_forward_cls(_hf_sd(m), ids, mask, num_heads=12, ln_eps=1e-5, return_hidden=True)
    enc = _mpnet_encoder(cabi, m, B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    e = out - ref
    assert e.abs().max() < 3e-4 and e.norm(dim=1).max() < 1e-3, (e.abs().max(), e.norm(dim=1).max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5
    if not cls_only:
        hidden = enc.last_hidden(B, S).cpu()
        keep = mask.bool()
        assert (hidden.view(B, S, -1)[keep] - ref_hidden[keep]).abs().max() < 5e-3
    enc.close()


def test_mpnet_base_at_the_benched_batch_matches_oracle_on_sampled_rows(cabi):
    """the all-mpnet-base-v2 shape (workload.mpnet_base, bias table scaled to O(1)) at B = 512 x S = 128: 8 sampled sequences
    against the fp32 CPU oracle"""
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.mpnet_base(1234)
    with torch.no_grad():
        m.encoder.relative_attention_bias.weight.mul_(50.0)
    B, S = 512, 128
    ids = eo.synthetic_ids(B, S, vocab=cfg.vocab_size, arch="roberta")
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda()).cpu()
    sel = torch.tensor([0, 1, 63, 127, 128, 300, 510, 511])
    ref = mo.mpnet_forward_cls(_hf_sd(m), ids[sel], None, num_heads=12, ln_eps=cfg.layer_norm_eps)
    e = out[sel] - ref
    assert e.norm(dim=1).max() < 1e-3 and e.abs().max() < 2e-4, (e.norm(dim=1).max(), e.abs().max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5 and bool(torch.isfinite(out).all())
    enc.close()


def test_mpnet_through_from_hf_matches_hf(cabi):
    """a seeded MPNetModel through Encoder.from_hf, against HF on the CPU"""
    m = mpnet_model(seed=11, num_hidden_layers=3, **WIDE)
    ids, mask = mpnet_ids(4, 150, True, vocab=WIDE["vocab_size"])
    with torch.no_grad():
        ref = torch.nn.functional.normalize(m(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=4 * 150)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check_cls(out, ref)
    enc.close()
