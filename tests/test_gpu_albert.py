"""GPU tests of the ALBERT (albert-base / large v1 / v2) and ELECTRA (discriminators) encoders: factorized embeddings with
the E -> H projection, ALBERT's shared layers packed once, and the tanh-approximated GELU of "gelu_new".  Against the fp32
oracle of oracle/albert_oracle.py (pinned to HF by tests/test_albert_cpu.py), HF itself on the CPU, an fp64 reference of the
activation alone.  The golden ALBERT / ELECTRA classifier runs, the CUDA-graph pipeline step and the drop-in classifier on
local checkpoints are tests/test_gpu_encoder_families.py's.

Encoder bounds are those of test_gpu_deberta.py: max abs < 3e-4 and max row norm < 1e-3 on the unit CLS rows.  The
768-wide test models keep HF's initial weight scale (LayerNorms and biases perturbed): with every weight matrix tripled, as
the 256-wide CPU oracle tests do, the fp16 operand rounding alone moves the CLS rows of 4 to 12 layers by 1.1e-3 to 1.9e-3
(row norm; max abs <= 2e-4), in ELECTRA's unshared erf layers as much as in ALBERT's shared tanh ones."""
import pytest
import torch

from oracle import albert_oracle as ao
from test_albert_cpu import albert_ids, albert_model, electra_model, fp16_grid, gelu_tanh64, tanh_gelu_bound
from test_gpu_minilm import _check_cls

pytestmark = pytest.mark.gpu

BASE = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=1000)


def _sd(m):
    return {k: v.detach().float() for k, v in m.state_dict().items()}


def _encoder(cabi, m, max_tokens, cls_only=True, clone_layers=False):
    fn = cabi.albert_to_bert_state_dict if m.config.model_type == "albert" else cabi.electra_to_bert_state_dict
    sd, dims = fn(dict(m.state_dict()), m.config)
    if clone_layers:   # every layer its own copy: defeats the sharing
        sd = {k: (v.clone() if k.startswith("encoder.layer.") else v) for k, v in sd.items()}
    return cabi.Encoder(sd, arch="bert", max_tokens=max_tokens, cls_only=cls_only, **dims)


def _check(out, ref):
    e = out - ref
    assert e.abs().max() < 3e-4 and e.norm(dim=1).max() < 1e-3, (e.abs().max(), e.norm(dim=1).max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5


# ------------------------------------------------------------------------------------------------ activation alone
def test_tanh_gelu_epilogue_on_every_fp16_value(cabi):
    """ac_linear_tc epi 3 on exact pre-activations: A = identity rows (K = 64), so output (m, n) is act(W[n, m] + 0) for one
    fp16 weight; W holds every fp16 value in [-10, 10].  Bound: tests/test_albert_cpu.py::tanh_gelu_bound"""
    x = fp16_grid()
    K = 64
    N = (x.numel() + K - 1) // K
    N = (N + 7) // 8 * 8
    W = torch.zeros(N * K, dtype=torch.float16)
    W[: x.numel()] = x
    W = W.view(N, K)
    X = torch.eye(K, dtype=torch.float16)
    Y = cabi.linear_tc(X.cuda(), W.cuda(), torch.zeros(N, device="cuda"), epi=3, out_half=True).cpu()
    out = Y.t().reshape(-1)[: x.numel()].double()
    ref = gelu_tanh64(x)
    frac = ((out - ref).abs() / tanh_gelu_bound(ref))
    worst = int(frac.argmax())
    # outputs below the fp16 normal range round absolutely (the 2^-25 term dominates their bound); over the normal ones the
    # fraction measures the relative terms, fp16 rounding plus the fp32 evaluation allowance
    normal = ref.abs() >= 2.0 ** -14
    fn = frac.masked_fill(~normal, 0.0)
    wn = int(fn.argmax())
    print(f"tanh GELU epilogue: {x.numel()} fp16 values, worst error / bound = {frac.max().item():.3f} at x = "
          f"{x[worst].item():.6g}; over the {int(normal.sum())} normal fp16 outputs {fn.max().item():.3f} at x = "
          f"{x[wn].item():.6g}")
    assert bool(torch.isfinite(out).all()) and frac.max().item() <= 1.0


# ------------------------------------------------------------------------------------------------ encoders
@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("B,S", [(3, 16), (5, 77), (4, 128), (3, 129), (3, 300), (2, 512)])
def test_albert_base_shape_matches_oracle(cabi, B, S, cls_only):
    """albert-base shape (768, 12 heads, I 3072, E 128, "gelu_new"), 4 shared layers, padded; full hidden state too"""
    m = albert_model(num_hidden_layers=4, scale=1.0, **BASE)
    ids, mask = albert_ids(B, S, True, vocab=BASE["vocab_size"])
    ref, ref_hidden = ao.factorized_forward_cls(_sd(m), ids, mask, m.config, return_hidden=True)
    enc = _encoder(cabi, m, B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ref)
    if not cls_only:
        # the hidden rows are LayerNorm outputs of norm ~sqrt(768) = 28 (elements O(1)), not unit rows: the CLS rows' 3e-4
        # bound per element of a unit row corresponds to ~8e-3 here.  5e-3 keeps that relative precision with margin.
        hidden = enc.last_hidden(B, S).cpu().view(B, S, -1)
        keep = mask.bool()
        assert (hidden[keep] - ref_hidden[keep]).abs().max() < 5e-3
    enc.close()


def test_projection_with_embedding_size_zero_means_hidden(cabi):
    """embedding_size = 0 means hidden also when a projection is given (an ALBERT with E = H): the handle computes the same
    bits as one built with embedding_size = H, and matches the oracle"""
    m = albert_model(num_hidden_layers=2, embedding_size=768, scale=1.0, **BASE)
    sd, dims = cabi.albert_to_bert_state_dict(dict(m.state_dict()), m.config)
    assert dims["embedding_size"] == 768 and "embeddings_project.weight" in sd
    ids, mask = albert_ids(3, 100, True, vocab=BASE["vocab_size"])
    outs = []
    for E in (768, 0):
        enc = cabi.Encoder(sd, arch="bert", max_tokens=3 * 100, **{**dims, "embedding_size": E})
        outs.append(enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu())
        enc.close()
    assert torch.equal(outs[0], outs[1])
    _check(outs[1], ao.factorized_forward_cls(_sd(m), ids, mask, m.config))


@pytest.mark.parametrize("over", [dict(num_hidden_layers=4, num_hidden_groups=2, inner_group_num=2),
                                  dict(num_hidden_layers=3, embedding_size=768), dict(num_hidden_layers=2, hidden_act="gelu"),
                                  dict(num_hidden_layers=1)])
def test_albert_variants_match_oracle(cabi, over):
    """groups x inner layers, E = H (the projection still runs), v1's erf GELU, and one layer (the CLS tail reads the
    projection's output directly)"""
    m = albert_model(scale=1.0, **{**BASE, **over})
    ids, mask = albert_ids(4, 150, True, vocab=BASE["vocab_size"])
    enc = _encoder(cabi, m, 4 * 150)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ao.factorized_forward_cls(_sd(m), ids, mask, m.config))
    enc.close()


def test_albert_base_at_the_benched_batch_matches_oracle_on_sampled_rows(cabi):
    """the seeded workload.albert_base (12 shared layers) at B = 512 x S = 128: 8 sampled sequences against the oracle"""
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.albert_base(1234)
    B, S = 512, 128
    ids, _ = albert_ids(B, S, False, vocab=cfg.vocab_size, seed=3)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda()).cpu()
    sel = torch.tensor([0, 1, 63, 127, 128, 300, 510, 511])
    _check(out[sel], ao.factorized_forward_cls(_sd(m), ids[sel], None, cfg))
    assert bool(torch.isfinite(out).all())
    enc.close()


def test_albert_large_shape_matches_oracle(cabi):
    from adaptive_classifier_b200 import workload as wl
    m, cfg = wl.albert_large(1234)
    ids, mask = albert_ids(3, 200, True, vocab=cfg.vocab_size, seed=4)
    enc = cabi.Encoder.from_hf(m, max_tokens=3 * 200)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ao.factorized_forward_cls(_sd(m), ids, mask, cfg))
    enc.close()


@pytest.mark.parametrize("cls_only", [True, False])
@pytest.mark.parametrize("B,S", [(3, 16), (5, 77), (3, 129), (3, 300), (2, 512)])
def test_electra_small_shape_matches_oracle(cabi, B, S, cls_only):
    """electra-small shape: hidden 256 (new to this library), 4 heads, E 128, I 1024, 4 layers"""
    m = electra_model(num_hidden_layers=4, intermediate_size=1024, vocab_size=1000)
    ids, mask = albert_ids(B, S, True, vocab=1000)
    enc = _encoder(cabi, m, B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ao.factorized_forward_cls(_sd(m), ids, mask, m.config))
    enc.close()


@pytest.mark.parametrize("family", ["electra_base", "bert_gelu_new"])
def test_from_hf_matches_hf(cabi, family):
    """an electra-base-shaped ElectraModel (E = H: no projection) and a BertModel with hidden_act "gelu_new", through
    Encoder.from_hf against HF on the CPU"""
    if family == "electra_base":
        m = electra_model(seed=11, num_hidden_layers=12, embedding_size=768, scale=1.0, **BASE)
    else:
        from transformers import BertConfig, BertModel
        torch.manual_seed(12)
        m = BertModel(BertConfig(num_hidden_layers=4, hidden_act="gelu_new", vocab_size=1000), add_pooling_layer=False).eval()
    ids, mask = albert_ids(4, 150, True, vocab=1000)
    with torch.no_grad():
        ref = torch.nn.functional.normalize(m(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=4 * 150)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check_cls(out, ref)
    enc.close()


# ------------------------------------------------------------------------------------------------ sharing
def _handle_bytes(make):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    enc = make()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return enc, free0 - torch.cuda.mem_get_info()[0]


def test_shared_layers_are_packed_once_and_compute_the_same_bits(cabi):
    """a 12-layer shared albert-base handle takes less device memory over a 1-layer handle (same max_tokens) than one layer's
    packed weights; its output is bitwise that of a handle built from cloned per-layer tensors"""
    from adaptive_classifier_b200 import workload as wl
    m12, _ = wl.albert_base(1234)
    m1 = albert_model(num_hidden_layers=1, scale=1.0, **{**BASE, "vocab_size": 30000})
    T = 8 * 128
    enc1, b1 = _handle_bytes(lambda: _encoder(cabi, m1, T))
    enc12, b12 = _handle_bytes(lambda: _encoder(cabi, m12, T))
    layer_bytes = (4 * 768 * 768 + 2 * 768 * 3072) * 2
    print(f"albert-base handles: 1 layer {b1 / 2**20:.1f} MiB, 12 shared layers {b12 / 2**20:.1f} MiB, one layer's packed "
          f"weights {layer_bytes / 2**20:.1f} MiB")
    assert b12 - b1 < layer_bytes, (b1, b12)
    enc1.close()
    encc, bc = _handle_bytes(lambda: _encoder(cabi, m12, T, clone_layers=True))
    assert bc - b12 > 10 * layer_bytes, (bc, b12)     # the unshared packing really is larger
    ids, mask = albert_ids(8, 128, True, vocab=30000, seed=9)
    a = enc12.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    b = encc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    assert torch.equal(a, b)
    enc12.close(); encc.close()
