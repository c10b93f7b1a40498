"""GPU tests of the head_dim-32 encoders (all-MiniLM-L6/L12-v2, BGE-small, E5-small, GTE-small: BertModel with 384 hidden =
12 heads of 32) against the fp32 oracle of oracle/encoder_oracle.py (pinned to HF BertModel at that shape by
tests/test_minilm_cpu.py) and HF itself on the CPU; then the D = 384 stages downstream of the encoder (kNN, head
training).  The golden classifier run, the CUDA-graph pipeline step and the drop-in classifier on a local checkpoint are
tests/test_gpu_encoder_families.py's."""
import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo
from oracle import head_oracle as ho
from oracle import knn_oracle as ko
from test_gpu_parity import _encoder, _head, _perturb_layernorms

pytestmark = pytest.mark.gpu

MINILM = dict(hidden_size=384, num_attention_heads=12, intermediate_size=1536)


def _minilm(layers=6, seed=1234):
    sd, cfg, _ = eo.make_bert_state_dict(seed, num_hidden_layers=layers, **MINILM)
    return sd, cfg


def _ids_mask(B, S, pad, vocab=30522):
    ids = eo.synthetic_ids(B, S, vocab=vocab)
    mask = torch.ones_like(ids)
    if pad:
        for b in range(1, B):
            n = max(2, S - (S * b) // (B + 1))
            mask[b, n:] = 0
            ids[b, n:] = 0
    return ids, mask


def _check_cls(out, ref, abs_bound=2e-4):
    """the bounds of test_gpu_parity.py::test_encoder_cls_matches_oracle"""
    e = out - ref
    assert e.abs().max() < abs_bound, e.abs().max()
    assert e.norm(dim=1).max() < 1e-3, e.norm(dim=1).max()
    P = torch.nn.functional.normalize(torch.randn(2048, out.shape[1], generator=torch.Generator().manual_seed(0)), dim=1)
    dd = (((out[:, None, :] - P[None]) ** 2).sum(-1) - ((ref[:, None, :] - P[None]) ** 2).sum(-1)).abs().max()
    assert dd < 1e-3, dd
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5


# ------------------------------------------------------------------------------------------------ encoder
@pytest.mark.parametrize("B,S,pad", [(2, 128, False), (3, 16, True), (5, 77, True), (8, 128, False),
                                     (3, 129, False), (2, 300, True), (1, 512, False)])
def test_minilm_l6_encoder_matches_oracle(cabi, B, S, pad):
    """6 x 384, 12 heads of 32; S <= 128 runs attention_kernel<32, ScorePlain>, 128 < S <= 512
    attention_stream_kernel<32, ScorePlain>"""
    sd, cfg = _minilm(6)
    ids, mask = _ids_mask(B, S, pad)
    ref = eo.encoder_forward_cls(sd, ids, mask, num_heads=12)
    enc = _encoder(cabi, sd, cfg, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check_cls(out, ref)
    enc.close()


@pytest.mark.parametrize("B,S,cls_only,pad", [(5, 96, False, True), (3, 200, False, True), (8, 128, True, False)])
def test_minilm_with_nontrivial_layernorms_matches_oracle(cabi, B, S, cls_only, pad):
    """non-unit gamma, non-zero beta and shifted row means at head_dim 32; with cls_only off the whole last hidden state too
    (bounds of test_gpu_parity.py::test_encoder_with_nontrivial_layernorms_matches_oracle)"""
    sd, cfg = _minilm(6)
    sd = _perturb_layernorms(sd)
    ids, mask = _ids_mask(B, S, pad)
    ref, ref_hidden = eo.encoder_forward_cls(sd, ids, mask, num_heads=12, return_hidden=True)
    enc = _encoder(cabi, sd, cfg, max_tokens=B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    e = out - ref
    assert e.abs().max() < 3e-4 and e.norm(dim=1).max() < 1e-3, (e.abs().max(), e.norm(dim=1).max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5
    if not cls_only:
        hidden = enc.last_hidden(B, S).cpu()
        keep = mask.bool()
        assert (hidden.view(B, S, -1)[keep] - ref_hidden[keep]).abs().max() < 5e-3
    enc.close()


def test_minilm_l12_shape_matches_oracle(cabi):
    """all-MiniLM-L12-v2 / paraphrase-multilingual-MiniLM-L12-v2 depth: 12 x 384"""
    sd, cfg = _minilm(12)
    ids, mask = _ids_mask(4, 128, True)
    ref = eo.encoder_forward_cls(sd, ids, mask, num_heads=12)
    enc = _encoder(cabi, sd, cfg, max_tokens=4 * 128)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check_cls(out, ref)
    enc.close()


def test_minilm_at_the_benched_batch_matches_oracle_on_sampled_rows(cabi):
    """B = 512 x S = 128 (the step tools/bench_minilm.py times): 8 sampled sequences against the fp32 CPU oracle"""
    sd, cfg = _minilm(6)
    B, S = 512, 128
    ids = eo.synthetic_ids(B, S)
    enc = _encoder(cabi, sd, cfg, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda()).cpu()
    sel = torch.tensor([0, 1, 63, 127, 128, 300, 510, 511])
    ref = eo.encoder_forward_cls(sd, ids[sel], None, num_heads=12)
    e = out[sel] - ref
    assert e.norm(dim=1).max() < 1e-3 and e.abs().max() < 2e-4, (e.norm(dim=1).max(), e.abs().max())
    assert (out.norm(dim=1) - 1).abs().max() < 1e-5 and bool(torch.isfinite(out).all())
    enc.close()


def test_minilm_roberta_arch_positions_and_padding(cabi):
    """RoBERTa position ids (cumsum of non-pad + pad_idx) with 12 heads of 32"""
    sd, cfg, _ = eo.make_bert_state_dict(5, arch="roberta", num_hidden_layers=2, hidden_size=384, num_attention_heads=12,
                                         intermediate_size=1536, vocab_size=300, max_position_embeddings=130)
    B, S = 4, 40
    ids = eo.synthetic_ids(B, S, vocab=300, arch="roberta")
    for b in range(B):
        ids[b, S - 3 * b:] = 1
    mask = (ids != 1).long()
    ref = eo.encoder_forward_cls(sd, ids, mask, arch="roberta", num_heads=12, ln_eps=cfg.layer_norm_eps, pad_idx=1)
    enc = _encoder(cabi, sd, cfg, B * S, arch="roberta")
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    assert (out - ref).norm(dim=1).max() < 1e-3
    enc.close()


def test_minilm_distilbert_through_from_hf(cabi):
    """DistilBERT with 4 heads of 32 (dim 128) through Encoder.from_hf vs HF itself on the CPU"""
    from transformers import DistilBertConfig, DistilBertModel
    torch.manual_seed(3)
    cfg = DistilBertConfig(vocab_size=400, dim=128, n_heads=4, n_layers=2, hidden_dim=256, max_position_embeddings=64)
    m = DistilBertModel(cfg).eval()
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "LayerNorm" in n or "layer_norm" in n or n.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape))
    ids = eo.synthetic_ids(5, 40, vocab=400)
    mask = torch.ones_like(ids)
    mask[1, 30:] = 0
    mask[4, 11:] = 0
    with torch.no_grad():
        ref = torch.nn.functional.normalize(m(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=5 * 40)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    assert (out - ref).norm(dim=1).max() < 1e-3
    enc.close()


def test_minilm_bert_through_from_hf_matches_hf(cabi):
    """a seeded BertModel(BertConfig(hidden_size=384, num_attention_heads=12, intermediate_size=1536, num_hidden_layers=6))
    through Encoder.from_hf, against HF on the CPU"""
    from transformers import BertConfig, BertModel
    torch.manual_seed(11)
    m = BertModel(BertConfig(num_hidden_layers=6, **MINILM)).eval()
    ids, mask = _ids_mask(4, 64, True)
    with torch.no_grad():
        ref = torch.nn.functional.normalize(m(input_ids=ids, attention_mask=mask).last_hidden_state[:, 0, :], dim=1)
    enc = cabi.Encoder.from_hf(m, max_tokens=4 * 64)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check_cls(out, ref)
    enc.close()


# ------------------------------------------------------------------------------------------------ D = 384 downstream
@pytest.mark.parametrize("k", [5, 1000])
def test_knn_tensor_path_at_d384_equals_oracle(cabi, k):
    """1M-class-structured rows are not needed for the property: 120k x 384 rows, 1000 classes; bit-identical ids and
    distances against the oracle (16 queries) and the exact scan (32 queries)"""
    from adaptive_classifier_b200 import workload as wl
    N, D, C, B = 120_000, 384, 1000, 256
    P = wl.synthetic_rows(0, N, D, C, seed=0, device="cuda")
    Q = wl.synthetic_queries_embeddings(B, D, C, device="cuda")
    Ph = cabi.knn_make_shadow(P)
    stats = torch.zeros(4, dtype=torch.int32, device="cuda")
    d1, i1 = cabi.knn_l2_topk(Q, P, k, p_sqnorm=cabi.row_sqnorm(P), p_half=Ph, algo=cabi.AC_KNN_TENSOR, stats=stats)
    sel = torch.arange(0, B, B // 32)[:32].cuda()
    d0, i0 = cabi.knn_l2_topk(Q[sel].contiguous(), P, k, algo=cabi.AC_KNN_EXACT)
    torch.cuda.synchronize()
    assert stats.cpu().tolist()[1] == 0
    assert torch.equal(i1[sel], i0) and torch.equal(d1[sel], d0)
    assert bool((d1[:, 1:] >= d1[:, :-1]).all())
    d_ref, i_ref = ko.knn_l2(Q[sel[:16]].cpu().numpy(), P.cpu().numpy(), k)
    assert np.array_equal(i1[sel[:16]].cpu().numpy(), i_ref) and np.array_equal(d1[sel[:16]].cpu().numpy(), d_ref)


def test_head_train_steps_match_oracle_at_d384(cabi):
    """3 optimizer steps of the 384 -> 384 -> 192 -> C head (fwd with injected dropout masks, CE loss, bwd, clip, AdamW)
    against the torch-CPU restatement; batches are drawn until every |pre-activation| > 1e-6 (ReLU' is discontinuous at 0)"""
    B, D, C = 32, 384, 12
    g = torch.Generator().manual_seed(19)
    p, pg = _head(D, C)
    m = {k: torch.zeros_like(v) for k, v in p.items()}
    v = {k: torch.zeros_like(v2) for k, v2 in p.items()}
    mg = {k: torch.zeros_like(t) for k, t in pg.items()}
    vg = {k: torch.zeros_like(t) for k, t in pg.items()}
    for step in range(1, 4):
        while True:
            X = torch.nn.functional.normalize(torch.randn(B, D, generator=g), dim=1)
            masks = tuple(((torch.rand(B, n, generator=g) >= 0.1).float() / 0.9) for n in (D, D // 2))
            a0 = X @ p["W0"].t() + p["b0"]
            a1 = (torch.relu(a0) * masks[0]) @ p["W1"].t() + p["b1"]
            if min(a0.abs().min().item(), a1.abs().min().item()) > 1e-6:
                break
        y = torch.randint(0, C, (B,), generator=g)
        loss_ref, grads, _ = ho.head_grads(X, y, p, masks, "ce")
        norm_ref = ho.clip_and_adamw(p, grads, m, v, step)
        stats = cabi.head_train_step(X.cuda(), y.cuda(), pg, mg, vg, step=step, loss_kind=cabi.AC_LOSS_CE,
                                     masks=(masks[0].cuda(), masks[1].cuda())).cpu()
        assert abs(stats[0].item() - loss_ref.item()) < 1e-5
        assert abs(stats[2].item() - norm_ref.item()) < 1e-4 * max(1.0, norm_ref.item())
        for k in ho.PARAM_ORDER:
            diff = (pg[k].cpu() - p[k]).abs()
            solid = grads[k].abs() > 1e-6 * grads[k].abs().max()
            assert diff[solid].max() < 2e-5, (step, k, float(diff[solid].max()))
            assert diff.max() <= 2.1e-3 * step, (step, k)
