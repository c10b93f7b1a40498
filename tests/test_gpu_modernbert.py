"""GPU tests of the ModernBERT encoder (pre-LN blocks, RoPE and GeGLU epilogues, sliding-window attention) against the fp32
oracle of oracle/modernbert_oracle.py (pinned to HF ModernBertModel by tests/test_modernbert_cpu.py).  The reference's
classifier outputs on the golden ModernBERT checkpoint and the CUDA-graph replay of the pipeline step are
tests/test_gpu_encoder_families.py's."""
import pytest
import torch

from oracle import modernbert_oracle as eo

pytestmark = pytest.mark.gpu


def _model(seed, gamma_noise=0.3, **over):
    kw = dict(vocab_size=300, hidden_size=128, num_hidden_layers=4, num_attention_heads=2, intermediate_size=192,
              local_attention=16, max_position_embeddings=512, pad_token_id=0)
    kw.update(over)
    sd, cfg, m = eo.make_modernbert(seed, **kw)
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "norm" in n and gamma_noise:
                p.add_(gamma_noise * torch.randn(p.shape, generator=g))
    return m


def _oracle(m, ids, mask):
    from adaptive_classifier_b200._cabi import modernbert_settings
    c = m.config
    s = modernbert_settings(c)
    sd = {k: v.detach().float() for k, v in m.state_dict().items()}
    with torch.no_grad():
        return eo.modernbert_forward_cls(sd, ids, mask, num_heads=c.num_attention_heads,
                                         layer_sliding=[bool(v) for v in s["layer_sliding"]], sliding_window=s["sliding_window"],
                                         rope_theta=s["rope_theta"], norm_eps=c.norm_eps, return_hidden=True)


def _ids(B, S, vocab, seed, pad):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(5, vocab, (B, S), generator=g)
    ids[:, 0] = 2
    mask = torch.ones(B, S, dtype=torch.int64)
    if pad:
        for b in range(1, B):
            n = max(2, S - (S * b) // (B + 1))
            mask[b, n:] = 0
            ids[b, n:] = 0
    return ids, mask


def _check(out, ref):
    e = out - ref
    assert e.norm(dim=1).max() < 1.5e-3, e.norm(dim=1).max()
    P = torch.nn.functional.normalize(torch.randn(1024, out.shape[1], generator=torch.Generator().manual_seed(0)), dim=1)
    dd = (((out[:, None, :] - P[None]) ** 2).sum(-1) - ((ref[:, None, :] - P[None]) ** 2).sum(-1)).abs().max()
    assert dd < 1e-3, dd


@pytest.mark.parametrize("B,S,pad", [(3, 77, True), (2, 128, False), (3, 300, True), (1, 512, False)])
@pytest.mark.parametrize("cls_only", [True, False])
def test_modernbert_tiny_matches_oracle(cabi, B, S, pad, cls_only):
    """hidden 128 / 2 heads, 4 layers (full, sliding, sliding, full), half-window 8: the band edge falls inside every
    sequence; non-unit norm gammas; attention_kernel at S <= 128, attention_stream_kernel at 128 < S <= 512 (sliding layers
    skip the key blocks outside the band); padded batches"""
    m = _model(7)
    ids, mask = _ids(B, S, 300, S + B, pad)
    ref, ref_hidden = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ref)
    if not cls_only:
        hid = enc.last_hidden(B, S).cpu().view(B, S, -1)
        keep = mask.bool()
        assert (hid[keep] - ref_hidden[keep]).abs().max() < 2e-2 * ref_hidden[keep].abs().max()
    else:
        with pytest.raises(cabi.AdaptiveB200Error):
            enc.last_hidden(B, S)
    enc.close()


def test_modernbert_large_residual_stream_with_row_mean(cabi):
    """residual sums of |y| ~ 1e2..1e3 with a non-zero row mean: the deferred attn_norm / mlp_norm correction
    r (acc - mu c1) subtracts two large, nearly equal terms"""
    m = _model(11, gamma_noise=0.0)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        m.embeddings.norm.weight.copy_(300.0 + 100.0 * torch.randn(128, generator=g))
        for l in m.layers:
            l.mlp.Wo.weight.add_(0.05)                             # every output column gets + 0.05 sum(h): row mean moves
            if l.attn_norm.__class__.__name__ != "Identity":
                l.attn_norm.weight.add_(0.3 * torch.randn(128, generator=g))
            l.mlp_norm.weight.add_(0.3 * torch.randn(128, generator=g))
    B, S = 3, 150
    ids, mask = _ids(B, S, 300, 9, True)
    with torch.no_grad():
        y0 = m.embeddings(input_ids=ids)
        hs = m(input_ids=ids, attention_mask=mask, output_hidden_states=True).hidden_states
    y = torch.stack(hs[1:])[:, mask.bool()]
    assert y0.abs().mean() > 100 and y.abs().max() > 1e3 and y.mean(-1).abs().mean() > 3
    ref, _ = _oracle(m, ids, mask)
    for cls_only in (True, False):
        enc = cabi.Encoder.from_hf(m, max_tokens=B * S, cls_only=cls_only)
        out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
        _check(out, ref)
        enc.close()


@pytest.mark.parametrize("name,B,S,pad", [("base", 4, 128, False), ("base", 3, 300, True), ("large", 2, 128, False)])
def test_modernbert_published_shapes(cabi, name, B, S, pad):
    """ModernBERT-base (22 x 768, 12 heads, I 1152) and -large (28 x 1024, 16 heads, I 2624), vocab 50368, seeded init"""
    over = dict(vocab_size=50368, max_position_embeddings=8192, pad_token_id=50283, local_attention=128)
    if name == "large":
        over.update(hidden_size=1024, num_hidden_layers=28, num_attention_heads=16, intermediate_size=2624)
    else:
        over.update(hidden_size=768, num_hidden_layers=22, num_attention_heads=12, intermediate_size=1152)
    m = _model(1234, gamma_noise=0.1, **over)
    g = torch.Generator().manual_seed(S)
    ids = torch.randint(1000, 50000, (B, S), generator=g)
    ids[:, 0] = 50281
    mask = torch.ones(B, S, dtype=torch.int64)
    if pad:
        mask[1, 200:] = 0
        mask[2, 37:] = 0
        ids[mask == 0] = 50283
    ref, _ = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ref)
    enc.close()
