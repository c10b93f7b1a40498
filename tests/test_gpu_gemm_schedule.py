"""The GEMM's epilogue warps drain tile i while the MMA warpgroup already runs tile i+1's mainloop, through one shared
accumulator tile.  A persistent launch with many tiles per CTA must therefore give, bit for bit, what launches with at
most one tile per CTA give: every 128-row block of the output is recomputed on its own and compared."""
import pytest
import torch

# (M, N, K) with a ragged last row block: 129 x 24 tiles (~23 per CTA on 132 SMs) and, ragged in N too, 385 x 7 tiles (~20)
SHAPES = [(16384 + 77, 3072, 768), (49152 + 77, 776, 3072)]
KINDS = [  # (operand dtype, epi, out_half)
    (torch.float16, 0, False), (torch.float16, 1, False), (torch.float16, 2, False),
    (torch.float16, 0, True), (torch.float16, 1, True),
    (torch.float32, 0, False), (torch.float32, 1, False), (torch.float32, 2, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,epi,out_half", KINDS)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_persistent_launch_equals_single_block_launches(cabi, M, N, K, dtype, epi, out_half):
    g = torch.Generator(device="cuda").manual_seed(N + K + epi)
    X = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dtype)
    W = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g) if epi == 2 else None
    Y = cabi.linear_tc(X, W, bias, res, epi=epi, out_half=out_half)
    blocks = M // 128 + 1
    for b in sorted({0, 1, 37, blocks // 2, blocks - 2, blocks - 1}):
        r0, r1 = 128 * b, min(128 * (b + 1), M)
        Yb = cabi.linear_tc(X[r0:r1], W, bias, None if res is None else res[r0:r1], epi=epi, out_half=out_half)
        torch.cuda.synchronize()
        assert torch.equal(Y[r0:r1], Yb), f"row block {b} differs"


@pytest.mark.gpu
def test_encoder_forward_is_deterministic_at_bench_batch(cabi):
    from oracle import encoder_oracle as eo
    B, S = 512, 128
    sd, cfg, _ = eo.make_bert_state_dict(1234)
    enc = cabi.Encoder(sd, arch="bert", layers=cfg.num_hidden_layers, hidden=768, heads=12, intermediate=3072,
                       vocab=cfg.vocab_size, max_pos=512, type_vocab=2, ln_eps=cfg.layer_norm_eps, max_tokens=B * S)
    ids = eo.synthetic_ids(B, S).to(torch.int32).cuda()
    a = enc.forward_cls(ids).clone()
    b = enc.forward_cls(ids).clone()
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    enc.close()


@pytest.mark.gpu
def test_modernbert_batch_equals_single_sequences(cabi):
    """The RoPE (Wqkv) and GeGLU (Wi) epilogues re-read partner columns of the accumulator tile after the chunk they
    write: at B = 512 every CTA drains ~70 such tiles back to back, a single sequence gives each CTA at most one"""
    from oracle import modernbert_oracle as mo
    B, S = 512, 128
    _, _, m = mo.make_modernbert(5, vocab_size=300, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                                 intermediate_size=1152, local_attention=128, max_position_embeddings=512, pad_token_id=0)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(5, 300, (B, S), generator=g, dtype=torch.int32)
    ids[:, 0] = 2
    mask = torch.ones(B, S, dtype=torch.int32)
    full = enc.forward_cls(ids.cuda(), mask.cuda()).clone()
    for b in (0, 1, 255, B - 1):
        one = enc.forward_cls(ids[b:b + 1].contiguous().cuda(), mask[b:b + 1].contiguous().cuda())
        torch.cuda.synchronize()
        assert torch.equal(full[b:b + 1], one), f"sequence {b} differs"
    enc.close()
