"""GPU tests of ModernBERT at 512 < S <= 8192 (the streamed one-pass attention kernel and max_pos-row RoPE tables) against
the query-block fp32 oracle of oracle/modernbert_long_oracle.py (pinned to HF ModernBertModel by
tests/test_modernbert_long_cpu.py), run on the GPU in fp32 with TF32 off; the unchanged S <= 512 results; the refusals.
The reference's classifier outputs with max_length 1024 and the CUDA-graph replay of the pipeline step at S = 1024 are
tests/test_gpu_encoder_families.py's."""
import pytest
import torch

from oracle.modernbert_long_oracle import modernbert_forward_cls_blocked
from test_gpu_modernbert import _check, _ids, _model

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_oracle():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _oracle(m, ids, mask):
    from adaptive_classifier_b200._cabi import modernbert_settings
    c = m.config
    s = modernbert_settings(c)
    sd = {k: v.detach().float().cuda() for k, v in m.state_dict().items()}
    with torch.no_grad():
        unit, hid = modernbert_forward_cls_blocked(sd, ids.cuda(), mask.cuda(), num_heads=c.num_attention_heads,
                                                   layer_sliding=[bool(v) for v in s["layer_sliding"]],
                                                   sliding_window=s["sliding_window"], rope_theta=s["rope_theta"],
                                                   norm_eps=c.norm_eps, return_hidden=True)
    return unit.cpu(), hid.cpu()


def _run(cabi, m, ids, mask, cls_only):
    B, S = ids.shape
    ref, ref_hidden = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S, cls_only=cls_only)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ref)
    if not cls_only:
        hid = enc.last_hidden(B, S).cpu().view(B, S, -1)
        keep = mask.bool()
        assert (hid[keep] - ref_hidden[keep]).abs().max() < 2e-2 * ref_hidden[keep].abs().max()
    enc.close()


@pytest.mark.parametrize("S,B,pad", [(513, 2, True), (640, 1, False), (1000, 3, True), (2048, 2, True), (8192, 1, False),
                                     (8192, 2, True)])
@pytest.mark.parametrize("local_attention", [16, 128])
@pytest.mark.parametrize("cls_only", [True, False])
def test_modernbert_long_tiny_matches_oracle(cabi, S, B, pad, local_attention, cls_only):
    """hidden 128 / 2 heads, 4 layers (full, sliding, sliding, full), half-window 8 or 64, non-unit norm gammas; padded
    sequences end at 128 n +- 1 and at other lengths (_ids)"""
    m = _model(7, local_attention=local_attention, max_position_embeddings=8192)
    ids, mask = _ids(B, S, 300, S + B, pad)
    if pad and B >= 2:
        mask[1, 128 * (S // 256) + 1:] = 0
        ids[1, 128 * (S // 256) + 1:] = 0
    _run(cabi, m, ids, mask, cls_only)


@pytest.mark.parametrize("local_attention", [16, 128])
@pytest.mark.parametrize("cls_only", [True, False])
def test_modernbert_long_mask_with_a_hole(cabi, local_attention, cls_only):
    """keys 130-400 of sequence 0 masked: query rows near the hole see key blocks with no valid key first"""
    m = _model(5, local_attention=local_attention, max_position_embeddings=8192)
    ids, mask = _ids(2, 1000, 300, 17, True)
    mask[0, 130:401] = 0
    ids[0, 130:401] = 0
    _run(cabi, m, ids, mask, cls_only)


@pytest.mark.parametrize("B,S,pad", [(1, 8192, False), (2, 2048, True)])
def test_modernbert_long_base_shape(cabi, B, S, pad):
    """ModernBERT-base (22 x 768, 12 heads, I 1152, half-window 64 on 2 of 3 layers), vocab 50368, seeded init"""
    over = dict(vocab_size=50368, max_position_embeddings=8192, pad_token_id=50283, local_attention=128, hidden_size=768,
                num_hidden_layers=22, num_attention_heads=12, intermediate_size=1152)
    m = _model(1234, gamma_noise=0.1, **over)
    g = torch.Generator().manual_seed(S)
    ids = torch.randint(1000, 50000, (B, S), generator=g)
    ids[:, 0] = 50281
    mask = torch.ones(B, S, dtype=torch.int64)
    if pad:
        mask[1, 1300:] = 0
        ids[mask == 0] = 50283
    ref, _ = _oracle(m, ids, mask)
    enc = cabi.Encoder.from_hf(m, max_tokens=B * S)
    out = enc.forward_cls(ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()).cpu()
    _check(out, ref)
    enc.close()


@pytest.mark.parametrize("S", [300, 512])
@pytest.mark.parametrize("cls_only", [True, False])
def test_8192_row_tables_leave_short_sequences_unchanged(cabi, S, cls_only):
    """the same weights with max_position_embeddings 512 and 8192: the encoders give the same bits at S <= 512"""
    short, long_ = _model(9, max_position_embeddings=512), _model(9, max_position_embeddings=8192)
    assert all(torch.equal(a, b) for a, b in zip(short.state_dict().values(), long_.state_dict().values()))
    ids, mask = _ids(3, S, 300, S, True)
    ids, mask = ids.to(torch.int32).cuda(), mask.to(torch.int32).cuda()
    outs = []
    for m in (short, long_):
        enc = cabi.Encoder.from_hf(m, max_tokens=3 * S, cls_only=cls_only)
        outs.append((enc.forward_cls(ids, mask).cpu(), None if cls_only else enc.last_hidden(3, S).cpu()))
        enc.close()
    assert torch.equal(outs[0][0], outs[1][0])
    if not cls_only:
        assert torch.equal(outs[0][1], outs[1][1])


def test_bert_past_512_and_modernbert_past_max_pos_are_refused(cabi):
    from transformers import BertConfig, BertModel
    torch.manual_seed(0)
    bert = BertModel(BertConfig(vocab_size=300, hidden_size=128, num_hidden_layers=1, num_attention_heads=2,
                                intermediate_size=256, max_position_embeddings=1024)).eval()
    enc = cabi.Encoder.from_hf(bert, max_tokens=2048)
    ids = torch.full((1, 513), 7, dtype=torch.int32, device="cuda")
    with pytest.raises(cabi.AdaptiveB200Error, match=r"S=513 > 512 is not supported \(the reference truncates at max_length"):
        enc.forward_cls(ids)
    enc.close()
    m = _model(3, max_position_embeddings=1024)
    enc = cabi.Encoder.from_hf(m, max_tokens=4096)
    enc.forward_cls(torch.full((1, 1024), 7, dtype=torch.int32, device="cuda"))
    with pytest.raises(cabi.AdaptiveB200Error, match="max_pos=1024"):
        enc.forward_cls(torch.full((1, 1025), 7, dtype=torch.int32, device="cuda"))
    enc.close()
