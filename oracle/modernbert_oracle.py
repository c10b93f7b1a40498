"""ORACLE (test infrastructure only -- never imported by the product path).

CPU fp32 restatement of the encoder stage E for ModernBERT checkpoints:

    AdaptiveClassifier._get_embeddings            /root/reference/src/adaptive_classifier/classifier.py:1249-1282
      -> HF ModernBertModel.forward (third-party `transformers`, 5.5.0 installed: models/modernbert/modeling_modernbert.py)
      -> last_hidden_state[:, 0, :]                 classifier.py:1272
      -> F.normalize(p=2, dim=1)  (eps 1e-12)       classifier.py:1275

Restated from the published algorithm (ModernBertEmbeddings, pre-LN ModernBertEncoderLayer with layer 0's Identity
attn_norm, ModernBertRotaryEmbedding, eager attention with the bidirectional sliding-window mask, GeGLU ModernBertMLP,
final_norm) and PINNED against the installed HF module by tests/test_modernbert_cpu.py (1e-5 on CLS rows and hidden states,
padded batches, sliding band edge, both RoPE theta) and against the reference's own _get_embeddings on
tests/golden/golden_classifier_modernbert*.npz (oracle/make_golden_encoders.py modernbert).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle.encoder_oracle import _gelu_erf, _ln

Tensor = torch.Tensor


def rope_cos_sin(theta: float, S: int, dh: int):
    """HF ModernBertRotaryEmbedding (default rope type): fp32 inv_freq, freqs = inv_freq (x) positions, emb = (freqs, freqs)"""
    inv_freq = 1.0 / (theta ** (torch.arange(0, dh, 2, dtype=torch.int64).to(dtype=torch.float) / dh))
    freqs = (inv_freq[None, :, None] @ torch.arange(S).float()[None, None, :]).transpose(1, 2)[0]
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos(), emb.sin()


def modernbert_forward_cls(
    sd: Dict[str, Tensor],
    input_ids: Tensor,                 # int64 [B, S]
    attention_mask: Optional[Tensor],  # int64 [B, S] (1 = keep) or None
    *,
    num_heads: int,
    layer_sliding,                     # per layer: True = sliding_attention, False = full_attention
    sliding_window: int,               # half-window: a sliding layer's query i sees keys |i - j| <= sliding_window
    rope_theta=(160000.0, 10000.0),    # (full_attention, sliding_attention)
    norm_eps: float = 1e-5,
    return_hidden: bool = False,
):
    """HF ModernBertModel.forward (eager attention, no biases) followed by the CLS row and F.normalize.
    Returns unit-norm CLS rows fp32 [B, H] (and optionally the last hidden state)."""
    B, S = input_ids.shape
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)
    H = sd["embeddings.tok_embeddings.weight"].shape[1]
    dh = H // num_heads
    zeros = torch.zeros(H)

    def ln(x, name):
        return _ln(x, sd[name], zeros, norm_eps)

    x = ln(sd["embeddings.tok_embeddings.weight"][input_ids], "embeddings.norm.weight")      # ModernBertEmbeddings
    key_ok = attention_mask.bool()[:, None, None, :]
    i = torch.arange(S)
    band = (i[:, None] - i[None, :]).abs() <= sliding_window
    minval = torch.finfo(torch.float32).min
    rope = {False: rope_cos_sin(rope_theta[0], S, dh), True: rope_cos_sin(rope_theta[1], S, dh)}

    def rot(t, cos, sin):
        # apply_rotary_pos_emb: t cos + rotate_half(t) sin, rotate_half = (-t[d/2:], t[:d/2])
        return t * cos + torch.cat((-t[..., dh // 2:], t[..., : dh // 2]), dim=-1) * sin

    for l, sliding in enumerate(layer_sliding):
        p = f"layers.{l}."
        a = x if l == 0 else ln(x, p + "attn_norm.weight")                                   # layer 0: Identity
        qkv = (a @ sd[p + "attn.Wqkv.weight"].t()).view(B, S, 3, num_heads, dh)
        q, k, v = (t.transpose(1, 2) for t in qkv.unbind(dim=2))
        cos, sin = rope[bool(sliding)]
        q, k = rot(q, cos, sin), rot(k, cos, sin)
        ok = key_ok & band if sliding else key_ok
        scores = (q @ k.transpose(-1, -2)) * dh ** -0.5 + torch.where(ok, 0.0, minval)
        ctx = (torch.softmax(scores, dim=-1) @ v).transpose(1, 2).reshape(B, S, H)
        x = x + ctx @ sd[p + "attn.Wo.weight"].t()
        inp, gate = (ln(x, p + "mlp_norm.weight") @ sd[p + "mlp.Wi.weight"].t()).chunk(2, dim=-1)
        x = x + (_gelu_erf(inp) * gate) @ sd[p + "mlp.Wo.weight"].t()
    x = ln(x, "final_norm.weight")
    cls = x[:, 0, :]
    unit = cls / cls.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if return_hidden:
        return unit, x
    return unit


def make_modernbert(seed: int = 1234, **cfg_over):
    """Seeded random-init ModernBertModel (eager attention, fp32, eval).  Returns (state_dict, config, model)."""
    from transformers import ModernBertConfig, ModernBertModel

    torch.manual_seed(seed)
    cfg = ModernBertConfig(**cfg_over)
    cfg._attn_implementation = "eager"
    m = ModernBertModel(cfg)
    m.eval()
    sd = {k: v.detach().clone().float() for k, v in m.state_dict().items()}
    return sd, cfg, m
