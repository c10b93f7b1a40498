"""ORACLE (test infrastructure only -- never imported by the product path).

Query-block form of oracle/modernbert_oracle.py for long ModernBERT inputs (S up to 8192).  modernbert_forward_cls there
builds B x heads x S x S scores, 3.2 GB per sequence at ModernBERT-base and S = 8192.  This form computes attention per
block of queries and, in sliding layers, only over that block's band of keys [q0 - w, q0 + n - 1 + w]: O(n S) memory.
Everything else (embeddings, pre-LN blocks, RoPE, GeGLU, final_norm, CLS row, F.normalize) is the same restatement.

A query row with no valid key in its band (only a masked row can have none: a valid row always sees itself) averages the
band here instead of every key as in HF; such rows are never attended to by a valid row, and tests compare valid rows.

PINNED to modernbert_oracle.modernbert_forward_cls at small S and to HF ModernBertModel (eager) at S > 512 by
tests/test_modernbert_long_cpu.py.  Runs on the device of its inputs (fp32; with TF32 off on a GPU).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle.encoder_oracle import _gelu_erf, _ln
from oracle.modernbert_oracle import rope_cos_sin

Tensor = torch.Tensor


def modernbert_forward_cls_blocked(
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
    q_block: int = 128,                # queries per attention block
):
    """modernbert_forward_cls with attention computed per block of q_block queries (band-limited in sliding layers).
    Returns unit-norm CLS rows fp32 [B, H] (and optionally the last hidden state)."""
    B, S = input_ids.shape
    dev = input_ids.device
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)
    H = sd["embeddings.tok_embeddings.weight"].shape[1]
    dh = H // num_heads
    zeros = torch.zeros(H, device=dev)
    w = sliding_window

    def ln(x, name):
        return _ln(x, sd[name], zeros, norm_eps)

    x = ln(sd["embeddings.tok_embeddings.weight"][input_ids], "embeddings.norm.weight")      # ModernBertEmbeddings
    key_ok = attention_mask.bool()[:, None, None, :]
    i = torch.arange(S, device=dev)
    minval = torch.finfo(torch.float32).min
    rope = {s: tuple(t.to(dev) for t in rope_cos_sin(rope_theta[int(s)], S, dh)) for s in (False, True)}

    def rot(t, cos, sin):
        # apply_rotary_pos_emb: t cos + rotate_half(t) sin, rotate_half = (-t[d/2:], t[:d/2])
        return t * cos + torch.cat((-t[..., dh // 2:], t[..., : dh // 2]), dim=-1) * sin

    def attend(q, k, v, sliding, q0, q1):
        k0, k1 = (max(0, q0 - w), min(S, q1 + w)) if sliding else (0, S)
        ok = key_ok[..., k0:k1]
        if sliding:
            ok = ok & ((i[q0:q1, None] - i[None, k0:k1]).abs() <= w)
        scores = (q[:, :, q0:q1] @ k[:, :, k0:k1].transpose(-1, -2)) * dh ** -0.5 + torch.where(ok, 0.0, minval)
        return torch.softmax(scores, dim=-1) @ v[:, :, k0:k1]

    for l, sliding in enumerate(layer_sliding):
        p = f"layers.{l}."
        a = x if l == 0 else ln(x, p + "attn_norm.weight")                                   # layer 0: Identity
        qkv = (a @ sd[p + "attn.Wqkv.weight"].t()).view(B, S, 3, num_heads, dh)
        q, k, v = (t.transpose(1, 2) for t in qkv.unbind(dim=2))
        cos, sin = rope[bool(sliding)]
        q, k = rot(q, cos, sin), rot(k, cos, sin)
        ctx = torch.cat([attend(q, k, v, sliding, q0, min(S, q0 + q_block)) for q0 in range(0, S, q_block)], dim=2)
        x = x + ctx.transpose(1, 2).reshape(B, S, H) @ sd[p + "attn.Wo.weight"].t()
        inp, gate = (ln(x, p + "mlp_norm.weight") @ sd[p + "mlp.Wi.weight"].t()).chunk(2, dim=-1)
        x = x + (_gelu_erf(inp) * gate) @ sd[p + "mlp.Wo.weight"].t()
    x = ln(x, "final_norm.weight")
    cls = x[:, 0, :]
    unit = cls / cls.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if return_hidden:
        return unit, x
    return unit
