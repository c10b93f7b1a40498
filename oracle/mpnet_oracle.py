"""ORACLE (test infrastructure only -- never imported by the product path).

CPU fp32 restatement of HF MPNetModel.forward (third-party `transformers`, models/mpnet/modeling_mpnet.py), the encoder of
sentence-transformers/all-mpnet-base-v2, multi-qa-mpnet-base-* and paraphrase-mpnet-base-v2, followed by the reference's
CLS row + F.normalize (classifier.py:1272-1275):

    embeddings   word + position (RoBERTa's rule, padding_idx 1), no token types, LayerNorm      (MPNetEmbeddings)
    layer        post-LN BERT block with exact-erf GELU; the attention scores get, after the 1/sqrt(d) scale and before
                 the mask, the relative position bias of MPNetEncoder.compute_position_bias
    bias         relative_attention_bias.weight[bucket(key - query), head], T5's bidirectional bucketing with 32 buckets
                 and max_distance 128 (relative_position_bucket; `num_buckets=32` is fixed in HF's forward call)

Restated from the published algorithm on MPNet's own parameter names and PINNED against the installed HF module by
tests/test_mpnet_cpu.py (last hidden state and unit CLS rows to 1e-6, padded batches, distances past the saturation).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from oracle.encoder_oracle import _gelu_erf, _ln

Tensor = torch.Tensor


def mpnet_position_bias(weight: Tensor, S: int) -> Tensor:
    """[heads, S, S] bias of (head, query, key): weight[bucket(key - query)], weight = [32, heads].  Keys after the query take
    buckets 16..31; distance n < 8 is its own bucket, farther ones 8 + floor(log(n / 8) / log(16) * 8), at most 15 (fp32)."""
    pos = torch.arange(S, dtype=torch.long)
    n = pos[:, None] - pos[None, :]                      # query - key
    half = 16
    bucket = (n < 0).to(torch.long) * half
    n = n.abs()
    far = 8 + (torch.log(n.float() / 8) / math.log(128 / 8) * (half - 8)).to(torch.long)
    far = torch.clamp(far, max=half - 1)
    bucket = bucket + torch.where(n < 8, n, far)
    return weight[bucket].permute(2, 0, 1).contiguous()


def mpnet_forward_cls(sd: Dict[str, Tensor], input_ids: Tensor, attention_mask: Optional[Tensor], *, num_heads: int,
                      ln_eps: float, return_hidden: bool = False, bias_scale: float = 1.0):
    """Unit-norm CLS rows fp32 [B, H] (and optionally the last hidden state [B, S, H]) from an HF MPNetModel state dict;
    bias_scale 0 drops the relative position bias (the tests' sensitivity check)."""
    B, S = input_ids.shape
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)

    def lin(x, prefix):
        return x @ sd[prefix + ".weight"].t() + sd[prefix + ".bias"]

    # MPNetEmbeddings: position ids = cumsum(ids != 1) * (ids != 1) + 1
    nonpad = (input_ids != 1).to(torch.int64)
    pos = torch.cumsum(nonpad, dim=1) * nonpad + 1
    x = sd["embeddings.word_embeddings.weight"][input_ids] + sd["embeddings.position_embeddings.weight"][pos]
    x = _ln(x, sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"], ln_eps)

    H = x.shape[-1]
    dh = H // num_heads
    scale = dh ** -0.5
    bias = mpnet_position_bias(sd["encoder.relative_attention_bias.weight"], S) * bias_scale
    addmask = (1.0 - attention_mask.to(torch.float32))[:, None, None, :] * torch.finfo(torch.float32).min

    L = 0
    while f"encoder.layer.{L}.attention.attn.q.weight" in sd:
        L += 1
    for l in range(L):
        p = f"encoder.layer.{l}."
        x2 = x.reshape(B * S, H)
        q = lin(x2, p + "attention.attn.q").view(B, S, num_heads, dh).transpose(1, 2)
        k = lin(x2, p + "attention.attn.k").view(B, S, num_heads, dh).transpose(1, 2)
        v = lin(x2, p + "attention.attn.v").view(B, S, num_heads, dh).transpose(1, 2)
        scores = (q @ k.transpose(-1, -2)) * scale + bias + addmask
        ctx = (torch.softmax(scores, dim=-1) @ v).transpose(1, 2).reshape(B * S, H)
        a = lin(ctx, p + "attention.attn.o")
        x2 = _ln(a + x2, sd[p + "attention.LayerNorm.weight"], sd[p + "attention.LayerNorm.bias"], ln_eps)
        h = _gelu_erf(lin(x2, p + "intermediate.dense"))
        o = lin(h, p + "output.dense")
        x2 = _ln(o + x2, sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"], ln_eps)
        x = x2.view(B, S, H)

    cls = x[:, 0, :]
    unit = cls / cls.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if return_hidden:
        return unit, x
    return unit
