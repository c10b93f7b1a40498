"""ORACLE (test infrastructure only -- never imported by the product path).

fp32 restatement of HF NomicBertModel (models/nomic_bert) and JinaEmbeddingsV3Model (models/jina_embeddings_v3) on their
own parameter names, plus the classifier's CLS row and F.normalize.  Both are the post-LN BERT block with:
  * embeddings LayerNorm(word + token_type), no position table (token_type_ids absent = 0)
  * RoPE on q and k after the projections (biases included), positions arange(S) whatever the padding, HF rotate_half
    form: t cos + (-t[32:], t[:32]) sin, with LlamaRotaryEmbedding's default-type table (attention scaling 1)
  * attention softmax(q k^T / sqrt(64) + key mask) v, then o_proj, residual, post_attention_layernorm
  * FFN: Nomic down(silu(gate_proj x) * up_proj x) (no biases), jina fc2(GELU_erf(fc1 x)) (biases), residual,
    post_mlp_layernorm
Attention runs per block of q_block queries (O(q_block S) memory), so S up to 8192 fits; it runs on the device of its inputs
(fp32; with TF32 off on a GPU).

PINNED to HF NomicBertModel / JinaEmbeddingsV3Model (eager attention) by tests/test_rotary_cpu.py.

`wrong` names one deliberately wrong rule (tests show that each one moves the embeddings far past the GPU bound):
  "no_rope"        RoPE dropped
  "gptj"           GPT-J interleaved pairs (2i, 2i + 1) instead of rotate_half
  "cumsum"         padding-aware positions cumsum(mask) - 1 instead of arange(S)
  "rope_v"         RoPE applied to v as well
  "swap_gate_up"   silu applied to up_proj instead of gate_proj (Nomic)
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle.encoder_oracle import _gelu_erf, _ln

Tensor = torch.Tensor
WRONG_RULES = ("no_rope", "gptj", "cumsum", "rope_v", "swap_gate_up")


def rope_inv_freq(theta: float, dh: int = 64) -> Tensor:
    """LlamaRotaryEmbedding's default inv_freq (fp32)"""
    return 1.0 / (theta ** (torch.arange(0, dh, 2, dtype=torch.int64).to(dtype=torch.float) / dh))


def rotary_forward_cls(
    sd: Dict[str, Tensor],
    input_ids: Tensor,                 # int64 [B, S]
    attention_mask: Optional[Tensor],  # int64 [B, S] (1 = keep) or None
    token_type_ids: Optional[Tensor] = None,
    *,
    family: str,                       # "nomic" (SwiGLU) or "jina" (GELU FFN)
    num_heads: int,
    rope_theta: float,
    ln_eps: float,
    return_hidden: bool = False,
    q_block: int = 512,
    wrong: Optional[str] = None,
):
    """Returns unit-norm CLS rows fp32 [B, H] (row 0 of every sequence, padded or not), and optionally the last hidden state."""
    assert family in ("nomic", "jina") and wrong in (None,) + WRONG_RULES
    B, S = input_ids.shape
    dev = input_ids.device
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    H = sd["embeddings.word_embeddings.weight"].shape[1]
    dh = H // num_heads
    half = dh // 2

    def lin(x, name):
        y = x @ sd[name + ".weight"].t()
        b = sd.get(name + ".bias")
        return y if b is None else y + b

    x = sd["embeddings.word_embeddings.weight"][input_ids] + sd["embeddings.token_type_embeddings.weight"][token_type_ids]
    x = _ln(x, sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"], ln_eps)

    if wrong == "cumsum":
        pos = (attention_mask.cumsum(1) - 1).clamp_min(0).float()                             # [B, S]
    else:
        pos = torch.arange(S, device=dev).float()[None].expand(B, S)
    freqs = pos[..., None] * rope_inv_freq(rope_theta, dh).to(dev)[None, None, :]           # [B, S, dh / 2]
    if wrong == "gptj":
        emb = torch.repeat_interleave(freqs, 2, dim=-1)
    else:
        emb = torch.cat((freqs, freqs), dim=-1)
    cos, sin = emb.cos()[:, None], emb.sin()[:, None]                                       # [B, 1, S, dh]

    def rot(t):
        if wrong == "no_rope":
            return t
        if wrong == "gptj":
            r = torch.stack((-t[..., 1::2], t[..., 0::2]), dim=-1).flatten(-2)
        else:
            r = torch.cat((-t[..., half:], t[..., :half]), dim=-1)
        return t * cos + r * sin

    key_ok = attention_mask.bool()[:, None, None, :]
    minval = torch.finfo(torch.float32).min
    for l in range(len([k for k in sd if k.endswith(".post_mlp_layernorm.weight")])):
        p = f"layers.{l}."
        heads = lambda t: t.view(B, S, num_heads, dh).transpose(1, 2)
        q = rot(heads(lin(x, p + "self_attn.q_proj")))
        k = rot(heads(lin(x, p + "self_attn.k_proj")))
        v = heads(lin(x, p + "self_attn.v_proj"))
        if wrong == "rope_v":
            v = rot(v)
        ctx = []
        for q0 in range(0, S, q_block):
            s = (q[:, :, q0:q0 + q_block] @ k.transpose(-1, -2)) * dh ** -0.5 + torch.where(key_ok, 0.0, minval)
            ctx.append(torch.softmax(s, dim=-1) @ v)
        ctx = torch.cat(ctx, dim=2).transpose(1, 2).reshape(B, S, H)
        x = _ln(x + lin(ctx, p + "self_attn.o_proj"), sd[p + "post_attention_layernorm.weight"],
                sd[p + "post_attention_layernorm.bias"], ln_eps)
        if family == "nomic":
            g, u = lin(x, p + "mlp.gate_proj"), lin(x, p + "mlp.up_proj")
            if wrong == "swap_gate_up":
                g, u = u, g
            f = lin(torch.nn.functional.silu(g) * u, p + "mlp.down_proj")
        else:
            f = lin(_gelu_erf(lin(x, p + "mlp.fc1")), p + "mlp.fc2")
        x = _ln(x + f, sd[p + "post_mlp_layernorm.weight"], sd[p + "post_mlp_layernorm.bias"], ln_eps)
    cls = x[:, 0, :]
    unit = cls / cls.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if return_hidden:
        return unit, x
    return unit


def rotary_forward_for(config, sd, input_ids, attention_mask, token_type_ids=None, **kw):
    """rotary_forward_cls with family, heads, theta and eps read from an HF NomicBertConfig / JinaEmbeddingsV3Config or its
    to_dict()"""
    c = config if isinstance(config, dict) else config.to_dict()
    return rotary_forward_cls(sd, input_ids, attention_mask, token_type_ids,
                              family="nomic" if c["model_type"] == "nomic_bert" else "jina",
                              num_heads=c["num_attention_heads"], rope_theta=float(c["rope_parameters"]["rope_theta"]),
                              ln_eps=c["layer_norm_eps"], **kw)
