"""ORACLE (test infrastructure only -- never imported by the product path).

fp32 restatement of HF EuroBertModel (models/eurobert) on its own parameter names, plus the classifier's CLS row and
F.normalize.  The block is Llama's decoder layer without the causal mask:
  * h = embed_tokens(ids): no scale, no embedding norm
  * per layer  h = h + o_proj(attn(RoPE(q_proj(n)), RoPE(k_proj(n)), v_proj(n))),  n = input_layernorm(h)
               h = h + down_proj(silu(gate_proj(m)) * up_proj(m)),                 m = post_attention_layernorm(h)
  * out = norm(h); every norm is EuroBertRMSNorm: weight * (x * rsqrt(mean(x^2) + eps))
  * RoPE in rotate_half form at positions arange(S) whatever the padding (default rope type, attention scaling 1)
  * attention softmax(q k^T / sqrt(64) + key mask) v; k and v of num_key_value_heads heads, query head h reading kv head
    h // (heads / kv_heads) (repeat_kv)
Attention runs per block of q_block queries (O(q_block S) memory), so S up to 8192 fits; it runs on the device of its inputs
(fp32; with TF32 off on a GPU).

PINNED to HF EuroBertModel (eager attention) by tests/test_eurobert_cpu.py.

`wrong` names one deliberately wrong rule (tests show that each one moves the embeddings far past the GPU bound):
  "layernorm"        LayerNorm (mean and variance, no bias) in place of every RMSNorm
  "rms_centred"      RMSNorm that subtracts the row mean from x but keeps the uncentred RMS
  "layer0_identity"  layer 0's input_layernorm treated as the identity (ModernBERT's layer-0 rule)
  "no_final_norm"    the final norm skipped
  "no_rope"          RoPE dropped
  "cumsum"           padding-aware positions cumsum(mask) - 1 instead of arange(S)
  "kv_tiled"         kv heads in repeat (tiled) order, query head h reading kv head h % kv_heads
  "swap_gate_up"     silu applied to up_proj instead of gate_proj
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle.rotary_oracle import rope_inv_freq

Tensor = torch.Tensor
WRONG_RULES = ("layernorm", "rms_centred", "layer0_identity", "no_final_norm", "no_rope", "cumsum", "kv_tiled",
               "swap_gate_up")


def _rms(x: Tensor, w: Tensor, eps: float, wrong: Optional[str]) -> Tensor:
    if wrong == "layernorm":
        return torch.nn.functional.layer_norm(x, x.shape[-1:], w, None, eps)
    var = x.pow(2).mean(-1, keepdim=True)
    if wrong == "rms_centred":
        x = x - x.mean(-1, keepdim=True)
    return w * (x * torch.rsqrt(var + eps))


def eurobert_forward_cls(
    sd: Dict[str, Tensor],
    input_ids: Tensor,                 # int64 [B, S]
    attention_mask: Optional[Tensor],  # int64 [B, S] (1 = keep) or None
    *,
    num_heads: int,
    num_kv_heads: int,
    rope_theta: float,
    eps: float,
    return_hidden: bool = False,
    q_block: int = 512,
    wrong: Optional[str] = None,
):
    """Returns unit-norm CLS rows fp32 [B, H] (row 0 of every sequence, padded or not), and optionally the last hidden state."""
    assert wrong in (None,) + WRONG_RULES
    B, S = input_ids.shape
    dev = input_ids.device
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)
    H = sd["embed_tokens.weight"].shape[1]
    dh = H // num_heads
    half, rep = dh // 2, num_heads // num_kv_heads
    norm_wrong = wrong if wrong in ("layernorm", "rms_centred") else None

    def lin(x, name):
        y = x @ sd[name + ".weight"].t()
        b = sd.get(name + ".bias")
        return y if b is None else y + b

    x = sd["embed_tokens.weight"][input_ids]
    if wrong == "cumsum":
        pos = (attention_mask.cumsum(1) - 1).clamp_min(0).float()                             # [B, S]
    else:
        pos = torch.arange(S, device=dev).float()[None].expand(B, S)
    freqs = pos[..., None] * rope_inv_freq(rope_theta, dh).to(dev)[None, None, :]           # [B, S, dh / 2]
    emb = torch.cat((freqs, freqs), dim=-1)
    cos, sin = emb.cos()[:, None], emb.sin()[:, None]                                       # [B, 1, S, dh]

    def rot(t):
        if wrong == "no_rope":
            return t
        return t * cos + torch.cat((-t[..., half:], t[..., :half]), dim=-1) * sin

    def kv_expand(t):                                                                       # [B, kv, S, dh] -> [B, heads, S, dh]
        if wrong == "kv_tiled":
            return t.repeat(1, rep, 1, 1)
        return t.repeat_interleave(rep, dim=1)

    key_ok = attention_mask.bool()[:, None, None, :]
    minval = torch.finfo(torch.float32).min
    layers = len([k for k in sd if k.endswith(".input_layernorm.weight")])
    for l in range(layers):
        p = f"layers.{l}."
        n = x if (l == 0 and wrong == "layer0_identity") else _rms(x, sd[p + "input_layernorm.weight"], eps, norm_wrong)
        heads = lambda t: t.view(B, S, -1, dh).transpose(1, 2)
        q = rot(heads(lin(n, p + "self_attn.q_proj")))
        k = kv_expand(rot(heads(lin(n, p + "self_attn.k_proj"))))
        v = kv_expand(heads(lin(n, p + "self_attn.v_proj")))
        ctx = []
        for q0 in range(0, S, q_block):
            s = (q[:, :, q0:q0 + q_block] @ k.transpose(-1, -2)) * dh ** -0.5 + torch.where(key_ok, 0.0, minval)
            ctx.append(torch.softmax(s, dim=-1) @ v)
        ctx = torch.cat(ctx, dim=2).transpose(1, 2).reshape(B, S, H)
        x = x + lin(ctx, p + "self_attn.o_proj")
        m = _rms(x, sd[p + "post_attention_layernorm.weight"], eps, norm_wrong)
        g, u = lin(m, p + "mlp.gate_proj"), lin(m, p + "mlp.up_proj")
        if wrong == "swap_gate_up":
            g, u = u, g
        x = x + lin(torch.nn.functional.silu(g) * u, p + "mlp.down_proj")
    if wrong != "no_final_norm":
        x = _rms(x, sd["norm.weight"], eps, norm_wrong)
    cls = x[:, 0, :]
    unit = cls / cls.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if return_hidden:
        return unit, x
    return unit


SPECIALS = ["<|begin_of_text|>", "<|end_of_text|>", "<|mask|>", "<unk>"]     # ids 0..3: bos, eos = pad, mask, unk


def eurobert_tokenizer(words):
    """PreTrainedTokenizerFast over SPECIALS + words (one id per whitespace-separated word) that, as the real EuroBERT
    tokenizer does, wraps a text in <|begin_of_text|> ... <|end_of_text|>, pads with <|end_of_text|> and returns input_ids
    and attention_mask only (EuroBertModel.forward takes no token_type_ids)"""
    from tokenizers import Tokenizer, models, pre_tokenizers, processors
    from transformers import PreTrainedTokenizerFast
    vocab = {w: i for i, w in enumerate(SPECIALS + list(words))}
    tok = Tokenizer(models.WordLevel(vocab=vocab, unk_token="<unk>"))
    tok.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    tok.post_processor = processors.TemplateProcessing(
        single="<|begin_of_text|> $A <|end_of_text|>", special_tokens=[("<|begin_of_text|>", 0), ("<|end_of_text|>", 1)])
    return PreTrainedTokenizerFast(tokenizer_object=tok, bos_token="<|begin_of_text|>", eos_token="<|end_of_text|>",
                                   pad_token="<|end_of_text|>", mask_token="<|mask|>", unk_token="<unk>",
                                   model_input_names=["input_ids", "attention_mask"])


def eurobert_forward_for(config, sd, input_ids, attention_mask, **kw):
    """eurobert_forward_cls with heads, kv heads, theta and eps read from an HF EuroBertConfig or its to_dict()"""
    c = config if isinstance(config, dict) else config.to_dict()
    heads = c["num_attention_heads"]
    return eurobert_forward_cls(sd, input_ids, attention_mask, num_heads=heads,
                                num_kv_heads=c.get("num_key_value_heads") or heads,
                                rope_theta=float(c["rope_parameters"]["rope_theta"]), eps=c["rms_norm_eps"], **kw)
