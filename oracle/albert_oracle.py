"""ORACLE (test infrastructure only -- never imported by the product path).

CPU fp32 restatement of HF AlbertModel.forward (models/albert/modeling_albert.py) and ElectraModel.forward
(models/electra/modeling_electra.py), the encoders of albert-base / large v1 / v2 and the ELECTRA discriminators, on their
own parameter names, followed by the reference's CLS row + F.normalize (classifier.py:1272-1275):

    embeddings   (word + token type) + absolute position at width embedding_size, LayerNorm at that width, times nothing
                 (AlbertEmbeddings / ElectraEmbeddings; the mask enters the attention only)
    projection   ALBERT encoder.embedding_hidden_mapping_in (always), ELECTRA embeddings_project (when embedding_size !=
                 hidden_size): a linear layer embedding_size -> hidden_size; its output is layer 0's input as it is
    layers       ALBERT: effective layer i runs group int(i / (num_hidden_layers / num_hidden_groups)), each group its
                 inner_group_num layers in order; ELECTRA: encoder.layer.l
    block        the post-LN BERT block with the configured GELU: "gelu" exact erf, "gelu_new" / "gelu_pytorch_tanh" tanh

PINNED against the installed HF modules by tests/test_albert_cpu.py (last hidden state and unit CLS rows to 1e-6, padded
batches, shared and grouped ALBERT layers, ELECTRA with and without the projection).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from oracle.encoder_oracle import _gelu_erf, _ln

Tensor = torch.Tensor


def gelu_tanh(x: Tensor) -> Tensor:
    # HF NewGELUActivation ("gelu_new"); GELUTanh ("gelu_pytorch_tanh") is the same function
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


ACTS = {"gelu": _gelu_erf, "gelu_new": gelu_tanh, "gelu_pytorch_tanh": gelu_tanh}


def albert_layer_prefixes(c) -> list:
    """parameter prefix of every effective layer of an ALBERT encoder (HF AlbertTransformer's group walk)"""
    out = []
    for i in range(c.num_hidden_layers):
        g = int(i / (c.num_hidden_layers / c.num_hidden_groups))
        out += [f"encoder.albert_layer_groups.{g}.albert_layers.{j}." for j in range(c.inner_group_num)]
    return out


def _block(sd, p, names, x2, addmask, B, S, heads, act, eps):
    """one post-LN block on x2 [B*S, H]; names = (query, key, value, attn out, attn LN, ffn in, ffn out, out LN)"""
    def lin(x, prefix):
        return x @ sd[p + prefix + ".weight"].t() + sd[p + prefix + ".bias"]

    H = x2.shape[-1]
    dh = H // heads
    q = lin(x2, names[0]).view(B, S, heads, dh).transpose(1, 2)
    k = lin(x2, names[1]).view(B, S, heads, dh).transpose(1, 2)
    v = lin(x2, names[2]).view(B, S, heads, dh).transpose(1, 2)
    probs = torch.softmax((q @ k.transpose(-1, -2)) * dh ** -0.5 + addmask, dim=-1)
    ctx = (probs @ v).transpose(1, 2).reshape(B * S, H)
    a = lin(ctx, names[3])
    x2 = _ln(a + x2, sd[p + names[4] + ".weight"], sd[p + names[4] + ".bias"], eps)
    h = act(lin(x2, names[5]))
    o = lin(h, names[6])
    return _ln(o + x2, sd[p + names[7] + ".weight"], sd[p + names[7] + ".bias"], eps)


ALBERT_NAMES = ("attention.query", "attention.key", "attention.value", "attention.dense", "attention.LayerNorm", "ffn",
                "ffn_output", "full_layer_layer_norm")
ELECTRA_NAMES = ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense",
                 "attention.output.LayerNorm", "intermediate.dense", "output.dense", "output.LayerNorm")


def factorized_forward_cls(sd: Dict[str, Tensor], input_ids: Tensor, attention_mask: Optional[Tensor], c, *,
                           token_type_ids: Optional[Tensor] = None, return_hidden: bool = False, act: Optional[str] = None):
    """Unit-norm CLS rows fp32 [B, H] (and optionally the last hidden state [B, S, H]) from an HF AlbertModel or ElectraModel
    state dict and its config (c.model_type "albert" / "electra").  act overrides c.hidden_act (the tests use it to show
    that the wrong GELU is told apart)."""
    B, S = input_ids.shape
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    albert = c.model_type == "albert"
    x = sd["embeddings.word_embeddings.weight"][input_ids] + sd["embeddings.token_type_embeddings.weight"][token_type_ids]
    x = x + sd["embeddings.position_embeddings.weight"][torch.arange(S)][None]
    x = _ln(x, sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"], c.layer_norm_eps)
    proj = "encoder.embedding_hidden_mapping_in" if albert else "embeddings_project"
    if proj + ".weight" in sd:
        x = x @ sd[proj + ".weight"].t() + sd[proj + ".bias"]
    H = x.shape[-1]
    addmask = (1.0 - attention_mask.to(torch.float32))[:, None, None, :] * torch.finfo(torch.float32).min
    fn = ACTS[act or c.hidden_act]
    if albert:
        prefixes, names = albert_layer_prefixes(c), ALBERT_NAMES
    else:
        prefixes, names = [f"encoder.layer.{l}." for l in range(c.num_hidden_layers)], ELECTRA_NAMES
    x2 = x.reshape(B * S, H)
    for p in prefixes:
        x2 = _block(sd, p, names, x2, addmask, B, S, c.num_attention_heads, fn, c.layer_norm_eps)
    x = x2.view(B, S, H)
    cls = x[:, 0, :]
    unit = cls / cls.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if return_hidden:
        return unit, x
    return unit
