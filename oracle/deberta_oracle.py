"""ORACLE (test infrastructure only -- never imported by the product path).

CPU fp32 restatement of HF DebertaV2Model.forward (third-party `transformers`, models/deberta_v2/modeling_deberta_v2.py),
the encoder of microsoft/deberta-v3-xsmall / -small / -base / -large and mdeberta-v3-base, followed by the reference's CLS
row + F.normalize (classifier.py:1272-1275):

    embeddings   word (+ absolute position when position_biased_input, + token type when type_vocab_size > 0),
                 LayerNorm, times the mask                                                    (DebertaV2Embeddings)
    layer        post-LN BERT block with exact-erf GELU; disentangled attention with the mask mask_i mask_j:
                     s(i, j) = (q_i . k_j + q_i . PosK[c2p(i, j)] + k_j . PosQ[p2c(j, i)]) / sqrt(3 dh)
                 c2p(i, j) = clamp(bucket(i - j) + span, 0, 2 span - 1) and p2c(j, i) = clamp(-bucket(j - i) + span, ...),
                 both gathered as HF gathers them (p2c on the key rows, then transposed)
    positions    rel_embeddings (LayerNorm-ed under norm_rel_ebd = layer_norm) through key_proj / query_proj
                 (share_att_key) or pos_key_proj / pos_query_proj; bucket = make_log_bucket_position

Restated on DeBERTa's own parameter names and PINNED against the installed HF module by tests/test_deberta_cpu.py (last
hidden state and unit CLS rows to 1e-6, padded batches, log buckets, both share_att_key settings).  The keyword flags
mutate one rule each so that the tests can show how far a wrong kernel would move the embeddings.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle.encoder_oracle import _gelu_erf, _ln

Tensor = torch.Tensor


def deberta_bucket(rel: Tensor, bucket_size: int, max_position: int) -> Tensor:
    """make_log_bucket_position: identity for |r| <= bucket_size / 2, log-spaced up to max_position beyond (fp32 log)"""
    sign = torch.sign(rel)
    mid = bucket_size // 2
    abs_pos = torch.where((rel < mid) & (rel > -mid), torch.tensor(mid - 1).type_as(rel), torch.abs(rel))
    log_pos = torch.ceil(torch.log(abs_pos / mid) / torch.log(torch.tensor((max_position - 1) / mid)) * (mid - 1)) + mid
    return torch.where(abs_pos <= mid, rel.type_as(log_pos), log_pos * sign).to(torch.long)


def deberta_spans(c):
    """(position_buckets, max_relative_positions, span) of a DebertaV2Config, with HF's defaults"""
    buckets = getattr(c, "position_buckets", -1)
    max_rel = getattr(c, "max_relative_positions", -1)
    if max_rel < 1:
        max_rel = c.max_position_embeddings
    return buckets, max_rel, (buckets if buckets > 0 else max_rel)


def deberta_relative_position(S: int, c) -> Tensor:
    """[S, S] bucket(i - j) of query i, key j (build_relative_position)"""
    buckets, max_rel, _ = deberta_spans(c)
    pos = torch.arange(S, dtype=torch.long)
    rel = pos[:, None] - pos[None, :]
    if buckets > 0 and max_rel > 0:
        rel = deberta_bucket(rel, buckets, max_rel)
    return rel


def deberta_forward_cls(sd: Dict[str, Tensor], input_ids: Tensor, attention_mask: Optional[Tensor], c, *,
                        return_hidden: bool = False, c2p: bool = True, p2c: bool = True, p2c_transposed: bool = True,
                        p2c_index_of_r: bool = False, scale_factor: int = 3):
    """Unit-norm CLS rows fp32 [B, H] (and optionally the last hidden state [B, S, H]) from an HF DebertaV2Model state dict
    and its config.  Mutations: c2p / p2c False drop a term; p2c_transposed False leaves the p2c product untransposed
    (key j's row used for query j); p2c_index_of_r gathers p2c at -bucket(i - j) instead of -bucket(j - i); scale_factor 1
    divides by sqrt(dh) instead of sqrt(3 dh)."""
    B, S = input_ids.shape
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)
    m = attention_mask.to(torch.float32)
    heads = c.num_attention_heads

    def lin(x, prefix):
        return x @ sd[prefix + ".weight"].t() + sd[prefix + ".bias"]

    x = sd["embeddings.word_embeddings.weight"][input_ids]
    if getattr(c, "position_biased_input", True):
        x = x + sd["embeddings.position_embeddings.weight"][torch.arange(S)][None]
    if c.type_vocab_size > 0:
        x = x + sd["embeddings.token_type_embeddings.weight"][0]
    x = _ln(x, sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"], c.layer_norm_eps) * m[..., None]

    H = x.shape[-1]
    dh = H // heads
    _, _, span = deberta_spans(c)
    rel = sd["encoder.rel_embeddings.weight"]
    if "layer_norm" in [t.strip() for t in getattr(c, "norm_rel_ebd", "none").lower().split("|")]:
        rel = _ln(rel, sd["encoder.LayerNorm.weight"], sd["encoder.LayerNorm.bias"], c.layer_norm_eps)
    rel = rel[:2 * span]
    rp = deberta_relative_position(S, c)                              # [S, S] bucket(i - j)
    c2p_idx = torch.clamp(rp + span, 0, 2 * span - 1)                 # [i, j]
    p2c_idx = torch.clamp((rp if p2c_index_of_r else -rp) + span, 0, 2 * span - 1)   # [j, i] HF: -bucket(j - i)
    scale = torch.sqrt(torch.tensor(float(dh) * scale_factor))
    keep = (m[:, None, :, None] * m[:, None, None, :]).bool()         # [B, 1, S, S] mask_i mask_j

    L = 0
    while f"encoder.layer.{L}.attention.self.query_proj.weight" in sd:
        L += 1
    for l in range(L):
        p = f"encoder.layer.{l}."
        sp = p + "attention.self."
        x2 = x.reshape(B * S, H)
        q = lin(x2, sp + "query_proj").view(B, S, heads, dh).transpose(1, 2)
        k = lin(x2, sp + "key_proj").view(B, S, heads, dh).transpose(1, 2)
        v = lin(x2, sp + "value_proj").view(B, S, heads, dh).transpose(1, 2)
        kq = ("key_proj", "query_proj") if getattr(c, "share_att_key", False) else ("pos_key_proj", "pos_query_proj")
        pos_k = lin(rel, sp + kq[0]).view(2 * span, heads, dh).transpose(0, 1)     # [heads, 2 span, dh]
        pos_q = lin(rel, sp + kq[1]).view(2 * span, heads, dh).transpose(0, 1)
        scores = q @ (k / scale).transpose(-1, -2)
        if c2p:
            c2p_att = q @ pos_k.transpose(-1, -2)                     # [B, heads, S (i), 2 span]
            scores = scores + torch.gather(c2p_att, -1, c2p_idx.expand(B, heads, S, S)) / scale
        if p2c:
            p2c_att = k @ pos_q.transpose(-1, -2)                     # [B, heads, S (j), 2 span]
            g = torch.gather(p2c_att, -1, p2c_idx.expand(B, heads, S, S))
            scores = scores + (g.transpose(-1, -2) if p2c_transposed else g) / scale
        scores = scores.masked_fill(~keep, torch.finfo(torch.float32).min)
        ctx = (torch.softmax(scores, dim=-1) @ v).transpose(1, 2).reshape(B * S, H)
        a = lin(ctx, p + "attention.output.dense")
        x2 = _ln(a + x2, sd[p + "attention.output.LayerNorm.weight"], sd[p + "attention.output.LayerNorm.bias"],
                 c.layer_norm_eps)
        h = _gelu_erf(lin(x2, p + "intermediate.dense"))
        o = lin(h, p + "output.dense")
        x2 = _ln(o + x2, sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"], c.layer_norm_eps)
        x = x2.view(B, S, H)

    cls = x[:, 0, :]
    unit = cls / cls.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if return_hidden:
        return unit, x
    return unit
