"""ORACLE (test infrastructure only -- never imported by the product path).

CPU fp32 restatement of the encoder stage E of the hot path:

    AdaptiveClassifier._get_embeddings            /root/reference/src/adaptive_classifier/classifier.py:1249-1282
      -> HF BertModel.forward / RobertaModel.forward (third-party `transformers`, 5.5.0 installed;
         the reference pins only `transformers>=4.30.0`, requirements.txt:2)
      -> last_hidden_state[:, 0, :]                 classifier.py:1272
      -> F.normalize(p=2, dim=1)  (eps 1e-12)       classifier.py:1275

The arithmetic lives in the third-party dependency, so it is restated here from its published
algorithm (HF `models/bert/modeling_bert.py`: embeddings :53-113, self-attention :143-207,
attention output + LayerNorm :287-298, FFN :330-356; `models/roberta/modeling_roberta.py:146-159`
for RoBERTa position ids) and PINNED against the installed HF module itself
(tests/test_oracle_cpu.py::test_encoder_oracle_matches_hf, max abs diff < 2e-6 on unit CLS rows).

`round_fn` lets the precision study (oracle/precision_study.py) emulate tensor-core operand
rounding (bf16 / tf32 / split-bf16) to choose the tensor-core operand format per GEMM.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional

import torch

Tensor = torch.Tensor


def _ln(x: Tensor, w: Tensor, b: Tensor, eps: float) -> Tensor:
    # torch.nn.LayerNorm: biased variance, eps inside the sqrt
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w + b


def _gelu_erf(x: Tensor) -> Tensor:
    # HF ACT2FN["gelu"] == exact erf GELU (modeling_bert.py:330-340)
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def encoder_forward_cls(
    sd: Dict[str, Tensor],
    input_ids: Tensor,                 # int64 [B, S]
    attention_mask: Optional[Tensor],  # int64 [B, S] (1 = keep) or None
    *,
    arch: str = "bert",                # "bert" | "roberta"
    num_heads: int = 12,
    ln_eps: float = 1e-12,
    pad_idx: int = 1,                  # roberta only
    token_type_ids: Optional[Tensor] = None,
    round_fn: Optional[Callable[[Tensor], Tensor]] = None,
    mm: Optional[Callable[[Tensor, Tensor], Tensor]] = None,
    return_hidden: bool = False,
):
    """Returns unit-norm CLS rows fp32 [B, H] (and optionally the last hidden state)."""
    B, S = input_ids.shape
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)
    if mm is None:
        if round_fn is None:
            mm = lambda a, bt: a @ bt.t()
        else:
            mm = lambda a, bt: round_fn(a) @ round_fn(bt).t()

    def lin(x, prefix):
        return mm(x, sd[prefix + ".weight"]) + sd[prefix + ".bias"]

    # --- embeddings (modeling_bert.py:53-113) ---
    if arch == "roberta":
        # modeling_roberta.py:146-159: position ids = cumsum(mask_nonpad) * mask + pad_idx
        nonpad = (input_ids != pad_idx).to(torch.int64)
        pos = torch.cumsum(nonpad, dim=1) * nonpad + pad_idx
    else:
        pos = torch.arange(S).unsqueeze(0).expand(B, S)
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    x = (
        sd["embeddings.word_embeddings.weight"][input_ids]
        + sd["embeddings.token_type_embeddings.weight"][token_type_ids]
    )
    x = x + sd["embeddings.position_embeddings.weight"][pos]
    x = _ln(x, sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"], ln_eps)

    H = x.shape[-1]
    dh = H // num_heads
    scale = dh ** -0.5
    # additive mask: 0 keep, -inf (finfo.min in HF) masked
    addmask = (1.0 - attention_mask.to(torch.float32))[:, None, None, :] * torch.finfo(torch.float32).min

    L = 0
    while f"encoder.layer.{L}.attention.self.query.weight" in sd:
        L += 1
    for l in range(L):
        p = f"encoder.layer.{l}."
        x2 = x.reshape(B * S, H)
        q = lin(x2, p + "attention.self.query").view(B, S, num_heads, dh).transpose(1, 2)
        k = lin(x2, p + "attention.self.key").view(B, S, num_heads, dh).transpose(1, 2)
        v = lin(x2, p + "attention.self.value").view(B, S, num_heads, dh).transpose(1, 2)
        if round_fn is not None:
            scores = (round_fn(q) @ round_fn(k).transpose(-1, -2)) * scale + addmask
        else:
            scores = (q @ k.transpose(-1, -2)) * scale + addmask
        probs = torch.softmax(scores, dim=-1)
        if round_fn is not None:
            ctx = round_fn(probs) @ round_fn(v)
        else:
            ctx = probs @ v
        ctx = ctx.transpose(1, 2).reshape(B * S, H)
        a = lin(ctx, p + "attention.output.dense")
        x2 = _ln(a + x2, sd[p + "attention.output.LayerNorm.weight"], sd[p + "attention.output.LayerNorm.bias"], ln_eps)
        h = _gelu_erf(lin(x2, p + "intermediate.dense"))
        o = lin(h, p + "output.dense")
        x2 = _ln(o + x2, sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"], ln_eps)
        x = x2.view(B, S, H)

    cls = x[:, 0, :]
    # F.normalize(p=2, dim=1, eps=1e-12): x / max(||x||, eps)
    unit = cls / cls.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if return_hidden:
        return unit, x
    return unit


# ---- operand rounding emulations for the precision study -------------------------------------

def round_bf16(t: Tensor) -> Tensor:
    return t.to(torch.bfloat16).to(torch.float32)


def round_tf32(t: Tensor) -> Tensor:
    """Round-to-nearest-even to 10 explicit mantissa bits (the tf32 MMA reads the top 19 bits:
    hardware TRUNCATES fp32 operands; see `trunc_tf32`)."""
    i = t.contiguous().view(torch.int32)
    bias = ((i >> 13) & 1) + 0x0FFF
    return ((i + bias) & ~0x1FFF).view(torch.float32)


def trunc_tf32(t: Tensor) -> Tensor:
    i = t.contiguous().view(torch.int32)
    return (i & ~0x1FFF).view(torch.float32)


def make_bert_state_dict(seed: int = 1234, arch: str = "bert", **cfg_over):
    """Seeded random-init checkpoint of the bert-base-uncased architecture (SURVEY.md section 8(d)):
    torch.manual_seed(seed); BertModel(BertConfig()).  Returns (state_dict, config)."""
    from transformers import BertConfig, BertModel, RobertaConfig, RobertaModel

    torch.manual_seed(seed)
    if arch == "bert":
        cfg = BertConfig(**cfg_over)
        m = BertModel(cfg, add_pooling_layer=True)
    else:
        base = dict(vocab_size=50265, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                    intermediate_size=4096, max_position_embeddings=514, type_vocab_size=1,
                    layer_norm_eps=1e-5, pad_token_id=1)
        base.update(cfg_over)
        cfg = RobertaConfig(**base)
        m = RobertaModel(cfg, add_pooling_layer=True)
    m.eval()
    sd = {k: v.detach().clone().float() for k, v in m.state_dict().items()}
    return sd, cfg, m


def synthetic_ids(B: int, S: int, vocab: int = 30522, seed: int = 7, arch: str = "bert") -> Tensor:
    """SURVEY.md section 8(d): Generator(seed=7), uniform in [1000, vocab), CLS at 0, SEP at S-1."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(min(1000, vocab // 2), vocab, (B, S), generator=g, dtype=torch.int64)
    if arch == "bert":
        ids[:, 0] = min(101, vocab - 1)
        ids[:, -1] = min(102, vocab - 1)
    else:
        ids[:, 0] = 0
        ids[:, -1] = 2
    return ids
