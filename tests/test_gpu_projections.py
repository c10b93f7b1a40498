"""The encoder projections with their fused epilogues run alone through Encoder.projection (ac_encoder_projection: the very
role functions the layer loop runs) and are compared, at every output element, with a plain fp64 reference of the same
operation computed from the fp32 HF-layout state dict (never from the packed operands):

    QKV, FFN1 (deferred-norm consumers)   z = N(y) W^T + b,   N(y) = (y - mu) r gamma + beta  (RMSNorm: mu = 0, beta = 0;
                                          the identity where the layer consumes none: post-LN and ModernBERT layer 0)
        QKV     q | k = RoPE(z[:, :2H]) per HF apply_rotary_pos_emb at position row mod S with the layer's own table;
                V^T[(b H + f) S_pad + key] = z[b S + key, 2H + f] at every (b, f, key < S)
        FFN1    gelu_erf(z), gelu_tanh(z) or, with W = [input; gate] rows, act(z_input) z_gate (GeGLU: gelu_erf,
                SwiGLU: silu(gate_proj) up_proj)
    FFN1_ROWS   the CLS-only tail's FFN1 on normalised rows: act(a W^T + b)
    WO, W2      y_new = a W^T + b + LN_pending(y), LN_pending the norm the forward leaves pending there (post-LN: the previous
                layer's output LayerNorm before Wo, nothing in layer 0, the attention-output LayerNorm before W2; pre-LN: none);
                fp16 y_new must equal fp16_rne(y_new) bit for bit, stats_out the fp64 statistics of the kernel's own y_new
    EMB         y = a Wp^T + bp (ALBERT), fp16 y bit for bit

The statistics a consumer applies are the fp64 ones of the fp32 y (rounded to fp32), so only the consumer is measured.

Whole-encoder tests cannot see most of this: randomly initialised rows have mean ~0 (a dropped mu c1 is invisible), beta = 0
hides a c0 without W beta, and a wrong element is averaged away by later LayerNorms.  Here rows carry mu / sigma up to 30
and single elements up to 3e4, every gamma / beta / bias is O(1) and differs per layer, and the check names the role, row
and column.  tests/test_projections_cpu.py mutates this reference the ways an epilogue goes wrong on these inputs: every
mutation exceeds the bound by >= 10x.

Error bounds, per output element (u = 2^-11 the fp16 unit roundoff, K the reduction length):

  consumers, pre-activation, with A = sum_k |y_k| |gamma_k W_nk|, D = sum_k |y_k - mu| |gamma_k W_nk|,
  Bt = sum_k |beta_k W_nk| + |b_n|, c_K = (K / 8 + 8) 2^-23:
      E = r (u (A + D) + c_K (A + D)) + c_K Bt + 2^-23 |z|
    * the kernel computes r (sum_k fp16(y_k) fp16(gamma_k W_nk) - mu c1) + c0 with c1 = sum_k fp16(gamma_k W_nk), which is
      r sum_k (fp16(y_k) - mu) fp16(gamma W): the fp16 roundings of y and of gamma W change it by at most
      r u sum_k (|y_k| (1 + u) |gamma W| + |y_k - mu| |gamma W|) -- the first term, which carries the |mu| / sigma growth
      (A ~ |mu| / sigma D): the kernel's error grows with the row mean, and the bound says by how much
    * fp32: the wgmma accumulation (K / 16 chained k-blocks plus the in-instruction sum, <= (K / 16 + 4) 2^-23 A), the
      warp-sum of c1 and the fp32 mu ((K / 32 + 6) 2^-24 (A + D), as |mu| sum |gamma W| <= A + D), the fmaf and the product
      with the fp32 r (2^-22 D), c0 = W beta + b in fp32 ((K / 32 + 6) 2^-24 Bt) and the last fma (2^-23 |z|): c_K covers all
  RoPE: |cos| E_d + |sin| E_partner + 2^-23 (|z_d cos| + |z_partner sin|)
  activations (documented at gelu_erf, gelu_tanh, silu in encoder.cu), slopes <= 1.13:
      gelu_erf   1.13 E + 2^-21 |z| + 2^-24 |out|   (Abramowitz-Stegun 7.1.26: 0.75e-7 |z|; ex2 / rcp .approx and the
                                                    polynomial's roundings: <= 12 2^-24 |z h|, h <= 1/2)
      gelu_tanh  1.13 E + 2^-15 |out|               (relative error < 2^-15)
      silu       1.13 E + (min(|z|, 89) 2^-23 + 5e-7) |out|
      GLU        (1.13 E_in + err_act) |z_gate| + |act(z_in)| E_gate + 2^-24 |out|
  residual roles, with S1 = sum_k |a_k| |W_nk| (a is fp16 already):
      E = u (1 + u) S1 + (K / 16 + 4) 2^-23 (1 + 2u) S1 + 2^-23 (|acc| + |b| + |N(y)| + |y_new|)
          + |gamma| r 2^-22 (|mu| + |y - mu|)       (the pending norm recomputed in fp32 from fp32 y, mu, r)
  every fp16 output: E (1 + u) + u |ref| + 2^-25 (half an ulp of the subnormals)
  stats_out (ln_stats_kernel, single pass in fp32): every square and sum passes at most n = 10 + H / 64 roundings (the
  product, the pairwise float4 sums, two chunks x two halves, two shuffles, H / 64 parts), so with Q = mean(y^2):
      |d mu| <= n 2^-24 mean|y| + 2^-24 |mu|
      |d var| <= 2^-24 ((n + 2) Q + 4 mu^2 + 2 n |mu| mean|y|)         (RMS: d of mean(y^2) <= (n + 1) 2^-24 Q)
      |d r| / r <= 1.01 (|d var| / (2 (var + eps)) + 2^-22)
    The single-pass variance loses ~(mu / sigma)^2 2^-24 n relative: the bound allows ~2e-3 of r at mu / sigma = 30, H = 768.

Tested ranges and documented limits (DESIGN.md section 3): rows with |mu| / sigma up to 30 and single elements up to 3e4.
ln_stats_kernel<Layer> meets that mean on ModernBERT (pre-LN) only: a post-LN Wo / W2 adds the normalised sums back.
The fp16 copy of the residual sums overflows past 65504, and nothing guards it; the error of r from the single-pass
variance grows as (mu / sigma)^2, so past mu / sigma ~ 100 the deferred norm is outside the tested range.  Neither is
changed here.

Largest error / bound per role, on an H100 80GB HBM3 at a 700 W power limit: DESIGN.md section 5.1.
"""
import functools
import math

import pytest
import torch

from adaptive_classifier_b200 import _cabi as cb

EMB, QKV, WO, FFN1, W2, ROWS = (cb.AC_PROJ_EMB, cb.AC_PROJ_QKV, cb.AC_PROJ_WO, cb.AC_PROJ_FFN1, cb.AC_PROJ_W2,
                                cb.AC_PROJ_FFN1_ROWS)
ROLE_NAMES = {EMB: "emb", QKV: "qkv", WO: "wo", FFN1: "ffn1", W2: "w2", ROWS: "ffn1_rows"}
MAX_TOKENS = 16512
U = 2.0 ** -11
SLOPE = 1.13          # max |d act / dz| of GELU (1.129) and SiLU (1.100)


# ------------------------------------------------------------------------------------------------
# families: seeded HF models with O(1) norms and biases that differ per layer
# ------------------------------------------------------------------------------------------------
def _perturb(m, seed):
    """gamma = 1 + 0.5 N, beta and every bias ~ N(0, 1): c0 = W beta + b and a pending norm of the wrong layer both show"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            low = n.lower()
            if "norm" in low and n.endswith("weight"):
                p.copy_(1.0 + 0.5 * torch.randn(p.shape, generator=g))
            elif n.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g))
    return m.eval()


class Family:
    """name, HF model, the HF-layout state dict under the names the Encoder reads, and the block's settings"""

    def __init__(self, name, model, sd, *, pre, rms, act, layers, hidden, intermediate, eps, rope=None, emb=0):
        self.name, self.model, self.sd = name, model, {k: v.detach().float() for k, v in sd.items()}
        self.pre, self.rms, self.act, self.L, self.H, self.I, self.eps = pre, rms, act, layers, hidden, intermediate, eps
        self.rope = rope or [None] * layers          # per layer: the fp32 cos | sin table [max_pos, 64] or None
        self.E = emb


@functools.lru_cache(maxsize=None)
def family(name):
    import transformers as tf
    from oracle import encoder_oracle as eo, modernbert_oracle as mo
    if name in ("bert", "bert_large", "minilm"):
        dims = {"bert": dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072),
                "bert_large": dict(hidden_size=1024, num_attention_heads=16, intermediate_size=4096),
                "minilm": dict(hidden_size=384, num_attention_heads=12, intermediate_size=1536)}[name]
        _, cfg, m = eo.make_bert_state_dict(21, num_hidden_layers=2, vocab_size=100, **dims)
        m = _perturb(m, 22)
        return Family(name, m, m.state_dict(), pre=False, rms=False, act="gelu", layers=2, hidden=cfg.hidden_size,
                      intermediate=cfg.intermediate_size, eps=cfg.layer_norm_eps)
    if name == "albert":
        torch.manual_seed(23)
        c = tf.AlbertConfig(vocab_size=100, embedding_size=128, hidden_size=768, num_hidden_layers=3, num_attention_heads=12,
                            intermediate_size=3072, hidden_act="gelu_new", max_position_embeddings=512)
        m = _perturb(tf.AlbertModel(c, add_pooling_layer=False), 24)
        sd, dims = cb.albert_to_bert_state_dict(dict(m.state_dict()), c)
        return Family(name, m, sd, pre=False, rms=False, act="gelu_tanh", layers=3, hidden=768, intermediate=3072,
                      eps=c.layer_norm_eps, emb=128)
    if name == "modernbert":
        _, c, m = mo.make_modernbert(25, vocab_size=100, hidden_size=768, intermediate_size=1152, num_hidden_layers=3,
                                     num_attention_heads=12, max_position_embeddings=8192, pad_token_id=99, bos_token_id=97,
                                     eos_token_id=98, cls_token_id=97, sep_token_id=98)
        m = _perturb(m, 26)
        d = cb.modernbert_settings(c)
        full, slide = (cb.modernbert_rope_table(t, 8192) for t in d["rope_theta"])
        rope = [slide if s else full for s in d["layer_sliding"]]
        assert d["layer_sliding"][0] == 0 and d["layer_sliding"][1] == 1
        return Family(name, m, m.state_dict(), pre=True, rms=False, act="geglu", layers=3, hidden=768, intermediate=1152,
                      eps=c.norm_eps, rope=rope)
    if name == "eurobert":
        torch.manual_seed(27)
        c = tf.EuroBertConfig(vocab_size=100, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                              num_key_value_heads=4, intermediate_size=2048, max_position_embeddings=8192,
                              rope_parameters={"rope_type": "default", "rope_theta": 250000.0}, bos_token_id=0,
                              eos_token_id=2, pad_token_id=1, mask_token_id=3)
        m = _perturb(tf.EuroBertModel(c), 28)
        sd, d = cb.eurobert_to_modernbert_names(dict(m.state_dict()), c)
        t = cb.modernbert_rope_table(float(d["rope_theta"]), 8192)
        return Family(name, m, sd, pre=True, rms=True, act="swiglu", layers=2, hidden=768, intermediate=2048,
                      eps=c.rms_norm_eps, rope=[t, t])
    assert name == "nomic"
    torch.manual_seed(29)
    c = tf.NomicBertConfig(vocab_size=100, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                           intermediate_size=3072, max_position_embeddings=2048, type_vocab_size=2)
    m = _perturb(tf.NomicBertModel(c), 30)
    sd, d = cb.nomic_bert_to_bert_state_dict(dict(m.state_dict()), c)
    t = cb.modernbert_rope_table(float(d["rope_theta"]), 2048)
    return Family(name, m, sd, pre=False, rms=False, act="swiglu", layers=2, hidden=768, intermediate=d["intermediate"],
                  eps=d["ln_eps"], rope=[t, t])


def role_params(fam, layer, role):
    """W [N, K], b [N] or None, the consumed norm (gamma, beta-or-None) or None = identity, the pending norm of a residual
    role, the activation and the RoPE table of the layer -- all read from the HF-layout state dict"""
    sd, L = fam.sd, fam.L
    get = lambda n: sd[n] if n in sd else None
    norm = lambda pre: (sd[pre + "weight"], get(pre + "bias"))
    if role == EMB:
        return dict(W=sd["embeddings_project.weight"], b=sd["embeddings_project.bias"])
    if fam.pre:
        p = f"layers.{layer}."
        if role == QKV:
            consumed = norm(p + "attn_norm.") if (layer or fam.rms) else None
            return dict(W=sd[p + "attn.Wqkv.weight"], b=None, norm=consumed, rope=fam.rope[layer])
        if role == FFN1:
            return dict(W=sd[p + "mlp.Wi.weight"], b=None, norm=norm(p + "mlp_norm."), act=fam.act)
        if role == ROWS:
            return dict(W=sd[f"layers.{L - 1}.mlp.Wi.weight"], b=None, norm=None, act=fam.act)
        return dict(W=sd[p + ("attn.Wo.weight" if role == WO else "mlp.Wo.weight")], b=None, pending=None)
    p = f"encoder.layer.{layer}."
    if role == QKV:
        qkv = ("attention.self.query.", "attention.self.key.", "attention.self.value.")
        return dict(W=torch.cat([sd[p + n + "weight"] for n in qkv]), b=torch.cat([sd[p + n + "bias"] for n in qkv]),
                    norm=norm(f"encoder.layer.{layer - 1}.output.LayerNorm.") if layer else None, rope=fam.rope[layer])
    if role == FFN1:
        return dict(W=sd[p + "intermediate.dense.weight"], b=sd[p + "intermediate.dense.bias"],
                    norm=norm(p + "attention.output.LayerNorm."), act=fam.act)
    if role == ROWS:
        q = f"encoder.layer.{L - 1}.intermediate.dense."
        return dict(W=sd[q + "weight"], b=sd[q + "bias"], norm=None, act=fam.act)
    if role == WO:
        return dict(W=sd[p + "attention.output.dense.weight"], b=sd[p + "attention.output.dense.bias"],
                    pending=norm(f"encoder.layer.{layer - 1}.output.LayerNorm.") if layer else None)
    return dict(W=sd[p + "output.dense.weight"], b=sd[p + "output.dense.bias"],
                pending=norm(p + "attention.output.LayerNorm."))


# ------------------------------------------------------------------------------------------------
# reference (device-agnostic fp64 torch; the CPU tests import it)
# ------------------------------------------------------------------------------------------------
def row_stats(y, eps, rms):
    """[M, 2] fp64 (mu, r) of the rows of y: LayerNorm (two-pass) or RMSNorm (mu = 0)"""
    y = y.double()
    if rms:
        return torch.stack([torch.zeros_like(y[:, 0]), 1.0 / torch.sqrt((y * y).mean(1) + eps)], 1)
    mu = y.mean(1)
    return torch.stack([mu, 1.0 / torch.sqrt(((y - mu[:, None]) ** 2).mean(1) + eps)], 1)


def identity_stats(M, device="cpu"):
    return torch.tensor([[0.0, 1.0]], dtype=torch.float64, device=device).expand(M, 2).contiguous()


def gelu_erf(z):
    return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))


def gelu_tanh(z):
    return 0.5 * z * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (z + 0.044715 * z ** 3)))


def silu(z):
    return z * torch.sigmoid(z)


def act_ref(act, z, E):
    """(act(z), bound) for an elementwise activation given the pre-activation bound E"""
    if act == "gelu":
        out = gelu_erf(z)
        return out, SLOPE * E + 2.0 ** -21 * z.abs() + 2.0 ** -24 * out.abs()
    if act == "gelu_tanh":
        out = gelu_tanh(z)
        return out, SLOPE * E + 2.0 ** -15 * out.abs()
    assert act == "silu"
    out = silu(z)
    return out, SLOPE * E + (z.abs().clamp_max(89.0) * 2.0 ** -23 + 5e-7) * out.abs()


def f16_tol(ref, E):
    return E * (1 + U) + U * ref.abs() + 2.0 ** -25


def rope_ref(z, E, table, S, H):
    """HF apply_rotary_pos_emb on q | k [M, 2H] at position row mod S: x cos + rotate_half(x) sin, head_dim 64"""
    M = z.shape[0]
    t = table.double().to(z.device)[torch.arange(M, device=z.device) % S]            # [M, 64] cos | sin
    cos, sin = t[:, None, :32].repeat(1, 1, 2), t[:, None, 32:].repeat(1, 1, 2)
    x, e = z.view(M, 2 * H // 64, 64), E.view(M, 2 * H // 64, 64)
    rot = torch.cat([-x[..., 32:], x[..., :32]], -1)
    erot = torch.cat([e[..., 32:], e[..., :32]], -1)
    out = x * cos + rot * sin
    tol = cos.abs() * e + sin.abs() * erot + 2.0 ** -23 * ((x * cos).abs() + (rot * sin).abs())
    return out.reshape(M, 2 * H), tol.reshape(M, 2 * H)


def consumer_pre(P, y, stats):
    """(z, E) [M, N] fp64: the pre-activation N(y) W^T + b of a consumer and its bound; y [M, K] fp32 (the kernel reads
    fp16(y)), stats [M, 2] the (mu, r) it applies"""
    dev = stats.device
    W = P["W"].double().to(dev)
    K = W.shape[1]
    gam, bet = P["norm"] if P.get("norm") is not None else (None, None)
    Wg = W * gam.double().to(dev)[None, :] if gam is not None else W
    yd = y.double().to(dev)
    mu, r = stats[:, :1], stats[:, 1:]
    z = ((yd - mu) * r) @ Wg.T
    Bt = torch.zeros(W.shape[0], dtype=torch.float64, device=dev)
    if bet is not None:
        z = z + bet.double().to(dev) @ W.T
        Bt = Bt + bet.double().to(dev).abs() @ W.abs().T
    if P["b"] is not None:
        z = z + P["b"].double().to(dev)
        Bt = Bt + P["b"].double().to(dev).abs()
    Wa = Wg.abs().T
    AD = yd.abs() @ Wa + (yd - mu).abs() @ Wa
    cK = (K / 8 + 8) * 2.0 ** -23
    return z, r * (U + cK) * AD + cK * Bt + 2.0 ** -23 * z.abs()


def consumer_ref(fam, P, role, y, stats, S):
    """reference outputs and bounds of a consumer role: QKV -> (qk, qk_tol, v, v_tol) with v [M, H]; FFN1 -> (ffn, tol)"""
    H = fam.H
    z, E = consumer_pre(P, y, stats)
    if role == QKV:
        qk, eqk = z[:, :2 * H], E[:, :2 * H]
        if P["rope"] is not None:
            qk, eqk = rope_ref(qk, eqk, P["rope"], S, H)
        return qk, f16_tol(qk, eqk), z[:, 2 * H:], f16_tol(z[:, 2 * H:], E[:, 2 * H:])
    act = P["act"]
    if act in ("geglu", "swiglu"):
        I = z.shape[1] // 2
        a, g = act_ref("gelu" if act == "geglu" else "silu", z[:, :I], E[:, :I])
        out = a * z[:, I:]
        return out, f16_tol(out, g * z[:, I:].abs() + a.abs() * E[:, I:] + 2.0 ** -24 * out.abs())
    out, tol = act_ref(act, z, E)
    return out, f16_tol(out, tol)


def pending_ref(P, y, stats):
    """(N_pending(y), its bound) [M, H] fp64"""
    yd = y.double().to(stats.device)
    if P.get("pending") is None:
        return yd, torch.zeros_like(yd)
    g, b = (t.double().to(stats.device) for t in P["pending"])
    mu, r = stats[:, :1], stats[:, 1:]
    n = (yd - mu) * r * g + b
    return n, g.abs() * r * 2.0 ** -22 * (mu.abs() + (yd - mu).abs())


def residual_ref(P, a, y, stats):
    """(y_new, bound) [M, H] fp64 of a residual role (EMB: y = None)"""
    dev = stats.device
    W = P["W"].double().to(dev)
    K = W.shape[1]
    ad = a.double().to(dev)
    acc = ad @ W.T
    S1 = ad.abs() @ W.abs().T
    b = P["b"].double().to(dev) if P["b"] is not None else torch.zeros(W.shape[0], dtype=torch.float64, device=dev)
    if y is None:
        n, En = torch.zeros_like(acc), torch.zeros_like(acc)
    else:
        n, En = pending_ref(P, y, stats)
    out = acc + b + n
    E = (U * (1 + U) + (K / 16 + 4) * 2.0 ** -23 * (1 + 2 * U)) * S1 + 2.0 ** -23 * (acc.abs() + b.abs() + n.abs() + out.abs()) + En
    return out, E


def stats_tol(y, rms, eps):
    """bound on |mu_kernel - mu|, |r_kernel - r| of ln_stats_kernel against the fp64 statistics of the same fp32 rows"""
    y = y.double()
    H = y.shape[1]
    n = 10 + H / 64
    Q, ma = (y * y).mean(1), y.abs().mean(1)
    ref = row_stats(y, eps, rms)
    mu = ref[:, 0]
    if rms:
        dvar, var, dmu = (n + 1) * 2.0 ** -24 * Q, Q, torch.full_like(Q, 1e-30)   # mu must be exactly 0
    else:
        dmu = n * 2.0 ** -24 * ma + 2.0 ** -24 * mu.abs()
        dvar = 2.0 ** -24 * ((n + 2) * Q + 4 * mu * mu + 2 * n * mu.abs() * ma)
        var = 1.0 / ref[:, 1] ** 2 - eps
    dr = 1.01 * (dvar / (2 * (var + eps)) + 2.0 ** -22) * ref[:, 1]
    return ref, torch.stack([dmu, dr], 1)


# ------------------------------------------------------------------------------------------------
# seeded inputs (built on the CPU in fp32: GPU and CPU tests see the same values)
# ------------------------------------------------------------------------------------------------
def residual_rows(M, H, mu_sigma=3.0, spike=0.0, seed=0):
    """[M, H] fp32 residual sums: row r = s_r (+-mu_sigma + N(0, 1)), s_r in [0.5, 2]; rows with r % 3 == 0 have mean 0 and
    rows with r % 3 == 1 half the mean, so every call mixes them.  spike: element (r, (37 r) % H) of every 5th row set to
    +-spike"""
    g = torch.Generator().manual_seed(seed)
    s = 0.5 + 1.5 * torch.rand(M, 1, generator=g)
    sign = torch.where(torch.rand(M, 1, generator=g) < 0.5, -1.0, 1.0)
    frac = torch.tensor([0.0, 0.5, 1.0]).repeat(M // 3 + 1)[:M, None]
    y = s * (sign * frac * mu_sigma + torch.randn(M, H, generator=g))
    if spike:
        rows = torch.arange(0, M, 5)
        y[rows, (37 * rows) % H] = spike * torch.where(rows % 2 == 0, 1.0, -1.0)
    return y


def fp16_rows(M, K, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(M, K, generator=g)).half()


# ------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------
WORST = {}      # "family role" -> largest |out - ref| / bound seen


@pytest.fixture(scope="module")
def encoders(cabi):
    made = {}

    def get(name):
        if name not in made:
            made[name] = cabi.Encoder.from_hf(family(name).model, max_tokens=MAX_TOKENS, cls_only=True)
        return made[name]
    yield get
    for e in made.values():
        e.close()
    print("\nlargest error / bound per role: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))


def compare(what, got, ref, tol):
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    ratio = (got.double() - ref).abs() / tol
    worst = ratio.max().item()
    key = what.split(" [")[0]
    WORST[key] = max(WORST.get(key, 0.0), worst)
    if worst > 1.0:
        idx = [int(i) for i in (ratio == ratio.max()).nonzero()[0]]
        pytest.fail(f"{what}: |out - ref| = {worst:.2f} x bound at {idx}: out {got[tuple(idx)].item():.6g} "
                    f"ref {ref[tuple(idx)].item():.6g} bound {tol[tuple(idx)].item():.3g}")


def consumer_stats(fam, P, y):
    """the fp64 statistics of the consumed norm, rounded to fp32 as the kernel reads them ((0, 1) for the identity)"""
    if P.get("norm") is None:
        return identity_stats(y.shape[0]).float()
    return row_stats(y, fam.eps, fam.rms).float()


def run_consumer(encoders, name, role, layer, B, S, mu_sigma=3.0, spike=0.0, seed=0):
    fam, enc = family(name), encoders(name)
    P = role_params(fam, layer, role)
    M, H = B * S, fam.H
    y = residual_rows(M, H, mu_sigma, spike, seed) if role != ROWS else fp16_rows(M, H, seed).float()
    st = consumer_stats(fam, P, y).cuda()
    outs = enc.projection(role, layer, B, S, y.cuda().half(), stats=st)
    tag = f"{name} {ROLE_NAMES[role]} [layer={layer} B={B} S={S} mu/sigma={mu_sigma} spike={spike}]"
    if role == QKV:
        qk, qk_tol, v, v_tol = consumer_ref(fam, P, role, y.cuda(), st.double(), S)
        compare(tag.replace(" [", " q|k ["), outs[0], qk, qk_tol)
        S_pad = (S + 7) // 8 * 8
        vT = outs[1].view(B, H, S_pad)[:, :, :S].permute(0, 2, 1).reshape(M, H)
        compare(tag.replace(" [", " v ["), vT, v, v_tol)
    else:
        ref, tol = consumer_ref(fam, P, role, y.cuda(), st.double(), S)
        compare(tag, outs[0], ref, tol)
    return outs


def run_residual(encoders, name, role, layer, B, S, mu_sigma=3.0, spike=0.0, seed=0):
    fam, enc = family(name), encoders(name)
    P = role_params(fam, layer, role)
    M, H = B * S, fam.H
    K = fam.E if role == EMB else fam.I if role == W2 else H
    a = fp16_rows(M, K, seed + 1)
    tag = f"{name} {ROLE_NAMES[role]} [layer={layer} B={B} S={S} mu/sigma={mu_sigma} spike={spike}]"
    if role == EMB:
        y_new, yh = enc.projection(role, layer, B, S, a.cuda())
        ref, E = residual_ref(P, a.cuda(), None, identity_stats(M, "cuda"))
    else:
        y = residual_rows(M, H, mu_sigma, spike, seed)
        st = row_stats(y, fam.eps, fam.rms).float().cuda()
        y_new, yh, st_out = enc.projection(role, layer, B, S, a.cuda(), y=y.cuda(), stats=st)
        ref, E = residual_ref(P, a.cuda(), y.cuda(), st.double())
        sref, stol = stats_tol(y_new, fam.rms, fam.eps)
        # recorded apart at |mu| / sigma = 30: the single-pass variance's (mu / sigma)^2 term is what that case measures
        compare(tag.replace(" [", " stats at mu/sigma 30 [" if mu_sigma == 30.0 else " stats ["), st_out, sref, stol)
        if fam.rms:
            assert (st_out[:, 0] == 0).all(), f"{tag}: RMSNorm statistics with mu != 0"
    compare(tag, y_new, ref, E)
    assert torch.equal(yh, y_new.half()), f"{tag}: fp16 copy differs from fp16_rne(y_new)"
    return y_new, yh


pytestmark = pytest.mark.gpu
SEAMS = [(3, 77), (2, 100), (3, 129)]          # B*S not a multiple of 128, sequences straddling 128-row tiles
LONG = [(2, 513)]                              # rotary families only (BERT positions stop at 512)


@pytest.mark.parametrize("B,S", SEAMS)
@pytest.mark.parametrize("role", [QKV, FFN1, WO, W2])
@pytest.mark.parametrize("name", ["bert", "bert_large", "minilm", "albert", "modernbert", "eurobert", "nomic"])
def test_every_family_and_role_at_the_tile_seams(encoders, name, role, B, S):
    layer = 1
    if role in (QKV, FFN1):
        run_consumer(encoders, name, role, layer, B, S, seed=S)
    else:
        run_residual(encoders, name, role, layer, B, S, seed=S)


@pytest.mark.parametrize("role", [QKV, FFN1, WO, W2])
@pytest.mark.parametrize("name", ["modernbert", "eurobert", "nomic"])
def test_rotary_families_past_512(encoders, name, role):
    for B, S in LONG:
        (run_consumer if role in (QKV, FFN1) else run_residual)(encoders, name, role, 0, B, S, seed=B + S)


@pytest.mark.parametrize("spike", [0.0, 1e3, 3e4])
@pytest.mark.parametrize("mu_sigma", [0.0, 3.0, 30.0])
@pytest.mark.parametrize("role", [QKV, FFN1, WO, W2])
@pytest.mark.parametrize("name", ["bert", "modernbert", "eurobert"])
def test_row_mean_and_single_large_elements(encoders, name, role, mu_sigma, spike):
    """|mu| / sigma in {0, 3, 30} (the deferred norm's cancellation in r (acc - mu c1)) and one element of 1e3 / 3e4 in
    every 5th row.  The residual roles of a post-LN block add the normalised sums back, so BERT's new sums have mean ~0;
    ModernBERT (pre-LN) keeps the mean, so its Wo / W2 statistics are ln_stats_kernel<Layer>'s single-pass variance at
    |mu| / sigma ~ 30 -- asserted below, so that the case keeps reaching that edge; EuroBERT carries the RMS statistics"""
    if role in (QKV, FFN1):
        run_consumer(encoders, name, role, 1, 2, 100, mu_sigma=mu_sigma, spike=spike, seed=int(mu_sigma) + int(spike))
        return
    y_new, _ = run_residual(encoders, name, role, 1, 2, 100, mu_sigma=mu_sigma, spike=spike,
                            seed=int(mu_sigma) + int(spike))
    if name == "modernbert" and mu_sigma == 30.0 and spike == 0.0:
        st = row_stats(y_new, family(name).eps, False)
        assert (st[:, 0].abs() * st[:, 1]).max() > 25.0, "the new sums no longer carry |mu| / sigma ~ 30"


@pytest.mark.parametrize("role", [QKV, FFN1, WO, W2])
@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("name", ["bert", "albert", "modernbert", "eurobert", "nomic"])
def test_each_layer_uses_its_own_norms_and_tables(encoders, name, layer, role):
    """layer 0 consumes the identity (post-LN, ModernBERT) or the real input_layernorm (EuroBERT); layer 1 the previous
    layer's output norm (post-LN) or its own attn_norm; Wo of layer 0 adds the raw sums, of layer 1 the pending norm"""
    fn = run_consumer if role in (QKV, FFN1) else run_residual
    fn(encoders, name, role, layer, 3, 77, mu_sigma=3.0, seed=10 + layer)


@pytest.mark.parametrize("S", [57, 66, 75, 84, 93, 102, 111])
def test_v_transpose_at_every_s_mod_8(encoders, S):
    """S = 1 .. 7 (mod 8): V^T rows are S_pad = roundup(S, 8) keys apart"""
    run_consumer(encoders, "bert", QKV, 1, 3, S, seed=S)
    run_consumer(encoders, "minilm", QKV, 1, 3, S, seed=S)


@pytest.mark.parametrize("layer,S", [(0, 8192), (1, 8192), (0, 4099), (1, 4099)])
def test_modernbert_rope_at_long_sequences_per_layer_table(encoders, layer, S):
    """layer 0 is global (rope theta 160000), layer 1 sliding (10000): each reads its own table at positions up to 8191"""
    run_consumer(encoders, "modernbert", QKV, layer, 1 if S > 4096 else 2, S, seed=layer)


@pytest.mark.parametrize("name,B,S", [("eurobert", 1, 8192), ("nomic", 1, 2048)])
def test_rotary_tables_at_their_longest(encoders, name, B, S):
    run_consumer(encoders, name, QKV, 1, B, S, seed=S)


PERSISTENT = (59, 279)          # M = 16461 = 16K + 77 rows at H = 768: every CTA drains >= 20 tiles


@pytest.mark.parametrize("role", [QKV, FFN1, WO, W2])
def test_persistent_size_bert(encoders, role):
    fn = run_consumer if role in (QKV, FFN1) else run_residual
    fn(encoders, "bert", role, 1, *PERSISTENT, mu_sigma=3.0, seed=5)


def test_persistent_size_embedding_projection(encoders):
    run_residual(encoders, "albert", EMB, 0, *PERSISTENT, seed=6)


@pytest.mark.parametrize("name", ["bert", "modernbert", "nomic"])
def test_persistent_size_cls_tail_ffn1(encoders, name):
    """EpiF16<ACT, false> on w1_last: ModernBERT's GeGLU is the only path to EpiF16<GeGLU, false>"""
    run_consumer(encoders, name, ROWS, family(name).L - 1, *PERSISTENT, seed=7)


@pytest.mark.parametrize("B,S", SEAMS + [(1, 1), (2, 7)])
@pytest.mark.parametrize("name", ["bert", "albert", "modernbert", "eurobert", "nomic"])
def test_cls_tail_ffn1_and_embedding_projection_at_the_seams(encoders, name, B, S):
    run_consumer(encoders, name, ROWS, family(name).L - 1, B, S, seed=S)
    if name == "albert":
        run_residual(encoders, "albert", EMB, 0, B, S, seed=S)


@pytest.mark.parametrize("role", [QKV, FFN1, WO, W2])
def test_albert_shared_layers_are_bitwise_equal(encoders, role):
    """ALBERT shares one layer's parameters: layers 1 and 2 (both consuming the shared output LayerNorm) give the same
    bits; layer 0's QKV consumes the identity instead"""
    enc, fam, B, S = encoders("albert"), family("albert"), 2, 100
    M, H = B * S, fam.H
    y = residual_rows(M, H, seed=3)
    st = row_stats(y, fam.eps, False).float().cuda()
    a = fp16_rows(M, fam.I if role == W2 else H, seed=4).cuda()
    args = (y.cuda().half(),) if role in (QKV, FFN1) else (a,)
    kw = dict(stats=st) if role in (QKV, FFN1) else dict(y=y.cuda(), stats=st)
    one, two = (enc.projection(role, layer, B, S, *args, **kw) for layer in (1, 2))
    for x, z in zip(one, two):
        assert torch.equal(x, z)


def test_projection_refuses_bad_arguments_by_name(cabi, encoders):
    bert, modern = encoders("bert"), encoders("modernbert")
    a = torch.zeros(100, 768, dtype=torch.float16, device="cuda")
    st = identity_stats(100, "cuda").float()
    with pytest.raises(cabi.AdaptiveB200Error, match="unknown role=9"):
        bert.projection(9, 0, 1, 100, a, stats=st)
    with pytest.raises(cabi.AdaptiveB200Error, match="layer=2 outside 0..1"):
        bert.projection(QKV, 2, 1, 100, a, stats=st)
    with pytest.raises(cabi.AdaptiveB200Error, match="AC_PROJ_EMB needs an encoder with an embedding projection"):
        bert.projection(EMB, 0, 1, 100, a)
    big = torch.zeros(3 * 8192, 768, dtype=torch.float16, device="cuda")
    with pytest.raises(cabi.AdaptiveB200Error, match="exceeds max_tokens|must be in 1..max_tokens"):
        modern.projection(FFN1, 0, 3, 8192, big, stats=identity_stats(3 * 8192, "cuda").float())
    with pytest.raises(cabi.AdaptiveB200Error, match=r"a is shape \(100, 768\); AC_PROJ_W2 needs \(100, 3072\)"):
        bert.projection(W2, 1, 1, 100, a, y=torch.zeros(100, 768, device="cuda"), stats=st)
    with pytest.raises(cabi.AdaptiveB200Error, match=r"stats is shape \(50, 2\); AC_PROJ_QKV needs \(100, 2\)"):
        bert.projection(QKV, 1, 1, 100, a, stats=st[:50])
    nocls = cabi.Encoder.from_hf(family("bert").model, max_tokens=256, cls_only=False)
    try:
        with pytest.raises(cabi.AdaptiveB200Error, match="AC_PROJ_FFN1_ROWS needs a cls_only encoder"):
            nocls.projection(ROWS, 1, 1, 100, a)
    finally:
        nocls.close()
