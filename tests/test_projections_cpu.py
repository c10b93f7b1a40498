"""Proof that tests/test_gpu_projections.py can fail.  Its fp64 reference is pinned to Hugging Face's own modules in fp64
(BertSelfAttention's q / k / v, BertIntermediate, BertOutput, ModernBERT's Wqkv with its rotary embedding and
apply_rotary_pos_emb, ModernBertMLP, EuroBERT's RMSNorm and MLP, NomicBERT's MLP), then mutated the way an epilogue goes
wrong, on the very seeded inputs the GPU tests use: every mutation must exceed the GPU bound by >= 10x.

The last test records why the file exists: in a randomly initialised 2-layer bert-base, leaving W beta out of every
consumer does not move the unit CLS row at all (beta = 0 at init) and dropping mu c1 moves it by 2.4e-3, 2.4x the 1e-3
whole-encoder tolerance (row means are small at init), while on this file's inputs both are >= 100x the bound."""
import pytest
import torch

import test_gpu_projections as gp

FACTOR = 10.0
QKV, FFN1, WO, W2, ROWS = gp.QKV, gp.FFN1, gp.WO, gp.W2, gp.ROWS
B, S = 3, 77


def excess(ref, tol, mutated):
    return float("inf") if not torch.isfinite(mutated).all() else ((mutated - ref).abs() / tol).max().item()


def consumer_case(name, layer, role, mu_sigma=3.0, seed=0, B=B, S=S):
    fam = gp.family(name)
    P = gp.role_params(fam, layer, role)
    y = gp.residual_rows(B * S, fam.H, mu_sigma, 0.0, seed)
    st = stats64(fam, P, y)
    return fam, P, y, st


def stats64(fam, P, y):
    """the consumed norm's fp64 statistics, unrounded (the pinning tests compare to 1e-9)"""
    return gp.identity_stats(y.shape[0]) if P.get("norm") is None else gp.row_stats(y, fam.eps, fam.rms)


def with_params(P, **over):
    return {**P, **over}


# ---- the reference against HF's modules -------------------------------------------------------------
def test_bert_consumers_and_outputs_equal_hf_modules():
    fam = gp.family("bert")
    lay = [l.double() for l in fam.model.encoder.layer]
    y = gp.residual_rows(B * S, fam.H, 3.0, 1e3, 1)
    yd = y.double()
    with torch.no_grad():
        x = lay[0].output.LayerNorm(yd)                 # QKV of layer 1 consumes layer 0's output LayerNorm
        qk, _, v, _ = gp.consumer_ref(fam, gp.role_params(fam, 1, QKV), role=QKV, y=y, stats=gp.row_stats(y, fam.eps, False), S=S)
        att = lay[1].attention.self
        assert (qk - torch.cat([att.query(x), att.key(x)], 1)).abs().max() < 1e-9
        assert (v - att.value(x)).abs().max() < 1e-9
        xi = lay[1].attention.output.LayerNorm(yd)
        ffn, _ = gp.consumer_ref(fam, gp.role_params(fam, 1, FFN1), FFN1, y, gp.row_stats(y, fam.eps, False), S)
        assert (ffn - lay[1].intermediate(xi)).abs().max() < 1e-9
        a = gp.fp16_rows(B * S, fam.I, 2)
        ynew, _ = gp.residual_ref(gp.role_params(fam, 1, W2), a, y, gp.row_stats(y, fam.eps, False))
        assert (lay[1].output.LayerNorm(ynew) - lay[1].output(a.double(), xi)).abs().max() < 1e-9
        c = gp.fp16_rows(B * S, fam.H, 3)
        ynew, _ = gp.residual_ref(gp.role_params(fam, 1, WO), c, y, gp.row_stats(y, fam.eps, False))
        assert (lay[1].attention.output.LayerNorm(ynew) - lay[1].attention.output(c.double(), x)).abs().max() < 1e-9


@pytest.mark.parametrize("layer", [0, 1])
def test_modernbert_qkv_rope_and_mlp_equal_hf_modules(layer):
    from transformers.models.modernbert.modeling_modernbert import apply_rotary_pos_emb
    fam = gp.family("modernbert")
    m = fam.model.double()
    ly = m.layers[layer]
    y = gp.residual_rows(B * S, fam.H, 3.0, 0.0, 4)
    yd = y.double()
    with torch.no_grad():
        x = ly.attn_norm(yd)
        P = gp.role_params(fam, layer, QKV)
        st = stats64(fam, P, y)
        qk, _, v, _ = gp.consumer_ref(fam, P, QKV, y, st, S)
        qkv = ly.attn.Wqkv(x).view(B, S, 3, 12, 64)
        pos = torch.arange(S)[None].expand(B, S)
        cos, sin = m.rotary_emb(qkv, pos, m.config.layer_types[layer])
        q, k = apply_rotary_pos_emb(qkv[:, :, 0].transpose(1, 2), qkv[:, :, 1].transpose(1, 2), cos, sin)
        want = torch.cat([q.transpose(1, 2).reshape(B * S, -1), k.transpose(1, 2).reshape(B * S, -1)], 1)
        assert (qk - want).abs().max() < 1e-5          # HF's own cos / sin are fp32: the table the kernel reads
        assert (v - qkv[:, :, 2].reshape(B * S, -1)).abs().max() < 1e-9
        P = gp.role_params(fam, layer, FFN1)
        ffn, _ = gp.consumer_ref(fam, P, FFN1, y, stats64(fam, P, y), S)
        assert (ffn @ ly.mlp.Wo.weight.T - ly.mlp(ly.mlp_norm(yd))).abs().max() < 1e-9
    fam.model.float()


@pytest.mark.parametrize("name", ["eurobert", "nomic"])
def test_swiglu_mlps_and_rms_norm_equal_hf_modules(name):
    fam = gp.family(name)
    m = fam.model.double()
    y = gp.residual_rows(B * S, fam.H, 3.0, 0.0, 5)
    yd = y.double()
    P = gp.role_params(fam, 1, FFN1)
    with torch.no_grad():
        if name == "eurobert":
            ly = m.layers[1]
            x, mlp = ly.post_attention_layernorm(yd), ly.mlp
            P0 = gp.role_params(fam, 0, QKV)            # layer 0's real input_layernorm (RMS)
            xa = m.layers[0].input_layernorm(yd)
            w = torch.cat([m.layers[0].self_attn.q_proj.weight, m.layers[0].self_attn.k_proj.weight.view(4, 64, -1)
                           .repeat_interleave(3, 0).reshape(768, -1)])
            # EuroBertRMSNorm computes in fp32 whatever its input: 1e-5, not 1e-9
            assert (gp.consumer_pre(P0, y, stats64(fam, P0, y))[0][:, :2 * fam.H] - xa @ w.T).abs().max() < 1e-5
        else:
            ly = m.layers[1] if hasattr(m, "layers") else m.encoder.layer[1]
            mods = dict(ly.named_modules())
            norm = next(v for k, v in mods.items() if "post_attention_layernorm" in k)
            mlp = next(v for k, v in mods.items() if k.endswith("mlp"))
            x = norm(yd)
        ffn, _ = gp.consumer_ref(fam, P, FFN1, y, stats64(fam, P, y), S)
        assert (ffn @ mlp.down_proj.weight.T + (mlp.down_proj.bias if mlp.down_proj.bias is not None else 0)
                - mlp(x)).abs().max() < (1e-5 if name == "eurobert" else 1e-9)
    fam.model.float()


# ---- consumer mutations -------------------------------------------------------------------------------
def mutated_consumer(fam, P, role, y, st, how, S=S):
    """the consumer's outputs with the pre-activation z mutated as `how` says, everything else as the reference"""
    H = fam.H
    z, E = gp.consumer_pre(P, y, st)
    W = P["W"].double()
    gam, bet = P["norm"] if P.get("norm") is not None else (torch.ones(W.shape[1]), None)
    mu, r = st[:, :1], st[:, 1:]
    c1 = (W * gam.double()[None]).sum(1)
    c0 = (bet.double() @ W.T if bet is not None else 0) + (P["b"].double() if P["b"] is not None else 0)
    part = torch.arange(W.shape[0]) ^ 32                   # the partner column of a GLU / RoPE chunk
    if how == "mu_c1_dropped":
        z = z + r * mu * c1
    elif how == "c1_partner":
        z = z - r * mu * (c1[part] - c1)
    elif how == "bias_partner":
        z = z + torch.as_tensor(c0)[part] - c0
    elif how == "no_w_beta":
        z = z - bet.double() @ W.T
    if role == QKV:
        qk = z[:, :2 * H]
        if P["rope"] is not None:
            table, M = P["rope"], qk.shape[0]
            rows = torch.arange(M)
            if how == "rope_pos_plus_one":
                table = table[torch.cat([torch.arange(1, table.shape[0]), torch.tensor([0])])]
            if how == "rope_row_not_mod_s":
                t = table.double()[rows]
                table = None
            else:
                t = table.double()[rows % S]
            cos, sin = t[:, None, :32].repeat(1, 1, 2), t[:, None, 32:].repeat(1, 1, 2)
            x = qk.view(M, -1, 64)
            src = torch.roll(x, -1, dims=1) if how == "rope_partner_next_head" else x
            rot = torch.cat([-src[..., 32:], src[..., :32]], -1)
            if how == "rope_sign":
                rot = -rot
            qk = (x * cos + rot * sin).reshape(M, -1)
        return qk, z[:, 2 * H:]
    I = z.shape[1] // 2
    act = P["act"]
    if act in ("geglu", "swiglu"):
        a, g = z[:, :I], z[:, I:]
        if how == "glu_swapped":
            a, g = g, a
        if how == "glu_interleave_32":
            a = torch.roll(a.view(a.shape[0], -1, 32), -1, dims=1).reshape(a.shape)
        f = gp.gelu_erf if act == "geglu" else gp.silu
        if how == "gelu_silu_swapped":
            f = gp.silu if act == "geglu" else gp.gelu_erf
        return (f(a) * g,)
    return ({"gelu": gp.gelu_erf, "gelu_tanh": gp.gelu_tanh}[act](z),)


CONSUMER_MUTATIONS = [
    ("bert", 1, QKV, "mu_c1_dropped"), ("bert", 1, FFN1, "mu_c1_dropped"), ("modernbert", 1, QKV, "mu_c1_dropped"),
    ("modernbert", 1, FFN1, "c1_partner"), ("nomic", 1, QKV, "c1_partner"), ("bert", 1, QKV, "bias_partner"),
    ("nomic", 1, FFN1, "bias_partner"), ("bert", 1, QKV, "no_w_beta"), ("bert", 1, FFN1, "no_w_beta"),
    ("albert", 1, FFN1, "no_w_beta"), ("modernbert", 1, QKV, "rope_pos_plus_one"), ("nomic", 1, QKV, "rope_pos_plus_one"),
    ("modernbert", 0, QKV, "rope_row_not_mod_s"), ("eurobert", 1, QKV, "rope_row_not_mod_s"), ("modernbert", 1, QKV, "rope_sign"),
    ("modernbert", 1, QKV, "rope_partner_next_head"), ("modernbert", 1, FFN1, "glu_swapped"),
    ("eurobert", 1, FFN1, "glu_swapped"), ("nomic", 1, FFN1, "gelu_silu_swapped"), ("modernbert", 1, FFN1, "gelu_silu_swapped"),
    ("modernbert", 1, FFN1, "glu_interleave_32"), ("eurobert", 1, FFN1, "glu_interleave_32"),
]


@pytest.mark.parametrize("name,layer,role,how", CONSUMER_MUTATIONS)
def test_consumer_mutations_exceed_the_gpu_bound(name, layer, role, how):
    """rows with mean 0 and with |mu| / sigma = 3 (a dropped mu c1 needs a mean to show)"""
    for mu_sigma in (3.0,) if how == "mu_c1_dropped" else (0.0, 3.0):
        fam, P, y, st = consumer_case(name, layer, role, mu_sigma)
        ref = gp.consumer_ref(fam, P, role, y, st, S)
        got = mutated_consumer(fam, P, role, y, st, how)
        worst = max(excess(ref[2 * i], ref[2 * i + 1], g) for i, g in enumerate(got))
        assert worst >= FACTOR, f"{name} {how} mu/sigma={mu_sigma}: {worst:.2f} x the bound"


def test_sliding_table_on_a_global_layer_exceeds_the_gpu_bound():
    fam, P, y, st = consumer_case("modernbert", 0, QKV, S=1000, B=1)
    ref = gp.consumer_ref(fam, P, QKV, y, st, 1000)
    wrong = gp.consumer_ref(fam, with_params(P, rope=fam.rope[1]), QKV, y, st, 1000)
    assert excess(ref[0], ref[1], wrong[0]) >= FACTOR


def test_v_transpose_mutations_exceed_the_gpu_bound():
    fam, P, y, st = consumer_case("bert", 1, QKV)
    _, _, v, vtol = gp.consumer_ref(fam, P, QKV, y, st, S)
    H, S_pad = fam.H, (S + 7) // 8 * 8
    vb = v.view(B, S, H)
    neighbour = torch.roll(vb, -1, dims=0).reshape(B * S, H)
    assert excess(v, vtol, neighbour) >= FACTOR
    flat = torch.zeros(B * H * S_pad, dtype=torch.float64)      # written with a stride of S, read with S_pad
    flat[:B * H * S] = vb.permute(0, 2, 1).reshape(-1)
    read = flat.view(B, H, S_pad)[:, :, :S].permute(0, 2, 1).reshape(B * S, H)
    assert excess(v, vtol, read) >= FACTOR


# ---- residual mutations ---------------------------------------------------------------------------
@pytest.mark.parametrize("name,role,wrong", [("bert", WO, "ffn"), ("bert", W2, "out"), ("albert", W2, "out"),
                                             ("nomic", WO, "ffn"), ("bert", WO, "none")])
def test_pending_norm_of_the_wrong_layer_exceeds_the_gpu_bound(name, role, wrong):
    fam = gp.family(name)
    P = gp.role_params(fam, 1, role)
    y = gp.residual_rows(B * S, fam.H, 3.0, 0.0, 6)
    a = gp.fp16_rows(B * S, fam.I if role == W2 else fam.H, 7)
    st = gp.row_stats(y, fam.eps, False)
    ref, E = gp.residual_ref(P, a, y, st)
    other = {"ffn": gp.role_params(fam, 1, W2)["pending"], "out": gp.role_params(fam, 1, WO)["pending"], "none": None}[wrong]
    if wrong == "out" and name == "bert":
        other = (fam.sd["encoder.layer.1.output.LayerNorm.weight"], fam.sd["encoder.layer.1.output.LayerNorm.bias"])
    got, _ = gp.residual_ref(with_params(P, pending=other), a, y, st)
    assert excess(ref, E, got) >= FACTOR


def partial_sums(y):
    """per-64-column (sum, sumsq) of the rows, fp64: [M, H / 64, 2]"""
    yp = y.double().view(y.shape[0], -1, 64)
    return torch.stack([yp.sum(2), (yp * yp).sum(2)], 2)


def stats_from_parts(parts, H, eps, rms):
    s, q = parts[..., 0].sum(1), parts[..., 1].sum(1)
    if rms:
        return torch.stack([torch.zeros_like(s), 1.0 / torch.sqrt(q / H + eps)], 1)
    mu = s / H
    return torch.stack([mu, 1.0 / torch.sqrt((q / H - mu * mu).clamp_min(0.0) + eps)], 1)


@pytest.mark.parametrize("name", ["bert", "eurobert", "minilm", "bert_large"])
@pytest.mark.parametrize("how", ["part_dropped", "part_twice", "norm_swapped"])
@pytest.mark.parametrize("mu_sigma", [0.0, 3.0, 30.0])
def test_statistics_mutations_exceed_the_gpu_bound(name, how, mu_sigma):
    fam = gp.family(name)
    y = gp.residual_rows(B * S, fam.H, mu_sigma, 0.0, 8)
    if how == "norm_swapped" and mu_sigma == 0.0:
        y = y + 0.5                                        # LN and RMS statistics coincide on rows with mean 0
    ref, tol = gp.stats_tol(y, fam.rms, fam.eps)
    parts = partial_sums(y)
    k = 5 % parts.shape[1]
    if how == "part_dropped":
        parts[:, k] = 0
    elif how == "part_twice":
        parts[:, k] *= 2
    got = stats_from_parts(parts, fam.H, fam.eps, fam.rms != (how == "norm_swapped"))
    assert excess(ref, tol, got) >= FACTOR


@pytest.mark.parametrize("name", ["modernbert", "eurobert"])
def test_eps_left_out_exceeds_the_gpu_bound(name):
    """rows whose variance (RMS: mean square) is about eps"""
    fam = gp.family(name)
    g = torch.Generator().manual_seed(9)
    y = fam.eps ** 0.5 * torch.randn(B * S, fam.H, generator=g, dtype=torch.float64)
    ref, tol = gp.stats_tol(y, fam.rms, fam.eps)
    got = stats_from_parts(partial_sums(y), fam.H, 0.0, fam.rms)
    assert excess(ref, tol, got) >= FACTOR


# ---- why this file exists -------------------------------------------------------------------------
def test_whole_encoder_tolerance_misses_what_the_bound_sees():
    """a randomly initialised bert-base (2 layers), forward through HF with a consumer's input replaced: dropping mu c1
    adds r mu gamma to every consumed row, leaving out W beta removes beta.  The unit CLS row moves by 0 and 2.4e-3
    against the 1e-3 whole-encoder tolerance, while on the GPU test's inputs the same mutations are >= 100x its bound"""
    from oracle import encoder_oracle as eo
    _, _, m = eo.make_bert_state_dict(1234, num_hidden_layers=2)
    m = m.double().eval()
    ids = eo.synthetic_ids(2, 64)
    stats = {}

    def keep_stats(mod, inp, out):
        x = inp[0]
        mu = x.mean(-1, keepdim=True)
        stats[mod] = (mu, 1.0 / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + mod.eps), mod.weight, mod.bias)

    def cls(how):
        hooks = []
        for l, lay in enumerate(m.encoder.layer):
            src = [(lay.attention.output.LayerNorm, [lay.intermediate.dense])]
            if l:
                prev = m.encoder.layer[l - 1].output.LayerNorm
                src.append((prev, [lay.attention.self.query, lay.attention.self.key, lay.attention.self.value]))
            for ln, consumers in src:
                hooks.append(ln.register_forward_hook(keep_stats))
                for c in consumers:
                    def pre(mod, inp, ln=ln):
                        mu, r, g, b = stats[ln]
                        return (inp[0] + r * mu * g if how == "mu_c1_dropped" else inp[0] - b,)
                    hooks.append(c.register_forward_pre_hook(pre))
        with torch.no_grad():
            out = m(ids).last_hidden_state[:, 0]
        for h in hooks:
            h.remove()
        return out / out.norm(dim=1, keepdim=True)

    with torch.no_grad():
        base = m(ids).last_hidden_state[:, 0]
    base = base / base.norm(dim=1, keepdim=True)
    moved = {how: (cls(how) - base).norm(dim=1).max().item() for how in ("mu_c1_dropped", "no_w_beta")}
    assert moved["no_w_beta"] == 0.0 and moved["mu_c1_dropped"] < 5e-3, moved
    fam, P, y, st = consumer_case("bert", 1, FFN1, 3.0)
    ref = gp.consumer_ref(fam, P, FFN1, y, st, S)
    for how in moved:
        assert excess(ref[0], ref[1], mutated_consumer(fam, P, FFN1, y, st, how)[0]) >= 100


def test_projection_wrapper_refuses_inputs_of_the_wrong_shape():
    """the C entry copies B*S rows of each input, so Encoder.projection checks every shape first (no device is touched)"""
    from adaptive_classifier_b200 import _cabi as cb
    enc = cb.Encoder.__new__(cb.Encoder)
    enc.handle, enc.hidden, enc.intermediate, enc.embedding_size = None, 768, 3072, 128
    a = torch.zeros(100, 768, dtype=torch.float16)
    st = torch.zeros(100, 2)
    with pytest.raises(cb.AdaptiveB200Error, match=r"a is shape \(100, 768\); AC_PROJ_W2 needs \(100, 3072\)"):
        enc.projection(W2, 1, 1, 100, a, y=torch.zeros(100, 768), stats=st)
    with pytest.raises(cb.AdaptiveB200Error, match=r"a is shape \(100, 768\); AC_PROJ_EMB needs \(100, 128\)"):
        enc.projection(gp.EMB, 0, 1, 100, a)
    with pytest.raises(cb.AdaptiveB200Error, match=r"y is None; AC_PROJ_WO needs \(100, 768\)"):
        enc.projection(WO, 1, 1, 100, a, stats=st)
    with pytest.raises(cb.AdaptiveB200Error, match=r"stats is shape \(99, 2\); AC_PROJ_FFN1 needs \(100, 2\)"):
        enc.projection(FFN1, 1, 1, 100, a, stats=st[:99])
    with pytest.raises(cb.AdaptiveB200Error, match=r"a is on cpu; AC_PROJ_QKV needs CUDA tensors"):
        enc.projection(QKV, 1, 2, 50, a, stats=st)
