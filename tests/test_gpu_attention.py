"""The two encoder attention kernels (attention_kernel for S <= 128, attention_stream_kernel with the online softmax above;
ScorePlain at head_dim 64 and 32, ScoreRelBias, the MPNet relative bias, at 64) run alone through Encoder.attention and are
compared with a plain fp64 reference of the same operation, on the fp16-rounded operands, at every row of every (sequence,
head):

    out[b, q, h, :] = softmax_key( q.k / sqrt(dh) + bias[h, 511 + key - q] + M[b, q, key] ) . v
    M = 0 where mask[b, key] != 0 and (window == 0 or |q - key| <= window), -inf elsewhere

A query with no attended key (a sequence that is all padding, a band that holds only padded keys) gets a context of exactly
0, never NaN: that is the kernels' rule (row sum 0 -> factor 0) and the reference states it the same way.  Padded *query*
rows are computed like any other row and are compared too.

Whole-encoder tests cannot see a subtly wrong attention: with randomly initialised weights the scaled scores have a standard
deviation of about 0.3, the softmax is nearly uniform and the context is diluted by the output projection and the residual.
Here the scores are peaked, the running maximum of the online softmax moves by tens between key blocks, and a probe with
q = 0 makes the output the plain mean of V over the attended set, so that one key too many or too few is far outside the
bound.  tests/test_attention_cpu.py proves that by mutating the reference on these very inputs.

Error bound (one for the whole file), per output element, with w = the fp64 softmax weights of the row:

    |out - ref| <= 2^-10 (w . |v|) + 2^-11 |ref| + 2^-25 sum_{attended keys} |v| + 2^-24

  * the kernels round P = exp(s - max) to fp16 before the PV product: relative error 2^-11 per key, so at most
    2^-11 (w . |v|) in the context (the row sum is taken from the unrounded fp32 values).  The first term allows twice
    that; the second 2^-11 (w . |v|) covers ex2.approx (2 ulp fp32), the fp32 rounding of the scaled score (|logit| 2^-24,
    which is 2^-15 at |logit| = 500) and the fp32 accumulation of QK^T, PV and the row sum, all far smaller
  * P below 2^-14 is a subnormal fp16 with absolute error 2^-25 (P = 1 at the row maximum, the row sum is >= 1, and the
    online rescale only shrinks earlier blocks): the third term
  * the context is rounded to fp16: 2^-11 |ref|, or 2^-25 once subnormal (last term)
  * w . |v| <= max |v|, so this is never looser than 2^-10 max|v| + 2^-11 |ref|, and it is much tighter where V is sparse,
    which the membership probes use.
Largest error seen, on an H100 80GB HBM3 at a 700 W power limit: 0.62 of the bound (per family in DESIGN.md section 5.2).
"""
import math

import pytest
import torch

MAX_S = 512           # AC_ENCODER_MAX_S: the bias table has 2 * MAX_S - 1 entries per head
INF = float("inf")

# kind -> (arch, head_dim): <64, ScorePlain>, <32, ScorePlain> and <64, ScoreRelBias> of each kernel, and ModernBERT
# (head_dim 64 with a band)
KINDS = {"dh64": ("bert", 64), "dh32": ("bert", 32), "bias": ("mpnet", 64), "modern": ("modernbert", 64)}
HEADS = {"dh64": 4, "dh32": 8, "bias": 4, "modern": 2}     # >= 3 heads where S stays <= 512: inner heads have two neighbours
BERT_KINDS = ["dh64", "dh32", "bias"]
ALL_KINDS = BERT_KINDS + ["modern"]


# ------------------------------------------------------------------------------------------------
# reference (device-agnostic fp64 torch; the CPU tests import it)
# ------------------------------------------------------------------------------------------------
def logits_ref(q, k, bias=None):
    """[B, heads, S, S] fp64: q . k / sqrt(dh) (+ bias[h, 511 + key - query]); q, k [B, S, heads, dh]"""
    q, k = q.double(), k.double()
    S, dh = q.shape[1], q.shape[3]
    x = torch.einsum("bqhd,bkhd->bhqk", q, k) / math.sqrt(dh)
    if bias is not None:
        pos = torch.arange(S, device=q.device)
        x = x + bias.double().to(q.device)[:, MAX_S - 1 + pos[None, :] - pos[:, None]][None]
    return x


def attended_ref(B, S, mask=None, window=0, device="cpu"):
    """[B, 1, S, S] bool: key is attended by query (not padded, inside the band)"""
    pos = torch.arange(S, device=device)
    att = torch.ones(B, 1, S, S, dtype=torch.bool, device=device)
    if mask is not None:
        att = att & (mask.to(device) != 0)[:, None, None, :]
    if window > 0:
        att = att & ((pos[:, None] - pos[None, :]).abs() <= window)[None, None]
    return att


def softmax_av(logits, att, v):
    """(context, error bound) [B, S, heads, dh] fp64 of softmax over the attended keys; rows without one are 0"""
    x = logits.masked_fill(~att, -INF)
    m = x.amax(-1, keepdim=True)
    p = torch.exp(x - torch.where(torch.isinf(m), torch.zeros_like(m), m))
    w = p / p.sum(-1, keepdim=True).clamp_min(1e-300)
    vv = v.double().permute(0, 2, 1, 3)
    out, wabs, reach = w @ vv, w @ vv.abs(), att.double() @ vv.abs()
    tol = 2.0 ** -10 * wabs + 2.0 ** -11 * out.abs() + 2.0 ** -25 * reach + 2.0 ** -24
    return out.permute(0, 2, 1, 3), tol.permute(0, 2, 1, 3)


def attention_ref(q, k, v, mask=None, window=0, bias=None):
    B, S = q.shape[:2]
    return softmax_av(logits_ref(q, k, bias), attended_ref(B, S, mask, window, q.device), v)


# ------------------------------------------------------------------------------------------------
# seeded inputs (built on the CPU in fp32, rounded to fp16: GPU and CPU tests see the same values)
# ------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def bias_table(heads, seed=3):
    """[heads, 1023] fp32, every entry distinct, spread of a few units: a bucketed table would hide an index that is off
    by one inside a bucket"""
    return 1.5 * torch.randn(heads, 2 * MAX_S - 1, generator=_gen(seed))


def random_qkv(B, S, heads, dh, logit_std, seed):
    """q, k, v [B, S, heads, dh] fp16; the scaled scores q.k / sqrt(dh) have standard deviation logit_std"""
    g = _gen(seed)
    a = math.sqrt(logit_std)
    q, k, v = (torch.randn(B, S, heads, dh, generator=g) for _ in range(3))
    return (a * q).half(), (a * k).half(), v.half()


def ramp_qkv(B, S, heads, dh, pattern, step, seed):
    """scores that follow the key index: `step` per 128-key block upwards ("rising": every block raises the running
    maximum), downwards ("falling": the maximum is in block 0) or up to a block in the middle and down again ("middle"),
    plus unit noise"""
    g = _gen(seed)
    u = torch.ones(dh)
    blk = torch.arange(S) / 128.0
    nblk = (S + 127) // 128
    level = {"rising": blk, "falling": S / 128.0 - blk, "middle": -(blk - (nblk // 2 + 0.4)).abs()}[pattern] * step
    q = u + 0.5 * torch.randn(B, S, heads, dh, generator=g)
    k = level[None, :, None, None] * u / dh ** 0.5 + torch.randn(B, S, heads, dh, generator=g)
    return q.half(), k.half(), torch.randn(B, S, heads, dh, generator=g).half()


def spike_qkv(B, S, heads, dh, key, seed, height=30.0):
    """unit-noise scores and one key about `height` above everything else"""
    g = _gen(seed)
    u = torch.ones(dh)
    q = u + 0.5 * torch.randn(B, S, heads, dh, generator=g)
    k = torch.randn(B, S, heads, dh, generator=g)
    k[:, key] += height / dh ** 0.5 * u
    return q.half(), k.half(), torch.randn(B, S, heads, dh, generator=g).half()


def probe_qkv(B, S, heads, dh, seed=0):
    """q = 0: P is exactly uniform over the attended keys (softmax of the bias row with MPNet).  V[b, key, h, :] is the
    unit vector (key + h + b) % dh, so output element d is the share of attended keys in residue class d: one key wrongly
    in or out moves it by a multiple of its own size once fewer than ~100 dh keys are attended"""
    q = torch.zeros(B, S, heads, dh)
    k = torch.randn(B, S, heads, dh, generator=_gen(seed))
    cls = (torch.arange(S)[None, :, None] + torch.arange(heads)[None, None, :] + torch.arange(B)[:, None, None]) % dh
    v = torch.nn.functional.one_hot(cls, dh).float()
    return q.half(), k.half(), v.half()


def make_mask(name, B, S):
    """[B, S] int32.  Sequence 0 is always full; the named pattern goes to the others (the last one for "empty")."""
    m = torch.ones(B, S, dtype=torch.int32)
    r = m[1:]
    if name == "right":                       # right padding, a different length per sequence
        for b in range(1, B):
            m[b, max(1, S - (S * b) // (B + 1)):] = 0
    elif name == "left":                      # left padding: for S > 256 the first two key blocks hold no valid key
        r[:, :(S * 5) // 8] = 0
    elif name == "hole":                      # whole key blocks missing in the middle
        r[:, S // 4:(S * 3) // 4] = 0
    elif name == "alternate":
        r[:, 1::2] = 0
    elif name.startswith("single"):           # one valid key: at 0, at the last key of the first key block, at S - 1
        at = {"single_first": 0, "single_block_end": min(127, S - 2), "single_last": S - 1}[name]
        r[:] = 0
        r[:, at] = 1
    elif name == "empty":                     # a sequence with no valid key next to normal ones
        m[B - 1] = 0
    else:
        assert name == "none"
        return None
    return m


# ------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------
def make_encoder(cabi, kind):
    """one dummy layer of tiny seeded weights: attention only needs heads, hidden, the arch and rel_bias"""
    arch, dh = KINDS[kind]
    heads = HEADS[kind]
    H, I, V = heads * dh, 64, 32
    g = _gen(11)
    r = lambda *s: (0.02 * torch.randn(*s, generator=g)).cuda()
    ones, zeros = (lambda n: torch.ones(n).cuda()), (lambda n: torch.zeros(n).cuda())
    common = dict(layers=1, hidden=H, heads=heads, intermediate=I, vocab=V, ln_eps=1e-5, max_tokens=16384)
    if arch == "modernbert":
        sd = {"embeddings.tok_embeddings.weight": r(V, H), "embeddings.norm.weight": ones(H), "final_norm.weight": ones(H),
              "layers.0.attn.Wqkv.weight": r(3 * H, H), "layers.0.attn.Wo.weight": r(H, H), "layers.0.mlp_norm.weight": ones(H),
              "layers.0.mlp.Wi.weight": r(2 * I, H), "layers.0.mlp.Wo.weight": r(H, I)}
        return cabi.Encoder(sd, arch=arch, max_pos=8192, sliding_window=64, layer_sliding=[1], rope_theta=(160000.0, 10000.0),
                            **common)
    p = "encoder.layer.0."
    sd = {"embeddings.word_embeddings.weight": r(V, H), "embeddings.position_embeddings.weight": r(MAX_S + 2, H),
          "embeddings.token_type_embeddings.weight": r(1, H), "embeddings.LayerNorm.weight": ones(H),
          "embeddings.LayerNorm.bias": zeros(H), p + "intermediate.dense.weight": r(I, H), p + "intermediate.dense.bias": zeros(I),
          p + "output.dense.weight": r(H, I), p + "output.dense.bias": zeros(H)}
    for n in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense"):
        sd[p + n + ".weight"], sd[p + n + ".bias"] = r(H, H), zeros(H)
    for n in ("attention.output.LayerNorm", "output.LayerNorm"):
        sd[p + n + ".weight"], sd[p + n + ".bias"] = ones(H), zeros(H)
    rel = bias_table(heads) if arch == "mpnet" else None
    return cabi.Encoder(sd, arch=arch, max_pos=MAX_S + 2, pad_idx=1 if arch == "mpnet" else 0, rel_bias=rel, **common)


WORST = {}      # family -> largest |out - ref| / bound seen


@pytest.fixture(scope="module")
def encoders(cabi):
    """kind -> handle, made on first use and shared by the module (so handles are reused across shapes all the time)"""
    made = {}

    def get(kind):
        if kind not in made:
            made[kind] = make_encoder(cabi, kind)
        return made[kind]
    yield get
    for e in made.values():
        e.close()
    print("\nlargest error / bound per family: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))


def run_case(enc, kind, q, k, v, mask=None, window=0, **kw):
    """kernel output [B, S, heads, dh] fp16; the pad keys of V^T hold 1000, which no correct kernel lets through"""
    dev = lambda t: None if t is None else t.cuda()
    return enc.attention(dev(q), dev(k), dev(v), dev(mask), window=window, pad_fill=1000.0, **kw)


def check(family, enc, kind, q, k, v, mask=None, window=0, rows=None):
    out = run_case(enc, kind, q, k, v, mask, window)
    bias = bias_table(HEADS[kind]) if kind == "bias" else None
    ref, tol = attention_ref(q.cuda(), k.cuda(), v.cuda(), mask, window, bias)
    assert torch.isfinite(out).all(), f"{family}: non-finite context"
    ratio = (out.double() - ref).abs() / tol
    worst = ratio.max().item()
    WORST[family] = max(WORST.get(family, 0.0), worst)
    if worst > 1.0:
        b, s, h, d = [int(i) for i in (ratio == ratio.max()).nonzero()[0]]
        pytest.fail(f"{family} {kind} S={q.shape[1]} window={window}: |out - ref| = {worst:.2f} x bound at (b={b}, q={s}, h={h}, "
                    f"d={d}): out {out[b, s, h, d].item():.6g} ref {ref[b, s, h, d].item():.6g}")
    return out


def shape(kind, B, S):
    return B, S, HEADS[kind], KINDS[kind][1]


pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("logit_std", [0.3, 8.0, 200.0])
@pytest.mark.parametrize("S", [100, 512])
@pytest.mark.parametrize("kind", ALL_KINDS)
def test_peaked_scores(encoders, kind, S, logit_std):
    """0.3 is what randomly initialised encoders produce (the control), 8 the range of trained ones, 200 the extreme"""
    q, k, v = random_qkv(*shape(kind, 3, S), logit_std, seed=S)
    check("peaked", encoders(kind), kind, q, k, v, make_mask("right", 3, S))


@pytest.mark.parametrize("pattern", ["rising", "falling", "middle"])
@pytest.mark.parametrize("kind,S,step", [("dh64", 512, 20.0), ("dh32", 512, 20.0), ("bias", 512, 20.0), ("modern", 1024, 20.0),
                                         ("modern", 8192, 20.0), ("modern", 8000, 3.0)])
def test_running_maximum_moves(encoders, kind, S, step, pattern):
    B = 1 if S > 1024 else 2
    q, k, v = ramp_qkv(*shape(kind, B, S), pattern, step, seed=S + len(pattern))
    check("max_moves", encoders(kind), kind, q, k, v)


@pytest.mark.parametrize("kind,S", [("dh64", 500), ("dh32", 500), ("bias", 500), ("modern", 1000)])
def test_one_dominant_key_in_each_key_block(encoders, kind, S):
    """the spike sits in every key block in turn, the last, partial one included, so the maximum jumps by ~30 there"""
    for blk in range((S + 127) // 128):
        key = min(128 * blk + 77, S - 1)
        q, k, v = spike_qkv(*shape(kind, 2, S), key, seed=blk)
        check("spike", encoders(kind), kind, q, k, v)


@pytest.mark.parametrize("key", [50, 31 * 128 + 127, 63 * 128 + 5, 8099])
def test_one_dominant_key_at_8192(encoders, key):
    q, k, v = spike_qkv(*shape("modern", 1, 8100), key, seed=key)
    check("spike", encoders("modern"), "modern", q, k, v)


@pytest.mark.parametrize("S", [100, 129, 300, 512, 513, 1000, 1025, 4096])
def test_band_membership_is_exact(encoders, S):
    """uniform probe: the output is the mean of V over the band, one key in or out is >= 10x the bound (test_attention_cpu)"""
    B = 1 if S > 1025 else 3
    q, k, v = probe_qkv(*shape("modern", B, S))
    for window in (1, 8, 63, 64, 127, 128, 129, S, S + 200):
        check("band", encoders("modern"), "modern", q, k, v, None, window)


@pytest.mark.parametrize("S", [100, 129, 300, 512])
def test_bias_row_is_exact_at_every_query_block(encoders, S):
    """q = 0 with MPNet: P is softmax(bias[h, 511 + key - query]); S = 512 covers the query blocks at 0, 128, 256, 384"""
    q, k, v = probe_qkv(*shape("bias", 3, S))
    check("bias_probe", encoders("bias"), "bias", q, k, v)
    check("bias_probe", encoders("bias"), "bias", q, k, v, make_mask("right", 3, S))


SHORT_S = [1, 7, 8, 9, 31, 33, 64, 100, 127, 128]
STREAM_S = [129, 136, 255, 256, 257, 384, 511, 512]


@pytest.mark.parametrize("S", SHORT_S + STREAM_S)
@pytest.mark.parametrize("kind", ALL_KINDS)
def test_sequence_length_seams(encoders, kind, S):
    """S that is not a multiple of 8 pads V^T; S < 8 runs like any other length"""
    q, k, v = random_qkv(*shape(kind, 3, S), 3.0, seed=1000 + S)
    check("seams", encoders(kind), kind, q, k, v, make_mask("right", 3, S))
    if kind == "modern":
        check("seams", encoders(kind), kind, q, k, v, make_mask("right", 3, S), window=5)


@pytest.mark.parametrize("S,B", [(513, 3), (1000, 3), (2049, 2), (8192, 1)])
def test_long_sequence_seams(encoders, S, B):
    q, k, v = random_qkv(*shape("modern", B, S), 3.0, seed=S)
    mask = make_mask("right", B, S)
    check("seams", encoders("modern"), "modern", q, k, v, mask)
    check("seams", encoders("modern"), "modern", q, k, v, mask, window=64)


MASKS = ["none", "right", "left", "hole", "alternate", "single_first", "single_block_end", "single_last", "empty"]


@pytest.mark.parametrize("name", MASKS)
@pytest.mark.parametrize("kind,S", [(kd, S) for kd in ALL_KINDS for S in (100, 500)] + [("modern", 1100)])
def test_masks(encoders, kind, S, name):
    q, k, v = random_qkv(*shape(kind, 3, S), 3.0, seed=S + len(name))
    out = check("masks", encoders(kind), kind, q, k, v, make_mask(name, 3, S))
    if name == "empty":
        assert (out[2] == 0).all()             # no valid key: exactly zero


@pytest.mark.parametrize("S,window", [(100, 8), (500, 64), (1100, 64), (1100, 200)])
def test_left_padding_under_a_band(encoders, S, window):
    """queries further than `window` before the first valid key see none (zeros) while their neighbours do"""
    mask = make_mask("left", 3, S)
    first = (S * 5) // 8
    q, k, v = probe_qkv(*shape("modern", 3, S))
    out = check("masks", encoders("modern"), "modern", q, k, v, mask, window)
    assert (out[1, :first - window] == 0).all() and (out[1, first - window:].float().abs().amax(-1) > 0).all()
    q, k, v = random_qkv(*shape("modern", 3, S), 8.0, seed=S)
    check("masks", encoders("modern"), "modern", q, k, v, mask, window)


@pytest.mark.parametrize("S", [100, 300])
@pytest.mark.parametrize("loud", [0, 1])
@pytest.mark.parametrize("kind", ALL_KINDS)
def test_heads_and_sequences_do_not_leak(encoders, kind, S, loud):
    """every second head (the TMA boxes of head_dim 32 carry the neighbouring head) and every second sequence is 10x
    louder in V and in the scores, both together 100x: a value read from a neighbour lands far outside a quiet head's
    bound.  loud = 0 / 1 swaps the roles, and the last head of the last sequence is quiet once and loud once"""
    B, _, heads, dh = shape(kind, 4, S)
    q, k, v = random_qkv(B, S, heads, dh, 1.0, seed=S + loud)
    for t, f in ((q, 10 ** 0.5), (k, 10 ** 0.5), (v, 10.0)):
        t[:, :, loud::2] *= f
        t[loud::2] *= f
    check("leak", encoders(kind), kind, q, k, v, make_mask("right", B, S))


@pytest.mark.parametrize("kind", ALL_KINDS)
def test_cls_rows_equal_the_full_launch_bitwise(encoders, kind):
    q, k, v = random_qkv(*shape(kind, 3, 300), 8.0, seed=5)
    mask = make_mask("right", 3, 300)
    full = run_case(encoders(kind), kind, q, k, v, mask)
    first = run_case(encoders(kind), kind, q, k, v, mask, cls_rows=True)
    assert torch.equal(first[:, :128], full[:, :128])


@pytest.mark.parametrize("kind", ALL_KINDS)
def test_handle_reuse_is_bitwise_stable(cabi, encoders, kind):
    """a large shape, a smaller S that is not a multiple of 8, the large one again: each equals a fresh handle's result
    (the V^T view is cached per (B, S); the smaller shape leaves the larger one's data behind its rows)"""
    cases = [(3, 512), (2, 77), (3, 512), (3, 512), (5, 77)]
    used = encoders(kind)
    for i, (B, S) in enumerate(cases):
        q, k, v = random_qkv(*shape(kind, B, S), 8.0, seed=S + B)
        mask = make_mask("right", B, S)
        fresh = make_encoder(cabi, kind)
        want = run_case(fresh, kind, q, k, v, mask)
        fresh.close()
        assert torch.equal(run_case(used, kind, q, k, v, mask), want), f"call {i}: B={B} S={S}"


def test_shapes_are_refused_by_name(cabi, encoders):
    q, k, v = random_qkv(*shape("dh64", 1, 513), 1.0, seed=0)
    with pytest.raises(cabi.AdaptiveB200Error, match="S=513 > 512 is not supported"):
        run_case(encoders("dh64"), "dh64", q, k, v)
    q, k, v = random_qkv(*shape("dh64", 1, 64), 1.0, seed=0)
    with pytest.raises(cabi.AdaptiveB200Error, match="window=4 needs an AC_ARCH_MODERNBERT encoder"):
        run_case(encoders("dh64"), "dh64", q, k, v, window=4)
    q, k, v = random_qkv(*shape("modern", 3, 8192), 1.0, seed=0)
    with pytest.raises(cabi.AdaptiveB200Error, match="exceeds max_tokens=16384"):
        run_case(encoders("modern"), "modern", q, k, v)
