// head.cu -- stage H: AdaptiveHead inference forward, the training / gradient entry points (one persistent cooperative
// kernel per call: head_train.cuh) and the stand-alone EWC penalty.  fp32 SIMT.
//
// Replaces (paths relative to /root/reference/src/adaptive_classifier/):
//   models.py:71-80                 AdaptiveHead.forward (Linear-ReLU-Dropout x2, Linear)
//   classifier.py:333-351,1489-1505 zero_grad / forward / CrossEntropyLoss / backward / clip_grad_norm_(1.0) / AdamW.step
//   multilabel.py:41-44,387-397     sigmoid head + BCELoss
//   ewc.py:67-92, :96-115           Fisher accumulation and penalty
#include "common.cuh"
#include "head_train.cuh"
#include <math_constants.h>

namespace ac {

enum { EPI_NONE = 0, EPI_BIAS = 1, EPI_BIAS_RELU = 2 };
struct SgemmEpi {
    int kind;
    const float *bias;     // [N]
};

// ------------------------------------------------------------------------------------------------
// inference forward: skinny linears (M = batch rows, 32 per pass)
// rowdot   Y[b,n] = epi( sum_k X[b,k] * W[n,k] + bias[n] )      W row-major [N,K] (nn.Linear layout)
//          warp = 4 output columns x 32 batch rows, lanes stride K, warp transpose-reduce at the end; fixed summation order
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float epi_apply(const SgemmEpi &epi, float v, int n, int64_t off) {
    switch (epi.kind) {
        case EPI_BIAS: v += epi.bias[n]; break;
        case EPI_BIAS_RELU: v = fmaxf(v + epi.bias[n], 0.f); break;
        default: break;
    }
    return v;
}

// after the call lane l holds the sum over all lanes of their v[l]
__device__ __forceinline__ float warp_transpose_reduce(float (&v)[32], int lane) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < off; ++i) {
            const float send = upper ? v[i] : v[i + off];
            const float keep = upper ? v[i + off] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
    }
    return v[0];
}

constexpr int RD_WARPS = 8;

// RD_COLS output columns per warp: 4 when there are many row blocks (re-use of the X loads), 1 for a single 32-row
// batch so that a 768-column layer still spreads over 96 CTAs
template <int RD_COLS>
__global__ void __launch_bounds__(RD_WARPS * 32)
rowdot_kernel(const float *__restrict__ X, const float *__restrict__ W, float *__restrict__ Y, int M, int N, int K,
              SgemmEpi epi) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = (blockIdx.x * RD_WARPS + warp) * RD_COLS;
    const int b0 = blockIdx.y * 32;
    if (n0 >= N) return;
    float acc[RD_COLS][32];
#pragma unroll
    for (int c = 0; c < RD_COLS; ++c)
#pragma unroll
        for (int b = 0; b < 32; ++b) acc[c][b] = 0.f;
    const int rows = min(32, M - b0);
#pragma unroll 2
    for (int k = lane; k < K; k += 32) {
        float w[RD_COLS];
#pragma unroll
        for (int c = 0; c < RD_COLS; ++c) w[c] = (n0 + c < N) ? __ldg(W + static_cast<int64_t>(n0 + c) * K + k) : 0.f;
#pragma unroll
        for (int b = 0; b < 32; ++b) {
            const float x = (b < rows) ? __ldg(X + static_cast<int64_t>(b0 + b) * K + k) : 0.f;
#pragma unroll
            for (int c = 0; c < RD_COLS; ++c) acc[c][b] = fmaf(x, w[c], acc[c][b]);
        }
    }
#pragma unroll
    for (int c = 0; c < RD_COLS; ++c) {
        const float s = warp_transpose_reduce(acc[c], lane);     // lane = batch row
        const int n = n0 + c, m = b0 + lane;
        if (n < N && lane < rows) {
            const int64_t off = static_cast<int64_t>(m) * N + n;
            Y[off] = epi_apply(epi, s, n, off);
        }
    }
}

// batched forward (M > 64 rows, the predict step at B = 512): Y[m,n] = epi( sum_k X[m,k] W[n,k] ), both operands K-major.
// 64 x 64 tile, 256 threads x (4 x 4) outputs, K in slabs of 16 staged transposed in shared memory ([k][row], padded), next slab
// prefetched into registers.  k is added in ascending order per output.  (rowdot_kernel<4> needs 255 registers -- a whole SM's
// register file per CTA, so on the side stream it could not share an SM with the prototype scan.)
constexpr int SG_T = 64, SG_K = 16;
__global__ void __launch_bounds__(256)
sgemm_nt_kernel(const float *__restrict__ X, const float *__restrict__ W, float *__restrict__ Y, int M, int N, int K, SgemmEpi epi) {
    __shared__ __align__(16) float sx[2][SG_K][SG_T + 4];
    __shared__ __align__(16) float sw[2][SG_K][SG_T + 4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * SG_T, n0 = blockIdx.x * SG_T;
    const int tx = tid & 15, ty = tid >> 4;                 // outputs: rows m0 + 4 ty .. +3, columns n0 + 4 tx .. +3
    const int lr = tid >> 2, lk = (tid & 3) * 4;            // loader: row lr of the tile, 4 consecutive k
    const bool vec = (K & 3) == 0;
    auto load4 = [&](const float *base, int row, int rows, int k) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < rows) {
            const float *p = base + static_cast<int64_t>(row) * K + k;
            if (vec && k + 4 <= K) v = __ldg(reinterpret_cast<const float4 *>(p));
            else {
                if (k + 0 < K) v.x = __ldg(p + 0);
                if (k + 1 < K) v.y = __ldg(p + 1);
                if (k + 2 < K) v.z = __ldg(p + 2);
                if (k + 3 < K) v.w = __ldg(p + 3);
            }
        }
        return v;
    };
    auto stage = [&](float (*dst)[SG_T + 4], const float4 &v) {
        dst[lk + 0][lr] = v.x; dst[lk + 1][lr] = v.y; dst[lk + 2][lr] = v.z; dst[lk + 3][lr] = v.w;
    };
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float4 rx = load4(X, m0 + lr, M, lk), rw = load4(W, n0 + lr, N, lk);
    const int nslab = (K + SG_K - 1) / SG_K;
    for (int sl = 0; sl < nslab; ++sl) {
        const int buf = sl & 1;
        stage(sx[buf], rx);
        stage(sw[buf], rw);
        __syncthreads();
        if (sl + 1 < nslab) {
            rx = load4(X, m0 + lr, M, (sl + 1) * SG_K + lk);
            rw = load4(W, n0 + lr, N, (sl + 1) * SG_K + lk);
        }
#pragma unroll
        for (int k = 0; k < SG_K; ++k) {
            const float4 a = *reinterpret_cast<const float4 *>(&sx[buf][k][4 * ty]);
            const float4 b = *reinterpret_cast<const float4 *>(&sw[buf][k][4 * tx]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        // the buffer written two slabs from now is this one: the barrier at the top of the next iteration orders it
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + 4 * ty + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + 4 * tx + j;
            if (n < N) {
                const int64_t off = static_cast<int64_t>(m) * N + n;
                Y[off] = epi_apply(epi, acc[i][j], n, off);
            }
        }
    }
}

static int rowdot(const float *X, const float *W, float *Y, int M, int N, int K, SgemmEpi epi, cudaStream_t s) {
    if (M <= 0 || N <= 0) return AC_OK;
    if (M <= 64) {
        dim3 grid((N + RD_WARPS - 1) / RD_WARPS, (M + 31) / 32);
        rowdot_kernel<1><<<grid, RD_WARPS * 32, 0, s>>>(X, W, Y, M, N, K, epi);
    } else {
        dim3 grid((N + SG_T - 1) / SG_T, (M + SG_T - 1) / SG_T);
        sgemm_nt_kernel<<<grid, 256, 0, s>>>(X, W, Y, M, N, K, epi);
    }
    AC_LAUNCH_CHECK();
    return AC_OK;
}

// y[m,n] = act(X W^T + b)
static int linear_fwd(const float *X, const float *W, const float *b, float *Y, int M, int N, int K, int kind, cudaStream_t s) {
    SgemmEpi e{kind, b};
    return rowdot(X, W, Y, M, N, K, e, s);
}

// ------------------------------------------------------------------------------------------------
// row-wise output activations / losses
// ------------------------------------------------------------------------------------------------
__global__ void softmax_rows_kernel(const float *__restrict__ z, int B, int C, float *__restrict__ out, int act) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= B) return;
    const float *zr = z + static_cast<int64_t>(row) * C;
    float *orow = out + static_cast<int64_t>(row) * C;
    if (act == AC_ACT_SIGMOID) {
        for (int j = lane; j < C; j += 32) orow[j] = 1.f / (1.f + expf(-zr[j]));
        return;
    }
    float mx = -CUDART_INF_F;
    for (int j = lane; j < C; j += 32) mx = fmaxf(mx, zr[j]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j < C; j += 32) sum += expf(zr[j] - mx);
    sum = warp_sum(sum);
    for (int j = lane; j < C; j += 32) orow[j] = expf(zr[j] - mx) / sum;
}

// ------------------------------------------------------------------------------------------------
// flat parameter views: 6 tensors {W0,b0,W1,b1,W2,b2}
// ------------------------------------------------------------------------------------------------
struct Flat6 {
    float *p[6];
    int64_t n[6];
};
static Flat6 flat_of(const ac_head_params *h) {
    Flat6 f;
    f.p[0] = h->W0; f.n[0] = static_cast<int64_t>(h->H0) * h->D;
    f.p[1] = h->b0; f.n[1] = h->H0;
    f.p[2] = h->W1; f.n[2] = static_cast<int64_t>(h->H1) * h->H0;
    f.p[3] = h->b1; f.n[3] = h->H1;
    f.p[4] = h->W2; f.n[4] = static_cast<int64_t>(h->C) * h->H1;
    f.p[5] = h->b2; f.n[5] = h->C;
    return f;
}

// EWC: g += 2*lam*invB * F * (theta - theta*) over the first `n_lim` elements of each tensor;
// penalty partial sums (F*(theta-theta*)^2) go to partial[blockIdx] for a deterministic second stage.
__global__ void ewc_grad_penalty_kernel(Flat6 theta, Flat6 fisher, Flat6 star, Flat6 grad, Flat6 lim, float scale2,
                                        float *__restrict__ partial, int add_grad) {
    __shared__ float red[256];
    float local = 0.f;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int t = 0; t < 6; ++t) {
        const int64_t n = lim.n[t];
        for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
            const float diff = theta.p[t][i] - star.p[t][i];
            const float f = fisher.p[t][i];
            local += f * diff * diff;
            if (add_grad) grad.p[t][i] += scale2 * f * diff;
        }
    }
    red[threadIdx.x] = local;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

// finalize: out[0] = scale * sum(partial) (ewc penalty) or sqrt(sum) (grad norm)
__global__ void finalize_kernel(const float *__restrict__ partial, int n, float scale, int take_sqrt,
                                float *__restrict__ out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < n; ++i) s += partial[i];
        out[0] = take_sqrt ? sqrtf(s) : scale * s;
    }
}

constexpr int RED_BLOCKS = 64;

static int check_params(const ac_head_params *p, const char *who) {
    AC_REQUIRE(p && p->D > 0 && p->H0 > 0 && p->H1 > 0 && p->C > 0, "%s: bad head dims", who);
    AC_REQUIRE(p->W0 && p->b0 && p->W1 && p->b1 && p->W2 && p->b2, "%s: null head parameter", who);
    return AC_OK;
}

// ------------------------------------------------------------------------------------------------
// launch plan of head_train_kernel (head_train.cuh): grid size, ownership slots, global scratch
// ------------------------------------------------------------------------------------------------
struct TrainPlan {
    int G, nst, res_mv;
    size_t off_h0d, off_h1d, off_z, off_dz, off_da1, off_rowloss, off_part, off_pen, off_bar, off_stats, total;
    size_t smem_bytes;
};

static void plan_args(ht::Args &a, int batch, const ac_head_params *p, int G) {
    const int rows[3] = {p->H0, p->H1, p->C}, K[3] = {p->D, p->H0, p->H1};
    a.batch = batch;
    for (int l = 0; l < 3; ++l) { a.L[l].rows = rows[l]; a.L[l].K = K[l]; }
    ht::ht_assign(a, G);
}

static int plan_training(int batch, const ac_head_params *p, int n_steps, bool update, TrainPlan &pl, const char *who) {
    AC_REQUIRE(batch >= 1 && batch <= ht::HT_MAXB, "%s: batch=%d outside [1,%d]", who, batch, ht::HT_MAXB);
    AC_REQUIRE(p->D % 4 == 0 && p->H0 % 4 == 0 && p->H1 % 4 == 0, "%s: D, H0, H1 must be multiples of 4 (D=%d H0=%d H1=%d)", who, p->D,
               p->H0, p->H1);
    AC_REQUIRE(p->D <= 2048 && p->H0 <= 2048 && p->H1 <= 2048, "%s: layer widths above 2048 are not supported", who);
    AC_REQUIRE(n_steps <= (1 << 20), "%s: at most 2^20 steps per launch", who);
    // one CTA per SM at most (cooperative launch: all CTAs resident).  The 8-row blocks of the three layers are dealt round robin:
    // the reference's head (768 -> 768 -> 384 -> C <= 32) has 96 + 48 + 4 = 148 blocks, dealt over the 132 SMs of an H100
    ht::Args a{};
    plan_args(a, batch, p, 1);
    int G = sm_count();
    if (a.items < G) G = a.items;               // tiny heads: no idle CTAs spinning in the barriers
    pl.G = G;
    plan_args(a, batch, p, G);
    // AdamW moments resident in shared memory if at least three ring stages still fit; then as many stages (<= 8) as there is room
    // for, but no more than the longest product has chunks plus one: a deeper ring is never filled and only takes shared memory
    const size_t limit = 220 * 1024;
    pl.smem_bytes = ~size_t(0);
    constexpr int res_min_nst = 3;      // resident moments must leave room for at least three ring stages; otherwise they stay in L2
    const int nst_useful = (a.kmax + ht::HT_KC - 1) / ht::HT_KC + 1;
    const int nst_max = nst_useful < res_min_nst ? res_min_nst : (nst_useful > 8 ? 8 : nst_useful);
    for (int res = update ? 1 : 0; res >= 0; --res) {
        a.res_mv = res;
        for (a.nst = nst_max; a.nst >= (res ? res_min_nst : 2); --a.nst) {
            const size_t bytes = static_cast<size_t>(ht::ht_smem_layout(a).total) * sizeof(float);
            if (bytes <= limit) { pl.smem_bytes = bytes; break; }
        }
        if (pl.smem_bytes <= limit) break;
    }
    if (pl.smem_bytes > limit) {
        a.res_mv = 0; a.nst = 2;
        set_error("%s: head %d -> %d -> %d -> %d needs %zu bytes of shared memory per CTA (limit 220 KB)", who, p->D, p->H0, p->H1, p->C,
                  static_cast<size_t>(ht::ht_smem_layout(a).total) * sizeof(float));
        return AC_E_UNSUPPORTED;
    }
    pl.nst = a.nst;
    pl.res_mv = a.res_mv;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
    pl.off_h0d = take(sizeof(float) * batch * p->H0);
    pl.off_h1d = take(sizeof(float) * batch * p->H1);
    pl.off_z = take(sizeof(float) * batch * p->C);
    pl.off_dz = take(sizeof(float) * batch * a.ldz);
    pl.off_da1 = take(sizeof(float) * batch * p->H1);
    pl.off_rowloss = take(sizeof(float) * batch);
    pl.off_part = take(sizeof(float) * 256);
    pl.off_pen = take(sizeof(float) * 256);
    pl.off_bar = take(256);
    pl.off_stats = take(sizeof(float) * 3 * (n_steps > 0 ? n_steps : 1));
    pl.total = off;
    return AC_OK;
}

static unsigned long long *g_head_timing_dev = nullptr;

struct TrainCall {
    const float *X; const void *targets; const int64_t *perm; int n, batch, n_steps, first_step;
    ac_head_params *p, *m, *v;                 // m, v NULL in gradient-only mode
    const ac_train_cfg *cfg;                   // NULL in gradient-only mode
    int loss_kind;
    ac_head_params *grad_out, *fisher; float fisher_scale;
    float *stats;                              // [n_steps, 3] device (nullable -> internal)
    float *loss_accum;
};

static int launch_training(const TrainCall &c, void *workspace, size_t workspace_bytes, cudaStream_t s, const char *who,
                           float **stats_out) {
    int rc = ac_device_check();
    if (rc) return rc;
    TrainPlan pl;
    const bool update = c.m && c.v;
    if ((rc = plan_training(c.batch, c.p, c.n_steps, update, pl, who))) return rc;
    uint8_t *w = reinterpret_cast<uint8_t *>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
    const size_t slack = w - static_cast<uint8_t *>(workspace);
    if (pl.total + slack > workspace_bytes) { set_error("%s: workspace needs %zu bytes", who, pl.total + 256); return AC_E_WORKSPACE; }
    ht::Args a{};
    a.X = c.X; a.targets = c.targets; a.perm = c.perm; a.n = c.n; a.batch = c.batch; a.n_steps = c.n_steps; a.first_step = c.first_step;
    const ac_head_params *P = c.p;
    float *Wp[3] = {P->W0, P->W1, P->W2}, *bp[3] = {P->b0, P->b1, P->b2};
    const int rows[3] = {P->H0, P->H1, P->C}, K[3] = {P->D, P->H0, P->H1};
    const ac_train_cfg *cfg = c.cfg;
    const bool ewc = cfg && cfg->ewc_fisher && cfg->ewc_star;
    for (int l = 0; l < 3; ++l) {
        ht::Layer &Lr = a.L[l];
        Lr.W = Wp[l]; Lr.b = bp[l]; Lr.rows = rows[l]; Lr.K = K[l]; Lr.ewc_rows = rows[l];
#define AC_PICK(hp, l) ((l) == 0 ? (hp)->W0 : (l) == 1 ? (hp)->W1 : (hp)->W2)
#define AC_PICKB(hp, l) ((l) == 0 ? (hp)->b0 : (l) == 1 ? (hp)->b1 : (hp)->b2)
        if (c.m && c.v) { Lr.mW = AC_PICK(c.m, l); Lr.mb = AC_PICKB(c.m, l); Lr.vW = AC_PICK(c.v, l); Lr.vb = AC_PICKB(c.v, l); }
        if (ewc) {
            Lr.fW = AC_PICK(cfg->ewc_fisher, l); Lr.fb = AC_PICKB(cfg->ewc_fisher, l);
            Lr.sW = AC_PICK(cfg->ewc_star, l); Lr.sb = AC_PICKB(cfg->ewc_star, l);
        }
        if (c.grad_out) { Lr.gW = AC_PICK(c.grad_out, l); Lr.gb = AC_PICKB(c.grad_out, l); }
        if (c.fisher) { Lr.qW = AC_PICK(c.fisher, l); Lr.qb = AC_PICKB(c.fisher, l); }
#undef AC_PICK
#undef AC_PICKB
    }
    // the head may have grown since theta* was taken: only the first C_old output rows are penalised (ewc.py:96-115 on the old head)
    if (ewc && cfg->ewc_C_old > 0 && cfg->ewc_C_old < P->C) a.L[2].ewc_rows = cfg->ewc_C_old;
    a.update = update ? 1 : 0;
    ht::ht_assign(a, pl.G);
    a.nst = pl.nst;
    a.res_mv = pl.res_mv;
    // 16-byte asynchronous copies stream X rows and gather W1 / W2 columns
    AC_REQUIRE((reinterpret_cast<uintptr_t>(c.X) | reinterpret_cast<uintptr_t>(P->W0) | reinterpret_cast<uintptr_t>(P->W1) |
                reinterpret_cast<uintptr_t>(P->W2)) % 16 == 0, "%s: X and the weight matrices must be 16-byte aligned", who);
    if (update) AC_REQUIRE((reinterpret_cast<uintptr_t>(c.m->W0) | reinterpret_cast<uintptr_t>(c.m->W1) | reinterpret_cast<uintptr_t>(c.m->W2) |
                            reinterpret_cast<uintptr_t>(c.v->W0) | reinterpret_cast<uintptr_t>(c.v->W1) | reinterpret_cast<uintptr_t>(c.v->W2)) % 16 == 0,
                           "%s: the moment matrices must be 16-byte aligned", who);
    if (ewc) AC_REQUIRE((reinterpret_cast<uintptr_t>(a.L[0].fW) | reinterpret_cast<uintptr_t>(a.L[1].fW) | reinterpret_cast<uintptr_t>(a.L[2].fW) |
                         reinterpret_cast<uintptr_t>(a.L[0].sW) | reinterpret_cast<uintptr_t>(a.L[1].sW) | reinterpret_cast<uintptr_t>(a.L[2].sW)) % 16 == 0,
                        "%s: the EWC matrices must be 16-byte aligned", who);
    if (cfg) {
        a.lr = cfg->lr; a.beta1 = cfg->beta1; a.beta2 = cfg->beta2; a.eps = cfg->eps; a.wd = cfg->weight_decay; a.max_norm = cfg->max_norm;
        a.dropout_p = cfg->dropout_p; a.seed = cfg->seed; a.mask0 = cfg->mask0; a.mask1 = cfg->mask1;
        if (cfg->dropout_p > 0.f && cfg->mask0 && cfg->mask1) a.dropout_p = cfg->dropout_p;      // injected masks carry their own scale
        a.use_ewc = ewc ? 1 : 0; a.ewc_lambda = cfg->ewc_lambda;
        a.n_regular = cfg->n_regular; a.strategic_lambda = cfg->strategic_lambda;
    }
    if (c.loss_kind == AC_LOSS_CE_STRATEGIC)
        AC_REQUIRE(cfg && c.n_steps == 1 && cfg->n_regular >= 1 && c.n == 2 * cfg->n_regular,
                   "%s: AC_LOSS_CE_STRATEGIC steps one batch of 2 * n_regular rows (n=%d, n_regular=%d)", who, c.n, cfg ? cfg->n_regular : 0);
    a.loss_kind = c.loss_kind;
    a.fisher_scale = c.fisher_scale;
    a.h0d = reinterpret_cast<float *>(w + pl.off_h0d); a.h1d = reinterpret_cast<float *>(w + pl.off_h1d);
    a.z = reinterpret_cast<float *>(w + pl.off_z); a.dz = reinterpret_cast<float *>(w + pl.off_dz);
    a.da1 = reinterpret_cast<float *>(w + pl.off_da1); a.rowloss = reinterpret_cast<float *>(w + pl.off_rowloss);
    a.part = reinterpret_cast<float *>(w + pl.off_part); a.pen = reinterpret_cast<float *>(w + pl.off_pen);
    a.bar = reinterpret_cast<unsigned *>(w + pl.off_bar);
    a.stats = c.stats ? c.stats : reinterpret_cast<float *>(w + pl.off_stats);
    a.loss_accum = c.loss_accum;
    if (stats_out) *stats_out = a.stats;
    AC_CUDA(cudaMemsetAsync(a.bar, 0, 256, s));
    if (g_head_timing_dev) {               // diagnostic: per-phase nanoseconds of CTA 0 (ac_head_phase_timing)
        a.timing = g_head_timing_dev;
    }
    const bool strat = c.loss_kind == AC_LOSS_CE_STRATEGIC;
    const void *kern = strat ? reinterpret_cast<const void *>(ht::head_train_kernel<true>) : reinterpret_cast<const void *>(ht::head_train_kernel<false>);
    static bool attr_set[2][64] = {};
    int dev = 0;
    AC_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !attr_set[strat][dev]) {
        AC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
        if (dev >= 0 && dev < 64) attr_set[strat][dev] = true;
    }
    void *args[] = {&a};
    AC_CUDA(cudaLaunchCooperativeKernel(kern, dim3(pl.G), dim3(ht::HT_THREADS), args,
                                        pl.smem_bytes, s));
    count_launch();
    return AC_OK;
}

}  // namespace ac

using namespace ac;

extern "C" int ac_head_forward(const float *X, int B, const ac_head_params *p, int act, float *out, float *scratch,
                               size_t scratch_floats, ac_stream_t stream) {
    int rc = check_params(p, "ac_head_forward");
    if (rc) return rc;
    AC_REQUIRE(X && out && B >= 0, "ac_head_forward: bad arguments");
    if (B == 0) return AC_OK;
    const size_t need = static_cast<size_t>(B) * (p->H0 + p->H1);
    if (!scratch || scratch_floats < need) {
        set_error("ac_head_forward: scratch needs %zu floats", need);
        return AC_E_WORKSPACE;
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    float *h0 = scratch, *h1 = scratch + static_cast<size_t>(B) * p->H0;
    if ((rc = linear_fwd(X, p->W0, p->b0, h0, B, p->H0, p->D, EPI_BIAS_RELU, s))) return rc;
    if ((rc = linear_fwd(h0, p->W1, p->b1, h1, B, p->H1, p->H0, EPI_BIAS_RELU, s))) return rc;
    if ((rc = linear_fwd(h1, p->W2, p->b2, out, B, p->C, p->H1, EPI_BIAS, s))) return rc;
    if (act == AC_ACT_SOFTMAX || act == AC_ACT_SIGMOID) {
        const int wpb = 4;
        softmax_rows_kernel<<<(B + wpb - 1) / wpb, wpb * 32, 0, s>>>(out, B, p->C, out, act);
        AC_LAUNCH_CHECK();
    }
    return AC_OK;
}

// diagnostic (tools/head_phase_times.py): enable != 0 starts accumulating, per training launch, the nanoseconds three observed CTAs
// (the first holder of a layer-0 block, of a layer-1 block, and the last CTA: layer 2) spend in every phase of head_train_kernel,
// in the grid barriers between them and inside the two product routines; out72_host (nullable) receives 3 x 24 counters so far
extern "C" int ac_head_phase_timing(int enable, unsigned long long *out72_host) {
    if (enable && !g_head_timing_dev) {
        AC_CUDA(cudaMalloc(reinterpret_cast<void **>(&g_head_timing_dev), 3 * ht::HT_TROW * sizeof(unsigned long long)));
        AC_CUDA(cudaMemset(g_head_timing_dev, 0, 3 * ht::HT_TROW * sizeof(unsigned long long)));
    }
    if (out72_host && g_head_timing_dev) {
        AC_CUDA(cudaDeviceSynchronize());
        AC_CUDA(cudaMemcpy(out72_host, g_head_timing_dev, 3 * ht::HT_TROW * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    }
    if (!enable && g_head_timing_dev) {
        cudaFree(g_head_timing_dev);
        g_head_timing_dev = nullptr;
    }
    return AC_OK;
}

// diagnostic: the launch plan of the training kernel for this head and batch size: grid size, ring stages, moments resident in
// shared memory (0/1), dynamic shared memory bytes, reserved
extern "C" int ac_head_train_plan(int batch, const ac_head_params *p, int *out5) {
    AC_REQUIRE(p && out5 && batch > 0, "ac_head_train_plan: bad arguments");
    TrainPlan pl;
    int rc = plan_training(batch, p, 1, true, pl, "ac_head_train_plan");
    if (rc) return rc;
    out5[0] = pl.G; out5[1] = pl.nst; out5[2] = pl.res_mv; out5[3] = static_cast<int>(pl.smem_bytes);
    out5[4] = 0;   // reserved
    return AC_OK;
}

extern "C" int ac_head_train_workspace_bytes(int batch, int n_steps, const ac_head_params *p, size_t *bytes) {
    AC_REQUIRE(p && bytes && batch > 0, "ac_head_train_workspace_bytes: bad arguments");
    TrainPlan pl;
    int rc = plan_training(batch, p, n_steps, true, pl, "ac_head_train_workspace_bytes");
    if (rc) return rc;
    *bytes = pl.total + 512;
    return AC_OK;
}

extern "C" int ac_head_train_step(const float *X, const void *targets, int B, ac_head_params *p, ac_head_params *m,
                                  ac_head_params *v, const ac_train_cfg *cfg, float *out_stats, void *workspace,
                                  size_t workspace_bytes, ac_stream_t stream) {
    int rc = check_params(p, "ac_head_train_step");
    if (rc) return rc;
    AC_REQUIRE(X && targets && B > 0 && m && v && cfg && out_stats && workspace, "ac_head_train_step: bad arguments");
    AC_REQUIRE(cfg->step >= 1, "ac_head_train_step: step must be >= 1");
    TrainCall c{X, targets, nullptr, B, B, 1, cfg->step, p, m, v, cfg, cfg->loss_kind, nullptr, nullptr, 0.f, out_stats, nullptr};
    return launch_training(c, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), "ac_head_train_step", nullptr);
}

extern "C" int ac_head_train_epoch(const float *X, const void *targets, const int64_t *perm, int n, int batch,
                                   ac_head_params *p, ac_head_params *m, ac_head_params *v, const ac_train_cfg *cfg,
                                   float *loss_accum, float *step_stats, void *workspace, size_t workspace_bytes, ac_stream_t stream) {
    int rc = check_params(p, "ac_head_train_epoch");
    if (rc) return rc;
    AC_REQUIRE(X && targets && n > 0 && batch > 0 && m && v && cfg && workspace, "ac_head_train_epoch: bad arguments");
    AC_REQUIRE(cfg->step >= 1 && !cfg->mask0 && !cfg->mask1, "ac_head_train_epoch: step >= 1 and no injected masks");
    const int steps = (n + batch - 1) / batch;      // DataLoader keeps the last partial batch
    TrainCall c{X, targets, perm, n, batch, steps, cfg->step, p, m, v, cfg, cfg->loss_kind, nullptr, nullptr, 0.f, step_stats, loss_accum};
    return launch_training(c, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), "ac_head_train_epoch", nullptr);
}

extern "C" int ac_head_grad(const float *X, const void *targets, int B, const ac_head_params *p, int loss_kind,
                            ac_head_params *grad_out, ac_head_params *fisher_accum, float inv_n_batches,
                            float *out_loss, void *workspace, size_t workspace_bytes, ac_stream_t stream) {
    int rc = check_params(p, "ac_head_grad");
    if (rc) return rc;
    AC_REQUIRE(X && targets && B > 0 && out_loss && workspace, "ac_head_grad: bad arguments");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    TrainCall c{X, targets, nullptr, B, B, 1, 1, const_cast<ac_head_params *>(p), nullptr, nullptr, nullptr, loss_kind, grad_out,
                fisher_accum, inv_n_batches, nullptr, nullptr};
    float *stats = nullptr;
    if ((rc = launch_training(c, workspace, workspace_bytes, s, "ac_head_grad", &stats))) return rc;
    AC_CUDA(cudaMemcpyAsync(out_loss, stats, sizeof(float), cudaMemcpyDeviceToDevice, s));
    return AC_OK;
}

// ------------------------------------------------------------------------------------------------
// strategic training (classifier.py:1602-1647, strategic.py:200-242): per step gather the batch, search its best responses in
// train mode (strategic.cu), one optimizer step on [x ; br]
// ------------------------------------------------------------------------------------------------
constexpr int ST_MAX_BATCH = 16;       // DataLoader(batch_size=min(16, N)) of the reference

// rows [0, Bt) of Xa / ta: the batch's rows and targets through the permutation; targets [Bt, 2 Bt) repeat them
__global__ void strategic_gather_kernel(const float *__restrict__ X, const int64_t *__restrict__ targets, const int64_t *__restrict__ perm,
                                        int Bt, int D, float *__restrict__ Xa, int64_t *__restrict__ ta) {
    const int r = blockIdx.x;
    const int64_t src = perm[r];
    for (int k = threadIdx.x; k < D; k += blockDim.x) Xa[static_cast<int64_t>(r) * D + k] = X[src * D + k];
    if (threadIdx.x == 0) { ta[r] = targets[src]; ta[Bt + r] = targets[src]; }
}

struct StLayout { size_t xa, ta, choice, util, train, search, total; };
static int st_layout(int n, const ac_head_params *p, StLayout &l, const char *who) {
    const int batch = n < ST_MAX_BATCH ? n : ST_MAX_BATCH;
    TrainPlan pl;
    int rc = plan_training(2 * batch, p, 1, true, pl, who);
    if (rc) return rc;
    size_t search = 0;
    if ((rc = ac_strategic_workspace_bytes(batch, p, &search))) return rc;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
    l.xa = take(sizeof(float) * 2 * batch * p->D);
    l.ta = take(sizeof(int64_t) * 2 * batch);
    l.choice = take(sizeof(int32_t) * batch);
    l.util = take(sizeof(float) * batch);
    l.train = take(pl.total + 512);
    l.search = take(search);
    l.total = off + 256;
    return AC_OK;
}

extern "C" int ac_head_train_strategic_workspace_bytes(int n, const ac_head_params *p, size_t *bytes) {
    int rc = check_params(p, "ac_head_train_strategic_workspace_bytes");
    if (rc) return rc;
    AC_REQUIRE(bytes && n > 0, "ac_head_train_strategic_workspace_bytes: bad arguments");
    StLayout l;
    if ((rc = st_layout(n, p, l, "ac_head_train_strategic_workspace_bytes"))) return rc;
    *bytes = l.total;
    return AC_OK;
}

extern "C" int ac_head_train_strategic(const float *X, const int64_t *targets, const int64_t *perms, int n, int n_epochs, ac_head_params *p,
                                       ac_head_params *m, ac_head_params *v, const ac_train_cfg *cfg, const ac_strategic_cfg *scfg,
                                       float *step_stats, void *workspace, size_t workspace_bytes, ac_stream_t stream) {
    const char *who = "ac_head_train_strategic";
    int rc = check_params(p, who);
    if (rc) return rc;
    AC_REQUIRE(X && targets && perms && n > 0 && n_epochs >= 0 && m && v && cfg && scfg && step_stats && workspace, "%s: bad arguments", who);
    AC_REQUIRE(cfg->step >= 1 && !cfg->mask0 && !cfg->mask1 && !cfg->ewc_fisher, "%s: step >= 1, no injected masks, no EWC", who);
    StLayout l;
    if ((rc = st_layout(n, p, l, who))) return rc;
    uint8_t *w = reinterpret_cast<uint8_t *>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
    if (l.total + (w - static_cast<uint8_t *>(workspace)) > workspace_bytes) { set_error("%s: workspace needs %zu bytes", who, l.total); return AC_E_WORKSPACE; }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    float *Xa = reinterpret_cast<float *>(w + l.xa);
    int64_t *ta = reinterpret_cast<int64_t *>(w + l.ta);
    const int batch = n < ST_MAX_BATCH ? n : ST_MAX_BATCH;
    const int steps_per_epoch = (n + batch - 1) / batch;
    ac_train_cfg tc = *cfg;
    ac_strategic_cfg sc = *scfg;
    for (int e = 0; e < n_epochs; ++e) {
        for (int t = 0; t < steps_per_epoch; ++t) {
            const int off = t * batch;
            const int Bt = n - off < batch ? n - off : batch;
            const int gstep = e * steps_per_epoch + t;
            strategic_gather_kernel<<<Bt, 128, 0, s>>>(X, targets, perms + static_cast<int64_t>(e) * n + off, Bt, p->D, Xa, ta);
            AC_LAUNCH_CHECK();
            sc.step = cfg->step + gstep;
            if ((rc = ac_strategic_best_response(Xa, Bt, p, &sc, reinterpret_cast<int32_t *>(w + l.choice), reinterpret_cast<float *>(w + l.util),
                                                 Xa + static_cast<int64_t>(Bt) * p->D, w + l.search, l.total - l.search, stream)))
                return rc;
            tc.step = cfg->step + gstep;
            tc.n_regular = Bt;
            TrainCall c{Xa, ta, nullptr, 2 * Bt, 2 * Bt, 1, tc.step, p, m, v, &tc, AC_LOSS_CE_STRATEGIC, nullptr, nullptr, 0.f,
                        step_stats + 3 * static_cast<int64_t>(gstep), nullptr};
            if ((rc = launch_training(c, w + l.train, l.search - l.train, s, who, nullptr))) return rc;
        }
    }
    return AC_OK;
}

static Flat6 ewc_limits(const ac_head_params *p, int C_old) {
    // the head may have grown since theta* was taken: only the first C_old output rows are penalised
    ac_head_params q = *p;
    Flat6 f = flat_of(&q);
    if (C_old > 0 && C_old < p->C) {
        f.n[4] = static_cast<int64_t>(C_old) * p->H1;
        f.n[5] = C_old;
    }
    return f;
}

extern "C" int ac_ewc_penalty(const ac_head_params *p, const ac_head_params *fisher, const ac_head_params *star,
                              float lambda, float inv_batch, int C_old, float *out, ac_stream_t stream) {
    int rc = check_params(p, "ac_ewc_penalty");
    if (rc) return rc;
    AC_REQUIRE(fisher && star && out, "ac_ewc_penalty: bad arguments");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    float *partial = nullptr;
    AC_CUDA(cudaMallocAsync(reinterpret_cast<void **>(&partial), RED_BLOCKS * sizeof(float), s));
    Flat6 lim = ewc_limits(p, C_old);
    ewc_grad_penalty_kernel<<<RED_BLOCKS, 256, 0, s>>>(flat_of(p), flat_of(fisher), flat_of(star), flat_of(p), lim, 0.f,
                                                       partial, 0);
    AC_LAUNCH_CHECK();
    finalize_kernel<<<1, 32, 0, s>>>(partial, RED_BLOCKS, lambda * inv_batch, 0, out);
    AC_LAUNCH_CHECK();
    AC_CUDA(cudaFreeAsync(partial, s));
    return AC_OK;
}
