// strategic.cu -- stage S: the best-response search of strategic mode (fp32 SIMT).
//
// Replaces (paths relative to /root/reference/src/adaptive_classifier/):
//   strategic.py:74-123   SeparableCostFunction.compute_best_response / _generate_candidates: per sample, 50 candidates, one
//                         head forward each, utility = max softmax - cost, first maximum wins
//
// For a chunk of Bq query rows the search is four launches with no host round trip:
//   strategic_prep     per candidate row m = 50 q + c: the changed coordinate i and dlt = fl(x_i + delta) - x_i; the five
//                      W0 columns 0..4 as rows (w0c[5, H0])
//   strategic_gemm<0>  z0 = X W0^T + b0, once per QUERY: a candidate differs from x in one coordinate, so its layer-0
//                      pre-activation is the rank-1 update z0 + dlt * W0[:, i] (49 of the 50 D x H0 products disappear)
//   strategic_gemm<1>  h1 = relu(relu(z0 + dlt W0[:, i]) W1^T + b1): [50 Bq, H0] x [H0, H1], the layer-0 activations are
//                      formed while the A tile is staged (never stored); this product is ~95% of the FLOP of the search
//   strategic_gemm<2>  z = h1 W2^T + b2
//   strategic_select   per query: max softmax = 1 / sum exp(z - max z), cost, first argmax over the 50 candidates, Y row
// All products are fp32 FMA (no TF32 / fp16): the result is an argmax over utilities that must agree with an fp32 evaluation
// except at genuine near-ties (DESIGN.md section 5.7).
#include "common.cuh"
#include <math_constants.h>

namespace ac {

constexpr int SC_NC = AC_STRATEGIC_CANDIDATES;
constexpr int SC_T = 64, SC_K = 16;          // 64 x 64 output tile, K in slabs of 16, 256 threads x (4 x 4) outputs

// dropout mask of the candidate forwards (0 or 1/(1-p)), keyed on (seed, step, layer, row, candidate, unit); the stream id has
// bit 40 set so that it never meets the training kernel's (2 step + layer) streams
__device__ __forceinline__ float sc_mask(float p, unsigned long long seed, int step, int layer, long long elem) {
    unsigned long long x = seed * 0x9E3779B97F4A7C15ULL + ((1ull << 40) + 2ull * static_cast<unsigned>(step) + layer) * 0xD1B54A32D192ED03ULL +
                           static_cast<unsigned long long>(elem);
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    const float u = (static_cast<uint32_t>(x) >> 8) * (1.0f / 16777216.0f);
    return (u < p) ? 0.f : 1.f / (1.f - p);
}

struct ScArgs {
    const float *X;          // [Bq, D] this chunk's query rows
    int Bq, D, H0, H1, C;
    int row0;                // global index of the chunk's first query (dropout key)
    const float *W0, *b0, *W1, *b1, *W2, *b2;
    const float *c1, *c2;
    int cost_kind;
    float delta[10];
    float p;                 // dropout probability (0: eval mode)
    unsigned long long seed;
    int step;
    // workspace
    float *z0;               // [Bq, H0]
    float *w0c;              // [5, H0]
    float *dlt;              // [50 Bq]
    int *coord;              // [50 Bq] (-1 for candidate 0)
    float *h1;               // [50 Bq, H1]
    float *z;                // [50 Bq, C]
};

__device__ __forceinline__ void sc_cand(int c, int &i, int &j) {
    i = c == 0 ? -1 : (c - 1) / 10;
    j = c == 0 ? 0 : (c - 1) % 10;
}

__global__ void __launch_bounds__(256) strategic_prep_kernel(const ScArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.Bq * SC_NC) {
        const int q = t / SC_NC, c = t % SC_NC;
        int i, j;
        sc_cand(c, i, j);
        float d = 0.f;
        if (i >= 0) {
            const float xi = a.X[static_cast<int64_t>(q) * a.D + i];
            d = __fsub_rn(__fadd_rn(xi, a.delta[j]), xi);          // candidate[i] += delta (fp32), then y_i - x_i
        }
        a.dlt[t] = d;
        a.coord[t] = i;
    }
    if (t < 5 * a.H0) {
        const int i = t / a.H0, k = t % a.H0;
        a.w0c[t] = a.W0[static_cast<int64_t>(k) * a.D + i];
    }
}

// Y[m, n] = epi(sum_k A[m, k] W[n, k] + bias[n]), k ascending per output.
//   MODE 0: A = X [Bq, D], W = W0, no activation (z0)
//   MODE 1: A[m, k] = relu(z0[m / 50, k] + dlt[m] * w0c[coord[m], k]) * mask0, W = W1, relu * mask1 (h1)
//   MODE 2: A = h1, W = W2, no activation (logits)
template <int MODE>
__global__ void __launch_bounds__(256) strategic_gemm_kernel(const ScArgs a) {
    __shared__ __align__(16) float sx[2][SC_K][SC_T + 4];
    __shared__ __align__(16) float sw[2][SC_K][SC_T + 4];
    const int M = MODE == 0 ? a.Bq : a.Bq * SC_NC;
    const int N = MODE == 0 ? a.H0 : (MODE == 1 ? a.H1 : a.C);
    const int K = MODE == 0 ? a.D : (MODE == 1 ? a.H0 : a.H1);
    const float *W = MODE == 0 ? a.W0 : (MODE == 1 ? a.W1 : a.W2);
    const float *bias = MODE == 0 ? a.b0 : (MODE == 1 ? a.b1 : a.b2);
    float *Y = MODE == 0 ? a.z0 : (MODE == 1 ? a.h1 : a.z);
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * SC_T, n0 = blockIdx.x * SC_T;
    const int tx = tid & 15, ty = tid >> 4;
    const int lr = tid >> 2, lk = (tid & 3) * 4;
    // per-thread constants of the A row this thread stages
    const int am = m0 + lr;
    const bool arow = am < M;
    int aq = 0, ai = -1;
    float ad = 0.f;
    if (MODE == 1 && arow) { aq = am / SC_NC; ai = a.coord[am]; ad = a.dlt[am]; }
    auto loadA = [&](int k) -> float4 {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!arow || k >= K) return v;
        if (MODE == 0) return __ldg(reinterpret_cast<const float4 *>(a.X + static_cast<int64_t>(am) * K + k));
        if (MODE == 2) return *reinterpret_cast<const float4 *>(a.h1 + static_cast<int64_t>(am) * K + k);
        const float4 z = *reinterpret_cast<const float4 *>(a.z0 + static_cast<int64_t>(aq) * K + k);
        float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ai >= 0) w = *reinterpret_cast<const float4 *>(a.w0c + static_cast<int64_t>(ai) * K + k);
        float h[4] = {fmaf(ad, w.x, z.x), fmaf(ad, w.y, z.y), fmaf(ad, w.z, z.z), fmaf(ad, w.w, z.w)};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            h[u] = fmaxf(h[u], 0.f);
            if (a.p > 0.f) h[u] *= sc_mask(a.p, a.seed, a.step, 0, (static_cast<long long>(a.row0) * SC_NC + am) * K + k + u);
        }
        return make_float4(h[0], h[1], h[2], h[3]);
    };
    auto loadW = [&](int k) -> float4 {
        const int n = n0 + lr;
        if (n >= N || k >= K) return make_float4(0.f, 0.f, 0.f, 0.f);
        return __ldg(reinterpret_cast<const float4 *>(W + static_cast<int64_t>(n) * K + k));
    };
    auto stage = [&](float (*dst)[SC_T + 4], const float4 &v) {
        dst[lk + 0][lr] = v.x; dst[lk + 1][lr] = v.y; dst[lk + 2][lr] = v.z; dst[lk + 3][lr] = v.w;
    };
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float4 rx = loadA(lk), rw = loadW(lk);
    const int nslab = (K + SC_K - 1) / SC_K;
    for (int sl = 0; sl < nslab; ++sl) {
        const int buf = sl & 1;
        stage(sx[buf], rx);
        stage(sw[buf], rw);
        __syncthreads();
        if (sl + 1 < nslab) {
            rx = loadA((sl + 1) * SC_K + lk);
            rw = loadW((sl + 1) * SC_K + lk);
        }
#pragma unroll
        for (int k = 0; k < SC_K; ++k) {
            const float4 av4 = *reinterpret_cast<const float4 *>(&sx[buf][k][4 * ty]);
            const float4 bv4 = *reinterpret_cast<const float4 *>(&sw[buf][k][4 * tx]);
            const float av[4] = {av4.x, av4.y, av4.z, av4.w}, bv[4] = {bv4.x, bv4.y, bv4.z, bv4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        // the buffer staged two slabs from now is this one: the barrier at the top of the next iteration orders it
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + 4 * ty + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + 4 * tx + j;
            if (n >= N) continue;
            float v = acc[i][j] + bias[n];
            if (MODE == 1) {
                v = fmaxf(v, 0.f);
                if (a.p > 0.f) v *= sc_mask(a.p, a.seed, a.step, 1, (static_cast<long long>(a.row0) * SC_NC + m) * N + n);
            }
            Y[static_cast<int64_t>(m) * N + n] = v;
        }
    }
}

// one CTA per query: 8 warps x the 50 candidates; utilities in shared memory, first argmax by thread 0
__global__ void __launch_bounds__(256) strategic_select_kernel(const ScArgs a, int32_t *out_choice, float *out_utility, float *out_Y) {
    __shared__ float u[SC_NC];
    const int q = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float *x = a.X + static_cast<int64_t>(q) * a.D;
    const int C = a.C, D = a.D;
    float c1x = 0.f;
    if (a.cost_kind == AC_COST_SEPARABLE) {
        for (int k = lane; k < D; k += 32) c1x = fmaf(a.c1[k], x[k], c1x);
        c1x = warp_sum(c1x);
    }
    for (int c = warp; c < SC_NC; c += 8) {
        const int m = q * SC_NC + c;
        const float *zr = a.z + static_cast<int64_t>(m) * C;
        float mx = -CUDART_INF_F;
        for (int j = lane; j < C; j += 32) mx = fmaxf(mx, zr[j]);
        mx = warp_max(mx);
        float s = 0.f;
        for (int j = lane; j < C; j += 32) s += expf(zr[j] - mx);
        s = warp_sum(s);
        const float prob = 1.f / s;                                // softmax at the largest logit: exp(0) / sum
        int i, jd;
        sc_cand(c, i, jd);
        float cost = 0.f;
        if (a.cost_kind == AC_COST_LINEAR) {
            if (i >= 0) cost = fmaxf(__fmul_rn(a.c1[i], a.dlt[m]), 0.f);
        } else {
            // c2 . y in the order of c1 . x: lane-strided partial sums, then the same shuffle tree
            float c2y = 0.f;
            for (int k = lane; k < D; k += 32) {
                const float yk = (k == i) ? __fadd_rn(x[k], a.delta[jd]) : x[k];
                c2y = fmaf(a.c2[k], yk, c2y);
            }
            c2y = warp_sum(c2y);
            cost = fmaxf(__fsub_rn(c2y, c1x), 0.f);
        }
        if (lane == 0) u[c] = __fsub_rn(prob, cost);
    }
    __syncthreads();
    __shared__ int best_c;
    if (threadIdx.x == 0) {
        float best = -CUDART_INF_F;
        int bc = 0;
        for (int c = 0; c < SC_NC; ++c)
            if (u[c] > best) { best = u[c]; bc = c; }             // strict: the first maximum wins, NaN never does
        out_choice[a.row0 + q] = bc;
        out_utility[a.row0 + q] = best;
        best_c = bc;
    }
    __syncthreads();
    if (out_Y) {
        int i, jd;
        sc_cand(best_c, i, jd);
        float *y = out_Y + (static_cast<int64_t>(a.row0) + q) * D;
        for (int k = threadIdx.x; k < D; k += blockDim.x) y[k] = (k == i) ? __fadd_rn(x[k], a.delta[jd]) : x[k];
    }
}

// queries per chunk: the candidate activations h1 and logits of a chunk stay under ~64 MB
static int sc_chunk(int B, const ac_head_params *p) {
    const size_t per_query = static_cast<size_t>(SC_NC) * (p->H1 + p->C) * sizeof(float);
    size_t q = (size_t(64) << 20) / per_query;
    if (q < 1) q = 1;
    return static_cast<int>(q < static_cast<size_t>(B) ? q : static_cast<size_t>(B));
}

struct ScLayout { size_t z0, w0c, dlt, coord, h1, z, total; };
static ScLayout sc_layout(int Bq, const ac_head_params *p) {
    ScLayout l;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align_up(bytes, 256); return o; };
    const size_t M = static_cast<size_t>(Bq) * SC_NC;
    l.z0 = take(sizeof(float) * Bq * p->H0);
    l.w0c = take(sizeof(float) * 5 * p->H0);
    l.dlt = take(sizeof(float) * M);
    l.coord = take(sizeof(int) * M);
    l.h1 = take(sizeof(float) * M * p->H1);
    l.z = take(sizeof(float) * M * p->C);
    l.total = off + 256;
    return l;
}

static int sc_check(int B, const ac_head_params *p, const char *who) {
    AC_REQUIRE(p && B >= 0, "%s: bad arguments", who);
    AC_REQUIRE(p->D > 0 && p->H0 > 0 && p->H1 > 0 && p->C > 0, "%s: bad head dims", who);
    AC_REQUIRE(p->D >= 5, "%s: the candidate set moves coordinates 0..4 and needs D >= 5 (D=%d)", who, p->D);
    AC_REQUIRE(p->D % 4 == 0 && p->H0 % 4 == 0 && p->H1 % 4 == 0, "%s: D, H0, H1 must be multiples of 4 (D=%d H0=%d H1=%d)", who,
               p->D, p->H0, p->H1);
    return AC_OK;
}

}  // namespace ac

using namespace ac;

extern "C" int ac_strategic_workspace_bytes(int B, const ac_head_params *p, size_t *bytes) {
    int rc = sc_check(B, p, "ac_strategic_workspace_bytes");
    if (rc) return rc;
    AC_REQUIRE(bytes, "ac_strategic_workspace_bytes: bad arguments");
    *bytes = sc_layout(B > 0 ? sc_chunk(B, p) : 1, p).total;
    return AC_OK;
}

extern "C" int ac_strategic_best_response(const float *X, int B, const ac_head_params *p, const ac_strategic_cfg *cfg,
                                          int32_t *out_choice, float *out_utility, float *out_Y, void *workspace,
                                          size_t workspace_bytes, ac_stream_t stream) {
    int rc = sc_check(B, p, "ac_strategic_best_response");
    if (rc) return rc;
    AC_REQUIRE(cfg && X && out_choice && out_utility && workspace, "ac_strategic_best_response: bad arguments");
    AC_REQUIRE(p->W0 && p->b0 && p->W1 && p->b1 && p->W2 && p->b2, "ac_strategic_best_response: null head parameter");
    AC_REQUIRE(cfg->cost_kind == AC_COST_LINEAR || cfg->cost_kind == AC_COST_SEPARABLE,
               "ac_strategic_best_response: unknown cost kind %d", cfg->cost_kind);
    AC_REQUIRE(cfg->c1 && (cfg->cost_kind == AC_COST_LINEAR || cfg->c2), "ac_strategic_best_response: null cost coefficients");
    AC_REQUIRE(cfg->dropout_p >= 0.f && cfg->dropout_p < 1.f, "ac_strategic_best_response: dropout_p outside [0, 1)");
    AC_REQUIRE((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(p->W0) | reinterpret_cast<uintptr_t>(p->W1) |
                reinterpret_cast<uintptr_t>(p->W2)) % 16 == 0, "ac_strategic_best_response: X and the weights must be 16-byte aligned");
    if (B == 0) return AC_OK;
    if ((rc = ac_device_check())) return rc;
    const int chunk = sc_chunk(B, p);
    const ScLayout l = sc_layout(chunk, p);
    uint8_t *w = reinterpret_cast<uint8_t *>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
    if (l.total + (w - static_cast<uint8_t *>(workspace)) > workspace_bytes) {
        set_error("ac_strategic_best_response: workspace needs %zu bytes", l.total + 256);
        return AC_E_WORKSPACE;
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    ScArgs a{};
    a.D = p->D; a.H0 = p->H0; a.H1 = p->H1; a.C = p->C;
    a.W0 = p->W0; a.b0 = p->b0; a.W1 = p->W1; a.b1 = p->b1; a.W2 = p->W2; a.b2 = p->b2;
    a.c1 = cfg->c1; a.c2 = cfg->cost_kind == AC_COST_SEPARABLE ? cfg->c2 : cfg->c1;
    a.cost_kind = cfg->cost_kind;
    for (int j = 0; j < 10; ++j) a.delta[j] = cfg->delta[j];
    a.p = cfg->dropout_p; a.seed = cfg->seed; a.step = cfg->step;
    a.z0 = reinterpret_cast<float *>(w + l.z0); a.w0c = reinterpret_cast<float *>(w + l.w0c);
    a.dlt = reinterpret_cast<float *>(w + l.dlt); a.coord = reinterpret_cast<int *>(w + l.coord);
    a.h1 = reinterpret_cast<float *>(w + l.h1); a.z = reinterpret_cast<float *>(w + l.z);
    for (int r0 = 0; r0 < B; r0 += chunk) {
        a.row0 = r0;
        a.Bq = B - r0 < chunk ? B - r0 : chunk;
        a.X = X + static_cast<int64_t>(r0) * p->D;
        const int M = a.Bq * SC_NC;
        const int prep = M > 5 * p->H0 ? M : 5 * p->H0;
        strategic_prep_kernel<<<(prep + 255) / 256, 256, 0, s>>>(a);
        AC_LAUNCH_CHECK();
        strategic_gemm_kernel<0><<<dim3((p->H0 + SC_T - 1) / SC_T, (a.Bq + SC_T - 1) / SC_T), 256, 0, s>>>(a);
        AC_LAUNCH_CHECK();
        strategic_gemm_kernel<1><<<dim3((p->H1 + SC_T - 1) / SC_T, (M + SC_T - 1) / SC_T), 256, 0, s>>>(a);
        AC_LAUNCH_CHECK();
        strategic_gemm_kernel<2><<<dim3((p->C + SC_T - 1) / SC_T, (M + SC_T - 1) / SC_T), 256, 0, s>>>(a);
        AC_LAUNCH_CHECK();
        // the select kernel indexes outputs by row0 + q: hand it the chunk-relative X and the global outputs
        strategic_select_kernel<<<a.Bq, 256, 0, s>>>(a, out_choice, out_utility, out_Y);
        AC_LAUNCH_CHECK();
    }
    return AC_OK;
}
