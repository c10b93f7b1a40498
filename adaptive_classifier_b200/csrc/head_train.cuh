// head_train.cuh -- the optimizer loop of the adaptive head as ONE persistent cooperative kernel (fp32 SIMT).
//
// Replaces, per optimizer step (paths relative to /root/reference/src/adaptive_classifier/):
//   classifier.py:333-351, :1489-1505   zero_grad / forward (train mode: Dropout 0.1) / CrossEntropyLoss / backward /
//                                       clip_grad_norm_(1.0) / AdamW(lr 1e-3, wd 0.01).step()
//   multilabel.py:387-397               the same with sigmoid outputs + BCELoss
//   ewc.py:67-92, :96-115               gradient of the sampled-label NLL (Fisher) and the EWC penalty gradient
// and the DataLoader batching around it (one launch runs all steps of an epoch from a shuffled index list).
//
// Why one kernel: the head is 0.9 M parameters and a batch is 32 rows -- 171 MFLOP and 25 MB of optimizer traffic per step,
// i.e. microseconds of work, which ~21 dependent kernel launches per step would dominate.  Here the grid stays resident for
// the whole epoch and a step is seven phases separated by six grid barriers (75 us per step on an H100 80GB HBM3, batch 32,
// 21 classes: `cfg4.head_step_us_batch32` in profiles/h100_bench.json):
//
//   ownership   the rows of every weight matrix are cut into blocks of HT_RB = 8 rows, and the blocks of all three layers form
//               ONE list of items dealt over the grid (item i -> CTA i % G).  The reference's head (768 -> 768 -> 384 -> C)
//               has 96 + 48 + ceil(C / 8) items: with C <= 32 that is at most 148.  On the 132 SMs of an H100 the first
//               items_total - 132 CTAs (15 at C = 21) own a layer-0 item and a layer-1 or layer-2 item, so in the phases where
//               several layers work those CTAs do two items' work; the others work for one layer, and the weight-gradient
//               work of different layers runs side by side.  A CTA keeps
//               the rows of ITS item(s) -- parameters, gradient, biases, and the AdamW moments when they fit (res_mv; for the
//               reference's head they stay owner-private in L2) -- in shared memory for the whole launch, computes the activations / gradients of exactly those rows and applies AdamW to them: parameters
//               never move between CTAs, gradients and moments never leave shared memory (moments: when they fit, res_mv),
//               AdamW of step t needs no barrier before the forward of step t+1.
//   P1  h0 = dropout(relu(X W0^T + b0))        layer-0 items; X rows gathered through the shuffled index list
//   P2  h1 = dropout(relu(h0 W1^T + b1))       layer-1 items
//   P3a z  = h1 W2^T + b2                      layer-2 items
//   P3b loss, dz per batch row                 one warp per row over the whole grid (softmax-CE or sigmoid-BCE)
//   P4  da1 = (dz W2) * relu' * mask of the own rows (layer-1 items)
//   P5  gW2, gb2 (layer-2 items) | gW1, gb1 (layer-1 items) | P6  da0 = (da1 W1) * relu' * mask, gW0, gb0 (layer-0 items)
//       [EWC: g += 2 lambda / B * F (theta - theta*)];  partial sum of squares of the own gradients
//   P7  global grad norm (every CTA adds the G partials in the same order), clip, AdamW on the own rows
//   Activations cross CTAs through small global (L2-resident) buffers; every product streams its [B x K] operand through a
//   ring of shared-memory stages in chunks of HT_KC columns by 16-byte cp.async.cg copies (L2 only: these buffers are rewritten
//   by other CTAs every step and must never be served from this SM's L1).
//   The grid barrier is one arrival counter that only grows; the AdamW bias corrections are tabulated 256 steps at a time.
//
// All sums have a fixed order: results are deterministic run to run and independent of the grid size up to fp32 rounding of
// the (grid-size dependent) partial-sum order of the gradient norm.  Parity: the CPU restatement of the optimizer step (tests/test_gpu_parity.py,
// tests/test_gpu_training_golden.py: the reference's own per-step losses to 1e-5 over 60 steps).
//
// This header is plain SIMT C++ (no inline PTX beyond the timer): tests/cpu_shim/head_train_emul.cpp compiles it for the CPU (every CUDA
// thread a fiber, grid barriers real) and checks it against a straightforward restatement before any GPU time is spent.
#pragma once
#include <stdint.h>
#if !defined(AC_CPU_SHIM)
#include <cuda_pipeline.h>
#endif

namespace ac {
namespace ht {

constexpr int HT_THREADS = 256;
constexpr int HT_RB = 8;              // rows per ownership block
#ifndef HT_KC_COLS
#define HT_KC_COLS 256
#endif
constexpr int HT_KC = HT_KC_COLS;     // columns per streamed chunk (128 or 256)
constexpr int HT_AS = HT_KC + 4;      // padded row stride of the chunk buffer (floats): conflict-free float4 rows
constexpr int HT_MAXB = 64;           // rows per batch
constexpr int HT_KPARTS = HT_THREADS / 32;   // 8 warps split a chunk's columns
constexpr int HT_WC = HT_KC / HT_KPARTS;     // columns of a chunk per warp (16 or 32)
constexpr int HT_JH = HT_THREADS / HT_KC;    // weight-gradient products: row groups (2 or 1) ...
constexpr int HT_JR = HT_RB / HT_JH;         // ... of 4 or 8 rows per thread
constexpr int HT_BCW = 256;           // AdamW bias corrections are tabulated for 256 steps at a time
constexpr int HT_TROW = 24;           // timing counters per observed CTA
static_assert(HT_KC == 128 || HT_KC == 256, "chunk width");

struct Layer {
    float *W, *b;                 // [rows, K], [rows]   parameters (global; updated in place)
    float *mW, *mb, *vW, *vb;     // AdamW moments (update mode)
    const float *fW, *fb, *sW, *sb;   // EWC Fisher / theta* (nullable)
    float *gW, *gb;               // gradient outputs (gradient-only mode, nullable)
    float *qW, *qb;               // Fisher accumulators: q += g^2 * fisher_scale (gradient-only mode, nullable)
    int rows, K, ewc_rows;        // ewc_rows: only the first ewc_rows rows carry the EWC term (the head may have grown)
};

struct Args {
    const float *X;               // [n, D]
    const void *targets;          // int64 [n] (CE) or float [n, C] (BCE)
    const int64_t *perm;          // [n] shuffled row order, NULL = identity
    int n, batch, n_steps, first_step;
    Layer L[3];
    float lr, beta1, beta2, eps, wd, max_norm, dropout_p;
    int loss_kind;                // 0 CE, 1 BCE, 2 CE_STRATEGIC
    unsigned long long seed;
    const float *mask0, *mask1;   // injected dropout masks [B,H0], [B,H1] (single step) or NULL
    int use_ewc;
    float ewc_lambda;
    int update;                   // 1: clip + AdamW;  0: gradient only (Fisher)
    float fisher_scale;
    // global scratch
    float *h0d, *h1d, *z, *dz, *da1, *rowloss, *part, *pen;     // dz rows are padded to ldz floats (16-byte copies)
    float *stats;                 // [n_steps, 3] (task loss, EWC penalty, grad norm before clipping), nullable
    float *loss_accum;            // [1] += loss + penalty per step, nullable
    unsigned *bar;                // [1] grid barrier arrival counter, zero-initialised
    // ownership (ht_assign): the 8-row blocks of the three layers form one list of `items`; item i lives on CTA i % G, slot i / G
    int nblk[3], items, slots, kmax, ldz;
    int res_mv;                   // AdamW moments of the own rows stay in shared memory for the whole launch
    int nst;                      // stages of the streamed-operand ring (2..8)
    unsigned long long *timing;   // nullable, [3][HT_TROW]: nanoseconds per phase of three observed CTAs (one per layer), summed over the steps
    // CE_STRATEGIC: rows [0, n_regular) are x, rows [n_regular, 2 n_regular) their best responses.  Row weights: 1 / n_regular for x,
    // strategic_lambda / n_regular for a best response whose first argmax differs from its target, 0 otherwise
    int n_regular;
    float strategic_lambda;
};

// ownership for a grid of G CTAs (host and emulator call this before ht_smem_layout)
__host__ __device__ inline void ht_assign(Args &a, int G) {
    a.items = 0;
    a.kmax = 4;
    for (int l = 0; l < 3; ++l) {
        a.nblk[l] = (a.L[l].rows + HT_RB - 1) / HT_RB;
        a.items += a.nblk[l];
        if (a.L[l].K > a.kmax) a.kmax = a.L[l].K;
    }
    a.slots = (a.items + G - 1) / G;
    a.ldz = (a.L[2].rows + 3) & ~3;
}
struct Item { int l, q; };
__device__ __forceinline__ Item ht_item(const Args &a, int i) {
    Item it;
    if (i < a.nblk[0]) { it.l = 0; it.q = i; }
    else if (i < a.nblk[0] + a.nblk[1]) { it.l = 1; it.q = i - a.nblk[0]; }
    else { it.l = 2; it.q = i - a.nblk[0] - a.nblk[1]; }
    return it;
}

// ---------------------------------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------------------------------
#if !defined(AC_CPU_SHIM)
#define HT_LDCG(p) __ldcg(p)      // L2 (coherent across CTAs): everything another CTA wrote inside this launch
#else
#define HT_LDCG(p) (*(p))
#endif

// asynchronous global -> shared copies of 16 bytes: cp.async.cg (L2 only -- the streamed operands are rewritten by other CTAs
// every step and must never be served from this SM's L1); `valid` = false zero-fills the destination
#if !defined(AC_CPU_SHIM)
__device__ __forceinline__ void ht_async16(float *dst, const float *src, bool valid) { __pipeline_memcpy_async(dst, src, 16, valid ? 0 : 16); }
__device__ __forceinline__ void ht_async_commit() { __pipeline_commit(); }
template <int N> __device__ __forceinline__ void ht_async_wait() { __pipeline_wait_prior(N); }
#else
static inline void ht_async16(float *dst, const float *src, bool valid) { for (int i = 0; i < 4; ++i) dst[i] = valid ? src[i] : 0.f; }
static inline void ht_async_commit() {}
template <int N> static inline void ht_async_wait() {}
#endif
__device__ __forceinline__ void ht_async_wait_n(int n) {       // n = stages - 2 in [0, 6]
    switch (n) {
        case 0: ht_async_wait<0>(); break;
        case 1: ht_async_wait<1>(); break;
        case 2: ht_async_wait<2>(); break;
        case 3: ht_async_wait<3>(); break;
        case 4: ht_async_wait<4>(); break;
        case 5: ht_async_wait<5>(); break;
        default: ht_async_wait<6>(); break;
    }
}

__device__ __forceinline__ uint32_t ht_mix32(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    return static_cast<uint32_t>(x);
}
// counter-hash dropout mask of element i of mask stream `stream_id` (0 or 1/(1-p))
__device__ __forceinline__ float ht_mask(float p, unsigned long long seed, unsigned long long stream_id, unsigned long long i) {
    const uint32_t r = ht_mix32(seed * 0x9E3779B97F4A7C15ULL + stream_id * 0xD1B54A32D192ED03ULL + i);
    const float u = (r >> 8) * (1.0f / 16777216.0f);
    return (u < p) ? 0.f : 1.f / (1.f - p);
}

// phase timing (diagnostic, tools/head_phase_times.py): thread 0 of an observed CTA accumulates global-timer deltas
#if !defined(AC_CPU_SHIM)
__device__ __forceinline__ unsigned long long ht_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#else
static inline unsigned long long ht_now() { return 0; }
#endif
#define HT_STAMP(i)                                              \
    do {                                                         \
        if (tm) {                                                \
            const unsigned long long now_ = ht_now();            \
            tm[i] += now_ - t_prev;                              \
            t_prev = now_;                                       \
        }                                                        \
    } while (0)
// finer counters inside the two product routines: tm[DT + 0..3] = wait, issue, multiply, combine of ht_rows_dot,
// tm[DT + 4..6] = wait, issue, multiply of ht_outer_acc
constexpr int HT_DT = 14;
#define HT_DSTAMP(i)                                             \
    do {                                                         \
        if (dt) {                                                \
            const unsigned long long now_ = ht_now();            \
            dt[i] += now_ - d_prev;                              \
            d_prev = now_;                                       \
        }                                                        \
    } while (0)

// grid barrier: all threads of all CTAs.  One arrival counter that only grows (barrier number x grid size is the release
// value), so a barrier is one atomic and a poll -- no reset, no second flag.  Cooperative launch guarantees co-residency; a
// watchdog turns a protocol bug into a launch error instead of a hung GPU.
__device__ __forceinline__ void ht_grid_sync(unsigned *bar, unsigned &target) {
#if !defined(AC_CPU_SHIM)
    __syncthreads();
    target += gridDim.x;
    if (threadIdx.x == 0) {
        __threadfence();                                        // publish this CTA's global writes
        atomicAdd(bar, 1u);
        unsigned spins = 0;
        while (*reinterpret_cast<volatile unsigned *>(bar) < target) {
            if (++spins > (1u << 28)) { printf("ac: head_train grid barrier watchdog (block %d)\n", blockIdx.x); __trap(); }
        }
        __threadfence();
    }
    __syncthreads();
#else
    (void)bar; (void)target;
    cooperative_groups::this_grid().sync();
#endif
}

// block-wide sum in a fixed tree order; red: HT_THREADS floats of shared memory; every thread gets the result
__device__ __forceinline__ float ht_block_sum(float v, float *red) {
    __syncthreads();
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = HT_THREADS / 2; s > 0; s >>= 1) {
        if (static_cast<int>(threadIdx.x) < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    const float r = red[0];
    __syncthreads();
    return r;
}

// ---------------------------------------------------------------------------------------------------------------------
// streamed operand: chunk [rows x HT_KC] of a row-major [*, K] matrix (rows direct or through ridx) -> a stage of the shared
// memory ring, by 16-byte asynchronous copies (K and ld are multiples of 4, bases 16-byte aligned: host-checked).  `nst`
// stages are in flight, whatever the resident rows leave room for.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ht_issue_chunk(float *stage, const float *src, int64_t ld, const int64_t *ridx, int rows, int k0, int K) {
    for (int e = threadIdx.x; e < rows * (HT_KC / 4); e += HT_THREADS) {
        const int row = e / (HT_KC / 4), c4 = e % (HT_KC / 4);
        const int k = k0 + 4 * c4;
        const float *p = src + (ridx ? ridx[row] : static_cast<int64_t>(row)) * ld + k;
        ht_async16(stage + row * HT_AS + 4 * c4, k < K ? p : src, k < K);
    }
}
// weight chunk of an input-gradient product, as it lies in memory: Wt[kk][0..7] = gW[(k0 + kk) * gld + gcol0 + 0..7] (zero
// outside the [krows x gld] matrix; gld is a multiple of 4 and gcol0 of 8, so a group of 4 columns is inside or outside)
__device__ __forceinline__ void ht_issue_wt(float *wt_stage, const float *gW, int64_t gld, int gcol0, int k0, int krows) {
#pragma unroll
    for (int e = threadIdx.x; e < 2 * HT_KC; e += HT_THREADS) {
        const int kk = e >> 1, h4 = 4 * (e & 1);
        const bool ok = k0 + kk < krows && gcol0 + h4 < gld;
        ht_async16(wt_stage + kk * HT_RB + h4, ok ? gW + static_cast<int64_t>(k0 + kk) * gld + gcol0 + h4 : gW, ok);
    }
}

// Y[b, j] = sum_k A[b, k] * W[j][k]  for the 8 rows j of one ownership block, A streamed in chunks.
//   A: [rows x K] global (ld, optional row index list)
//   GATHER = false: the weights are the block's resident parameter rows w_res[8][K] in shared memory (forward products)
//   GATHER = true:  W[j][k] = gW[k * gld + gcol0 + j], streamed chunk by chunk from global (input-gradient products); k < krows
// Result: out[b * 8 + j] in shared memory (valid for b < rows), summed over the 8 column parts in a fixed order.
template <bool GATHER>
__device__ __forceinline__ void ht_rows_dot(float *out, float *As, float *red, float *Wt, int nst, const float *A, int64_t ld,
                                            const int64_t *ridx, int rows, int K, const float *w_res, const float *gW, int64_t gld,
                                            int gcol0, int krows, unsigned long long *dt) {
    const int lane = threadIdx.x & 31, kpart = threadIdx.x >> 5;
    const int nb = (rows + 31) >> 5;
    const int stage_floats = rows * HT_AS;
    unsigned long long d_prev = dt ? ht_now() : 0;
    float acc[2][HT_RB];
#pragma unroll
    for (int bi = 0; bi < 2; ++bi)
#pragma unroll
        for (int j = 0; j < HT_RB; ++j) acc[bi][j] = 0.f;
    const int nchunks = (K + HT_KC - 1) / HT_KC;
    for (int p = 0; p < nst - 1; ++p) {
        if (p < nchunks) {
            ht_issue_chunk(As + p * stage_floats, A, ld, ridx, rows, p * HT_KC, K);
            if (GATHER) ht_issue_wt(Wt + p * HT_RB * HT_KC, gW, gld, gcol0, p * HT_KC, krows);
        }
        ht_async_commit();
    }
    HT_DSTAMP(1);
    for (int c = 0; c < nchunks; ++c) {
        const int k0 = c * HT_KC;
        ht_async_wait_n(nst - 2);                       // chunk c has landed (for this thread's copies) ...
        __syncthreads();                                // ... and for everybody's; the stage read in iteration c - 1 is free again
        HT_DSTAMP(0);
        const int nx = c + nst - 1;
        if (nx < nchunks) {
            ht_issue_chunk(As + (nx % nst) * stage_floats, A, ld, ridx, rows, nx * HT_KC, K);
            if (GATHER) ht_issue_wt(Wt + (nx % nst) * HT_RB * HT_KC, gW, gld, gcol0, nx * HT_KC, krows);
        }
        ht_async_commit();
        HT_DSTAMP(1);
        const float *Ac = As + (c % nst) * stage_floats;
        const float *wc = GATHER ? (Wt + (c % nst) * HT_RB * HT_KC) : (w_res + k0);
        const int kcols = (K - k0 < HT_KC) ? (K - k0) : HT_KC;                           // resident rows: stay inside the row
#pragma unroll
        for (int bi = 0; bi < 2; ++bi) {
            if (lane + 32 * bi < rows) {          // rows past the batch lie in the NEXT stage, which asynchronous copies are filling
                const int b = lane + 32 * bi;
                const float *ap = Ac + b * HT_AS + kpart * HT_WC;
#pragma unroll
                for (int q4 = 0; q4 < HT_WC / 4; ++q4) {
                    const int kk = kpart * HT_WC + 4 * q4;
                    if (kk < kcols) {
                        const float4 av = *reinterpret_cast<const float4 *>(ap + 4 * q4);
                        if (GATHER) {
                            // chunk rows kk .. kk+3 of Wt[kk][8]: two 16-byte broadcast loads per k
                            const float avs[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const float4 w0 = *reinterpret_cast<const float4 *>(wc + (kk + i) * HT_RB);
                                const float4 w1 = *reinterpret_cast<const float4 *>(wc + (kk + i) * HT_RB + 4);
                                acc[bi][0] = fmaf(avs[i], w0.x, acc[bi][0]);
                                acc[bi][1] = fmaf(avs[i], w0.y, acc[bi][1]);
                                acc[bi][2] = fmaf(avs[i], w0.z, acc[bi][2]);
                                acc[bi][3] = fmaf(avs[i], w0.w, acc[bi][3]);
                                acc[bi][4] = fmaf(avs[i], w1.x, acc[bi][4]);
                                acc[bi][5] = fmaf(avs[i], w1.y, acc[bi][5]);
                                acc[bi][6] = fmaf(avs[i], w1.z, acc[bi][6]);
                                acc[bi][7] = fmaf(avs[i], w1.w, acc[bi][7]);
                            }
                        } else {
#pragma unroll
                            for (int j = 0; j < HT_RB; ++j) {
                                // one 16-byte broadcast load per 4 weights (rows are 16-byte aligned: K and kk are multiples of 4)
                                const float4 wv = *reinterpret_cast<const float4 *>(wc + j * K + kk);
                                float s = acc[bi][j];
                                s = fmaf(av.x, wv.x, s);
                                s = fmaf(av.y, wv.y, s);
                                s = fmaf(av.z, wv.z, s);
                                s = fmaf(av.w, wv.w, s);
                                acc[bi][j] = s;
                            }
                        }
                    }
                }
            }
        }
        HT_DSTAMP(2);
    }
    // combine the 8 column parts in order.  `red` shares its floats with the ring (ht_smem_layout): every copy has landed (the
    // last wait covered the last chunk) and the barrier orders the last chunk's reads before the partials overwrite it
    __syncthreads();
#pragma unroll
    for (int bi = 0; bi < 2; ++bi)
        if (bi < nb) {
            const int b = lane + 32 * bi;
#pragma unroll
            for (int j = 0; j < HT_RB; ++j) red[(kpart * HT_MAXB + b) * HT_RB + j] = acc[bi][j];
        }
    __syncthreads();
    for (int e = threadIdx.x; e < rows * HT_RB; e += HT_THREADS) {
        const int b = e / HT_RB, j = e % HT_RB;
        float s = 0.f;
#pragma unroll
        for (int kp = 0; kp < HT_KPARTS; ++kp) s += red[(kp * HT_MAXB + b) * HT_RB + j];
        out[b * HT_RB + j] = s;
    }
    __syncthreads();
    HT_DSTAMP(3);
}

// g[j][k] = sum_b dA[b][j] * A[b][k]  for the 8 rows j of one ownership block (weight gradient), A streamed in chunks;
// g: the block's gradient rows [8][K] in shared memory (rows past the matrix get the zeros of dA); dA: shared memory [rows][8];
// batch rows are added in index order.
__device__ __forceinline__ void ht_outer_acc(float *g, float *As, int nst, const float *dA, const float *A, int64_t ld,
                                             const int64_t *ridx, int rows, int K, unsigned long long *dt) {
    const int kk = threadIdx.x % HT_KC, jh = threadIdx.x / HT_KC;      // columns x row groups
    const int nchunks = (K + HT_KC - 1) / HT_KC;
    const int stage_floats = rows * HT_AS;
    unsigned long long d_prev = dt ? ht_now() : 0;
    for (int p = 0; p < nst - 1; ++p) {
        if (p < nchunks) ht_issue_chunk(As + p * stage_floats, A, ld, ridx, rows, p * HT_KC, K);
        ht_async_commit();
    }
    HT_DSTAMP(5);
    for (int c = 0; c < nchunks; ++c) {
        const int k0 = c * HT_KC;
        ht_async_wait_n(nst - 2);
        __syncthreads();
        HT_DSTAMP(4);
        const int nx = c + nst - 1;
        if (nx < nchunks) ht_issue_chunk(As + (nx % nst) * stage_floats, A, ld, ridx, rows, nx * HT_KC, K);
        ht_async_commit();
        HT_DSTAMP(5);
        const float *Ac = As + (c % nst) * stage_floats;
        float ac[HT_JR];
#pragma unroll
        for (int j = 0; j < HT_JR; ++j) ac[j] = 0.f;
        for (int b = 0; b < rows; ++b) {
            const float av = Ac[b * HT_AS + kk];
#pragma unroll
            for (int j4 = 0; j4 < HT_JR / 4; ++j4) {
                const float4 d = *reinterpret_cast<const float4 *>(dA + b * HT_RB + HT_JR * jh + 4 * j4);
                ac[4 * j4 + 0] = fmaf(d.x, av, ac[4 * j4 + 0]);
                ac[4 * j4 + 1] = fmaf(d.y, av, ac[4 * j4 + 1]);
                ac[4 * j4 + 2] = fmaf(d.z, av, ac[4 * j4 + 2]);
                ac[4 * j4 + 3] = fmaf(d.w, av, ac[4 * j4 + 3]);
            }
        }
        if (k0 + kk < K) {
#pragma unroll
            for (int j = 0; j < HT_JR; ++j) g[(HT_JR * jh + j) * K + k0 + kk] = ac[j];
        }
        HT_DSTAMP(6);
    }
    __syncthreads();
}

// shared-memory carve-up (floats), identical on host and device.  Per slot s: parameter rows th + s * 8 * kmax, gradient rows
// g + s * 8 * kmax, moments mv + s * 16 * kmax (m then v; only with res_mv), biases bs + 8 s, bias gradients gb + 8 s, relu' * mask
// factors (later the input gradients of the own rows) fac + s * batch * 8, bias moments bm + 16 s (m then v).
// The column-part partials `red` of ht_rows_dot are only written after a product's last chunk has been consumed, so they
// share their floats with the streamed-operand ring As (sized for the larger of the two): 16 KB that lets a 1024-wide head
// with two slots train at batch 32.
struct Smem {
    int th, g, mv, bs, gb, bm, fac;
    int dA, out, As, Wt, red, rsum, ridx /* int64 */, bc, scal, total;
};
__host__ __device__ inline Smem ht_smem_layout(const Args &a) {
    Smem s;
    int off = 0;
    auto take = [&](int n) { const int o = off; off += (n + 3) & ~3; return o; };
    s.th = take(a.slots * HT_RB * a.kmax);
    s.g = take(a.slots * HT_RB * a.kmax);
    s.mv = take(a.res_mv ? a.slots * 2 * HT_RB * a.kmax : 0);
    s.bs = take(a.slots * HT_RB);
    s.gb = take(a.slots * HT_RB);
    s.bm = take(a.slots * 2 * HT_RB);
    s.fac = take(a.slots * a.batch * HT_RB);
    s.dA = take(a.batch * HT_RB);
    s.out = take(a.batch * HT_RB);
    const int ring = a.nst * a.batch * HT_AS, red = HT_KPARTS * HT_MAXB * HT_RB;
    s.As = take(ring > red ? ring : red);
    s.red = s.As;
    s.Wt = take(a.nst * HT_RB * HT_KC);
    s.rsum = take(HT_THREADS);
    s.ridx = take(2 * HT_MAXB);
    s.bc = take(2 * HT_BCW);
    s.scal = take(16);
    s.total = off;
    return s;
}

// AdamW on the n4 float4 groups of one ownership block (its rows are contiguous in global memory and in shared memory).
// RES: the moments live in shared memory (m, v point there); otherwise in global memory -- all loads of a round of HT_ADAMW_U
// groups per thread are issued before the arithmetic so that the block costs about one L2 round trip per round.
constexpr int HT_ADAMW_U = 6;
template <bool RES>
__device__ __forceinline__ void ht_adamw_block(float *th, const float *g, float *m, float *v, float *Wg, int n4, float coef, float decay,
                                               float lr_c, float bc2s, float beta1, float beta2, float eps) {
    const float omb1 = 1.f - beta1, omb2 = 1.f - beta2;
    float4 *th4 = reinterpret_cast<float4 *>(th), *m4 = reinterpret_cast<float4 *>(m), *v4 = reinterpret_cast<float4 *>(v),
           *W4 = reinterpret_cast<float4 *>(Wg);
    const float4 *g4 = reinterpret_cast<const float4 *>(g);
    for (int base = 0; base < n4; base += HT_ADAMW_U * HT_THREADS) {
        float4 mi[HT_ADAMW_U], vi[HT_ADAMW_U];
#pragma unroll
        for (int u = 0; u < HT_ADAMW_U; ++u) {
            const int e = base + u * HT_THREADS + static_cast<int>(threadIdx.x);
            if (e < n4) { mi[u] = m4[e]; vi[u] = v4[e]; }
        }
#pragma unroll
        for (int u = 0; u < HT_ADAMW_U; ++u) {
            const int e = base + u * HT_THREADS + static_cast<int>(threadIdx.x);
            if (e < n4) {
                const float4 gq = g4[e], pq = th4[e];
                const float gs[4] = {gq.x, gq.y, gq.z, gq.w}, ps[4] = {pq.x, pq.y, pq.z, pq.w};
                const float ms[4] = {mi[u].x, mi[u].y, mi[u].z, mi[u].w}, vs[4] = {vi[u].x, vi[u].y, vi[u].z, vi[u].w};
                float po[4], mo[4], vo[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float gv = gs[i] * coef;
                    float p = ps[i] * decay;
                    const float m1 = ms[i] * beta1 + gv * omb1;
                    const float v1 = vs[i] * beta2 + gv * gv * omb2;
                    const float denom = sqrtf(v1) / bc2s + eps;
                    p = p - lr_c * (m1 / denom);
                    po[i] = p; mo[i] = m1; vo[i] = v1;
                }
                const float4 p4 = make_float4(po[0], po[1], po[2], po[3]);
                th4[e] = p4;
                W4[e] = p4;
                m4[e] = make_float4(mo[0], mo[1], mo[2], mo[3]);
                v4[e] = make_float4(vo[0], vo[1], vo[2], vo[3]);
            }
        }
    }
    (void)RES;
}

// ---------------------------------------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------------------------------------
// STRAT: the AC_LOSS_CE_STRATEGIC instantiation (row weights of P3b); the other loss kinds run head_train_kernel<false>
template <bool STRAT = false>
__global__ void __launch_bounds__(HT_THREADS, 1) head_train_kernel(const Args a) {
#if !defined(AC_CPU_SHIM)
    extern __shared__ __align__(16) float ht_smem[];
#else
    float *ht_smem = reinterpret_cast<float *>(shim_dyn_smem());
#endif
    const Smem sm = ht_smem_layout(a);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = gridDim.x, cta = blockIdx.x;
    const int D = a.L[0].K, H0 = a.L[0].rows, H1 = a.L[1].rows, C = a.L[2].rows;
    const int KM = a.kmax, ldz = a.ldz;
    float *As = ht_smem + sm.As, *Wt = ht_smem + sm.Wt, *red = ht_smem + sm.red, *rsum = ht_smem + sm.rsum;
    float *dA = ht_smem + sm.dA, *out = ht_smem + sm.out, *scal = ht_smem + sm.scal, *bc = ht_smem + sm.bc;
    int64_t *ridx = reinterpret_cast<int64_t *>(ht_smem + sm.ridx);
    unsigned bar_target = 0;
    const bool res_mv = a.res_mv && a.update;
    // observed CTAs of the phase timing: the first holder of a layer-0 block, of a layer-1 block, and the last CTA (layer 2)
    const int trow = cta == 0 ? 0 : ((cta == a.nblk[0] && cta < G - 1) ? 1 : (cta == G - 1 ? 2 : -1));
    unsigned long long *tm = (a.timing && trow >= 0 && tid == 0) ? a.timing + trow * HT_TROW : nullptr;
    unsigned long long *dt = tm ? tm + HT_DT : nullptr;

    // ---- resident rows of the own blocks: parameters (and AdamW moments)
    for (int s = 0; s < a.slots; ++s) {
        const int i = cta + s * G;
        if (i >= a.items) break;
        const Item it = ht_item(a, i);
        const Layer &L = a.L[it.l];
        const int K = L.K;
        const int nrow = (L.rows - it.q * HT_RB < HT_RB) ? (L.rows - it.q * HT_RB) : HT_RB;
        const int64_t g00 = static_cast<int64_t>(it.q) * HT_RB * K;
        float *th = ht_smem + sm.th + s * HT_RB * KM;
        for (int e = tid; e < HT_RB * K; e += HT_THREADS) {
            const bool in = e < nrow * K;
            th[e] = in ? L.W[g00 + e] : 0.f;
            if (res_mv) {
                ht_smem[sm.mv + s * 2 * HT_RB * KM + e] = in ? L.mW[g00 + e] : 0.f;
                ht_smem[sm.mv + s * 2 * HT_RB * KM + HT_RB * KM + e] = in ? L.vW[g00 + e] : 0.f;
            }
        }
        if (tid < HT_RB) {
            const bool in = tid < nrow;
            ht_smem[sm.bs + s * HT_RB + tid] = in ? L.b[it.q * HT_RB + tid] : 0.f;
            ht_smem[sm.bm + s * 2 * HT_RB + tid] = (in && a.update) ? L.mb[it.q * HT_RB + tid] : 0.f;
            ht_smem[sm.bm + s * 2 * HT_RB + HT_RB + tid] = (in && a.update) ? L.vb[it.q * HT_RB + tid] : 0.f;
        }
    }
    __syncthreads();

    unsigned long long t_prev = ht_now();
    for (int t = 0; t < a.n_steps; ++t) {
        const int step = a.first_step + t;
        const int off = t * a.batch;
        const int Bt = (a.n - off < a.batch) ? (a.n - off) : a.batch;
        if (tid < Bt) ridx[tid] = a.perm ? a.perm[off + tid] : static_cast<int64_t>(off + tid);
        if (a.update && (t % HT_BCW) == 0) {
            // AdamW bias corrections of the next 256 steps, one step per thread (double precision like Python's 1 - beta ** step)
            const double st = static_cast<double>(step + tid);
            bc[2 * tid] = static_cast<float>(1.0 - pow(static_cast<double>(a.beta1), st));
            bc[2 * tid + 1] = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(a.beta2), st)));
        }
        __syncthreads();
        const bool drop = a.dropout_p > 0.f;

        // ================= P1 / P2 / P3a: forward of the own rows =================
        for (int l = 0; l < 3; ++l) {
            const Layer &L = a.L[l];
            const float *A = l == 0 ? a.X : (l == 1 ? a.h0d : a.h1d);
            float *dst = l == 0 ? a.h0d : (l == 1 ? a.h1d : a.z);
            const float *inj = l == 0 ? a.mask0 : a.mask1;
            for (int s = 0; s < a.slots; ++s) {
                const int i = cta + s * G;
                if (i >= a.items) break;
                const Item it = ht_item(a, i);
                if (it.l != l) continue;
                const int q = it.q;
                float *fac = ht_smem + sm.fac + s * a.batch * HT_RB;
                ht_rows_dot<false>(out, As, red, Wt, a.nst, A, L.K, l == 0 ? ridx : nullptr, Bt, L.K, ht_smem + sm.th + s * HT_RB * KM, nullptr,
                                   0, 0, 0, dt);
                for (int e = tid; e < Bt * HT_RB; e += HT_THREADS) {
                    const int b = e / HT_RB, j = e % HT_RB;
                    const int r = q * HT_RB + j;
                    if (r >= L.rows) continue;
                    const float pre = out[e] + ht_smem[sm.bs + s * HT_RB + j];
                    if (l == 2) {
                        dst[static_cast<int64_t>(b) * C + r] = pre;
                    } else {
                        float mk = 1.f;
                        if (drop) mk = inj ? inj[static_cast<int64_t>(b) * L.rows + r]
                                           : ht_mask(a.dropout_p, a.seed, 2ull * step + l, static_cast<unsigned long long>(b) * L.rows + r);
                        const float h = pre > 0.f ? pre : 0.f;
                        dst[static_cast<int64_t>(b) * L.rows + r] = h * mk;
                        fac[b * HT_RB + j] = pre > 0.f ? mk : 0.f;
                    }
                }
                __syncthreads();
            }
            HT_STAMP(2 * l);
            ht_grid_sync(a.bar, bar_target);
            HT_STAMP(2 * l + 1);
        }

        // ================= P3b: loss and dz, one warp per batch row =================
        for (int b = cta + G * warp; b < Bt; b += G * HT_KPARTS) {
            const float *zr = a.z + static_cast<int64_t>(b) * C;
            float *dr = a.dz + static_cast<int64_t>(b) * ldz;
            if (STRAT || a.loss_kind == 0) {
                const int64_t y = static_cast<const int64_t *>(a.targets)[ridx[b]];
                // the first 128 logits of the row are fetched once (one L2 round trip), wider rows re-read the tail
                float zc[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) zc[u] = lane + 32 * u < C ? HT_LDCG(zr + lane + 32 * u) : -3.402823466e38f;
                const float zy = (y >= 0 && y < C) ? HT_LDCG(zr + y) : 0.f;
                float mx = fmaxf(fmaxf(zc[0], zc[1]), fmaxf(zc[2], zc[3]));
                for (int j = lane + 128; j < C; j += 32) mx = fmaxf(mx, HT_LDCG(zr + j));
                for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
                float sum = 0.f;
#pragma unroll
                for (int u = 0; u < 4; ++u) if (lane + 32 * u < C) sum += expf(zc[u] - mx);
                for (int j = lane + 128; j < C; j += 32) sum += expf(HT_LDCG(zr + j) - mx);
                for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                const float lse = mx + logf(sum);
                float invB = 1.f / static_cast<float>(Bt);          // the row's weight in the batch loss
                if (STRAT) {
                    const float invR = 1.f / static_cast<float>(a.n_regular);
                    invB = invR;
                    if (b >= a.n_regular) {
                        // first argmax of the row's logits (the same dropout masks as its loss): lanes scan their columns in
                        // ascending order, the shuffle tree keeps the smaller column on equal values
                        float bv = zc[0];
                        int bi = lane;
#pragma unroll
                        for (int u = 1; u < 4; ++u)
                            if (lane + 32 * u < C && zc[u] > bv) { bv = zc[u]; bi = lane + 32 * u; }
                        for (int j = lane + 128; j < C; j += 32) {
                            const float zv = HT_LDCG(zr + j);
                            if (zv > bv) { bv = zv; bi = j; }
                        }
                        for (int o = 16; o > 0; o >>= 1) {
                            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
                            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
                        }
                        invB = (bi != y) ? a.strategic_lambda * invR : 0.f;
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int j = lane + 32 * u;
                    if (j < C) dr[j] = (expf(zc[u] - mx) / sum - (j == y ? 1.f : 0.f)) * invB;
                    else if (j < ldz) dr[j] = 0.f;
                }
                for (int j = lane + 128; j < ldz; j += 32) {
                    if (j < C) {
                        const float p = expf(HT_LDCG(zr + j) - mx) / sum;
                        dr[j] = (p - (j == y ? 1.f : 0.f)) * invB;
                    } else {
                        dr[j] = 0.f;
                    }
                }
                if (lane == 0) a.rowloss[b] = (y >= 0 && y < C) ? (STRAT ? invB * (lse - zy) : (lse - zy)) : 0.f;
            } else {
                const float *yr = static_cast<const float *>(a.targets) + ridx[b] * C;
                const float numel = static_cast<float>(Bt) * static_cast<float>(C);
                float l = 0.f;
                for (int j = lane; j < ldz; j += 32) {
                    if (j < C) {
                        const float s = 1.f / (1.f + expf(-HT_LDCG(zr + j)));
                        const float y = yr[j];
                        l -= y * fmaxf(logf(s), -100.f) + (1.f - y) * fmaxf(logf(1.f - s), -100.f);   // nn.BCELoss clamps log at -100
                        // ATen's BCE backward (s - y) / max(s (1 - s), 1e-12) / (B C), then sigmoid's backward times (1 - s) s:
                        // not (s - y) / (B C), which differs where s rounds to 1 (z > 16.6) or s (1 - s) < 1e-12 (z < -27.6)
                        const float sp = (1.f - s) * s;
                        dr[j] = (s - y) / fmaxf(sp, 1e-12f) / numel * (1.f - s) * s;
                    } else {
                        dr[j] = 0.f;
                    }
                }
                for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
                if (lane == 0) a.rowloss[b] = l / static_cast<float>(C);
            }
        }
        HT_STAMP(6);
        ht_grid_sync(a.bar, bar_target);
        HT_STAMP(7);

        // ================= P4: da1 of the own rows (layer-1 blocks).  The layer-2 weight gradients need nothing newer than dz
        // either, but they wait for the next phase: there the layer-2 CTAs would idle while layer 0 works, here they would be
        // the critical path =================
        for (int s = 0; s < a.slots; ++s) {
            const int i = cta + s * G;
            if (i >= a.items) break;
            const Item it = ht_item(a, i);
            const int q = it.q;
            if (it.l == 1) {
                ht_rows_dot<true>(out, As, red, Wt, a.nst, a.dz, ldz, nullptr, Bt, ldz, nullptr, a.L[2].W, H1, q * HT_RB, C, dt);
                float *f1 = ht_smem + sm.fac + s * a.batch * HT_RB;
                for (int e = tid; e < Bt * HT_RB; e += HT_THREADS) {
                    const int b = e / HT_RB, j = e % HT_RB, r = q * HT_RB + j;
                    const float d = out[e] * f1[e];
                    f1[e] = r < H1 ? d : 0.f;                                   // da1 of the own rows (for gW1 in P5)
                    if (r < H1) a.da1[static_cast<int64_t>(b) * H1 + r] = d;
                }
                __syncthreads();
            }
        }
        HT_STAMP(8);
        ht_grid_sync(a.bar, bar_target);
        HT_STAMP(9);

        // ================= P5: layer-1 weight gradients (layer-1 blocks).  P6: da0 and layer-0 weight gradients (layer-0 blocks) ====
        for (int s = 0; s < a.slots; ++s) {
            const int i = cta + s * G;
            if (i >= a.items) break;
            const Item it = ht_item(a, i);
            const int q = it.q;
            float *fs = ht_smem + sm.fac + s * a.batch * HT_RB;
            if (it.l == 2) {
                for (int e = tid; e < Bt * HT_RB; e += HT_THREADS) {
                    const int b = e / HT_RB, r = q * HT_RB + e % HT_RB;
                    dA[e] = r < C ? HT_LDCG(a.dz + static_cast<int64_t>(b) * ldz + r) : 0.f;
                }
                __syncthreads();
                if (tid < HT_RB) {
                    float sb = 0.f;
                    for (int b = 0; b < Bt; ++b) sb += dA[b * HT_RB + tid];
                    ht_smem[sm.gb + s * HT_RB + tid] = sb;
                }
                ht_outer_acc(ht_smem + sm.g + s * HT_RB * KM, As, a.nst, dA, a.h1d, H1, nullptr, Bt, H1, dt);
            } else if (it.l == 1) {
                if (tid < HT_RB) {
                    float sb = 0.f;
                    for (int b = 0; b < Bt; ++b) sb += fs[b * HT_RB + tid];
                    ht_smem[sm.gb + s * HT_RB + tid] = sb;
                }
                ht_outer_acc(ht_smem + sm.g + s * HT_RB * KM, As, a.nst, fs, a.h0d, H0, nullptr, Bt, H0, dt);
            } else if (it.l == 0) {
                ht_rows_dot<true>(out, As, red, Wt, a.nst, a.da1, H1, nullptr, Bt, H1, nullptr, a.L[1].W, H0, q * HT_RB, H1, dt);
                for (int e = tid; e < Bt * HT_RB; e += HT_THREADS) {
                    const int r = q * HT_RB + e % HT_RB;
                    fs[e] = r < H0 ? out[e] * fs[e] : 0.f;                      // da0 of the own rows
                }
                __syncthreads();
                if (tid < HT_RB) {
                    float sb = 0.f;
                    for (int b = 0; b < Bt; ++b) sb += fs[b * HT_RB + tid];
                    ht_smem[sm.gb + s * HT_RB + tid] = sb;
                }
                ht_outer_acc(ht_smem + sm.g + s * HT_RB * KM, As, a.nst, fs, a.X, D, ridx, Bt, D, dt);
            }
        }
        __syncthreads();

        // ---- EWC gradient on the own rows, partial sum of squares of the own gradients (a block's rows are one linear range)
        float ss = 0.f, pen = 0.f;
        const float ewc2 = a.use_ewc ? 2.f * a.ewc_lambda / static_cast<float>(Bt) : 0.f;
        for (int s = 0; s < a.slots; ++s) {
            const int i = cta + s * G;
            if (i >= a.items) break;
            const Item it = ht_item(a, i);
            const Layer &L = a.L[it.l];
            const int K = L.K, q = it.q;
            const int nrow = (L.rows - q * HT_RB < HT_RB) ? (L.rows - q * HT_RB) : HT_RB;
            int erow = a.use_ewc ? (L.ewc_rows - q * HT_RB) : 0;
            erow = erow < 0 ? 0 : (erow > nrow ? nrow : erow);
            const int64_t g00 = static_cast<int64_t>(q) * HT_RB * K;
            float4 *g4 = reinterpret_cast<float4 *>(ht_smem + sm.g + s * HT_RB * KM);
            const float4 *th4 = reinterpret_cast<const float4 *>(ht_smem + sm.th + s * HT_RB * KM);
            const int n4 = nrow * K / 4, n4e = erow * K / 4;
            for (int e = tid; e < n4; e += HT_THREADS) {
                float4 gq = g4[e];
                if (e < n4e) {
                    const float4 tq = th4[e];
                    const float4 sq = *reinterpret_cast<const float4 *>(L.sW + g00 + 4 * e), fq = *reinterpret_cast<const float4 *>(L.fW + g00 + 4 * e);
                    float dl;
                    dl = tq.x - sq.x; gq.x = fmaf(ewc2 * fq.x, dl, gq.x); pen = fmaf(fq.x * dl, dl, pen);
                    dl = tq.y - sq.y; gq.y = fmaf(ewc2 * fq.y, dl, gq.y); pen = fmaf(fq.y * dl, dl, pen);
                    dl = tq.z - sq.z; gq.z = fmaf(ewc2 * fq.z, dl, gq.z); pen = fmaf(fq.z * dl, dl, pen);
                    dl = tq.w - sq.w; gq.w = fmaf(ewc2 * fq.w, dl, gq.w); pen = fmaf(fq.w * dl, dl, pen);
                    g4[e] = gq;
                }
                ss = fmaf(gq.x, gq.x, ss);
                ss = fmaf(gq.y, gq.y, ss);
                ss = fmaf(gq.z, gq.z, ss);
                ss = fmaf(gq.w, gq.w, ss);
            }
            if (tid < nrow) {
                const int r = q * HT_RB + tid;
                float gv = ht_smem[sm.gb + s * HT_RB + tid];
                if (tid < erow) {
                    const float dlt = ht_smem[sm.bs + s * HT_RB + tid] - L.sb[r];
                    const float f = L.fb[r];
                    gv = fmaf(ewc2 * f, dlt, gv);
                    pen = fmaf(f * dlt, dlt, pen);
                    ht_smem[sm.gb + s * HT_RB + tid] = gv;
                }
                ss = fmaf(gv, gv, ss);
            }
        }
        ss = ht_block_sum(ss, rsum);
        if (a.use_ewc) pen = ht_block_sum(pen, rsum);
        if (tid == 0) { a.part[cta] = ss; a.pen[cta] = pen; }
        HT_STAMP(10);
        ht_grid_sync(a.bar, bar_target);
        HT_STAMP(11);

        // ================= P7: global norm, clip, AdamW on the own rows =================
        float tot = 0.f, pt = 0.f, ls = 0.f;
        const bool stats_cta = cta == G - 1;              // the last CTA holds the fewest / shortest rows: it also reports the step
        if (warp == 0) {
            // every CTA adds the G partials in the same fixed order: lane-strided sums, then a shuffle tree
            for (int i = lane; i < G; i += 32) { tot += HT_LDCG(a.part + i); if (a.use_ewc) pt += HT_LDCG(a.pen + i); }
            for (int o = 16; o > 0; o >>= 1) { tot += __shfl_xor_sync(0xffffffffu, tot, o); pt += __shfl_xor_sync(0xffffffffu, pt, o); }
            if (tid == 0) {
                const float norm = sqrtf(tot);
                float coef = a.max_norm / (norm + 1e-6f);
                coef = coef < 1.f ? coef : 1.f;
                if (!(a.max_norm > 0.f)) coef = 1.f;
                scal[0] = coef;
                scal[3] = norm;
            }
        }
        __syncthreads();
        const float coef = scal[0], bc1 = bc[2 * (t % HT_BCW)], bc2s = bc[2 * (t % HT_BCW) + 1];
        const float decay = 1.f - a.lr * a.wd, lr_c = a.lr / bc1;
        for (int s = 0; s < a.slots; ++s) {
            const int i = cta + s * G;
            if (i >= a.items) break;
            const Item it = ht_item(a, i);
            const Layer &L = a.L[it.l];
            const int K = L.K, q = it.q;
            const int nrow = (L.rows - q * HT_RB < HT_RB) ? (L.rows - q * HT_RB) : HT_RB;
            const int64_t g00 = static_cast<int64_t>(q) * HT_RB * K;
            float *th = ht_smem + sm.th + s * HT_RB * KM;
            const float *g = ht_smem + sm.g + s * HT_RB * KM;
            const int n4 = nrow * K / 4;
            if (a.update) {
                if (res_mv) {
                    float *m = ht_smem + sm.mv + s * 2 * HT_RB * KM;
                    ht_adamw_block<true>(th, g, m, m + HT_RB * KM, L.W + g00, n4, coef, decay, lr_c, bc2s, a.beta1, a.beta2, a.eps);
                } else {
                    ht_adamw_block<false>(th, g, L.mW + g00, L.vW + g00, L.W + g00, n4, coef, decay, lr_c, bc2s, a.beta1, a.beta2, a.eps);
                }
            } else {
                for (int e = tid; e < nrow * K; e += HT_THREADS) {
                    const float graw = g[e];
                    if (L.gW) L.gW[g00 + e] = graw;
                    if (L.qW) L.qW[g00 + e] += graw * graw * a.fisher_scale;
                }
            }
            if (tid < nrow) {
                const int r = q * HT_RB + tid;
                const float graw = ht_smem[sm.gb + s * HT_RB + tid];
                if (a.update) {
                    const float gv = graw * coef;
                    float p = ht_smem[sm.bs + s * HT_RB + tid] * decay;
                    float *bmom = ht_smem + sm.bm + s * 2 * HT_RB;
                    const float m1 = bmom[tid] * a.beta1 + gv * (1.f - a.beta1);
                    const float v1 = bmom[HT_RB + tid] * a.beta2 + gv * gv * (1.f - a.beta2);
                    const float denom = sqrtf(v1) / bc2s + a.eps;
                    p = p - lr_c * (m1 / denom);
                    ht_smem[sm.bs + s * HT_RB + tid] = p;
                    L.b[r] = p;
                    bmom[tid] = m1;
                    bmom[HT_RB + tid] = v1;
                } else {
                    if (L.gb) L.gb[r] = graw;
                    if (L.qb) L.qb[r] += graw * graw * a.fisher_scale;
                }
            }
        }
        if (stats_cta && warp == 0) {
            // batch loss: the row losses are fetched in parallel, added in row order (after this CTA's own update: off the critical path)
            float r0 = lane < Bt ? HT_LDCG(a.rowloss + lane) : 0.f, r1 = lane + 32 < Bt ? HT_LDCG(a.rowloss + lane + 32) : 0.f;
            for (int b = 0; b < 32; ++b) ls += __shfl_sync(0xffffffffu, r0, b);
            for (int b = 0; b < 32; ++b) ls += __shfl_sync(0xffffffffu, r1, b);
            if (tid == 0) {
                const float loss = STRAT ? ls : ls / static_cast<float>(Bt);     // CE_STRATEGIC rows carry their weights
                const float penalty = a.use_ewc ? a.ewc_lambda / static_cast<float>(Bt) * pt : 0.f;
                if (a.stats) { a.stats[3 * t + 0] = loss; a.stats[3 * t + 1] = penalty; a.stats[3 * t + 2] = scal[3]; }
                if (a.loss_accum) a.loss_accum[0] += loss + penalty;
            }
        }
        __syncthreads();
        HT_STAMP(12);
    }

    // ---- resident moments go back to global memory
    if (a.update) {
        for (int s = 0; s < a.slots; ++s) {
            const int i = cta + s * G;
            if (i >= a.items) break;
            const Item it = ht_item(a, i);
            const Layer &L = a.L[it.l];
            const int K = L.K;
            const int nrow = (L.rows - it.q * HT_RB < HT_RB) ? (L.rows - it.q * HT_RB) : HT_RB;
            const int64_t g00 = static_cast<int64_t>(it.q) * HT_RB * K;
            if (res_mv)
                for (int e = tid; e < nrow * K; e += HT_THREADS) {
                    L.mW[g00 + e] = ht_smem[sm.mv + s * 2 * HT_RB * KM + e];
                    L.vW[g00 + e] = ht_smem[sm.mv + s * 2 * HT_RB * KM + HT_RB * KM + e];
                }
            if (tid < nrow) {
                L.mb[it.q * HT_RB + tid] = ht_smem[sm.bm + s * 2 * HT_RB + tid];
                L.vb[it.q * HT_RB + tid] = ht_smem[sm.bm + s * 2 * HT_RB + HT_RB + tid];
            }
        }
    }
}

}  // namespace ht
}  // namespace ac
