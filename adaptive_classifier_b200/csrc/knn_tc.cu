// knn_tc.cu -- stage K, tensor path: brute-force squared-L2 kNN over a large prototype matrix.
//
//   pass 1        d~(q,p) = ||q||^2 + ||p||^2 - 2 q.p   with q.p on wgmma (.f16 over the fp16 shadow of the rows, or
//                 .tf32 on the fp32 rows) through the GEMM mainloop of gemm_tc.cuh: M = queries (128 per CTA, fixed per
//                 CTA), N = prototype rows streamed ONCE from HBM by TMA, fp32 accumulators staged in shared memory.
//                 Epilogue EpiKnn: thread = query row; running top-16 (coarse key, row id) per (query, CTA, column half).
//   k <= 16       merge the lists, exact fp32 re-rank of the best KP = 32 candidates in the oracle's lane order
//                 (knn_exact.cu), CERTIFY: T = smallest coarse distance any non-candidate row can have, eps = rigorous bound
//                 on |d~ - d|; d_exact[k-1] < T - eps => no excluded row can enter or tie the top-k.
//   pass 2        for the queries pass 1 could not certify, and for every query when k > 16: with tau = the k-th smallest
//                 coarse distance among the merged candidates (real rows, so the exact k-th distance is <= tau + eps), a
//                 second tensor pass (EpiKnnCollect) appends EVERY row with d~ <= tau + 2 eps to a per-query buffer -- a
//                 superset of the true top-k -- which is then re-ranked exactly and selected by (d, id).
//                 The pass is launched unconditionally and exits at once when a device-side counter says nobody needs it:
//                 no host synchronisation anywhere, the whole search is capturable in a CUDA graph, and the worst case
//                 (every query uncertified, e.g. near-duplicate rows closer than eps) costs one more scan instead of a
//                 full fp32 SIMT scan per query.
//   overflow      a query with more than `cap` rows inside the 2 eps band (thousands of near-identical rows) is reported
//                 in stats[1]; without a stats pointer the call synchronises and recomputes those queries by the exact scan.
// Result: (d, id) bit-identical to the exact path / the oracle.
//
// Replaces faiss.IndexFlatL2.search (/root/reference/src/adaptive_classifier/memory.py:110-114) for the
// batched, large-N configurations of BASELINE.json (configs[1], configs[2], configs[4]); k = num_classes (predict(),
// classifier.py:424-425) stays on the tensor path up to k = 1024.
#include "gemm_tc.cuh"
#include <cuda_fp16.h>
#include <math_constants.h>

namespace ac {

int launch_knn_rerank(const float *Q, const float *P, int B, int64_t N, int D, int kc, const int32_t *cand, float *out_d,
                      int64_t *out_i, int64_t row_offset, cudaStream_t stream);
size_t topk_select_workspace(int B, int64_t L, int k);
int topk_select(const float *d, const int64_t *idx, int B, int64_t L, int64_t in_stride, int64_t id_offset, int k,
                float *out_d, int64_t *out_i, void *ws, size_t ws_bytes, cudaStream_t stream, const float *row_gate = nullptr);
int knn_exact_subset(const float *Q, const float *P, int B, int64_t N, int D, int k, float *out_d, int64_t *out_i,
                     int64_t row_offset, void *ws, size_t ws_bytes, cudaStream_t s);
size_t knn_exact_workspace_pub(int B, int64_t N, int k);

constexpr int KNN_KC = 16;   // candidates kept per (query, CTA)
constexpr int KNN_KP = 32;   // candidates re-ranked per query

// ------------------------------------------------------------------------------------------------
// coarse-pass epilogue
// ------------------------------------------------------------------------------------------------
// order-preserving map float -> uint32 (and back) so that atomicMin works on signed keys
__device__ __forceinline__ uint32_t key_to_ord(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord_to_key(uint32_t o) {
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

struct EpiKnn {
    const float *p_sqnorm;   // [N]
    float *cand_key;         // [B, slots, KC]  coarse key = ||p||^2 - 2 q.p  (||q||^2 added later)
    int32_t *cand_idx;       // [B, slots, KC]  local row id, -1 = empty
    uint32_t *gthr;          // [Bp] per query: smallest "worst kept key" published by any list so far (ordered uint)
    int B;                   // queries
    int64_t N;               // rows
    int tiles_m, slots;      // grid = slots/2 * tiles_m CTAs; every CTA owns one query tile and two lists per query
    int kt;                  // a list publishes its kt-th best key (k + 3 <= kt <= KC): see prefetch()

    static constexpr int kUnrollChunks = 1;
    static constexpr int kPrefetchDist = 1;
    struct State {
        float key[KNN_KC];
        int32_t idx[KNN_KC];
        float pn[2];          // ||p||^2 of the 32 rows of a chunk, one per lane, requested one chunk ahead
        float gt;             // global bound for this thread's query, refreshed once per tile
    };

    __device__ __forceinline__ bool skip_kernel() const { return false; }
    __device__ __forceinline__ void begin_cta(State &st, int, int) const {
#pragma unroll
        for (int i = 0; i < KNN_KC; ++i) { st.key[i] = CUDART_INF_F; st.idx[i] = -1; }
        st.pn[0] = st.pn[1] = CUDART_INF_F;
        st.gt = CUDART_INF_F;
    }

    // Every list (2 x (SMs / query tiles) per query) would on its own perform ~KC ln(n/KC) sorted inserts; sharing a bound
    // across lists makes all of them reject what cannot matter any more.  Each list publishes its kt-th best key;
    // gt = min over lists.  Exclusion bound for the certification: T = min over lists of their FINAL kt-th best
    // (<= every published value, gt only decreases).  A row with key < T is never rejected (key < T <= gt(t) and
    // key < T <= list's kt-th best <= list's KC-th best) and never evicted (eviction would put KC better rows in its
    // list, i.e. that list's kt-th best < key, contradicting key < T).  T >= the global kt-th smallest key, so the
    // certification is at least as strong as with one global top-kt list.
    __device__ __forceinline__ void prefetch(State &st, const GemmTileInfo &, int row, int col0, int lane, int buf) const {
        const int64_t n = static_cast<int64_t>(col0) + lane;
        const float x = (n < N) ? __ldg(p_sqnorm + n) : CUDART_INF_F;
        if (buf) st.pn[1] = x; else st.pn[0] = x;
        if (buf == 0) {        // first chunk of a tile: publish this list's bound, pick up the others'
            float pub = CUDART_INF_F;
#pragma unroll
            for (int i = 0; i < KNN_KC; ++i) pub = (i == kt - 1) ? st.key[i] : pub;
            if (pub < CUDART_INF_F) atomicMin(gthr + row, key_to_ord(pub));
            st.gt = ord_to_key(*reinterpret_cast<volatile uint32_t *>(gthr + row));
        }
    }

    __device__ __forceinline__ void insert(State &st, float key, int32_t n) const {
        // sorted insertion (ascending); strict '<' keeps the earlier (lower id) row on ties.  Slots are visited from the
        // tail towards the head, so every read sees the pre-insertion value.
#pragma unroll
        for (int i = KNN_KC - 1; i > 0; --i) {
            const bool shift = key < st.key[i - 1];
            const bool here = !shift && (key < st.key[i]);
            const float nk = shift ? st.key[i - 1] : (here ? key : st.key[i]);
            const int32_t ni = shift ? st.idx[i - 1] : (here ? n : st.idx[i]);
            st.key[i] = nk;
            st.idx[i] = ni;
        }
        if (key < st.key[0]) { st.key[0] = key; st.idx[0] = n; }
    }

    __device__ __forceinline__ void tile(State &st, const GemmTileInfo &, int /*row*/, int col0, const float (&v)[32],
                                         uint8_t * /*stage*/, int /*lane*/, int buf, const float *acc) const {
        // fast path: all lanes walk the same 32 prototype rows and only record which ones beat their query's bound
        const float pn_lane = buf ? st.pn[1] : st.pn[0];
        const float thr = fminf(st.key[KNN_KC - 1], st.gt);
        uint32_t hits = 0;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const float pn = __shfl_sync(0xffffffffu, pn_lane, j);
            const float key = fmaf(-2.f, v[j], pn);
            hits |= (key < thr) ? (1u << j) : 0u;
        }
        // slow path (rare once the bounds are tight): one copy of the insert network, the hit column is read again
        // from the shared-memory accumulator tile because v[] cannot be indexed dynamically
        uint32_t uni = __reduce_or_sync(0xffffffffu, hits);
        while (uni) {
            const int j = __ffs(uni) - 1;
            uni &= uni - 1;
            const float key = fmaf(-2.f, acc[j], __shfl_sync(0xffffffffu, pn_lane, j));
            const int64_t n = static_cast<int64_t>(col0) + j;
            if (((hits >> j) & 1u) && key < fminf(st.key[KNN_KC - 1], st.gt) && n < N) insert(st, key, static_cast<int32_t>(n));
        }
    }

    __device__ __forceinline__ void end_cta(State &st, int q, int lane) const {
        // two epilogue warps share a query row (one per column half of every tile): each owns a slot
        const int chalf = gemm_epi_chalf();
        const int mt = blockIdx.x % tiles_m;
        const int slot = (blockIdx.x / tiles_m) * 2 + chalf;
        const int row = mt * GEMM_BLOCK_M + q * 32 + lane;
        if (row >= B) return;
        float *ck = cand_key + (static_cast<int64_t>(row) * slots + slot) * KNN_KC;
        int32_t *ci = cand_idx + (static_cast<int64_t>(row) * slots + slot) * KNN_KC;
#pragma unroll
        for (int i = 0; i < KNN_KC; ++i) { ck[i] = st.key[i]; ci[i] = st.idx[i]; }
    }
};

// pass 2: append every row whose coarse key is <= thr[query] to the query's candidate buffer (thr = -inf: query not flagged).
// Hits are rare (about k per query over the whole scan), so the fast path is one FFMA + compare per accumulator element.
struct EpiKnnCollect {
    const float *p_sqnorm;   // [N]
    const float *thr;        // [Bp] key-domain threshold: tau_key + 2 eps, or -inf
    int32_t *buf;            // [B, cap] local row ids
    int32_t *cnt;            // [Bp] rows found (may exceed cap: overflow, reported by the re-rank)
    const int32_t *need;     // [0] = number of flagged queries; 0 => the whole kernel exits at once
    int cap, B;
    int64_t N;
    int tiles_m;

    static constexpr int kUnrollChunks = 1;
    static constexpr int kPrefetchDist = 1;
    struct State {
        float pn[2];
        float thr;
    };
    __device__ __forceinline__ bool skip_kernel() const { return *reinterpret_cast<const volatile int32_t *>(need) == 0; }
    __device__ __forceinline__ void begin_cta(State &st, int q, int lane) const {
        const int row = (blockIdx.x % tiles_m) * GEMM_BLOCK_M + q * 32 + lane;     // a CTA keeps one query tile (kMFastest)
        st.thr = (row < B) ? thr[row] : -CUDART_INF_F;
        st.pn[0] = st.pn[1] = CUDART_INF_F;
    }
    __device__ __forceinline__ void prefetch(State &st, const GemmTileInfo &, int, int col0, int lane, int buf_) const {
        const int64_t n = static_cast<int64_t>(col0) + lane;
        const float x = (n < N) ? __ldg(p_sqnorm + n) : CUDART_INF_F;
        if (buf_) st.pn[1] = x; else st.pn[0] = x;
    }
    __device__ __forceinline__ void tile(State &st, const GemmTileInfo &, int row, int col0, const float (&v)[32], uint8_t *,
                                         int, int buf_, const float *) const {
        const float pn_lane = buf_ ? st.pn[1] : st.pn[0];
        uint32_t hits = 0;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const float pn = __shfl_sync(0xffffffffu, pn_lane, j);
            const float key = fmaf(-2.f, v[j], pn);
            hits |= (key <= st.thr) ? (1u << j) : 0u;
        }
        while (hits) {                                   // per-lane: this thread's own hits, ascending row order
            const int j = __ffs(hits) - 1;
            hits &= hits - 1;
            const int64_t n = static_cast<int64_t>(col0) + j;
            if (n < N) {
                const int pos = atomicAdd(cnt + row, 1);
                if (pos < cap) buf[static_cast<int64_t>(row) * cap + pos] = static_cast<int32_t>(n);
            }
        }
    }
    __device__ __forceinline__ void end_cta(State &, int, int) const {}
};


// ------------------------------------------------------------------------------------------------
// small kernels around the coarse pass
// ------------------------------------------------------------------------------------------------
// Qr = tf32(RNE)(Q), qn[b] = ||Q_b||^2 (fp32), one warp per query
__global__ void knn_prep_queries_kernel(const float *__restrict__ Q, int B, int D, float *__restrict__ Qr,
                                        __half *__restrict__ Qh, float *__restrict__ qn) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= B) return;
    float s = 0.f;
    for (int i = lane; i < D; i += 32) {
        const float x = Q[static_cast<int64_t>(row) * D + i];
        if (Qh) Qh[static_cast<int64_t>(row) * D + i] = __float2half_rn(x);
        else Qr[static_cast<int64_t>(row) * D + i] = round_tf32(x);
        s = fmaf(x, x, s);
    }
    s = warp_sum(s);
    if (lane == 0) qn[row] = s;
}

// pn[n] = ||P_n||^2 (only when the caller did not pass the cached norms)
__global__ void knn_prep_rows_kernel(const float *__restrict__ P, int64_t N, int D, float *__restrict__ pn) {
    const int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= N) return;
    const float *p = P + row * D;
    float s = 0.f;
    for (int i = lane; i < D; i += 32) s = fmaf(p[i], p[i], s);
    s = warp_sum(s);
    if (lane == 0) pn[row] = s;
}

// max_n ||p_n||^2 (for the error bound) -> out[0] (zeroed by the caller); non-negative floats order like their bit patterns.
// One grid-stride pass over the norms, kept out of the scan epilogue, whose per-chunk work is on the scan's critical path.
__global__ void knn_max_norm_kernel(const float *__restrict__ pn, int64_t N, float *__restrict__ out) {
    float m = 0.f;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < N; i += stride) m = fmaxf(m, __ldg(pn + i));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int *>(out), __float_as_int(m));
}

// widen the int32 candidate ids of the per-CTA lists for the (key, id) sort
__global__ void knn_widen_kernel(const int32_t *__restrict__ in, int64_t n, int64_t *__restrict__ out) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i];
}

// after the (key,id) sort of all per-CTA candidates: take the best KP ids for the re-rank and compute
//   T[b] = ||q||^2 + min( key of the first entry NOT re-ranked, min over CTAs of their worst kept key )
// sorted_*: [B, KP+1] ascending.  cand_key: [B, slots, KC] (entry kt-1 = the bound that list published).
__global__ void knn_pick_kernel(const float *__restrict__ sorted_key, const int64_t *__restrict__ sorted_idx,
                                const float *__restrict__ cand_key, const float *__restrict__ qn, int B, int slots, int kt,
                                int32_t *__restrict__ rerank_idx /*[B,KP]*/, float *__restrict__ T) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float *sk = sorted_key + static_cast<int64_t>(b) * (KNN_KP + 1);
    const int64_t *si = sorted_idx + static_cast<int64_t>(b) * (KNN_KP + 1);
    for (int j = 0; j < KNN_KP; ++j) rerank_idx[static_cast<int64_t>(b) * KNN_KP + j] = static_cast<int32_t>(si[j]);
    float t = (si[KNN_KP] >= 0) ? sk[KNN_KP] : CUDART_INF_F;
    for (int s = 0; s < slots; ++s) t = fminf(t, cand_key[(static_cast<int64_t>(b) * slots + s) * KNN_KC + (kt - 1)]);
    T[b] = t + qn[b];
}

// rigorous bound on |coarse - exact| for query b: 2*rel*||q||*max||p|| * 1.02 + 4e-5*(1+||q||^2+max||p||^2) with
//   rel = 2^-10 + 2^-11 + 2^-21 (fp32 rows truncated to tf32 by the MMA, queries rounded RNE), or
//   rel = 2^-11 + 2^-11 + 2^-22 (fp16 shadow rows and fp16 queries, both RNE; the subnormal tail adds < 1e-6)
__device__ __forceinline__ float knn_eps(float qn2, float pm2, float rel) {
    return 2.f * rel * 1.02f * sqrtf(qn2) * sqrtf(pm2) + 4e-5f * (1.f + qn2 + pm2);
}

// k <= 16: certified[b] = out_d[b,k-1] < T[b] - eps(b).  An uncertified query is flagged for pass 2 with the key-domain
// threshold  thr = (k-th smallest coarse key among the merged candidates) + 2 eps  (see the header: a superset of the top-k).
// sorted_key / sorted_idx: [B, KP+1] merged candidates ascending.
__global__ void knn_certify_kernel(const float *__restrict__ out_d, const int64_t *__restrict__ out_i, const float *__restrict__ T,
                                   const float *__restrict__ qn, const float *__restrict__ pmax2, const float *__restrict__ sorted_key,
                                   const int64_t *__restrict__ sorted_idx, int B, int Bp, int k, float rel, float *__restrict__ thr,
                                   int32_t *__restrict__ cnt, int32_t *__restrict__ need) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= Bp) return;
    cnt[b] = 0;
    if (b >= B) { thr[b] = -CUDART_INF_F; return; }
    const float eps = knn_eps(qn[b], pmax2[0], rel);
    const float dk = out_d[static_cast<int64_t>(b) * k + (k - 1)];
    const bool full = out_i[static_cast<int64_t>(b) * k + (k - 1)] >= 0;
    // T == +inf: every row of the index was a candidate (nothing excluded) -> exact by construction
    const bool ok = (T[b] == CUDART_INF_F) || (full && dk < T[b] - eps);
    if (ok) { thr[b] = -CUDART_INF_F; return; }
    const bool have_k = sorted_idx[static_cast<int64_t>(b) * (KNN_KP + 1) + (k - 1)] >= 0;
    thr[b] = have_k ? sorted_key[static_cast<int64_t>(b) * (KNN_KP + 1) + (k - 1)] + 2.f * eps : CUDART_INF_F;
    atomicAdd(need, 1);
}

// k > 16: every query takes pass 2; sorted_key / sorted_idx: [B, k] merged candidates ascending
__global__ void knn_threshold_kernel(const float *__restrict__ sorted_key, const int64_t *__restrict__ sorted_idx,
                                     const float *__restrict__ qn, const float *__restrict__ pmax2, int B, int Bp, int k, float rel,
                                     float *__restrict__ thr, int32_t *__restrict__ cnt, int32_t *__restrict__ need) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= Bp) return;
    cnt[b] = 0;
    if (b >= B) { thr[b] = -CUDART_INF_F; return; }
    const bool have_k = sorted_idx[static_cast<int64_t>(b) * k + (k - 1)] >= 0;
    thr[b] = have_k ? sorted_key[static_cast<int64_t>(b) * k + (k - 1)] + 2.f * knn_eps(qn[b], pmax2[0], rel) : CUDART_INF_F;
    if (b == 0) need[0] = B;
}

// exact distance (oracle lane order, as knn_rerank_kernel) of the rows pass 2 collected; one 8-lane group per buffer slot.
// Slots >= cnt[b] are written as padding; queries that were not flagged are skipped.  Overflowing queries are counted.
__global__ void knn_rerank_collected_kernel(const float *__restrict__ Q, const float *__restrict__ P, int B, int64_t N, int D, int cap,
                                            const float *__restrict__ thr, const int32_t *__restrict__ cnt,
                                            const int32_t *__restrict__ buf, float *__restrict__ out_d, int64_t *__restrict__ out_i,
                                            int64_t row_offset, int32_t *__restrict__ stats, int32_t *__restrict__ over_list) {
    const int b = blockIdx.y;
    if (thr[b] == -CUDART_INF_F) return;                                         // block-uniform
    const int slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const int j = threadIdx.x & 7;
    const int have = cnt[b];
    const int n_use = have < cap ? have : cap;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        atomicAdd(stats + 0, 1);
        atomicMax(stats + 2, have);
        if (have > cap) over_list[atomicAdd(stats + 1, 1)] = b;
    }
    const bool valid = slot < cap;
    int32_t r = -1;
    if (valid && slot < n_use) r = buf[static_cast<int64_t>(b) * cap + slot];
    float acc = 0.f;
    if (r >= 0 && r < N) {
        const float *q = Q + static_cast<int64_t>(b) * D;
        const float *p = P + static_cast<int64_t>(r) * D;
        for (int i = j; i < D; i += 8) {
            const float t = __fsub_rn(q[i], p[i]);
            acc = __fadd_rn(acc, __fmul_rn(t, t));
        }
    }
    const unsigned m = 0xffffffffu;
    const float s4 = __fadd_rn(acc, __shfl_xor_sync(m, acc, 4));
    const float s1 = __fadd_rn(s4, __shfl_xor_sync(m, s4, 1));
    const float s2 = __fadd_rn(s1, __shfl_xor_sync(m, s1, 2));
    if (valid && j == 0) {
        const bool ok = (r >= 0 && r < N);
        out_d[static_cast<int64_t>(b) * cap + slot] = ok ? s2 : CUDART_INF_F;
        out_i[static_cast<int64_t>(b) * cap + slot] = ok ? (static_cast<int64_t>(r) + row_offset) : -1;
    }
}

__global__ void knn_gather_rows_kernel(const float *__restrict__ src, const int32_t *__restrict__ list, int n, int D,
                                       float *__restrict__ dst) {
    const int r = blockIdx.x;
    if (r >= n) return;
    const float *s = src + static_cast<int64_t>(list[r]) * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) dst[static_cast<int64_t>(r) * D + i] = s[i];
}
__global__ void knn_scatter_results_kernel(const float *__restrict__ d, const int64_t *__restrict__ idx,
                                           const int32_t *__restrict__ list, int n, int k, float *__restrict__ out_d,
                                           int64_t *__restrict__ out_i) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * k) return;
    const int r = t / k, j = t % k;
    out_d[static_cast<int64_t>(list[r]) * k + j] = d[t];
    out_i[static_cast<int64_t>(list[r]) * k + j] = idx[t];
}
__global__ void knn_add_stats_kernel(const int32_t *__restrict__ in, int32_t *__restrict__ out) {
    if (threadIdx.x == 0) { out[0] += in[0]; out[1] += in[1]; out[2] = max(out[2], in[2]); out[3] += 1; }
}

// ------------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------------
constexpr int KNN_SMALL_K = 16;        // certification path (lists of KNN_KC per (query, CTA, half))
// k > 16: queries per pass.  tau (the bound on the k-th distance) is the k-th smallest key among the merged lists, so it is
// tight only if no list had to drop a top-k row for lack of room (16 entries).  A list sees ~k / (lists per query) top-k rows.
// Two query tiles per pass give every query 2 x (SMs / 2) = 132 lists on an H100 over interleaved row tiles: at k = 1000 a list
// holds ~7.6 top-k rows on average, well under 16.  Four tiles per pass would halve the lists per query (~15 rows per list, so
// lists overflow and tau loosens); one tile per pass would scan the prototype matrix twice as often.  On an H100 80GB HBM3,
// 256 queries per pass run the k = 1000 search of 512 queries over 1 M x 768 rows in 4.7 ms with no overflowing query
// (`k_equals_C` in profiles/h100_bench.json).
#ifndef AC_KNN_QUERY_BLOCK
#define AC_KNN_QUERY_BLOCK 256
#endif
constexpr int KNN_QUERY_BLOCK = AC_KNN_QUERY_BLOCK;
static int knn_cap(int k) { return k <= KNN_SMALL_K ? 256 : 4096; }

struct KnnTcPlan {
    int tiles_m, slots, grid_ctas, cap, ksel;
    size_t off_qr, off_qn, off_gthr, off_pn, off_pmax, off_ckey, off_cidx, off_cidx64, off_skey, off_sidx, off_ridx, off_T,
        off_rd, off_ri, off_thr, off_cnt, off_stats, off_over, off_buf, off_rd2, off_ri2, off_sel, sel_bytes, total;
};

static KnnTcPlan plan_knn_tc(int B, int64_t N, int D, int k) {
    KnnTcPlan p;
    p.tiles_m = (B + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
    const int sms = sm_count();
    p.slots = sms / p.tiles_m;
    if (p.slots < 1) p.slots = 1;
    const int64_t tiles_n = (N + GEMM_BLOCK_N - 1) / GEMM_BLOCK_N;
    if (p.slots > tiles_n) p.slots = static_cast<int>(tiles_n);
    p.grid_ctas = p.slots * p.tiles_m;
    p.slots *= 2;   // candidate lists per query: one per (CTA, accumulator column half)
    p.cap = knn_cap(k);
    p.ksel = k <= KNN_SMALL_K ? KNN_KP + 1 : k;      // how many merged candidates are kept sorted
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes, 256); return o; };
    const size_t Bp = static_cast<size_t>(p.tiles_m) * GEMM_BLOCK_M;
    p.off_qr = take(Bp * D * 4);
    p.off_qn = take(Bp * 4);
    p.off_gthr = take(Bp * 4);
    p.off_pn = take(static_cast<size_t>(N) * 4);
    p.off_pmax = take(256);
    const size_t nc = static_cast<size_t>(B) * p.slots * KNN_KC;
    p.off_ckey = take(nc * 4);
    p.off_cidx = take(nc * 4);
    p.off_cidx64 = take(nc * 8);
    p.off_skey = take(static_cast<size_t>(B) * p.ksel * 4);
    p.off_sidx = take(static_cast<size_t>(B) * p.ksel * 8);
    p.off_ridx = take(static_cast<size_t>(B) * KNN_KP * 4);
    p.off_T = take(static_cast<size_t>(B) * 4);
    p.off_rd = take(static_cast<size_t>(B) * KNN_KP * 4);
    p.off_ri = take(static_cast<size_t>(B) * KNN_KP * 8);
    p.off_thr = take(Bp * 4);
    p.off_cnt = take(Bp * 4);
    p.off_stats = take(256);                          // [0] flagged, [1] overflowed, [2] max collected, [4] need (pass-2 gate)
    p.off_over = take(static_cast<size_t>(B) * 4);
    p.off_buf = take(static_cast<size_t>(B) * p.cap * 4);
    p.off_rd2 = take(static_cast<size_t>(B) * p.cap * 4);
    p.off_ri2 = take(static_cast<size_t>(B) * p.cap * 8);
    size_t sel = topk_select_workspace(B, static_cast<int64_t>(p.slots) * KNN_KC, p.ksel);
    const size_t sel2 = topk_select_workspace(B, p.cap, k);
    if (sel2 > sel) sel = sel2;
    p.sel_bytes = sel + 256;
    p.off_sel = take(p.sel_bytes);
    p.total = off;
    return p;
}

static int knn_block(int B, int k) { return (k > KNN_SMALL_K && B > KNN_QUERY_BLOCK) ? KNN_QUERY_BLOCK : B; }

size_t knn_tc_workspace(int B, int64_t N, int D, int k) {
    const int Bb = knn_block(B, k);
    KnnTcPlan p = plan_knn_tc(Bb, N, D, k);
    // exact-scan staging for overflowed queries (synchronous mode only): gathered queries + their results + the scan's scratch
    const size_t fb = align_up(static_cast<size_t>(Bb) * D * 4, 256) + align_up(static_cast<size_t>(Bb) * k * 4, 256) +
                      align_up(static_cast<size_t>(Bb) * k * 8, 256);
    return p.total + fb + knn_exact_workspace_pub(Bb, N, k) + 1024;
}

template <class Epi>
static int launch_scan(const float *Qr, const float *P, const void *p_half, size_t Bp, int64_t N, int D, const Epi &epi, int grid_ctas,
                       int prof_cls, cudaStream_t s) {
    CUtensorMap ta, tb;
    int rc;
    // algorithmic work of the scan: 2.B.N.D flops, one read of the fp32 prototype matrix (4.N.D bytes); with the fp16 shadow
    // the kernel actually streams 2.N.D bytes (the exact re-rank still reads fp32 rows): both are reported by bench.py
    const double bytes = 4.0 * static_cast<double>(N) * D;
    if (p_half) {
        if ((rc = make_tmap_2d(&ta, Qr, 2, Bp, D, static_cast<uint64_t>(D) * 2, GEMM_BLOCK_M, 64))) return rc;
        if ((rc = make_tmap_2d(&tb, p_half, 2, static_cast<uint64_t>(N), D, static_cast<uint64_t>(D) * 2, GEMM_BLOCK_N, 64))) return rc;
        return launch_gemm_tc<Epi, true, GEMM_KIND_F16>(ta, tb, static_cast<int>(Bp), static_cast<int>(N), D, epi, s, grid_ctas, prof_cls, bytes);
    }
    if ((rc = make_tmap_2d(&ta, Qr, 4, Bp, D, static_cast<uint64_t>(D) * 4, GEMM_BLOCK_M, GEMM_BLOCK_K))) return rc;
    if ((rc = make_tmap_2d(&tb, P, 4, static_cast<uint64_t>(N), D, static_cast<uint64_t>(D) * 4, GEMM_BLOCK_N, GEMM_BLOCK_K))) return rc;
    return launch_gemm_tc<Epi, true, GEMM_KIND_TF32>(ta, tb, static_cast<int>(Bp), static_cast<int>(N), D, epi, s, grid_ctas, prof_cls, bytes);
}

static int knn_tc_block(const float *Q, const float *P, const float *p_sqnorm, const void *p_half, int B, int64_t N, int D, int k,
                        float *out_d, int64_t *out_i, int64_t row_offset, void *ws, size_t ws_bytes, int32_t *stats_out,
                        cudaStream_t s) {
    int rc;
    KnnTcPlan pl = plan_knn_tc(B, N, D, k);
    const size_t fb_q = align_up(static_cast<size_t>(B) * D * 4, 256), fb_d = align_up(static_cast<size_t>(B) * k * 4, 256),
                 fb_i = align_up(static_cast<size_t>(B) * k * 8, 256);
    const size_t exact_ws = knn_exact_workspace_pub(B, N, k);
    if (pl.total + fb_q + fb_d + fb_i + exact_ws > ws_bytes) {
        set_error("knn_tc_search: workspace needs %zu bytes, have %zu", pl.total + fb_q + fb_d + fb_i + exact_ws, ws_bytes);
        return AC_E_WORKSPACE;
    }
    uint8_t *w = static_cast<uint8_t *>(ws);
    float *Qr = reinterpret_cast<float *>(w + pl.off_qr);
    float *qn = reinterpret_cast<float *>(w + pl.off_qn);
    uint32_t *gthr = reinterpret_cast<uint32_t *>(w + pl.off_gthr);
    float *pn = reinterpret_cast<float *>(w + pl.off_pn);
    float *pmax = reinterpret_cast<float *>(w + pl.off_pmax);
    float *ckey = reinterpret_cast<float *>(w + pl.off_ckey);
    int32_t *cidx = reinterpret_cast<int32_t *>(w + pl.off_cidx);
    int64_t *cidx64 = reinterpret_cast<int64_t *>(w + pl.off_cidx64);
    float *skey = reinterpret_cast<float *>(w + pl.off_skey);
    int64_t *sidx = reinterpret_cast<int64_t *>(w + pl.off_sidx);
    int32_t *ridx = reinterpret_cast<int32_t *>(w + pl.off_ridx);
    float *T = reinterpret_cast<float *>(w + pl.off_T);
    float *rd = reinterpret_cast<float *>(w + pl.off_rd);
    int64_t *ri = reinterpret_cast<int64_t *>(w + pl.off_ri);
    float *thr = reinterpret_cast<float *>(w + pl.off_thr);
    int32_t *cnt = reinterpret_cast<int32_t *>(w + pl.off_cnt);
    int32_t *stats = reinterpret_cast<int32_t *>(w + pl.off_stats);
    int32_t *need = stats + 4;
    int32_t *over = reinterpret_cast<int32_t *>(w + pl.off_over);
    int32_t *buf = reinterpret_cast<int32_t *>(w + pl.off_buf);
    float *rd2 = reinterpret_cast<float *>(w + pl.off_rd2);
    int64_t *ri2 = reinterpret_cast<int64_t *>(w + pl.off_ri2);
    uint8_t *selws = w + pl.off_sel;
    uint8_t *fbq = w + pl.total;
    uint8_t *fbd = fbq + fb_q;
    uint8_t *fbi = fbd + fb_d;
    uint8_t *exws = fbi + fb_i;

    const size_t Bp = static_cast<size_t>(pl.tiles_m) * GEMM_BLOCK_M;
    AC_CUDA(cudaMemsetAsync(Qr, 0, Bp * D * 4, s));
    AC_CUDA(cudaMemsetAsync(stats, 0, 32, s));
    AC_CUDA(cudaMemsetAsync(gthr, 0xFF, Bp * 4, s));   // ordered-uint +max: no bound published yet
    __half *Qh = p_half ? reinterpret_cast<__half *>(Qr) : nullptr;   // the fp16 queries reuse the fp32 query slot
    knn_prep_queries_kernel<<<(B + 3) / 4, 128, 0, s>>>(Q, B, D, Qr, Qh, qn);
    AC_LAUNCH_CHECK();
    const float *pn_use = p_sqnorm;
    if (!p_sqnorm) {
        knn_prep_rows_kernel<<<static_cast<unsigned>((N + 7) / 8), 256, 0, s>>>(P, N, D, pn);
        AC_LAUNCH_CHECK();
        pn_use = pn;
    }
    AC_CUDA(cudaMemsetAsync(pmax, 0, sizeof(float), s));
    knn_max_norm_kernel<<<sm_count() * 2, 256, 0, s>>>(pn_use, N, pmax);
    AC_LAUNCH_CHECK();

    // ---- pass 1 on the tensor cores: per-(query, CTA, half) top-16 lists
    const bool small_k = k <= KNN_SMALL_K;
    // kt = 0 (k > 16): no shared bound -- every list keeps its own true top-16, the merged lists bound the k-th distance
    int kt = 0;
    if (small_k) { kt = k + 3 > 8 ? k + 3 : 8; if (kt > KNN_KC) kt = KNN_KC; }
    EpiKnn epi{pn_use, ckey, cidx, gthr, B, N, pl.tiles_m, pl.slots, kt};
    if ((rc = launch_scan(Qr, P, p_half, Bp, N, D, epi, pl.grid_ctas, PROF_KNN_COARSE, s))) return rc;

    // ---- merge the lists (sorted by (key, id))
    const int64_t nc = static_cast<int64_t>(B) * pl.slots * KNN_KC;
    knn_widen_kernel<<<static_cast<unsigned>((nc + 255) / 256), 256, 0, s>>>(cidx, nc, cidx64);
    AC_LAUNCH_CHECK();
    const int64_t L = static_cast<int64_t>(pl.slots) * KNN_KC;
    if ((rc = topk_select(ckey, cidx64, B, L, L, 0, pl.ksel, skey, sidx, selws, pl.sel_bytes, s))) return rc;
    const float rel = p_half ? (2.f * 4.8828125e-4f + 2.4e-7f) : (9.765625e-4f + 4.8828125e-4f + 4.8e-7f);
    const unsigned bp_blocks = static_cast<unsigned>((Bp + 127) / 128);
    if (small_k) {
        // exact re-rank of the best KP candidates, final (d, id) order, certification
        knn_pick_kernel<<<(B + 127) / 128, 128, 0, s>>>(skey, sidx, ckey, qn, B, pl.slots, kt, ridx, T);
        AC_LAUNCH_CHECK();
        if ((rc = launch_knn_rerank(Q, P, B, N, D, KNN_KP, ridx, rd, ri, row_offset, s))) return rc;
        if ((rc = topk_select(rd, ri, B, KNN_KP, KNN_KP, 0, k, out_d, out_i, selws, pl.sel_bytes, s))) return rc;
        knn_certify_kernel<<<bp_blocks, 128, 0, s>>>(out_d, out_i, T, qn, pmax, skey, sidx, B, static_cast<int>(Bp), k, rel, thr, cnt,
                                                     need);
    } else {
        knn_threshold_kernel<<<bp_blocks, 128, 0, s>>>(skey, sidx, qn, pmax, B, static_cast<int>(Bp), k, rel, thr, cnt, need);
    }
    AC_LAUNCH_CHECK();

    // ---- pass 2 (device-conditional): collect the superset, exact re-rank, final selection for the flagged queries
    EpiKnnCollect epi2{pn_use, thr, buf, cnt, need, pl.cap, B, N, pl.tiles_m};
    if ((rc = launch_scan(Qr, P, p_half, Bp, N, D, epi2, pl.grid_ctas, PROF_KNN_PASS2, s))) return rc;
    knn_rerank_collected_kernel<<<dim3(static_cast<unsigned>((pl.cap * 8 + 255) / 256), B), 256, 0, s>>>(
        Q, P, B, N, D, pl.cap, thr, cnt, buf, rd2, ri2, row_offset, stats, over);
    AC_LAUNCH_CHECK();
    if ((rc = topk_select(rd2, ri2, B, pl.cap, pl.cap, 0, k, out_d, out_i, selws, pl.sel_bytes, s, thr))) return rc;

    if (stats_out) {
        knn_add_stats_kernel<<<1, 32, 0, s>>>(stats, stats_out);
        AC_LAUNCH_CHECK();
        return AC_OK;
    }
    // synchronous mode: queries whose 2-eps band overflowed the buffer are recomputed by the exact scan
    int32_t h[4] = {0, 0, 0, 0};
    AC_CUDA(cudaMemcpyAsync(h, stats, sizeof(h), cudaMemcpyDeviceToHost, s));
    AC_CUDA(cudaStreamSynchronize(s));
    const int nover = h[1];
    if (nover > 0) {
        float *gq = reinterpret_cast<float *>(fbq);
        float *gd = reinterpret_cast<float *>(fbd);
        int64_t *gi = reinterpret_cast<int64_t *>(fbi);
        knn_gather_rows_kernel<<<nover, 128, 0, s>>>(Q, over, nover, D, gq);
        AC_LAUNCH_CHECK();
        if ((rc = knn_exact_subset(gq, P, nover, N, D, k, gd, gi, row_offset, exws, exact_ws, s))) return rc;
        knn_scatter_results_kernel<<<(nover * k + 127) / 128, 128, 0, s>>>(gd, gi, over, nover, k, out_d, out_i);
        AC_LAUNCH_CHECK();
    }
    return AC_OK;
}

int knn_tc_search(const float *Q, const float *P, const float *p_sqnorm, const void *p_half, int B, int64_t N, int D, int k,
                  float *out_d, int64_t *out_i, int64_t row_offset, void *ws, size_t ws_bytes, int32_t *stats_out, cudaStream_t s) {
    int rc = ac_device_check();
    if (rc) return rc;
    const int Bb = knn_block(B, k);
    for (int b0 = 0; b0 < B; b0 += Bb) {
        const int nb = (B - b0 < Bb) ? B - b0 : Bb;
        if ((rc = knn_tc_block(Q + static_cast<int64_t>(b0) * D, P, p_sqnorm, p_half, nb, N, D, k, out_d + static_cast<int64_t>(b0) * k,
                               out_i + static_cast<int64_t>(b0) * k, row_offset, ws, ws_bytes, stats_out, s)))
            return rc;
    }
    return AC_OK;
}

__global__ void knn_to_half_kernel(const float *__restrict__ in, __half *__restrict__ out, int64_t n) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = __float2half_rn(in[i]);
}

}  // namespace ac

extern "C" int ac_knn_make_shadow(const float *P, int64_t N, int D, void *out_half, ac_stream_t stream) {
    AC_REQUIRE(P && out_half && N >= 0 && D > 0, "ac_knn_make_shadow: bad arguments");
    if (N == 0) return AC_OK;
    ac::knn_to_half_kernel<<<1184, 256, 0, static_cast<cudaStream_t>(stream)>>>(P, static_cast<__half *>(out_half), N * D);
    AC_LAUNCH_CHECK();
    return AC_OK;
}

