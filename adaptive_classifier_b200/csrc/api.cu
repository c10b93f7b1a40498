// api.cu -- C-ABI plumbing: error text, device check, TMA descriptor creation, kNN orchestration,
// and the host-buffer pipeline used for the end-to-end measurement.
#include "common.cuh"
#include <cstdarg>
#include <cudaTypedefs.h>
#include <atomic>
#include <mutex>
#include <vector>

namespace ac {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_cuda(cudaError_t e, const char *what) {
    if (e == cudaSuccess) return AC_OK;
    set_error("CUDA error %d (%s) at %s", static_cast<int>(e), cudaGetErrorString(e), what);
    return AC_E_CUDA;
}

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
void count_launch_n(long long n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_count_now() { return g_launches.load(std::memory_order_relaxed); }

struct ProfSlot { cudaEvent_t a, b; int cls; double flops, bytes; };
static bool g_prof_on = false;
bool prof_is_on() { return g_prof_on; }
static std::vector<ProfSlot> g_prof_slots;
static size_t g_prof_used = 0;
static double g_prof_ms[PROF_NUM], g_prof_flops[PROF_NUM], g_prof_bytes[PROF_NUM];
static long long g_prof_n[PROF_NUM];

static void prof_harvest() {
    cudaDeviceSynchronize();
    for (size_t i = 0; i < g_prof_used; ++i) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, g_prof_slots[i].a, g_prof_slots[i].b) == cudaSuccess) {
            const int c = g_prof_slots[i].cls;
            g_prof_ms[c] += ms; g_prof_flops[c] += g_prof_slots[i].flops; g_prof_bytes[c] += g_prof_slots[i].bytes;
            g_prof_n[c] += 1;
        }
    }
    g_prof_used = 0;
}

int prof_begin(int cls, double flops, double bytes, cudaStream_t s) {
    if (!g_prof_on) return -1;
    if (g_prof_used == g_prof_slots.size()) {
        if (g_prof_slots.size() >= 8192) {
            prof_harvest();
        } else {
            ProfSlot p{};
            if (cudaEventCreate(&p.a) != cudaSuccess || cudaEventCreate(&p.b) != cudaSuccess) return -1;
            g_prof_slots.push_back(p);
        }
    }
    ProfSlot &p = g_prof_slots[g_prof_used];
    p.cls = cls; p.flops = flops; p.bytes = bytes;
    cudaEventRecord(p.a, s);
    return static_cast<int>(g_prof_used++);
}
void prof_end(int slot, cudaStream_t s) {
    if (slot < 0) return;
    cudaEventRecord(g_prof_slots[slot].b, s);
}

int sm_count() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

int make_tmap_2d(CUtensorMap *out, const void *gptr, int elem_bytes, uint64_t rows, uint64_t cols,
                 uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols) {
    static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
    });
    if (!encode) {
        set_error("cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
        return AC_E_CUDA;
    }
    AC_REQUIRE((reinterpret_cast<uintptr_t>(gptr) & 15) == 0 && row_stride_bytes % 16 == 0,
               "make_tmap_2d: base pointer and row stride must be 16-byte aligned");
    AC_REQUIRE(box_cols * static_cast<uint32_t>(elem_bytes) == 128 && box_rows <= 256,
               "make_tmap_2d: box must be 128 bytes wide and <= 256 rows");
    const CUtensorMapDataType dt = (elem_bytes == 4) ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {row_stride_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(out, dt, 2, const_cast<void *>(gptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%llu cols=%llu)", static_cast<int>(r),
                  static_cast<unsigned long long>(rows), static_cast<unsigned long long>(cols));
        return AC_E_CUDA;
    }
    return AC_OK;
}

// from knn_exact.cu
int launch_knn_dist_exact(const float *Q, const float *P, int nq, int64_t N, int D, float *Dout, cudaStream_t stream);
int launch_knn_rerank(const float *Q, const float *P, int B, int64_t N, int D, int kc, const int32_t *cand, float *out_d,
                      int64_t *out_i, int64_t row_offset, cudaStream_t stream);
size_t topk_select_workspace(int B, int64_t L, int k);
int topk_select(const float *d, const int64_t *idx, int B, int64_t L, int64_t in_stride, int64_t id_offset, int k,
                float *out_d, int64_t *out_i, void *ws, size_t ws_bytes, cudaStream_t stream, const float *row_gate = nullptr);
// from knn_tc.cu
size_t knn_tc_workspace(int B, int64_t N, int D, int k);
int knn_tc_search(const float *Q, const float *P, const float *p_sqnorm, const void *p_half, int B, int64_t N, int D, int k,
                  float *out_d, int64_t *out_i, int64_t row_offset, void *ws, size_t ws_bytes, int32_t *stats, cudaStream_t stream);

// exact path processes the queries in blocks so the [qb, N] distance slab stays bounded
static int exact_query_block(int B, int64_t N) {
    const int64_t budget = 256ll << 20;   // bytes of distances per block
    int64_t qb = budget / (4 * (N > 0 ? N : 1));
    if (qb < 1) qb = 1;
    if (qb > B) qb = B;
    if (qb > 64) qb = 64;
    return static_cast<int>(qb);
}

static size_t knn_exact_workspace(int B, int64_t N, int k) {
    const int qb = exact_query_block(B, N);
    return align_up(static_cast<size_t>(qb) * N * sizeof(float), 256) + topk_select_workspace(qb, N, k) + 256;
}

static int knn_exact(const float *Q, const float *P, int B, int64_t N, int D, int k, float *out_d, int64_t *out_i,
                     int64_t row_offset, void *ws, size_t ws_bytes, cudaStream_t s) {
    const int qb = exact_query_block(B, N);
    const size_t dist_bytes = align_up(static_cast<size_t>(qb) * N * sizeof(float), 256);
    if (dist_bytes > ws_bytes) { set_error("ac_knn_l2_topk: workspace too small"); return AC_E_WORKSPACE; }
    float *dist = static_cast<float *>(ws);
    uint8_t *sel_ws = static_cast<uint8_t *>(ws) + dist_bytes;
    const size_t sel_bytes = ws_bytes - dist_bytes;
    for (int b0 = 0; b0 < B; b0 += qb) {
        const int nb = (B - b0 < qb) ? B - b0 : qb;
        int rc = launch_knn_dist_exact(Q + static_cast<int64_t>(b0) * D, P, nb, N, D, dist, s);
        if (rc) return rc;
        rc = topk_select(dist, nullptr, nb, N, N, row_offset, k, out_d + static_cast<int64_t>(b0) * k,
                         out_i + static_cast<int64_t>(b0) * k, sel_ws, sel_bytes, s);
        if (rc) return rc;
    }
    return AC_OK;
}

static int resolve_algo(int algo, int B, int64_t N, int D, int k) {
    if (algo != AC_KNN_AUTO) return algo;
    // tensor path pays off once the scan is compute-bound on the SIMT pipes (B >~ 8) and the index is big
    if (B >= 16 && k <= AC_KNN_TENSOR_MAX_K && N >= 4096 && N >= 8ll * k && D % 32 == 0) return AC_KNN_TENSOR;
    return AC_KNN_EXACT;
}

}  // namespace ac

using namespace ac;

extern "C" int ac_version(void) { return 1; }
extern "C" long long ac_launch_count(void) { return g_launches.load(); }
extern "C" int ac_profile_enable(int on) {
    if (on && !g_prof_on) {
        for (int c = 0; c < PROF_NUM; ++c) { g_prof_ms[c] = g_prof_flops[c] = g_prof_bytes[c] = 0; g_prof_n[c] = 0; }
        g_prof_used = 0;
    }
    if (!on && g_prof_on) prof_harvest();
    g_prof_on = on != 0;
    return AC_OK;
}
extern "C" int ac_profile_read(int cls, double *ms, double *flops, double *bytes, long long *launches) {
    AC_REQUIRE(cls >= 0 && cls < PROF_NUM, "ac_profile_read: bad class");
    prof_harvest();
    if (ms) *ms = g_prof_ms[cls];
    if (flops) *flops = g_prof_flops[cls];
    if (bytes) *bytes = g_prof_bytes[cls];
    if (launches) *launches = g_prof_n[cls];
    return AC_OK;
}
extern "C" const char *ac_last_error(void) { return g_err; }

extern "C" int ac_device_check(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        set_error("no CUDA device visible (%s); this library has no CPU fallback", cudaGetErrorString(e));
        return AC_E_CUDA;
    }
    int dev = 0, major = 0, minor = 0;
    AC_CUDA(cudaGetDevice(&dev));
    AC_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    AC_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (major != 9 || minor != 0) {
        set_error("device compute capability %d.%d is not sm_90 (H100); kernels are sm_90a only", major, minor);
        return AC_E_CUDA;
    }
    return AC_OK;
}

extern "C" int ac_knn_workspace_bytes(int B, int64_t N, int D, int k, int algo, size_t *bytes) {
    AC_REQUIRE(bytes && B >= 0 && N >= 0 && D > 0 && k >= 1, "ac_knn_workspace_bytes: bad arguments");
    AC_REQUIRE(k <= AC_KNN_MAX_K, "ac_knn_workspace_bytes: k=%d > %d", k, AC_KNN_MAX_K);
    const int a = resolve_algo(algo, B, N, D, k);
    size_t need = knn_exact_workspace(B, N, k);      // the tensor path may fall back per query
    if (a == AC_KNN_TENSOR) need += knn_tc_workspace(B, N, D, k);
    *bytes = need + 256;
    return AC_OK;
}

extern "C" int ac_knn_l2_topk(const float *Q, const float *P, const float *p_sqnorm, const void *p_half, int B, int64_t N,
                              int D, int k, float *out_d, int64_t *out_i, int64_t row_offset, void *workspace,
                              size_t workspace_bytes, int algo, int32_t *stats, ac_stream_t stream) {
    AC_REQUIRE(Q && out_d && out_i && B >= 0 && N >= 0 && D > 0, "ac_knn_l2_topk: bad arguments");
    AC_REQUIRE(k >= 1 && k <= AC_KNN_MAX_K, "ac_knn_l2_topk: k=%d outside [1,%d]", k, AC_KNN_MAX_K);
    AC_REQUIRE(N == 0 || P, "ac_knn_l2_topk: null index");
    AC_REQUIRE(N < (1ll << 31), "ac_knn_l2_topk: shards are limited to 2^31-1 rows");
    if (B == 0) return AC_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int a = resolve_algo(algo, B, N, D, k);
    uint8_t *ws = static_cast<uint8_t *>(workspace);
    ws = reinterpret_cast<uint8_t *>(align_up(reinterpret_cast<uintptr_t>(ws), 256));
    const size_t slack = static_cast<size_t>(ws - static_cast<uint8_t *>(workspace));
    AC_REQUIRE(workspace && workspace_bytes > slack, "ac_knn_l2_topk: null/empty workspace");
    const size_t avail = workspace_bytes - slack;
    if (a == AC_KNN_TENSOR) {
        AC_REQUIRE(k <= AC_KNN_TENSOR_MAX_K && D % 32 == 0, "ac_knn_l2_topk: tensor path needs k <= %d and D %% 32 == 0", AC_KNN_TENSOR_MAX_K);
        AC_REQUIRE(!p_half || D % 64 == 0, "ac_knn_l2_topk: the fp16 shadow path needs D %% 64 == 0");
        return knn_tc_search(Q, P, p_sqnorm, p_half, B, N, D, k, out_d, out_i, row_offset, ws, avail, stats, s);
    }
    return knn_exact(Q, P, B, N, D, k, out_d, out_i, row_offset, ws, avail, s);
}

// exact search entry used by the tensor path for queries it could not certify
namespace ac {
int knn_exact_subset(const float *Q, const float *P, int B, int64_t N, int D, int k, float *out_d, int64_t *out_i,
                     int64_t row_offset, void *ws, size_t ws_bytes, cudaStream_t s) {
    return knn_exact(Q, P, B, N, D, k, out_d, out_i, row_offset, ws, ws_bytes, s);
}
size_t knn_exact_workspace_pub(int B, int64_t N, int k) { return knn_exact_workspace(B, N, k); }
}  // namespace ac

