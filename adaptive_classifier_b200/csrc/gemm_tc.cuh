// gemm_tc.cuh -- persistent warp-specialised wgmma GEMM mainloop for sm_90a (H100).
//
//   D[M,N] (fp32) = A[M,K] * B[N,K]^T      K-major operands, either
//       kKind = GEMM_KIND_TF32 : fp32 containers holding tf32 values (wgmma .tf32, 32 elements per 128-byte k-block)
//       kKind = GEMM_KIND_F16  : fp16 values                         (wgmma .f16,  64 elements per 128-byte k-block)
//   (same bytes per stage, same descriptors; fp16 has tf32's 10-bit mantissa at twice the tensor rate)
//
//   warpgroup 3 : TMA producer (one thread: cp.async.bulk.tensor.2d, 128B swizzle, 4-stage mbarrier ring)
//   warpgroup 2 : MMA.  Issues both wgmma m64n128 chains of a 128 x 128 tile (rows 0-63 and 64-127, 2 x 64 fp32
//                 accumulator registers per thread) and stores the finished accumulators into a shared-memory tile.
//   warpgroups 0, 1 : epilogue.  Warpgroup g runs the fused epilogue functor on tile rows [64 g, 64 g + 64): warp w of the
//                 warpgroup drains rows 32 (2 g + w % 2) .. + 32 and the column half w / 2 (64 columns = two chunks of
//                 32), thread = one accumulator row.
//
// Hand-off through the single accumulator tile: the MMA warpgroup runs the mainloop of tile i, waits on acc_empty (the
// epilogue of tile i-1 has read the tile for the last time), stores, arrives on acc_full and goes on with the mainloop of
// tile i+1, so tile i's epilogue runs under tile i+1's mainloop.  The producer keeps loading stages throughout.  Registers:
// 128 per thread at launch (512 threads); setmaxnreg moves them from the producer (24) to the MMA warpgroup (160: the 128
// accumulators plus addressing; at 152 ptxas spills the accumulators) and the epilogue (160).  This one kernel serves the
// encoder linears and the kNN scans (running per-query top-k' lists / threshold collection over prototype tiles).
#pragma once
#include "common.cuh"

namespace ac {

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_N = 128;
constexpr int GEMM_BLOCK_K = 32;                    // tf32: fp32 elements per 128-byte swizzle row
constexpr int GEMM_KIND_TF32 = 0, GEMM_KIND_F16 = 1;
__host__ __device__ constexpr int gemm_block_k(int kind) { return kind == GEMM_KIND_F16 ? 64 : 32; }
constexpr int GEMM_STAGES = 4;
constexpr int GEMM_EPI_COLS = GEMM_BLOCK_N / 2;     // accumulator columns one epilogue warp drains per tile
constexpr int GEMM_EPI_WARPS = 8;                   // the epilogue warps (threads 0-255)
constexpr int GEMM_MMA_THREAD0 = 32 * GEMM_EPI_WARPS;   // first thread of the MMA warpgroup
constexpr int GEMM_PRODUCER_THREAD = GEMM_MMA_THREAD0 + 128;
constexpr int GEMM_THREADS = GEMM_PRODUCER_THREAD + 128; // 512: two epilogue warpgroups + MMA + producer
// per-thread registers of each role after setmaxnreg: 128 * 24 + 128 * 160 + 256 * 160 = 64512 of 65536
constexpr int GEMM_EPI_REGS = 160, GEMM_MMA_REGS = 160, GEMM_PRODUCER_REGS = 24;
static_assert(128 * GEMM_PRODUCER_REGS + 128 * GEMM_MMA_REGS + 256 * GEMM_EPI_REGS <= 65536, "register split exceeds the file");
constexpr int GEMM_A_STAGE_BYTES = GEMM_BLOCK_M * 128;  // 16 KB
constexpr int GEMM_B_STAGE_BYTES = GEMM_BLOCK_N * 128;  // 16 KB
constexpr int GEMM_STAGE_BYTES = GEMM_A_STAGE_BYTES + GEMM_B_STAGE_BYTES;
// accumulator tile row stride: +4 floats keeps the thread-per-row 16-byte reads conflict-free
constexpr int GEMM_ACC_LD = GEMM_BLOCK_N + 4;
constexpr int GEMM_ACC_BYTES = GEMM_BLOCK_M * GEMM_ACC_LD * 4;  // 66 KB
// per-epilogue-warp staging tile for the thread-row -> coalesced-row transpose: 32 rows x 80 bytes
// (16 fp32 or 32 fp16 payload + 16 B pad: conflict-free 16-byte accesses for both the row writes and the
// transposed reads)
constexpr int GEMM_EPI_STAGE_ROW_BYTES = 80;
constexpr int GEMM_EPI_STAGE_BYTES = 32 * GEMM_EPI_STAGE_ROW_BYTES;   // 2560 B per warp
constexpr int GEMM_SMEM_BYTES = GEMM_STAGES * GEMM_STAGE_BYTES + GEMM_ACC_BYTES + GEMM_EPI_WARPS * GEMM_EPI_STAGE_BYTES +
                                1024 /*align slack*/ + 256 /*barriers*/;
static_assert(GEMM_SMEM_BYTES <= 227 * 1024, "stage ring + accumulator tile do not fit");

#ifndef AC_MBAR_WATCHDOG
#define AC_MBAR_WATCHDOG 1
#endif

__device__ __forceinline__ void mbar_wait_guarded(uint64_t *bar, uint32_t parity) {
#if AC_MBAR_WATCHDOG
    // a broken pipeline must surface as a launch failure, never as a hung GPU.  No printf here: a function call in a
    // kernel that issues wgmma makes ptxas serialise every wgmma of that kernel.
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) __trap();
    }
#else
    mbar_wait(bar, parity);
#endif
}

struct GemmTileInfo {
    int m0, n0;       // tile origin
    int tile_iter;    // how many tiles this CTA has processed before this one
};

// column half (0 or 1) of the accumulator tile that the calling epilogue warp drains
__device__ __forceinline__ int gemm_epi_chalf() { return ((threadIdx.x >> 5) >> 1) & 1; }

// Epilogue concept (parameters live in the functor, per-thread running state in Epi::State):
//   struct Epi { struct State {...};
//                static constexpr int kUnrollChunks, kPrefetchDist;
//                __device__ bool skip_kernel() const;   (true => every thread returns immediately)
//                __device__ void begin_cta(State&, int warp_q, int lane) const;
//                __device__ void prefetch(State&, const GemmTileInfo&, int row, int col0, int lane, int buf) const;
//                      (issue the global loads chunk (col0) will need into State buffer `buf`; called kPrefetchDist chunks ahead)
//                __device__ void tile(State&, const GemmTileInfo&, int row /*global m*/, int col0 /*global n of v[0]*/,
//                                     const float (&v)[32], uint8_t *stage, int lane, int buf, const float *acc) const;
//                      (2x per tile per thread; acc = this thread's accumulator row in shared memory at column v[0], for
//                       re-reading single columns; stage = this warp's private 32 x 80-byte smem tile for transposing to
//                       coalesced rows; the 32 lanes of a warp hold rows row - lane .. row - lane + 31)
//                __device__ void end_cta(State&, int warp_q, int lane) const; };
//
// Tile order: kMFastest = false -> n fastest (tiles of the same A row-block run concurrently and share A
// through L2: encoder linears, A = activations); kMFastest = true -> m fastest (consecutive CTAs share the
// same B tile: kNN, B = prototype rows streamed once from HBM).
template <class Epi, bool kMFastest = false, int kKind = GEMM_KIND_TF32>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               int M, int N, int K, Epi epi) {
    // device-conditional launch: an epilogue may declare the whole launch unnecessary (kNN pass 2 when every query was
    // certified) from a device-side counter, before any barrier state exists -- uniform over the grid
    if (epi.skip_kernel()) return;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *smem_a = smem;
    uint8_t *smem_b = smem + GEMM_STAGES * GEMM_A_STAGE_BYTES;
    float *acc_tile = reinterpret_cast<float *>(smem + GEMM_STAGES * GEMM_STAGE_BYTES);
    uint8_t *epi_stage = smem + GEMM_STAGES * GEMM_STAGE_BYTES + GEMM_ACC_BYTES;
    uint64_t *bars = reinterpret_cast<uint64_t *>(epi_stage + GEMM_EPI_WARPS * GEMM_EPI_STAGE_BYTES);
    uint64_t *full_bar = bars;                        // [STAGES]
    uint64_t *empty_bar = bars + GEMM_STAGES;         // [STAGES]
    uint64_t *acc_full = bars + 2 * GEMM_STAGES;      // accumulator tile stored (MMA -> epilogue)
    uint64_t *acc_empty = acc_full + 1;               // accumulator tile read for the last time (epilogue -> MMA)

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int tiles_m = (M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
    const int tiles_n = (N + GEMM_BLOCK_N - 1) / GEMM_BLOCK_N;
    const int num_tiles = tiles_m * tiles_n;
    constexpr int BK = gemm_block_k(kKind);            // elements per 128-byte k-block
    const int num_kb = (K + BK - 1) / BK;
    // tiles blockIdx.x, blockIdx.x + gridDim.x, ... : the MMA and epilogue loops count them instead of carrying tile ids
    const int my_tiles = (num_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);

    if (threadIdx.x == GEMM_PRODUCER_THREAD) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        for (int s = 0; s < GEMM_STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 4);                // one arrival per MMA warp
        }
        mbar_init(acc_full, 128);                       // every MMA thread, after its own accumulator stores
        mbar_init(acc_empty, 32 * GEMM_EPI_WARPS);      // every epilogue thread, after its last read of the tile
        fence_mbar_init();
    }
    __syncthreads();

    if (threadIdx.x >= GEMM_PRODUCER_THREAD) {
        // ---------------- TMA producer ----------------
        setmaxnreg_dec<GEMM_PRODUCER_REGS>();          // the whole warpgroup, idle threads included
        if (threadIdx.x == GEMM_PRODUCER_THREAD) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int m0 = (kMFastest ? tile % tiles_m : tile / tiles_n) * GEMM_BLOCK_M;
                const int n0 = (kMFastest ? tile / tiles_m : tile % tiles_n) * GEMM_BLOCK_N;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait_guarded(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], GEMM_STAGE_BYTES);
                    tma_load_2d(smem_a + stage * GEMM_A_STAGE_BYTES, &tmap_a, &full_bar[stage], kb * BK, m0);
                    tma_load_2d(smem_b + stage * GEMM_B_STAGE_BYTES, &tmap_b, &full_bar[stage], kb * BK, n0);
                    if (++stage == GEMM_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;     // no CTA-wide barrier follows: the other roles synchronise through mbarriers
    }

    if (threadIdx.x >= GEMM_MMA_THREAD0) {
        // ---------------- MMA warpgroup: both 64-row wgmma chains of every tile, then the accumulator store ----------------
        setmaxnreg_inc<GEMM_MMA_REGS>();
        // the 128 accumulators leave 32 registers: keep the loop state small (a tile count instead of tile ids, stage
        // descriptors as base + offset)
        const uint64_t a_desc0 = wgmma_desc_sw128(smem_u32(smem_a));
        const uint64_t b_desc0 = wgmma_desc_sw128(smem_u32(smem_b));
        int stage = 0;
        uint32_t phase = 0;
        for (int it = 0; it < my_tiles; ++it) {
            float acc0[64], acc1[64];                // tile rows 0-63 and 64-127
#pragma unroll
            for (int j = 0; j < 64; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }
            // one wgmma group stays in flight: the stage of k-block kb-1 is released once the group of kb has been issued
            // and the group of kb-1 has retired
            int prev_stage = -1;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait_guarded(&full_bar[stage], phase);
                const uint64_t a_desc = a_desc0 + stage * (GEMM_A_STAGE_BYTES >> 4);
                const uint64_t b_desc = b_desc0 + stage * (GEMM_B_STAGE_BYTES >> 4);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    // advance 32 bytes inside the 128B swizzle row: +2 in the (addr >> 4) field; rows 64-127 of the A
                    // stage start 8192 B further: +512
                    if (kKind == GEMM_KIND_F16) {
                        wgmma_m64n128_f16(acc0, a_desc + 2 * k, b_desc + 2 * k, 1u);
                        wgmma_m64n128_f16(acc1, a_desc + 512 + 2 * k, b_desc + 2 * k, 1u);
                    } else {
                        wgmma_m64n128_tf32(acc0, a_desc + 2 * k, b_desc + 2 * k, 1u);
                        wgmma_m64n128_tf32(acc1, a_desc + 512 + 2 * k, b_desc + 2 * k, 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();
                __syncwarp();
                if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);   // this warp's share has been consumed
                prev_stage = stage;
                if (++stage == GEMM_STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

            mbar_wait_guarded(acc_empty, (it & 1) ^ 1);  // the epilogue of tile it-1 is done with the accumulator tile
            wgmma_store_acc(acc0, acc_tile, GEMM_ACC_LD);
            wgmma_store_acc(acc1, acc_tile + 64 * GEMM_ACC_LD, GEMM_ACC_LD);
            mbar_arrive(acc_full);                       // releases this thread's stores
        }
        return;
    }

    // ---------------- epilogue warpgroups: the fused epilogue of rows [64 wg, 64 wg + 64) of every tile ----------------
    setmaxnreg_inc<GEMM_EPI_REGS>();
    const int wg = warp >> 2;                        // 0 or 1: tile rows [64 wg, 64 wg + 64)
    const int q = 2 * wg + (warp & 1);               // 32-row quarter of the tile this warp drains
    const int chalf = gemm_epi_chalf();
    typename Epi::State est;
    epi.begin_cta(est, q, lane);
    const float *acc_row = acc_tile + (q * 32 + lane) * GEMM_ACC_LD;
    for (int it = 0; it < my_tiles; ++it) {
        const int tile = static_cast<int>(blockIdx.x) + it * static_cast<int>(gridDim.x);
        GemmTileInfo ti;
        ti.m0 = (kMFastest ? tile % tiles_m : tile / tiles_n) * GEMM_BLOCK_M;
        ti.n0 = (kMFastest ? tile / tiles_m : tile % tiles_n) * GEMM_BLOCK_N;
        ti.tile_iter = it;
        const int row = ti.m0 + q * 32 + lane;
        const int c_lo = chalf * GEMM_EPI_COLS;
        // operands the epilogue needs from global memory (residual rows) are requested kDist chunks ahead into kDist + 1
        // register buffers; the first requests go out while the tile's mainloop still runs
        constexpr int kDist = Epi::kPrefetchDist, kBufs = kDist + 1, kChunks = GEMM_EPI_COLS / 32;
#pragma unroll
        for (int d = 0; d < kDist; ++d)
            if (d < kChunks) epi.prefetch(est, ti, row, ti.n0 + c_lo + 32 * d, lane, d % kBufs);

        mbar_wait_guarded(acc_full, it & 1);
#pragma unroll (Epi::kUnrollChunks)
        for (int ci = 0; ci < kChunks; ++ci) {
            const int c = c_lo + 32 * ci;
            if (ci + kDist < kChunks) epi.prefetch(est, ti, row, ti.n0 + c + 32 * kDist, lane, (ci + kDist) % kBufs);
            float v[32];
            acc_row_ld32(acc_row + c, v);
            epi.tile(est, ti, row, ti.n0 + c, v, epi_stage + warp * GEMM_EPI_STAGE_BYTES, lane, ci % kBufs, acc_row + c);
        }
        mbar_arrive(acc_empty);                      // tile() re-reads acc (RoPE / GeGLU partners, kNN hits): only now done
    }
    epi.end_cta(est, q, lane);
}

// host-side launcher.  ta: A map with a GEMM_BLOCK_M-row box, tb: B map with a GEMM_BLOCK_N-row box (128-byte rows).
template <class Epi, bool kMFastest = false, int kKind = GEMM_KIND_TF32>
int launch_gemm_tc(const CUtensorMap &ta, const CUtensorMap &tb, int M, int N, int K, const Epi &epi,
                   cudaStream_t stream, int max_ctas = 0, int prof_cls = PROF_GEMM_LINEAR, double prof_bytes = 0.0) {
    auto kern = gemm_tc_kernel<Epi, kMFastest, kKind>;
    static bool attr_set[64] = {};   // per instantiation and per device
    int dev = 0;
    AC_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !attr_set[dev]) {
        AC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM_BYTES));
        if (dev >= 0 && dev < 64) attr_set[dev] = true;
    }
    const int tiles = ((M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M) * ((N + GEMM_BLOCK_N - 1) / GEMM_BLOCK_N);
    int ctas = sm_count();
    if (max_ctas > 0 && max_ctas < ctas) ctas = max_ctas;
    if (tiles < ctas) ctas = tiles;
    if (ctas <= 0) return AC_OK;
    const int slot = prof_begin(prof_cls, 2.0 * M * static_cast<double>(N) * K, prof_bytes, stream);
    kern<<<ctas, GEMM_THREADS, GEMM_SMEM_BYTES, stream>>>(ta, tb, M, N, K, epi);
    prof_end(slot, stream);
    AC_LAUNCH_CHECK();
    return AC_OK;
}

}  // namespace ac
