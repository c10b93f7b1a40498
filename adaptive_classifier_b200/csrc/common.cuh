// common.cuh -- error plumbing and sm_90a PTX wrappers (mbarrier, TMA, wgmma).
// Hand-written for H100; no CUTLASS/CuTe dependency.
#pragma once

#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>

#include "../../include/adaptive_b200.h"

namespace ac {

// ---------------------------------------------------------------- error handling
void set_error(const char *fmt, ...);
int check_cuda(cudaError_t e, const char *what);

#define AC_CUDA(call)                                                \
    do {                                                             \
        int _rc = ::ac::check_cuda((call), #call);                   \
        if (_rc != 0) return _rc;                                    \
    } while (0)

#define AC_REQUIRE(cond, ...)                                        \
    do {                                                             \
        if (!(cond)) {                                               \
            ::ac::set_error(__VA_ARGS__);                            \
            return AC_E_INVALID;                                     \
        }                                                            \
    } while (0)

// every kernel launch of the library passes through here: the counter backs bench.py's `gpu_launches`
void count_launch();
void count_launch_n(long long n);      // kernels replayed by a CUDA graph launch
long long launch_count_now();
bool prof_is_on();
#define AC_LAUNCH_CHECK()                                            \
    do {                                                             \
        ::ac::count_launch();                                        \
        AC_CUDA(cudaGetLastError());                                 \
    } while (0)

// optional CUDA-event timing of individual launches on their own stream (roofline numbers of bench.py)
enum { PROF_GEMM_LINEAR = 0, PROF_ATTENTION = 1, PROF_KNN_COARSE = 2, PROF_KNN_EXACT = 3, PROF_KNN_PASS2 = 4, PROF_NUM = 5 };
int prof_begin(int cls, double flops, double bytes, cudaStream_t s);   // slot id or -1 when disabled
void prof_end(int slot, cudaStream_t s);

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
int sm_count();

// ---------------------------------------------------------------- small device helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// round fp32 to tf32 (10 explicit mantissa bits), round-to-nearest-even, keep fp32 container
__device__ __forceinline__ float round_tf32(float x) {
    uint32_t u = __float_as_uint(x);
    u += 0x0FFFu + ((u >> 13) & 1u);
    u &= 0xFFFFE000u;
    return __uint_as_float(u);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ---------------------------------------------------------------- TMA (cp.async.bulk.tensor)
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load global -> shared, completion on an mbarrier (complete_tx::bytes)
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *m, uint64_t *bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// generic-proxy writes to smem that the async proxy (wgmma / TMA) will read
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// barrier over `nthreads` threads of the CTA (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// per-thread register budget of the calling warpgroup (warpgroup-collective; N a multiple of 8 in [24, 256]).  inc blocks
// until the CTA's pool has the registers, which other warpgroups return with dec.
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// Shared-memory matrix descriptor, K-major operand in the canonical 128-byte-swizzled layout that TMA writes with
// CU_TENSOR_MAP_SWIZZLE_128B (rows of 128 B, 8-row groups of 1024 B): start>>4 | LBO 1 (unused) | SBO 1024>>4 | SWIZZLE_128B.
// Advancing K by 32 bytes inside the swizzle row is +2 on the descriptor; 64 rows further down is +8192 B (+512).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>(1) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x K] * B[N x K]^T, A and B K-major in shared memory, D fp32 in registers; the whole warpgroup issues.
// kind f16: K = 16 per instruction; kind tf32: K = 8 (fp32 containers, the MMA reads the top 19 bits).
__device__ __forceinline__ void wgmma_m64n128_f16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n128_tf32(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n64_f16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n32_f16(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T with A in REGISTERS (f16x2 a[0..3]: rows 16 (t/32) + (t%32)/4 (+8) and
// columns 2 (t%4) (+8) of the warp's 16 rows, the layout of an accumulator's columns 16 k .. 16 k + 15), B K-major in
// shared memory
__device__ __forceinline__ void wgmma_m64n64_f16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc,
                                                    uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}

// Accumulator fragment of an m64nN wgmma -> rows of a row-major fp32 tile (ld floats per row).  Thread t of the warpgroup
// holds, for every 8-column group j, rows 16 (t/32) + (t%32)/4 (+8) and columns 8 j + 2 (t%4) (+1).
template <int NREG>
__device__ __forceinline__ void wgmma_store_acc(const float (&d)[NREG], float *tile, int ld) {
    const int t = threadIdx.x & 127;
    const int r0 = 16 * (t >> 5) + ((t & 31) >> 2), c0 = 2 * (t & 3);
#pragma unroll
    for (int j = 0; j < NREG / 4; ++j) {
        *reinterpret_cast<float2 *>(tile + r0 * ld + 8 * j + c0) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2 *>(tile + (r0 + 8) * ld + 8 * j + c0) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
}
// 32 consecutive fp32 of one accumulator row (16-byte aligned) -> registers
__device__ __forceinline__ void acc_row_ld32(const float *p, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
        const float4 x = *reinterpret_cast<const float4 *>(p + j);
        v[j] = x.x; v[j + 1] = x.y; v[j + 2] = x.z; v[j + 3] = x.w;
    }
}

// ---------------------------------------------------------------- host: TMA descriptor creation
// 2-D row-major fp32/bf16 matrix [rows, cols] (cols contiguous); box = [box_rows, box_cols], 128B swizzle.
// Uses the driver entry point resolved at run time (no link-time libcuda dependency).
int make_tmap_2d(CUtensorMap *out, const void *gptr, int elem_bytes, uint64_t rows, uint64_t cols,
                 uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols);

}  // namespace ac
