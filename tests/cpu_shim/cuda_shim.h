// cuda_shim.h -- just enough of the CUDA execution model to run SIMT device code (no tensor cores, no TMA) on the CPU.
//
// TEST INFRASTRUCTURE ONLY.  Kernels written after the GPU budget of a round is spent cannot be run, but their control
// flow can: every CUDA thread becomes a fiber (ucontext), __syncthreads / __syncwarp / cooperative grid.sync are fiber
// barriers, warp shuffles exchange through a per-warp array between two warp barriers, and the scheduler visits the fibers
// in a shuffled order so that missing barriers show up as wrong results.  Device source is compiled as ordinary C++ with
// the CUDA keywords defined away (head_train.cuh is written to be included as it is: AC_CPU_SHIM selects the few CPU stand-ins).
#pragma once
#include <ucontext.h>
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <random>
#include <vector>

// CUDA's own host-usable headers supply dim3 / float4 / uint4 / __half ...; their execution-space keywords are then
// redefined to nothing for the device code compiled as C++
#include <cuda_fp16.h>
#include <vector_functions.h>
#include <vector_types.h>
#undef __global__
#undef __device__
#undef __host__
#undef __forceinline__
#undef __restrict__
#undef __launch_bounds__
#undef __shared__
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static          /* kernels launched block by block; the cooperative kernel gets per-block arrays from the extractor */
#ifndef CUDART_INF_F
#define CUDART_INF_F (__builtin_inff())
#endif

static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
template <class T> static inline T __ldg(const T *p) { return *p; }
static inline float rsqrtf(float x) { return 1.f / sqrtf(x); }
static inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

namespace shim {

struct FiberBarrier {
    int n = 0, arrived = 0;
    unsigned gen = 0;
};
struct Warp {
    FiberBarrier bar;
    uint32_t xchg[32];
};
struct Block {
    FiberBarrier bar;
    std::vector<Warp> warps;
    // resources of the functional tensor-path model (tc_emul.h): dynamic shared memory (1024-byte aligned), tensor memory, and the
    // position of this CTA inside its cluster (all blocks of one run_blocks() call form the cluster)
    uint8_t *dyn_smem = nullptr;
    float (*tmem)[512] = nullptr;
    int cluster_rank = 0;
    std::vector<Block *> *cluster = nullptr;
};
struct Fiber {
    ucontext_t ctx;
    std::unique_ptr<char[]> stack;
    bool done = false;
    dim3 tid, bid;
    Block *blk = nullptr;
    Warp *warp = nullptr;
    int lane = 0;
};

extern Fiber *g_cur;
extern ucontext_t g_sched;
extern dim3 g_block_dim, g_grid_dim;
extern FiberBarrier g_grid_bar;
extern long long g_progress;       // barriers released + fibers finished (deadlock detection)

inline void yield() { swapcontext(&g_cur->ctx, &g_sched); }
inline void barrier_wait(FiberBarrier &b) {
    const unsigned g = b.gen;
    if (++b.arrived == b.n) {
        b.arrived = 0;
        b.gen++;
        ++g_progress;
    } else {
        while (b.gen == g) yield();
    }
}

// runs `blocks` (a set of block indices) concurrently, every thread executing `body`
void run_blocks(const std::vector<dim3> &blocks, dim3 grid, dim3 block, const std::function<void()> &body, unsigned seed);

// ordinary launch: blocks one after the other (static __shared__ is then per block)
inline void launch(dim3 grid, dim3 block, const std::function<void()> &body, unsigned seed = 1) {
    for (unsigned by = 0; by < grid.y; ++by)
        for (unsigned bx = 0; bx < grid.x; ++bx) run_blocks({dim3(bx, by, 0)}, grid, block, body, seed + bx + 977 * by);
}
// cluster launch: the `csize` CTAs of a cluster run concurrently (cluster barriers, peer shared memory), clusters one by one
inline void launch_cluster(dim3 grid, dim3 block, unsigned csize, const std::function<void()> &body, unsigned seed = 1) {
    for (unsigned c = 0; c < grid.x / csize; ++c) {
        std::vector<dim3> blocks;
        for (unsigned r = 0; r < csize; ++r) blocks.push_back(dim3(c * csize + r, 0, 0));
        run_blocks(blocks, grid, block, body, seed + 31 * c);
    }
}
// cooperative launch: all blocks resident at once (grid.sync works)
inline void launch_cooperative(dim3 grid, dim3 block, const std::function<void()> &body, unsigned seed = 1) {
    std::vector<dim3> all;
    for (unsigned bx = 0; bx < grid.x; ++bx) all.push_back(dim3(bx, 0, 0));
    run_blocks(all, grid, block, body, seed);
}

}  // namespace shim

#define threadIdx (shim::g_cur->tid)
#define blockIdx (shim::g_cur->bid)
#define blockDim (shim::g_block_dim)
#define gridDim (shim::g_grid_dim)

static inline void __syncthreads() { shim::barrier_wait(shim::g_cur->blk->bar); }
static inline void __syncwarp(unsigned = 0xffffffffu) { shim::barrier_wait(shim::g_cur->warp->bar); }
template <class T>
static inline T shim_shfl(T v, int src_lane) {
    static_assert(sizeof(T) == 4, "32-bit shuffles only");
    shim::Warp *w = shim::g_cur->warp;
    memcpy(&w->xchg[shim::g_cur->lane], &v, 4);
    shim::barrier_wait(w->bar);
    T r;
    memcpy(&r, &w->xchg[src_lane & 31], 4);
    shim::barrier_wait(w->bar);
    return r;
}
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int lanemask) { return shim_shfl(v, shim::g_cur->lane ^ lanemask); }
template <class T> static inline T __shfl_sync(unsigned, T v, int src) { return shim_shfl(v, src); }

namespace cooperative_groups {
struct grid_group {
    void sync() const { shim::barrier_wait(shim::g_grid_bar); }
};
inline grid_group this_grid() { return {}; }
}  // namespace cooperative_groups
