// cuda_shim.cpp -- fiber scheduler of tests/cpu_shim/cuda_shim.h (test infrastructure only)
#include "cuda_shim.h"

namespace shim {

Fiber *g_cur = nullptr;
ucontext_t g_sched;
dim3 g_block_dim, g_grid_dim;
FiberBarrier g_grid_bar;
long long g_progress = 0;

static const std::function<void()> *g_body = nullptr;

static void fiber_entry() {
    (*g_body)();
    g_cur->done = true;
    swapcontext(&g_cur->ctx, &g_sched);
}

void run_blocks(const std::vector<dim3> &blocks, dim3 grid, dim3 block, const std::function<void()> &body, unsigned seed) {
    constexpr size_t kStack = 128 * 1024;
    static std::vector<std::unique_ptr<char[]>> stack_pool;      // stacks are reused across launches (no mmap churn)
    size_t pool_next = 0;
    g_block_dim = block;
    g_grid_dim = grid;
    g_body = &body;
    const int tpb = static_cast<int>(block.x * block.y * block.z);
    if (tpb % 32 != 0) { fprintf(stderr, "cuda_shim: block size must be a multiple of 32\n"); abort(); }
    std::vector<std::unique_ptr<Block>> blks;
    std::vector<std::unique_ptr<Fiber>> fibers;
    static std::vector<uint8_t *> smem_pool;                    // 256 KB of "shared memory" per resident block
    static std::vector<float (*)[512]> tmem_pool;
    static std::vector<Block *> cluster_members;
    cluster_members.clear();
    for (const dim3 &b : blocks) {
        blks.emplace_back(new Block());
        Block *blk = blks.back().get();
        const size_t slot = blks.size() - 1;
        if (slot == smem_pool.size()) {
            smem_pool.push_back(static_cast<uint8_t *>(aligned_alloc(1024, 1024 * 1024)));
            tmem_pool.push_back(reinterpret_cast<float (*)[512]>(aligned_alloc(64, sizeof(float) * 128 * 512)));
        }
        blk->dyn_smem = smem_pool[slot];
        blk->tmem = tmem_pool[slot];
        blk->cluster_rank = static_cast<int>(slot);
        blk->cluster = &cluster_members;
        cluster_members.push_back(blk);
        blk->bar.n = tpb;
        blk->warps.resize(tpb / 32);
        for (auto &w : blk->warps) w.bar.n = 32;
        for (int t = 0; t < tpb; ++t) {
            fibers.emplace_back(new Fiber());
            Fiber *f = fibers.back().get();
            if (pool_next == stack_pool.size()) stack_pool.emplace_back(new char[kStack]);
            char *stk = stack_pool[pool_next++].get();
            f->tid = dim3(t % block.x, (t / block.x) % block.y, t / (block.x * block.y));
            f->bid = b;
            f->blk = blk;
            f->warp = &blk->warps[t / 32];
            f->lane = t % 32;
            getcontext(&f->ctx);
            f->ctx.uc_stack.ss_sp = stk;
            f->ctx.uc_stack.ss_size = kStack;
            f->ctx.uc_link = &g_sched;
            makecontext(&f->ctx, fiber_entry, 0);
        }
    }
    g_grid_bar = FiberBarrier();
    g_grid_bar.n = static_cast<int>(fibers.size());
    std::mt19937 rng(seed);
    std::vector<int> order(fibers.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = static_cast<int>(i);
    size_t alive = fibers.size();
    while (alive) {
        const long long before = g_progress;
        std::shuffle(order.begin(), order.end(), rng);          // any interleaving between barriers must give the same result
        for (int i : order) {
            Fiber *f = fibers[i].get();
            if (f->done) continue;
            g_cur = f;
            swapcontext(&g_sched, &f->ctx);
            if (f->done) { --alive; ++g_progress; }
        }
        // fibers only yield inside a barrier: a whole pass without a released barrier or a finished fiber is a deadlock
        if (alive && g_progress == before) { fprintf(stderr, "cuda_shim: deadlock (threads wait in barriers that can never fill)\n"); abort(); }
    }
    g_cur = nullptr;
}

}  // namespace shim
