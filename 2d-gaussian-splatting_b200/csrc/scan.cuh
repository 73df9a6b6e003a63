// scan.cuh — the single-pass decoupled look-back scan that chains a count across a whole grid in one launch, shared
// by preprocess_fwd.cu (tile offsets and R), densify.cu (the plan's four counters), mcubes.cu (count and merge),
// meshpost.cu, chamfer.cu and cull.cu.  grid_exclusive_scan is the whole protocol for one count per thread; kernels
// that scan several counters, or (preprocess) publish early and look back late, call the parts it is built from.
//
// Each block owns one 64-bit status word per counter: bits 0-31 hold a count, bit 32 (kFlagAgg) marks it as the
// block's own aggregate and bit 33 (kFlagPrefix) as the inclusive prefix of every block up to and including it; a
// word of 0 is not yet published.  A block publishes its aggregate (block 0 its prefix) as soon as it has it, then
// one warp walks back 32 predecessors at a time, summing aggregates until it meets a prefix, and publishes its own
// inclusive prefix.  The protocol holds only under these conditions:
//  * the grid has one status word per counter per block (grid_blocks sizes both), and the status words and the
//    ticket word are zeroed before the launch (the callers' cudaMemsetAsync);
//  * block indices come from a ticket (block_ticket), not from blockIdx: a block then waits only on blocks that have
//    already started, so the spin always ends, whatever order the hardware schedules blocks in;
//  * relaxed loads and stores suffice because the count travels in the same 64-bit word as its flag: a reader
//    that sees the flag sees the count, and no other data is passed from block to block;
//  * a count, and so the grid-wide total, must fit the 32-bit field.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace surfel {

constexpr unsigned long long kFlagAgg = 1ull << 32, kFlagPrefix = 2ull << 32;

// Blocks of `threads` that cover n items, at least one (a scan over nothing still has a block to write its zero
// total): the grid of a scan and the number of its status words per counter.
inline unsigned grid_blocks(long long n, int threads) { return n > 0 ? (unsigned)((n + threads - 1) / threads) : 1u; }

// The block's index in ticket order: thread 0 draws it from the zeroed word `ticket`, and every thread of the block
// calls this and gets it.
__device__ __forceinline__ uint32_t block_ticket(uint32_t* ticket) {
    __shared__ uint32_t s_bid;
    if (threadIdx.x == 0) s_bid = atomicAdd(ticket, 1u);
    __syncthreads();
    return s_bid;
}

__device__ __forceinline__ unsigned long long ld_status(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_status(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Block `bid` publishes its aggregate `total` (block 0 its inclusive prefix).  One thread calls it.
__device__ __forceinline__ void publish_aggregate(unsigned long long* status, uint32_t bid, uint32_t total) {
    st_status(status + bid, (bid == 0 ? kFlagPrefix : kFlagAgg) | total);
}

// The look-back of block `bid`, whose aggregate `total` is already published: returns the sum of the counts of
// blocks 0 .. bid-1 to every lane and publishes the block's inclusive prefix.  One whole warp calls it.
__device__ __forceinline__ uint32_t warp_lookback(unsigned long long* status, uint32_t bid, uint32_t total) {
    const int lane = threadIdx.x & 31;
    uint32_t excl = 0;
    if (bid != 0) {
        int look = (int)bid - 1;
        while (true) {
            const int j = look - lane;
            unsigned long long s = kFlagPrefix;
            if (j >= 0) {
                s = ld_status(status + j);
                while ((s >> 32) == 0) s = ld_status(status + j);
            }
            const unsigned pm = __ballot_sync(0xffffffffu, (s >> 32) == 2ull);
            const int first = pm ? (__ffs(pm) - 1) : 32;
            uint32_t x = (lane <= first) ? (uint32_t)(s & 0xffffffffull) : 0u;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
            excl += x;
            if (pm) break;
            look -= 32;
        }
        if (lane == 0) st_status(status + bid, kFlagPrefix | (unsigned long long)(excl + total));
    }
    return excl;
}

// Block-wide exclusive scan of `mine` over kThreads threads; T may pack several counters in fields that cannot
// overflow within a block.  Returns the thread's exclusive prefix and sets `total` to the block's sum.  s_warp holds
// kThreads / 32 values; every thread calls it.
template <int kThreads, typename T>
__device__ __forceinline__ T block_exclusive_scan(T mine, T* s_warp, T& total) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    T v = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += n;
    }
    if (lane == 31) s_warp[warp] = v;
    __syncthreads();
    if (warp == 0) {
        T w = lane < kThreads / 32 ? s_warp[lane] : T(0);
#pragma unroll
        for (int o = 1; o < kThreads / 32; o <<= 1) {
            const T n = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += n;
        }
        if (lane < kThreads / 32) s_warp[lane] = w;
    }
    __syncthreads();
    total = s_warp[kThreads / 32 - 1];
    return v - mine + (warp > 0 ? s_warp[warp - 1] : T(0));
}

// The look-back of C counters of block `bid` of `nb`, with status words laid out [C][nb]: publishes the block's
// totals, and warp c sums the totals of the blocks before it for counter c into s_excl[c].  Every thread of the
// block calls it; it ends with a barrier, so s_excl is ready on return.
template <int C>
__device__ __forceinline__ void block_lookback(unsigned long long* status, int nb, uint32_t bid, const uint32_t* total,
                                               uint32_t* s_excl) {
    const int tid = threadIdx.x, warp = tid >> 5;
    if (tid < C) publish_aggregate(status + (size_t)tid * nb, bid, total[tid]);
    if (warp < C) {
        const uint32_t excl = warp_lookback(status + (size_t)warp * nb, bid, total[warp]);
        if ((tid & 31) == 0) s_excl[warp] = excl;
    }
    __syncthreads();
}

struct GridScan {
    uint32_t rank;    // the thread's exclusive prefix over the whole grid
    uint32_t base;    // the sum over the blocks before this one
    uint32_t total;   // this block's sum
    bool last;        // this is the grid's last block, whose base + total is the grid's total
};

// Grid-wide exclusive scan of one count per thread over kThreads-thread blocks, block `bid` from block_ticket and
// status the grid's gridDim.x zeroed words.  Every thread of the block calls it.
template <int kThreads>
__device__ __forceinline__ GridScan grid_exclusive_scan(uint32_t mine, uint32_t bid, unsigned long long* status) {
    __shared__ uint32_t s_warp[kThreads / 32], s_excl[1];
    uint32_t total;
    const uint32_t excl = block_exclusive_scan<kThreads>(mine, s_warp, total);
    block_lookback<1>(status, gridDim.x, bid, &total, s_excl);
    return GridScan{s_excl[0] + excl, s_excl[0], total, bid == gridDim.x - 1};
}

}  // namespace surfel
