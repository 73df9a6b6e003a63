// radix_sort.cu — CUB-free stable LSD radix sort of (u64 key, u32 value) pairs for sm_90a.
//
// Replaces cub::DeviceRadixSort::SortPairs in upstream's binning step (SURVEY §8a row a9): sort the
// (tile | depth-bits) keys ascending on bits [0, 32 + msb(tiles)), STABLE, so every tile's splats
// end up front-to-back with ties in emission (splat index) order.
//
// Structure ("onesweep"): one histogram launch computes the digit histograms of ALL passes, one
// tiny launch turns them into global digit bases, then each 8-bit pass is a single launch in
// which every block (a) ranks its 4096-item tile stably with warp-wide match_any, (b) chains its
// per-digit counts to its predecessors with a decoupled look-back (one thread per digit), and
// (c) reorders the tile through shared memory so the global scatter writes contiguous runs.
// Per pass the pairs are read once and written once (24 B per pair).
#include <algorithm>
#include <utility>
#include "common.cuh"
#include "kernels.h"
#include "profile.h"

namespace surfel {

constexpr int kRadixBits = 8;
constexpr int kRadix = 1 << kRadixBits;
constexpr int kSortThreads = 256;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kItems = 16;
constexpr int kTile = kSortThreads * kItems;   // 4096 pairs per block
constexpr int kMaxPasses = 8;

constexpr uint32_t kStAgg = 1u << 30, kStPrefix = 2u << 30, kStMask = (1u << 30) - 1u;
static_assert(kRadixSortMaxPairs <= kStMask, "a digit's running count must fit the 30 bits of a look-back status word");

struct SortTemp {
    uint32_t* hist;       // [kMaxPasses][kRadix] -> exclusive global digit bases after scan
    uint32_t* tickets;    // [kMaxPasses]
    uint32_t* status;     // [passes][tiles][kRadix]
};

static inline size_t sort_tiles(size_t n) { return (n + kTile - 1) / kTile; }

size_t radix_sort_temp_bytes(size_t n) {
    size_t b = align_up((size_t)kMaxPasses * kRadix * 4, 256);
    b += 256;
    b += align_up((size_t)kMaxPasses * sort_tiles(n) * kRadix * 4, 256);
    return b + 256;
}

static SortTemp carve_temp(void* temp, size_t n) {
    SortTemp t;
    char* c = (char*)temp;
    t.hist = (uint32_t*)c;            c += align_up((size_t)kMaxPasses * kRadix * 4, 256);
    t.tickets = (uint32_t*)c;         c += 256;
    t.status = (uint32_t*)c;
    (void)n;
    return t;
}

__device__ __forceinline__ uint32_t digit_of(uint64_t key, int shift, uint32_t mask) {
    return (uint32_t)(key >> shift) & mask;
}

__global__ void __launch_bounds__(256)
radix_histogram_kernel(const uint64_t* __restrict__ keys, size_t n, int passes, int end_bit,
                       uint32_t* __restrict__ hist) {
    __shared__ uint32_t s_hist[kMaxPasses * kRadix];
    for (int i = threadIdx.x; i < passes * kRadix; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint64_t k = keys[i];
        for (int ps = 0; ps < passes; ps++) {
            const int shift = ps * kRadixBits;
            const uint32_t mask = (1u << min(kRadixBits, end_bit - shift)) - 1u;
            atomicAdd(&s_hist[ps * kRadix + digit_of(k, shift, mask)], 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < passes * kRadix; i += blockDim.x) {
        const uint32_t v = s_hist[i];
        if (v) atomicAdd(&hist[i], v);
    }
}

// one block per pass: exclusive scan of the 256 digit counts (in place)
__global__ void __launch_bounds__(kRadix) radix_scan_hist_kernel(uint32_t* __restrict__ hist) {
    __shared__ uint32_t s_w[kRadix / 32];
    uint32_t* h = hist + blockIdx.x * kRadix;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t v = h[t];
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t pre = 0;
    for (int w = 0; w < warp; w++) pre += s_w[w];
    h[t] = pre + incl - v;
}

__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

struct __align__(16) SortSmem {
    uint64_t keys[kTile];
    uint32_t vals[kTile];
    uint32_t warp_hist[kSortWarps][kRadix];
    uint32_t local_start[kRadix];   // first position of digit d inside the sorted tile
    uint32_t scatter_off[kRadix];   // global_start[d] - local_start[d] (mod 2^32)
    uint32_t scan_tmp[kSortWarps];
    uint32_t tile_id;
};

__global__ void __launch_bounds__(kSortThreads)
radix_onesweep_kernel(const uint64_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                      uint64_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out, size_t n,
                      int shift, uint32_t mask, const uint32_t* __restrict__ digit_base,
                      uint32_t* __restrict__ ticket, uint32_t* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SortSmem& s = *reinterpret_cast<SortSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    if (tid == 0) s.tile_id = atomicAdd(ticket, 1u);
    for (int i = tid; i < kSortWarps * kRadix; i += kSortThreads) (&s.warp_hist[0][0])[i] = 0;
    __syncthreads();
    const uint32_t tile = s.tile_id;
    const size_t tile_base = (size_t)tile * kTile;
    const uint32_t valid = (uint32_t)min((size_t)kTile, n - tile_base);

    // ---- load (warp-striped: linear order == (warp, item, lane)) and rank stably ----
    uint64_t key[kItems];
    uint32_t val[kItems];
    uint32_t rank[kItems];
    const uint32_t warp_off = warp * (32 * kItems);
#pragma unroll
    for (int i = 0; i < kItems; i++) {
        const uint32_t local = warp_off + i * 32 + lane;
        if (local < valid) {
            key[i] = keys_in[tile_base + local];
            val[i] = vals_in[tile_base + local];
        } else {
            key[i] = ~0ull;   // digit == mask (largest), ranks after every valid item
            val[i] = 0;
        }
    }
    const unsigned lt_mask = (1u << lane) - 1u;
    uint32_t* wh = s.warp_hist[warp];
#pragma unroll
    for (int i = 0; i < kItems; i++) {
        const uint32_t d = digit_of(key[i], shift, mask);
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        uint32_t prev = 0;
        if (lane == leader) { prev = wh[d]; wh[d] = prev + __popc(peers); }
        prev = __shfl_sync(0xffffffffu, prev, leader);
        rank[i] = prev + __popc(peers & lt_mask);
        __syncwarp();
    }
    __syncthreads();

    // ---- per digit (thread == digit): exclusive scan over warps, block count ----
    uint32_t count = 0;
    {
        const int d = tid;
#pragma unroll
        for (int w = 0; w < kSortWarps; w++) {
            const uint32_t c = s.warp_hist[w][d];
            s.warp_hist[w][d] = count;
            count += c;
        }
        if ((uint32_t)d == mask) count -= (kTile - valid);   // padding items are not real
    }
    // block exclusive scan over digits -> local_start
    {
        uint32_t incl = count;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        if (lane == 31) s.scan_tmp[warp] = incl;
        __syncthreads();
        uint32_t pre = 0;
        for (int w = 0; w < warp; w++) pre += s.scan_tmp[w];
        s.local_start[tid] = pre + incl - count;
    }

    // ---- decoupled look-back, one thread per digit ----
    {
        const int d = tid;
        uint32_t* my = status + (size_t)tile * kRadix + d;
        uint32_t excl = 0;
        if (tile == 0) {
            st_relaxed_u32(my, kStPrefix | count);
        } else {
            st_relaxed_u32(my, kStAgg | count);
            int look = (int)tile - 1;
            while (true) {
                const uint32_t* q = status + (size_t)look * kRadix + d;
                uint32_t v = ld_relaxed_u32(q);
                while ((v >> 30) == 0) v = ld_relaxed_u32(q);
                excl += v & kStMask;
                if ((v >> 30) == 2u) break;
                look--;
            }
            st_relaxed_u32(my, kStPrefix | (excl + count));
        }
        s.scatter_off[d] = digit_base[d] + excl - s.local_start[d];
    }
    __syncthreads();

    // ---- reorder through shared memory, then write contiguous runs ----
#pragma unroll
    for (int i = 0; i < kItems; i++) {
        const uint32_t d = digit_of(key[i], shift, mask);
        const uint32_t pos = s.local_start[d] + s.warp_hist[warp][d] + rank[i];
        if (pos < (uint32_t)kTile) { s.keys[pos] = key[i]; s.vals[pos] = val[i]; }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kItems; i++) {
        const uint32_t pos = i * kSortThreads + tid;
        if (pos < valid) {
            const uint64_t k = s.keys[pos];
            const uint32_t dst = pos + s.scatter_off[digit_of(k, shift, mask)];
            keys_out[dst] = k;
            vals_out[dst] = s.vals[pos];
        }
    }
}

static int radix_sort_passes(int end_bit) { return (end_bit + kRadixBits - 1) / kRadixBits; }

int radix_key_bits(unsigned long long max_key) { return max_key ? 64 - __builtin_clzll(max_key) : 1; }

// keys A, keys B, values A, values B
size_t radix_sort_pairs_bytes(size_t capacity) { return 2 * align_up(capacity * 8, 256) + 2 * align_up(capacity * 4, 256); }

size_t radix_sort_workspace_bytes(size_t capacity) {
    return radix_sort_pairs_bytes(capacity) + radix_sort_temp_bytes(capacity);
}

RadixSortWs radix_sort_ws(SortPairs a, SortPairs b, void* temp, int end_bit) {
    // each pass moves the pairs to the other buffer: after an odd number of passes they are in B
    const bool in_b = radix_sort_passes(end_bit) & 1;
    return RadixSortWs{a, in_b ? b : a, in_b ? a : b, temp, end_bit};
}

RadixSortWs radix_sort_ws(void* base, size_t capacity, int end_bit, void* temp) {
    char* c = (char*)base;
    const size_t keys = align_up(capacity * 8, 256), vals = align_up(capacity * 4, 256);
    const SortPairs a{(uint64_t*)c, (uint32_t*)(c + 2 * keys)};
    const SortPairs b{(uint64_t*)(c + keys), (uint32_t*)(c + 2 * keys + vals)};
    return radix_sort_ws(a, b, temp ? temp : c + radix_sort_pairs_bytes(capacity), end_bit);
}

int launch_radix_sort_pairs(const RadixSortWs& ws, size_t n, cudaStream_t stream) {
    if (n == 0) return 0;
    const int end_bit = ws.end_bit;
    if (n > (size_t)kRadixSortMaxPairs) { surfel_set_error("radix sort: n=%zu exceeds 2^30", n); return 1; }
    if (end_bit < 1 || end_bit > 64) { surfel_set_error("radix sort: bad end_bit %d", end_bit); return 1; }
    const int passes = radix_sort_passes(end_bit);
    const size_t tiles = sort_tiles(n);
    SortTemp t = carve_temp(ws.temp, n);
    SURFEL_CUDA_OK(cudaMemsetAsync(t.hist, 0, (size_t)kMaxPasses * kRadix * 4, stream));
    SURFEL_CUDA_OK(cudaMemsetAsync(t.tickets, 0, 256, stream));
    SURFEL_CUDA_OK(cudaMemsetAsync(t.status, 0, (size_t)passes * tiles * kRadix * 4, stream));

    static bool attr_set[kMaxDevices] = {};
    const int slot = current_device_slot();
    if (slot < 0 || !attr_set[slot]) {
        SURFEL_CUDA_OK(cudaFuncSetAttribute(radix_onesweep_kernel,
                                            cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)sizeof(SortSmem)));
        if (slot >= 0) attr_set[slot] = true;
    }
    const int hist_blocks = (int)std::min((size_t)current_device_sm_count() * 8, (n + 255) / 256);
    { LaunchScope scope(kStSortHist, stream);
    radix_histogram_kernel<<<hist_blocks, 256, 0, stream>>>(ws.in.keys, n, passes, end_bit, t.hist);
    SURFEL_CUDA_OK(cudaGetLastError());
    prof_count_launch();
    radix_scan_hist_kernel<<<passes, kRadix, 0, stream>>>(t.hist); }
    SURFEL_CUDA_OK(cudaGetLastError());

    // ping-pong A -> B -> A ...: radix_sort_ws() made `out` the buffer the last pass writes, so no copy follows
    SortPairs src = ws.in, dst = (passes & 1) ? ws.out : ws.spare;
    for (int ps = 0; ps < passes; ps++) {
        const int shift = ps * kRadixBits;
        const uint32_t mask = (1u << std::min(kRadixBits, end_bit - shift)) - 1u;
        LaunchScope scope(kStSortPass, stream);
        radix_onesweep_kernel<<<(unsigned)tiles, kSortThreads, sizeof(SortSmem), stream>>>(
            src.keys, src.vals, dst.keys, dst.vals, n, shift, mask, t.hist + ps * kRadix, t.tickets + ps,
            t.status + (size_t)ps * tiles * kRadix);
        SURFEL_CUDA_OK(cudaGetLastError());
        std::swap(src, dst);
    }
    return 0;
}

}  // namespace surfel
