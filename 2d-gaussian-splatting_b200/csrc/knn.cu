// knn.cu — simple_knn.distCUDA2 of the reference's model initialisation
// (/root/reference/scene/gaussian_model.py:20, :134-135): for every point, the mean of the squared
// distances to its three nearest OTHER points.  Upstream's source is not available; the rules below are
// what this library computes (DESIGN.md §7g).
//
//  1. Exact: the three neighbours are the true three nearest points under the float32 distance of rule 2.
//     The query is excluded by INDEX, so an exact duplicate of it is a neighbour at distance 0.
//  2. Fixed arithmetic, bit-reproducible: dx = xi - xj (dy, dz alike), d2 = (dx*dx + dy*dy) + dz*dz, every
//     operation rounded to nearest with no FMA contraction (the __f*_rn intrinsics below, and -fmad=false
//     for the file).  With a <= b <= c the three smallest d2, the result is ((a + b) + c) / 3.0f (IEEE
//     division).  It depends only on the multiset of d2 values, so tie-breaking cannot change it.
//  3. (this project's convention) Fewer than three eligible neighbours: the mean over the k = min(3, n - 1)
//     that exist (n = number of finite points), summed in ascending order and divided by (float)k; k = 0
//     gives 0.
//  4. (this project's convention) A row with a NaN or +-inf coordinate is nobody's neighbour and its own
//     result is NaN.  It takes no part in the bounding box or the Morton keys.
//  5. P = 0 launches nothing.
//
// Algorithm (all on the caller's stream, no host round trip):
//  (a) bounding box and count n of the finite points (order-preserving u32 encoding + atomics);
//  (b) 63-bit Morton keys (3 x 21 bits, one common scale for all axes) with the index as value; non-finite
//      rows get the key 2^63, above every Morton key, so the finite points form the prefix [0, n) after
//  (c) the library's stable LSD radix sort (radix_sort.cu);
//  (d) gather into sorted order as float4 (x, y, z, index bits);
//  (e) AABBs of every run of kBox = 32 sorted points (level 0), then of every 32 consecutive boxes of the
//      level below, up to a level of at most 32 boxes: an implicit 32-ary tree over the sorted order;
//  (f) one warp per level-0 box, one lane per query: seed the best three from the query's own box and
//      the two boxes beside it in Morton order, then walk the tree depth first.  A child is entered only
//      if its lower bound is below the third-best distance of some lane; a leaf is scanned by
//      broadcasting its 32 points lane by lane.  The walk stops as soon as every lane's third-best is 0
//      (thousands of copies of one point end after the seed).
//
// Exactness of the pruning.  Box bounds are the exact min / max of float32 coordinates.  The lower bound
// of a box is computed with the same rounded operations as d2: per axis g = max(lo - q, q - hi, 0) (for
// two boxes, the gap between them), lb = (g.x*g.x + g.y*g.y) + g.z*g.z.  For any point p of the box,
// |p - q| >= g exactly on every axis, and rounding to nearest is monotone, so each rounded step of d2 is
// >= the matching step of lb: lb <= d2 in float32, bit for bit, with no slack needed.  A box is skipped
// only when lb >= the current third-best c, and a point with d2 >= c cannot change the result.  Morton
// quantisation only decides the order and so the speed; it never decides which points are compared.
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/surfel_rasterizer.h"
#include "common.cuh"
#include "kernels.h"
#include "profile.h"

namespace surfel {

constexpr int kBox = 32;              // points per level-0 box == lanes per warp
constexpr int kMaxLevels = 8;         // 32^7 boxes of 32 points > 2^30 points
constexpr int kKnnThreads = 256;
constexpr uint64_t kNonFiniteKey = 1ull << 63;
constexpr int kKnnMaxP = (int)kRadixSortMaxPairs;   // indices fit in u32

struct KnnLevels {
    int count;                    // levels allocated for P points (the tree of the n finite ones may be shorter)
    uint32_t off[kMaxLevels];     // first box of each level in the box array
};

struct KnnLayout {
    size_t ctrl, sort, pts, boxes, total;
    KnnLevels lv;
};

static size_t ceil_box(size_t n) { return (n + kBox - 1) / kBox; }

static KnnLayout knn_layout(int P) {
    KnnLayout L;
    const size_t p = P > 0 ? (size_t)P : 1;
    size_t o = 0;
    L.ctrl = o;      o = align_up(o + 64, 256);          // [0..2] lo (ordered u32), [3..5] hi, [6] n finite
    L.sort = o;      o = align_up(o + radix_sort_workspace_bytes(p), 256);
    L.pts = o;       o = align_up(o + p * 16, 256);
    size_t nb = 0, n = ceil_box(p);
    L.lv.count = 0;
    while (true) {
        L.lv.off[L.lv.count++] = (uint32_t)nb;
        nb += n;
        if (n <= (size_t)kBox) break;
        n = ceil_box(n);
    }
    L.boxes = o;     o = align_up(o + nb * 32, 256);     // (lo, hi) float4 pair per box
    L.total = o;
    return L;
}

// float <-> u32 with the same order (for atomicMin / atomicMax on floats)
__device__ __forceinline__ uint32_t ord_of(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_of_ord(uint32_t u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
__device__ __forceinline__ bool finite3(float x, float y, float z) {
    return isfinite(x) && isfinite(y) && isfinite(z);
}

__global__ void __launch_bounds__(kKnnThreads)
knn_bbox_kernel(int P, const float* __restrict__ xyz, uint32_t* __restrict__ ctrl) {
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    uint32_t n = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
        const float x = xyz[3 * (size_t)i], y = xyz[3 * (size_t)i + 1], z = xyz[3 * (size_t)i + 2];
        if (!finite3(x, y, z)) continue;
        lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
        hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
        n++;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
        n += __shfl_xor_sync(0xffffffffu, n, o);
    }
    if ((threadIdx.x & 31) == 0 && n > 0) {
        for (int a = 0; a < 3; a++) {
            atomicMin(&ctrl[a], ord_of(lo[a]));
            atomicMax(&ctrl[3 + a], ord_of(hi[a]));
        }
        atomicAdd(&ctrl[6], n);
    }
}

__device__ __forceinline__ uint64_t spread21(uint32_t v) {   // bit i -> bit 3i
    uint64_t x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

__global__ void __launch_bounds__(kKnnThreads)
knn_morton_kernel(int P, const float* __restrict__ xyz, const uint32_t* __restrict__ ctrl,
                  uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float x = xyz[3 * (size_t)i], y = xyz[3 * (size_t)i + 1], z = xyz[3 * (size_t)i + 2];
    uint64_t key = kNonFiniteKey;
    if (finite3(x, y, z)) {
        const float lx = float_of_ord(ctrl[0]), ly = float_of_ord(ctrl[1]), lz = float_of_ord(ctrl[2]);
        // one scale for all axes keeps the cells cubes on flat or elongated clouds; the extent is computed in
        // double so that a box wider than FLT_MAX cannot overflow it
        const double ext = fmax(fmax((double)float_of_ord(ctrl[3]) - lx, (double)float_of_ord(ctrl[4]) - ly),
                                (double)float_of_ord(ctrl[5]) - lz);
        const double s = ext > 0.0 ? 2097151.0 / ext : 0.0;
        auto q = [&](float v, float l) {
            const double t = ((double)v - (double)l) * s;
            return (uint32_t)fmin(fmax(t, 0.0), 2097151.0);
        };
        key = spread21(q(x, lx)) | spread21(q(y, ly)) << 1 | spread21(q(z, lz)) << 2;
    }
    keys[i] = key;
    vals[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(kKnnThreads)
knn_gather_kernel(int P, const float* __restrict__ xyz, const uint32_t* __restrict__ vals_sorted,
                  float4* __restrict__ pts) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= P) return;
    const uint32_t i = vals_sorted[j];
    pts[j] = make_float4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], __uint_as_float(i));
}

// boxes of level `level` (one warp per box): over points when level == 0, else over the boxes of level - 1
__global__ void __launch_bounds__(kKnnThreads)
knn_box_kernel(int level, const __grid_constant__ KnnLevels lv, const uint32_t* __restrict__ ctrl,
               const float4* __restrict__ pts, float4* __restrict__ boxes) {
    const int lane = threadIdx.x & 31;
    const uint32_t box = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    uint32_t n_below = ctrl[6];                              // items of the level below: points, then boxes
    for (int l = 0; l < level; l++) n_below = (n_below + kBox - 1) / kBox;
    const uint32_t n = (n_below + kBox - 1) / kBox;
    if (box >= n) return;
    const uint32_t c = box * kBox + lane;
    float4 lo = make_float4(INFINITY, INFINITY, INFINITY, 0.f), hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f);
    if (c < n_below) {
        if (level == 0) {
            lo = hi = pts[c];
        } else {
            const float4* src = boxes + 2 * ((size_t)lv.off[level - 1] + c);
            lo = src[0]; hi = src[1];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, o));
        lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, o));
        lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, o));
        hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, o));
        hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, o));
        hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, o));
    }
    if (lane == 0) {
        float4* dst = boxes + 2 * ((size_t)lv.off[level] + box);
        dst[0] = make_float4(lo.x, lo.y, lo.z, 0.f);
        dst[1] = make_float4(hi.x, hi.y, hi.z, 0.f);
    }
}

// d2 of rule 2 and the lower bounds that are provably <= it (see the header comment)
__device__ __forceinline__ float sq_dist(float4 a, float4 b) {
    const float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y), dz = __fsub_rn(a.z, b.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
__device__ __forceinline__ float gap(float lo, float hi, float qlo, float qhi) {   // interval to interval
    return fmaxf(fmaxf(__fsub_rn(lo, qhi), __fsub_rn(qlo, hi)), 0.0f);
}
__device__ __forceinline__ float box_lb(float4 lo, float4 hi, float4 qlo, float4 qhi) {
    const float gx = gap(lo.x, hi.x, qlo.x, qhi.x), gy = gap(lo.y, hi.y, qlo.y, qhi.y), gz = gap(lo.z, hi.z, qlo.z, qhi.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz));
}

struct Best3 {
    float a, b, c;
    __device__ __forceinline__ void insert(float d) {
        if (d < c) {
            if (d < b) {
                c = b;
                if (d < a) { b = a; a = d; } else b = d;
            } else c = d;
        }
    }
};

// every lane compares its query with the (up to 32) points of level-0 box `leaf`
__device__ __forceinline__ void scan_leaf(uint32_t leaf, uint32_t n, const float4* __restrict__ pts, bool active,
                                          uint32_t self, float4 q, Best3& best) {
    const int lane = threadIdx.x & 31;
    const uint32_t first = leaf * kBox;
    const int cnt = (int)min((uint32_t)kBox, n - first);
    const float4 p = lane < cnt ? pts[first + lane] : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int t = 0; t < cnt; t++) {
        float4 o;
        o.x = __shfl_sync(0xffffffffu, p.x, t);
        o.y = __shfl_sync(0xffffffffu, p.y, t);
        o.z = __shfl_sync(0xffffffffu, p.z, t);
        if (active && first + t != self) best.insert(sq_dist(q, o));
    }
}

__global__ void __launch_bounds__(kKnnThreads)
knn_query_kernel(int P, const __grid_constant__ KnnLevels lv, const uint32_t* __restrict__ ctrl,
                 const float4* __restrict__ pts, const float4* __restrict__ boxes, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const uint32_t leaf = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t j = leaf * kBox + lane;                   // this lane's query, in sorted order
    if (leaf * kBox >= (uint32_t)P) return;
    const uint32_t n = ctrl[6];
    if (j >= n) {                                            // non-finite rows sort last (rule 4)
        if (j < (uint32_t)P) out[__float_as_uint(pts[j].w)] = __int_as_float(0x7fc00000);   // quiet NaN
        if (leaf * kBox >= n) return;
    }
    const bool active = j < n;
    const float4 q = active ? pts[j] : make_float4(0.f, 0.f, 0.f, 0.f);

    uint32_t cnt[kMaxLevels];                                // boxes per level of the tree over n points
    int top = 0;
    cnt[0] = (n + kBox - 1) / kBox;
    while (cnt[top] > (uint32_t)kBox) { cnt[top + 1] = (cnt[top] + kBox - 1) / kBox; top++; }
    auto box_lo = [&](int l, uint32_t b) { return __ldg(boxes + 2 * ((size_t)lv.off[l] + b)); };
    auto box_hi = [&](int l, uint32_t b) { return __ldg(boxes + 2 * ((size_t)lv.off[l] + b) + 1); };

    Best3 best{INFINITY, INFINITY, INFINITY};
    // seed: the query's own box and its two neighbours in Morton order
    scan_leaf(leaf, n, pts, active, j, q, best);
    if (leaf > 0) scan_leaf(leaf - 1, n, pts, active, j, q, best);
    if (leaf + 1 < cnt[0]) scan_leaf(leaf + 1, n, pts, active, j, q, best);
    const float4 qlo = box_lo(0, leaf), qhi = box_hi(0, leaf);   // bounds every query of this warp
    auto warp_cmax = [&]() {
        float c = active ? best.c : 0.0f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c = fmaxf(c, __shfl_xor_sync(0xffffffffu, c, o));
        return c;
    };

    // depth-first walk; mask[l] = children (boxes of level l - 1) of box parent[l] still to visit; the
    // virtual root sits at level top + 1 with the cnt[top] boxes of the top level as children
    uint32_t mask[kMaxLevels + 1], parent[kMaxLevels + 1];
    float cmax = warp_cmax();
    int l = top + 1;
    parent[l] = 0;
    {
        const bool in = (uint32_t)lane < cnt[top] && box_lb(box_lo(top, lane), box_hi(top, lane), qlo, qhi) < cmax;
        mask[l] = __ballot_sync(0xffffffffu, in);
    }
    while (cmax > 0.0f) {
        if (mask[l] == 0) {
            if (l == top + 1) break;
            l++;
            continue;
        }
        const int i = __ffs(mask[l]) - 1;
        mask[l] &= mask[l] - 1;
        const uint32_t child = parent[l] * kBox + i;         // a box of level l - 1
        const float4 lo = box_lo(l - 1, child), hi = box_hi(l - 1, child);
        const bool need = active && box_lb(lo, hi, q, q) < best.c;
        if (!__any_sync(0xffffffffu, need)) continue;
        if (l == 1) {
            if (child + 1 >= leaf && child <= leaf + 1) continue;   // seeded already
            scan_leaf(child, n, pts, active, j, q, best);
            cmax = warp_cmax();
        } else {
            l--;
            parent[l] = child;
            const uint32_t g = child * kBox + lane;
            const bool in = g < cnt[l - 1] && box_lb(box_lo(l - 1, g), box_hi(l - 1, g), qlo, qhi) < cmax;
            mask[l] = __ballot_sync(0xffffffffu, in);
        }
    }
    if (!active) return;
    const uint32_t k = min(n - 1, 3u);                       // rule 3
    float r = 0.0f;
    if (k == 3) r = __fdiv_rn(__fadd_rn(__fadd_rn(best.a, best.b), best.c), 3.0f);
    else if (k == 2) r = __fdiv_rn(__fadd_rn(best.a, best.b), 2.0f);
    else if (k == 1) r = best.a;
    out[__float_as_uint(q.w)] = r;
}

}  // namespace surfel

using namespace surfel;

extern "C" {

size_t surfel_knn_workspace_bytes(int P) {
    if (P < 0 || P > kKnnMaxP) return 0;
    return knn_layout(P).total;
}

int surfel_knn_mean_sq_dist(int P, const float* xyz, float* out, void* workspace, size_t workspace_bytes,
                            void* stream) {
    if (P < 0) { surfel_set_error("surfel_knn_mean_sq_dist: P < 0"); return 1; }
    if (P > kKnnMaxP) { surfel_set_error("surfel_knn_mean_sq_dist: P = %d exceeds %d", P, kKnnMaxP); return 1; }
    if (P == 0) return 0;
    if (!xyz || !out) { surfel_set_error("surfel_knn_mean_sq_dist: NULL pointer"); return 1; }
    const KnnLayout L = knn_layout(P);
    if (!workspace_ok("surfel_knn_mean_sq_dist", workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    uint32_t* ctrl = (uint32_t*)(w + L.ctrl);
    const RadixSortWs sort = radix_sort_ws(w + L.sort, (size_t)P, 64);
    float4* pts = (float4*)(w + L.pts);
    float4* boxes = (float4*)(w + L.boxes);
    const unsigned blocks = (unsigned)((P + kKnnThreads - 1) / kKnnThreads);

    SURFEL_CUDA_OK(cudaMemsetAsync(ctrl, 0xff, 12, st));          // lo: the largest ordered value
    SURFEL_CUDA_OK(cudaMemsetAsync(ctrl + 3, 0, 16, st));         // hi: the smallest; n = 0
    { LaunchScope scope(kStKnn, st);
      knn_bbox_kernel<<<(unsigned)min((size_t)blocks, (size_t)current_device_sm_count() * 8), kKnnThreads, 0, st>>>(P, xyz, ctrl); }
    SURFEL_CUDA_OK(cudaGetLastError());
    { LaunchScope scope(kStKnn, st);
      knn_morton_kernel<<<blocks, kKnnThreads, 0, st>>>(P, xyz, ctrl, sort.in.keys, sort.in.vals); }
    SURFEL_CUDA_OK(cudaGetLastError());
    if (launch_radix_sort_pairs(sort, (size_t)P, st)) return 1;
    { LaunchScope scope(kStKnn, st);
      knn_gather_kernel<<<blocks, kKnnThreads, 0, st>>>(P, xyz, sort.out.vals, pts); }
    SURFEL_CUDA_OK(cudaGetLastError());
    // one warp per box; the grids are sized for P points, the kernels read the finite count n
    size_t nboxes = ceil_box((size_t)P);
    for (int l = 0; l < L.lv.count; l++) {
        LaunchScope scope(kStKnn, st);
        knn_box_kernel<<<(unsigned)((nboxes * 32 + kKnnThreads - 1) / kKnnThreads), kKnnThreads, 0, st>>>(l, L.lv, ctrl, pts, boxes);
        SURFEL_CUDA_OK(cudaGetLastError());
        nboxes = ceil_box(nboxes);
    }
    { LaunchScope scope(kStKnn, st);
      knn_query_kernel<<<(unsigned)((ceil_box((size_t)P) * 32 + kKnnThreads - 1) / kKnnThreads), kKnnThreads, 0, st>>>(
          P, L.lv, ctrl, pts, boxes, out); }
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
