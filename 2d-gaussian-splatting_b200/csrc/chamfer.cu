// chamfer.cu — the DTU Chamfer evaluation of the reference's scripts/eval_dtu/eval.py (mesh sampling, greedy radius
// downsampling, the box and observation masks, the two bounded nearest-neighbour passes, the means and the colours of
// the two visualisation clouds) on the device, all in float64.  DESIGN.md §7m has the rules; tests/chamfer_ref.py
// restates them.  The file is compiled with -fmad=false and every operation the rules fix is a __d*_rn intrinsic.
//
//  * surfel_chamfer_sample_count / _emit: one warp per triangle.  The rows i <= n1 of a triangle go to the lanes, and
//    each row's points are a prefix j < c_i of 0..n2 (b_j and the rounded a + b_j are non-decreasing in j), so c_i
//    is found by bisection.  The count pass sums the rows; the emit pass ranks the triangles with the single-pass
//    look-back scan of scan.cuh and writes each row's points with the whole warp, coalesced, in row-major order.
//  * Point structure (three instances: the shuffled cloud, the STL cloud, data_in): 63-bit Morton keys over the
//    cloud's float64 box, the library's radix sort, float64 points gathered into sorted order with their original
//    index in .w, and the implicit 32-ary box tree of knn.cu (boxes of 32 sorted points, then of 32 boxes, ...).
//    Queries that are not in the tree are sorted the same way, so a warp's 32 queries are neighbours.
//  * Exactness of the pruning (knn.cu's argument in float64).  Box bounds are exact min / max of the coordinates.  A
//    box's lower bound uses the same rounded operations as rdist: per axis g = max(lo - q, q - hi, 0), lb =
//    (gx*gx + gy*gy) + gz*gz.  For a point p of the box |p - q| >= g exactly on each axis and rounding is monotone,
//    so lb <= rdist(p, q) bit for bit.  The radius walk skips a box only when lb > r*r, so no pair within r is
//    missed; the 1-NN walk skips it only when sqrt(lb) >= max_dist or lb > the current best, and neither can change
//    a result below max_dist.  Morton order and the box layout decide which pairs are compared, never the outcome.
//  * Greedy downsampling in rounds: an undecided point becomes removed as soon as an earlier (in shuffled order)
//    neighbour is kept, and kept once every earlier neighbour is removed.  Decisions are final, so a round may read
//    states another warp writes in the same round; each round decides at least the earliest undecided point.
//  * Masks and compaction: one look-back scan over the shuffled cloud with three counters (kept, inbound, observed)
//    and one over the STL (above the plane); order is kept, so the outputs are the reference's row order.
//  * Masked means: fixed-order tree sums per block and a one-block final pass; no float atomics.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "../../include/surfel_rasterizer.h"
#include "common.cuh"
#include "kernels.h"
#include "profile.h"
#include "scan.cuh"

namespace surfel {
namespace {

constexpr int kChThreads = 256;
constexpr int kBox = 32;                          // points per level-0 box == lanes per warp
constexpr int kMaxLevels = 8;                     // 32^7 boxes of 32 points > 2^30 points
constexpr long long kChMaxPoints = kRadixSortMaxPairs;   // indices fit in u32
constexpr int kRoundBatch = 8;                    // greedy rounds launched per read of the undecided count
constexpr uint8_t kUndecided = 0, kKept = 1, kRemoved = 2;

// ---------------------------------------------------------------------------------------------- mesh sampling

struct Tri {
    double t0[3], v1[3], v2[3];
    double n1, n2;                                // floor(l / thr); 0 for a dropped triangle
    bool kept;                                    // area2 > 0
};

__device__ __forceinline__ double norm3(const double* v) {
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])), __dmul_rn(v[2], v[2])));
}

// rule 1 up to n1, n2; `ok` is false when a vertex index lies outside [0, M)
__device__ __forceinline__ Tri load_tri(long long f, long long M, const long long* faces, const double* verts,
                                        double thresh, bool& ok) {
    Tri t;
    long long v[3];
    ok = true;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        v[k] = faces[3 * f + k];
        ok &= v[k] >= 0 && v[k] < M;
    }
    t.kept = false;
    t.n1 = t.n2 = 0.0;
    if (!ok) return t;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        t.t0[k] = verts[3 * v[0] + k];
        t.v1[k] = __dsub_rn(verts[3 * v[1] + k], t.t0[k]);
        t.v2[k] = __dsub_rn(verts[3 * v[2] + k], t.t0[k]);
    }
    const double l1 = norm3(t.v1), l2 = norm3(t.v2);
    const double* a = t.v1;
    const double* b = t.v2;
    const double cr[3] = {__dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1])),
                          __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2])),
                          __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]))};
    const double area2 = norm3(cr);
    t.kept = area2 > 0.0;
    if (!t.kept) return t;
    const double thr = __dmul_rn(thresh, __dsqrt_rn(__ddiv_rn(__dmul_rn(l1, l2), area2)));
    t.n1 = floor(__ddiv_rn(l1, thr));
    t.n2 = floor(__ddiv_rn(l2, thr));
    return t;
}

// the number of points row i of a triangle emits: the first j in [0, n2] with (i+0.5)/d1 + (j+0.5)/d2 >= 1
__device__ __forceinline__ uint32_t row_count(double i, double n1, double n2) {
    const double a = __ddiv_rn(__dadd_rn(i, 0.5), fmax(n1, 1e-7)), d2 = fmax(n2, 1e-7);
    long long lo = 0, hi = (long long)n2 + 1;           // a + b_j < 1 for j < lo; >= 1 for j >= hi
    while (lo < hi) {
        const long long mid = lo + (hi - lo) / 2;
        if (__dadd_rn(a, __ddiv_rn(__dadd_rn((double)mid, 0.5), d2)) < 1.0) lo = mid + 1;
        else hi = mid;
    }
    return (uint32_t)lo;
}

// a triangle whose n1 * n2 exceeds this emits more than the limit of points: it is counted as the saturated value
constexpr double kChMaxGrid = 8589934592.0;       // 2^33
constexpr unsigned long long kChSaturated = 1ull << 31;

__device__ __forceinline__ bool too_many(const Tri& t) {
    return t.n1 > (double)kChMaxPoints || t.n2 > (double)kChMaxPoints || t.n1 * t.n2 > kChMaxGrid;
}

// one warp per triangle: count[f] (clamped to 2^31), and into info: [0] the sum of counts, [1] a bad index flag,
// [2] a non-finite vertex flag (set by the vertex pass), [3] the number of triangles of positive area
__global__ void __launch_bounds__(kChThreads) ch_count_kernel(long long F, long long M, const long long* __restrict__ faces,
                                                              const double* __restrict__ verts, double thresh,
                                                              uint32_t* __restrict__ count,
                                                              unsigned long long* __restrict__ info) {
    const long long f = ((long long)blockIdx.x * kChThreads + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (f >= F) return;
    bool ok;
    const Tri t = load_tri(f, M, faces, verts, thresh, ok);
    unsigned long long c = 0;
    if (t.kept && t.n1 > 0.0 && t.n2 > 0.0) {
        if (too_many(t)) {
            c = kChSaturated;
        } else {
            for (double i = lane; i <= t.n1; i += 32.0) c += row_count(i, t.n1, t.n2);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
            c = c < kChSaturated ? c : kChSaturated;
        }
    }
    if (lane == 0) {
        count[f] = (uint32_t)c;
        if (c) atomicAdd(info, c);
        if (!ok) atomicOr(info + 1, 1ull);
        if (t.kept) atomicAdd(info + 3, 1ull);
    }
}

__global__ void __launch_bounds__(kChThreads) ch_finite_kernel(long long n, const double* __restrict__ xyz,
                                                               unsigned long long* flag) {
    const long long i = (long long)blockIdx.x * kChThreads + threadIdx.x;
    if (i < n && !(isfinite(xyz[3 * i]) && isfinite(xyz[3 * i + 1]) && isfinite(xyz[3 * i + 2]))) atomicOr(flag, 1ull);
}

// the triangles of a block are ranked by the look-back scan; then each warp writes the points of 32 of them
__global__ void __launch_bounds__(kChThreads) ch_emit_kernel(long long F, long long M, const long long* __restrict__ faces,
                                                             const double* __restrict__ verts, double thresh,
                                                             const uint32_t* __restrict__ count, uint32_t* ctrl,
                                                             unsigned long long* status, double* __restrict__ out) {
    __shared__ uint32_t s_off[kChThreads];
    const uint32_t bid = block_ticket(ctrl);
    const long long f0 = (long long)bid * kChThreads;
    const uint32_t mine = f0 + threadIdx.x < F ? count[f0 + threadIdx.x] : 0u;
    const GridScan s = grid_exclusive_scan<kChThreads>(mine, bid, status);
    s_off[threadIdx.x] = s.rank;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = warp; k < kChThreads && f0 + k < F; k += kChThreads / 32) {
        if (s_off[k] == (k + 1 < kChThreads ? s_off[k + 1] : s.base + s.total)) continue;   // no points
        bool ok;
        const Tri t = load_tri(f0 + k, M, faces, verts, thresh, ok);
        unsigned long long base = (unsigned long long)M + s_off[k];
        const double d1 = fmax(t.n1, 1e-7), d2 = fmax(t.n2, 1e-7);
        for (double i0 = 0.0; i0 <= t.n1; i0 += 32.0) {
            const double i = i0 + lane;
            const uint32_t c = i <= t.n1 ? row_count(i, t.n1, t.n2) : 0u;
            uint32_t incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += n;
            }
            const uint32_t chunk = __shfl_sync(0xffffffffu, incl, 31);
            for (int r = 0; r < 32; r++) {
                const uint32_t cr = __shfl_sync(0xffffffffu, c, r);
                if (cr == 0) continue;
                const unsigned long long row = base + __shfl_sync(0xffffffffu, incl - c, r);
                const double a = __ddiv_rn(__dadd_rn(i0 + r, 0.5), d1);
                for (uint32_t j = lane; j < cr; j += 32) {
                    const double b = __ddiv_rn(__dadd_rn((double)j, 0.5), d2);
                    double* q = out + 3 * (row + j);
#pragma unroll
                    for (int e = 0; e < 3; e++)
                        q[e] = __dadd_rn(__dadd_rn(__dmul_rn(t.v1[e], a), __dmul_rn(t.v2[e], b)), t.t0[e]);
                }
            }
            base += chunk;
        }
    }
}

// ---------------------------------------------------------------------------------------------- point structure

struct Tree {
    uint32_t n;                                   // points
    int top;                                      // level with at most 32 boxes
    uint32_t cnt[kMaxLevels];                     // boxes per level
    uint32_t off[kMaxLevels];                     // first box of each level in the box array
    const double4* pts;                           // sorted points, original index in .w
    const double4* boxes;                         // (lo, hi) pair per box
};

size_t ceil_box(size_t n) { return (n + kBox - 1) / kBox; }

size_t boxes_for(size_t n) {
    size_t nb = 0, c = ceil_box(std::max<size_t>(n, 1));
    while (true) {
        nb += c;
        if (c <= (size_t)kBox) break;
        c = ceil_box(c);
    }
    return nb;
}

Tree tree_of(uint32_t n, const double4* pts, const double4* boxes) {
    Tree t;
    t.n = n;
    t.pts = pts;
    t.boxes = boxes;
    uint32_t c = (uint32_t)ceil_box(std::max<uint32_t>(n, 1)), o = 0;
    t.top = 0;
    while (true) {
        t.cnt[t.top] = c;
        t.off[t.top] = o;
        o += c;
        if (c <= (uint32_t)kBox) break;
        c = (uint32_t)ceil_box(c);
        t.top++;
    }
    return t;
}

__device__ __forceinline__ unsigned long long ord_of(double d) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(d);
    return (u >> 63) ? ~u : (u | (1ull << 63));
}
__device__ __forceinline__ double double_of_ord(unsigned long long u) {
    return __longlong_as_double((long long)((u >> 63) ? (u & ~(1ull << 63)) : ~u));
}

// bb: [0..2] min, [3..5] max as ordered u64 (inputs are finite: the wrapper checks before any structure is built)
__global__ void __launch_bounds__(kChThreads) ch_bbox_kernel(uint32_t n, const double* __restrict__ xyz,
                                                             unsigned long long* bb) {
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const double v = xyz[3 * (size_t)i + a];
            lo[a] = fmin(lo[a], v);
            hi[a] = fmax(hi[a], v);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            lo[a] = fmin(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmax(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
        for (int a = 0; a < 3; a++) {
            atomicMin(&bb[a], ord_of(lo[a]));
            atomicMax(&bb[3 + a], ord_of(hi[a]));
        }
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

// the key only orders the points (and so sets the speed); any rounding here is harmless
__global__ void __launch_bounds__(kChThreads) ch_morton_kernel(uint32_t n, const double* __restrict__ xyz,
                                                               const unsigned long long* __restrict__ bb,
                                                               uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double lo[3], ext = 0.0;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        lo[a] = double_of_ord(bb[a]);
        ext = fmax(ext, double_of_ord(bb[3 + a]) - lo[a]);
    }
    const double s = ext > 0.0 && ext < INFINITY ? 2097151.0 / ext : 0.0;
    uint64_t key = 0;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const double t = (xyz[3 * (size_t)i + a] - lo[a]) * s;
        key |= spread21((uint32_t)fmin(fmax(t, 0.0), 2097151.0)) << a;
    }
    keys[i] = key;
    vals[i] = i;
}

__global__ void __launch_bounds__(kChThreads) ch_gather_kernel(uint32_t n, const double* __restrict__ xyz,
                                                               const uint32_t* __restrict__ vals_sorted,
                                                               double4* __restrict__ pts) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t i = vals_sorted[j];
    pts[j] = make_double4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], (double)i);
}

// boxes of `level` (one warp per box): over points when level == 0, else over the boxes of level - 1
__global__ void __launch_bounds__(kChThreads) ch_box_kernel(int level, const __grid_constant__ Tree t,
                                                            double4* __restrict__ boxes) {
    const int lane = threadIdx.x & 31;
    const uint32_t box = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (box >= t.cnt[level]) return;
    const uint32_t n_below = level == 0 ? t.n : t.cnt[level - 1];
    const uint32_t c = box * kBox + lane;
    double4 lo = make_double4(INFINITY, INFINITY, INFINITY, 0.0), hi = make_double4(-INFINITY, -INFINITY, -INFINITY, 0.0);
    if (c < n_below) {
        if (level == 0) {
            lo = hi = t.pts[c];
        } else {
            const double4* src = boxes + 2 * ((size_t)t.off[level - 1] + c);
            lo = src[0];
            hi = src[1];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo.x = fmin(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, o));
        lo.y = fmin(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, o));
        lo.z = fmin(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, o));
        hi.x = fmax(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, o));
        hi.y = fmax(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, o));
        hi.z = fmax(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, o));
    }
    if (lane == 0) {
        double4* dst = boxes + 2 * ((size_t)t.off[level] + box);
        dst[0] = make_double4(lo.x, lo.y, lo.z, 0.0);
        dst[1] = make_double4(hi.x, hi.y, hi.z, 0.0);
    }
}

// rdist of rule 3 / 6 and the lower bounds that are provably <= it (see the header comment)
__device__ __forceinline__ double rdist(double4 a, double4 b) {
    const double dx = __dsub_rn(a.x, b.x), dy = __dsub_rn(a.y, b.y), dz = __dsub_rn(a.z, b.z);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}
__device__ __forceinline__ double gap(double lo, double hi, double qlo, double qhi) {   // interval to interval
    return fmax(fmax(__dsub_rn(lo, qhi), __dsub_rn(qlo, hi)), 0.0);
}
__device__ __forceinline__ double box_lb(double4 lo, double4 hi, double4 qlo, double4 qhi) {
    const double gx = gap(lo.x, hi.x, qlo.x, qhi.x), gy = gap(lo.y, hi.y, qlo.y, qhi.y), gz = gap(lo.z, hi.z, qlo.z, qhi.z);
    return __dadd_rn(__dadd_rn(__dmul_rn(gx, gx), __dmul_rn(gy, gy)), __dmul_rn(gz, gz));
}

// the bounding box of the warp's active queries (every lane gets it); an empty warp gets an empty box
__device__ __forceinline__ void warp_box(bool active, double4 q, double4& lo, double4& hi) {
    lo = active ? q : make_double4(INFINITY, INFINITY, INFINITY, 0.0);
    hi = active ? q : make_double4(-INFINITY, -INFINITY, -INFINITY, 0.0);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo.x = fmin(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, o));
        lo.y = fmin(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, o));
        lo.z = fmin(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, o));
        hi.x = fmax(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, o));
        hi.y = fmax(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, o));
        hi.z = fmax(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, o));
    }
}

__device__ __forceinline__ double4 box_lo(const Tree& t, int l, uint32_t b) { return t.boxes[2 * ((size_t)t.off[l] + b)]; }
__device__ __forceinline__ double4 box_hi(const Tree& t, int l, uint32_t b) { return t.boxes[2 * ((size_t)t.off[l] + b) + 1]; }

// Depth-first walk of the tree by the whole warp.  warp_need(lo, hi): whether the box may hold a pair for some query
// of the warp (a conservative test against the warp's query box); lane_need(lo, hi): this lane's own test; a box is
// entered when some lane needs it.  leaf(b) visits level-0 box b; the walk ends early when busy() is false on every
// lane.  mask[l] holds the children (boxes of level l - 1) of box parent[l] still to visit; the virtual root sits at
// level top + 1.
template <class WarpNeed, class LaneNeed, class Leaf, class Busy>
__device__ __forceinline__ void tree_walk(const Tree& t, WarpNeed warp_need, LaneNeed lane_need, Leaf leaf, Busy busy) {
    const int lane = threadIdx.x & 31;
    uint32_t mask[kMaxLevels + 1], parent[kMaxLevels + 1];
    int l = t.top + 1;
    parent[l] = 0;
    mask[l] = __ballot_sync(0xffffffffu, (uint32_t)lane < t.cnt[t.top] &&
                                             warp_need(box_lo(t, t.top, lane), box_hi(t, t.top, lane)));
    while (__any_sync(0xffffffffu, busy())) {
        if (mask[l] == 0) {
            if (l == t.top + 1) break;
            l++;
            continue;
        }
        const int i = __ffs(mask[l]) - 1;
        mask[l] &= mask[l] - 1;
        const uint32_t child = parent[l] * kBox + i;         // a box of level l - 1
        if (!__any_sync(0xffffffffu, lane_need(box_lo(t, l - 1, child), box_hi(t, l - 1, child)))) continue;
        if (l == 1) {
            leaf(child);
        } else {
            l--;
            parent[l] = child;
            const uint32_t g = child * kBox + lane;
            mask[l] = __ballot_sync(0xffffffffu, g < t.cnt[l - 1] && warp_need(box_lo(t, l - 1, g), box_hi(t, l - 1, g)));
        }
    }
}

// the points of leaf b, one per lane (count returned); the caller broadcasts them with __shfl_sync
__device__ __forceinline__ int load_leaf(const Tree& t, uint32_t b, double4& p) {
    const int lane = threadIdx.x & 31;
    const uint32_t first = b * kBox;
    const int cnt = (int)min((uint32_t)kBox, t.n - first);
    p = lane < cnt ? t.pts[first + lane] : make_double4(0.0, 0.0, 0.0, 0.0);
    return cnt;
}
__device__ __forceinline__ double4 bcast(double4 p, int src) {
    return make_double4(__shfl_sync(0xffffffffu, p.x, src), __shfl_sync(0xffffffffu, p.y, src),
                        __shfl_sync(0xffffffffu, p.z, src), __shfl_sync(0xffffffffu, p.w, src));
}

__device__ __forceinline__ uint8_t ld_state(const uint8_t* p) {
    return *(const volatile uint8_t*)p;
}

// One greedy round (rule 3), one warp per level-0 box of the shuffled cloud's tree: every undecided point looks for
// earlier neighbours (shuffled position below its own, rdist <= r2).  A kept one removes it; if every one it finds
// is removed it is kept; otherwise it stays undecided.  undecided[round] counts the points left; a round after one
// that left none returns at once.
__global__ void __launch_bounds__(kChThreads, 4) ch_round_kernel(const __grid_constant__ Tree t, double r2, uint8_t* state,
                                                              uint32_t* undecided, int round) {
    if (round > 0 && undecided[round - 1] == 0) return;
    const int lane = threadIdx.x & 31;
    const uint32_t leaf = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (leaf >= t.cnt[0]) return;
    const uint32_t j = leaf * kBox + lane;
    const double4 q = j < t.n ? t.pts[j] : make_double4(0.0, 0.0, 0.0, 0.0);
    const uint32_t pos = (uint32_t)q.w;
    const bool mine = j < t.n && ld_state(state + pos) == kUndecided;
    if (!__any_sync(0xffffffffu, mine)) return;
    bool live = mine, blocked = false;
    double4 qlo, qhi;
    warp_box(mine, q, qlo, qhi);
    tree_walk(
        t, [&](double4 lo, double4 hi) { return box_lb(lo, hi, qlo, qhi) <= r2; },
        [&](double4 lo, double4 hi) { return live && box_lb(lo, hi, q, q) <= r2; },
        [&](uint32_t b) {
            double4 p;
            const int cnt = load_leaf(t, b, p);
            for (int s = 0; s < cnt; s++) {
                const double4 o = bcast(p, s);
                if (live && (uint32_t)o.w < pos && rdist(q, o) <= r2) {
                    const uint8_t st = ld_state(state + (uint32_t)o.w);
                    if (st == kKept) live = false;
                    else if (st == kUndecided) blocked = true;
                }
            }
        },
        [&]() { return live; });
    if (mine) {
        if (!live) state[pos] = kRemoved;
        else if (!blocked) state[pos] = kKept;
    }
    const unsigned left = __ballot_sync(0xffffffffu, mine && live && blocked);
    if (lane == 0 && left) atomicAdd(undecided + round, (uint32_t)__popc(left));
}

// Bounded 1-NN (rule 6), one warp per 32 sorted queries: d = sqrt(rdist to the nearest tree point) when it is below
// max_dist, else +inf.  The query's distance goes to dist[query index], its colour (rule 8) to color[target[index]].
__global__ void __launch_bounds__(kChThreads) ch_nn_kernel(uint32_t nq, const double4* __restrict__ queries,
                                                           const __grid_constant__ Tree t, double max_dist, double vis,
                                                           const uint32_t* __restrict__ target, double* __restrict__ dist,
                                                           double* __restrict__ color) {
    const int lane = threadIdx.x & 31;
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w * kBox >= nq) return;
    const uint32_t j = w * kBox + lane;
    const bool active = j < nq;
    const double4 q = active ? queries[j] : make_double4(0.0, 0.0, 0.0, 0.0);
    double best = INFINITY;
    double4 qlo, qhi;
    warp_box(active, q, qlo, qhi);
    auto scan = [&](uint32_t b) {
        double4 p;
        const int cnt = load_leaf(t, b, p);
        for (int s = 0; s < cnt; s++) {
            const double d = rdist(q, bcast(p, s));
            if (active && d < best) best = d;
        }
    };
    // seed: descend to the leaf nearest the warp's first query (lane 0 is always active), so that the walk starts
    // with a tight bound; the seed leaf may be scanned again by the walk, which changes nothing
    {
        const double4 s = bcast(q, 0);
        uint32_t b = 0;
        for (int l = t.top; l >= 0; l--) {
            const uint32_t g = b * kBox + lane;
            const double lb = g < t.cnt[l] ? box_lb(box_lo(t, l, g), box_hi(t, l, g), s, s) : INFINITY;
            double m = lb;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
            b = b * kBox + (__ffs(__ballot_sync(0xffffffffu, lb == m)) - 1);
        }
        scan(b);
    }
    auto far = [&](double lb, double bound) { return __dsqrt_rn(lb) >= max_dist || lb > bound; };
    auto warp_bound = [&]() {
        double m = active ? best : -INFINITY;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
        return m;
    };
    double wb = warp_bound();
    tree_walk(
        t, [&](double4 lo, double4 hi) { return !far(box_lb(lo, hi, qlo, qhi), wb); },
        [&](double4 lo, double4 hi) { return active && !far(box_lb(lo, hi, q, q), best); },
        [&](uint32_t b) {
            scan(b);
            wb = warp_bound();
        },
        [&]() { return active; });
    if (!active) return;
    const uint32_t qi = (uint32_t)q.w;
    const double d = __dsqrt_rn(best);
    const bool near = d < max_dist;
    dist[qi] = near ? d : INFINITY;
    double* c = color + 3 * (size_t)target[qi];
    if (near) {
        const double alpha = __ddiv_rn(fmin(d, vis), vis), beta = __dsub_rn(1.0, alpha);
        c[0] = __dadd_rn(__dmul_rn(1.0, alpha), __dmul_rn(1.0, beta));
        c[1] = __dadd_rn(__dmul_rn(0.0, alpha), __dmul_rn(1.0, beta));
        c[2] = __dadd_rn(__dmul_rn(0.0, alpha), __dmul_rn(1.0, beta));
    } else {
        c[0] = 0.0; c[1] = 1.0; c[2] = 0.0;
    }
}

// ---------------------------------------------------------------------------------------------- masks

struct SelectParams {
    double lo[3], hi[3];                          // rule 4, already rounded to float32 and widened
    double bb0[3], res;                           // rule 5
    int shape[3];
};

// over the shuffled cloud: kept -> data_down, inbound -> data_in, observed -> data_in_obs (+ its data_down row);
// info[0..2] the three counts
__global__ void __launch_bounds__(kChThreads) ch_select_kernel(uint32_t n, const double* __restrict__ xyz,
                                                               const uint8_t* __restrict__ state,
                                                               const __grid_constant__ SelectParams sp,
                                                               const uint8_t* __restrict__ obs, uint32_t* ctrl,
                                                               unsigned long long* status, double* __restrict__ down,
                                                               double* __restrict__ in, double* __restrict__ in_obs,
                                                               uint32_t* __restrict__ obs_down, long long* info) {
    __shared__ uint32_t s_warp[3][kChThreads / 32], s_excl[3];
    const uint32_t bid = block_ticket(ctrl);
    const uint32_t i = bid * kChThreads + threadIdx.x;
    double x[3] = {0.0, 0.0, 0.0};
    bool kept = false, inb = false, ob = false;
    if (i < n && state[i] == kKept) {
        kept = inb = true;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            x[a] = xyz[3 * (size_t)i + a];
            inb &= x[a] >= sp.lo[a] && x[a] < sp.hi[a];
        }
        if (inb) {
            long long g[3];
            bool gin = true;
#pragma unroll
            for (int a = 0; a < 3; a++) {
                const double v = rint(__ddiv_rn(__dsub_rn(x[a], sp.bb0[a]), sp.res));
                gin &= v >= 0.0 && v < (double)sp.shape[a];
                g[a] = gin ? (long long)v : 0;
            }
            ob = gin && obs[((size_t)g[0] * sp.shape[1] + (size_t)g[1]) * sp.shape[2] + (size_t)g[2]] != 0;
        }
    }
    uint32_t total[3], excl[3];
    excl[0] = block_exclusive_scan<kChThreads>(kept ? 1u : 0u, s_warp[0], total[0]);
    excl[1] = block_exclusive_scan<kChThreads>(inb ? 1u : 0u, s_warp[1], total[1]);
    excl[2] = block_exclusive_scan<kChThreads>(ob ? 1u : 0u, s_warp[2], total[2]);
    block_lookback<3>(status, gridDim.x, bid, total, s_excl);
    const uint32_t r0 = s_excl[0] + excl[0], r1 = s_excl[1] + excl[1], r2 = s_excl[2] + excl[2];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        if (kept) down[3 * (size_t)r0 + a] = x[a];
        if (inb) in[3 * (size_t)r1 + a] = x[a];
        if (ob) in_obs[3 * (size_t)r2 + a] = x[a];
    }
    if (ob) obs_down[r2] = r0;
    if (bid == gridDim.x - 1 && threadIdx.x < 3) info[threadIdx.x] = (long long)s_excl[threadIdx.x] + total[threadIdx.x];
}

// rule 7: STL points above the plane, in order, with their STL row; info[0] the count
__global__ void __launch_bounds__(kChThreads) ch_plane_kernel(uint32_t n, const double* __restrict__ stl, double p0,
                                                              double p1, double p2, double p3, uint32_t* ctrl,
                                                              unsigned long long* status, double* __restrict__ above,
                                                              uint32_t* __restrict__ above_idx, long long* info) {
    const uint32_t bid = block_ticket(ctrl);
    const uint32_t i = bid * kChThreads + threadIdx.x;
    double x[3] = {0.0, 0.0, 0.0};
    bool up = false;
    if (i < n) {
#pragma unroll
        for (int a = 0; a < 3; a++) x[a] = stl[3 * (size_t)i + a];
        const double h = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p0, x[0]), __dmul_rn(p1, x[1])), __dmul_rn(p2, x[2])),
                                   __dmul_rn(p3, 1.0));
        up = h > 0.0;
    }
    const GridScan s = grid_exclusive_scan<kChThreads>(up ? 1u : 0u, bid, status);
    if (up) {
#pragma unroll
        for (int a = 0; a < 3; a++) above[3 * (size_t)s.rank + a] = x[a];
        above_idx[s.rank] = i;
    }
    if (s.last && threadIdx.x == 0) info[0] = (long long)s.base + s.total;
}

__global__ void __launch_bounds__(kChThreads) ch_fill_blue_kernel(long long n, double* __restrict__ color) {
    const long long i = (long long)blockIdx.x * kChThreads + threadIdx.x;
    if (i >= n) return;
    color[3 * i] = 0.0;
    color[3 * i + 1] = 0.0;
    color[3 * i + 2] = 1.0;
}

// ---------------------------------------------------------------------------------------------- masked means

// block b sums the distances below max_dist of its 2048-entry slice in a fixed tree; partial[b] = (sum, count)
constexpr int kSumPer = 8;
__global__ void __launch_bounds__(kChThreads) ch_sum_kernel(uint32_t n, const double* __restrict__ dist, double max_dist,
                                                            double2* __restrict__ partial) {
    __shared__ double s_sum[kChThreads], s_cnt[kChThreads];
    const size_t base = (size_t)blockIdx.x * kChThreads * kSumPer;
    double sum = 0.0, cnt = 0.0;
#pragma unroll
    for (int k = 0; k < kSumPer; k++) {
        const size_t i = base + (size_t)k * kChThreads + threadIdx.x;
        if (i < n && dist[i] < max_dist) {
            sum = __dadd_rn(sum, dist[i]);
            cnt += 1.0;
        }
    }
    s_sum[threadIdx.x] = sum;
    s_cnt[threadIdx.x] = cnt;
    __syncthreads();
    for (int s = kChThreads / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            s_sum[threadIdx.x] = __dadd_rn(s_sum[threadIdx.x], s_sum[threadIdx.x + s]);
            s_cnt[threadIdx.x] += s_cnt[threadIdx.x + s];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = make_double2(s_sum[0], s_cnt[0]);
}

// one block: out = (sum, count) over the partials, each thread a fixed strided slice, then a fixed tree
__global__ void __launch_bounds__(kChThreads) ch_sum_final_kernel(int nb, const double2* __restrict__ partial,
                                                                  double* __restrict__ out) {
    __shared__ double s_sum[kChThreads], s_cnt[kChThreads];
    double sum = 0.0, cnt = 0.0;
    for (int b = threadIdx.x; b < nb; b += kChThreads) {
        sum = __dadd_rn(sum, partial[b].x);
        cnt += partial[b].y;
    }
    s_sum[threadIdx.x] = sum;
    s_cnt[threadIdx.x] = cnt;
    __syncthreads();
    for (int s = kChThreads / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            s_sum[threadIdx.x] = __dadd_rn(s_sum[threadIdx.x], s_sum[threadIdx.x + s]);
            s_cnt[threadIdx.x] += s_cnt[threadIdx.x + s];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        out[0] = s_sum[0];
        out[1] = s_cnt[0];
    }
}

// ---------------------------------------------------------------------------------------------- host side

// sample workspace: [ctrl 64 B][status][count u32 per triangle]
struct SampleLayout { size_t ctrl, status, count, total; };
SampleLayout sample_layout(long long F) {
    SampleLayout L;
    const size_t f = (size_t)std::max<long long>(F, 1);
    size_t o = 0;
    L.ctrl = o;   o = align_up(o + 64, 256);
    L.status = o; o = align_up(o + (size_t)grid_blocks(F, kChThreads) * 8, 256);
    L.count = o;  o = align_up(o + f * 4, 256);
    L.total = o;
    return L;
}

// evaluation workspace for a cloud of N points and an STL of S points; T = max(N, S)
struct EvalLayout {
    size_t ctrl, rounds, status_n, status_s, sort, state, pts_a, boxes_a, pts_b, boxes_b, pts_q, partial, total;
    size_t t;   // pairs the sort has room for
};
EvalLayout eval_layout(long long N, long long S) {
    EvalLayout L;
    const size_t n = (size_t)std::max<long long>(N, 1), s = (size_t)std::max<long long>(S, 1), t = std::max(n, s);
    size_t o = 0;
    L.ctrl = o;     o = align_up(o + 256, 256);         // [0..1] tickets, [8..13] box (u64 at byte 64)
    L.rounds = o;   o = align_up(o + kRoundBatch * 4, 256);
    L.status_n = o; o = align_up(o + (size_t)3 * grid_blocks(N, kChThreads) * 8, 256);
    L.status_s = o; o = align_up(o + (size_t)grid_blocks(S, kChThreads) * 8, 256);
    L.sort = o;     o = align_up(o + radix_sort_workspace_bytes(t), 256);
    L.state = o;    o = align_up(o + n, 256);
    L.pts_a = o;    o = align_up(o + n * 32, 256);
    L.boxes_a = o;  o = align_up(o + boxes_for(n) * 64, 256);
    L.pts_b = o;    o = align_up(o + s * 32, 256);
    L.boxes_b = o;  o = align_up(o + boxes_for(s) * 64, 256);
    L.pts_q = o;    o = align_up(o + t * 32, 256);
    L.partial = o;  o = align_up(o + (size_t)grid_blocks((long long)t, kChThreads * kSumPer) * 16, 256);
    L.total = o;
    L.t = t;
    return L;
}

struct EvalBufs {
    char* w;
    const EvalLayout* L;
    cudaStream_t st;
    unsigned long long* bb() const { return (unsigned long long*)(w + L->ctrl + 64); }
};

// n points of xyz (n x 3 float64) gathered into Morton order in pts (.w = row); n >= 1
int sort_points(const EvalBufs& B, uint32_t n, const double* xyz, double4* pts, int stage) {
    cudaStream_t st = B.st;
    SURFEL_CUDA_OK(cudaMemsetAsync(B.bb(), 0xff, 24, st));
    SURFEL_CUDA_OK(cudaMemsetAsync(B.bb() + 3, 0, 24, st));
    const unsigned nb = grid_blocks(n, kChThreads);
    {
        LaunchScope scope(stage, st);
        ch_bbox_kernel<<<std::min<unsigned>(nb, (unsigned)current_device_sm_count() * 8), kChThreads, 0, st>>>(
            n, xyz, B.bb());
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    const RadixSortWs sort = radix_sort_ws(B.w + B.L->sort, B.L->t, 63);
    {
        LaunchScope scope(stage, st);
        ch_morton_kernel<<<nb, kChThreads, 0, st>>>(n, xyz, B.bb(), sort.in.keys, sort.in.vals);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    if (launch_radix_sort_pairs(sort, n, st)) return 1;
    {
        LaunchScope scope(stage, st);
        ch_gather_kernel<<<nb, kChThreads, 0, st>>>(n, xyz, sort.out.vals, pts);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

int build_tree(const EvalBufs& B, uint32_t n, const double* xyz, double4* pts, double4* boxes, Tree& t, int stage) {
    if (sort_points(B, n, xyz, pts, stage)) return 1;
    t = tree_of(n, pts, boxes);
    for (int l = 0; l <= t.top; l++) {
        LaunchScope scope(stage, B.st);
        ch_box_kernel<<<grid_blocks((long long)t.cnt[l] * 32, kChThreads), kChThreads, 0, B.st>>>(l, t, boxes);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

bool eval_sizes_ok(const char* who, long long N, long long S) {
    if (N < 1 || S < 1) { surfel_set_error("%s: empty cloud (%lld points, %lld STL points)", who, N, S); return false; }
    if (N > kChMaxPoints || S > kChMaxPoints) {
        surfel_set_error("%s: %lld points and %lld STL points; at most %lld each are supported", who, N, S, kChMaxPoints);
        return false;
    }
    return true;
}

}  // namespace
}  // namespace surfel

using namespace surfel;

extern "C" {

long long surfel_chamfer_max_points(void) { return kChMaxPoints; }

size_t surfel_chamfer_sample_workspace_bytes(long long n_faces) {
    if (n_faces < 0 || n_faces > kChMaxPoints) return 0;
    return sample_layout(n_faces).total;
}

int surfel_chamfer_sample_count(long long n_verts, long long n_faces, const double* verts, const long long* faces,
                                double thresh, void* workspace, size_t workspace_bytes, long long* info,
                                void* stream) {
    const char* who = "surfel_chamfer_sample_count";
    if (n_verts < 0 || n_faces < 0 || n_verts > kChMaxPoints || n_faces > kChMaxPoints) {
        surfel_set_error("%s: %lld vertices, %lld faces; 0 to %lld of each are supported", who, n_verts, n_faces,
                         kChMaxPoints);
        return 1;
    }
    if (!info || (n_verts > 0 && !verts) || (n_faces > 0 && !faces)) {
        surfel_set_error("%s: NULL vertices, faces or info", who);
        return 1;
    }
    const SampleLayout L = sample_layout(n_faces);
    if (!workspace_ok(who, workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    SURFEL_CUDA_OK(cudaMemsetAsync(info, 0, 4 * sizeof(long long), st));
    if (n_verts > 0) {
        LaunchScope scope(kStChamferSample, st);
        ch_finite_kernel<<<grid_blocks(n_verts, kChThreads), kChThreads, 0, st>>>(n_verts, verts,
                                                                                  (unsigned long long*)info + 2);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    if (n_faces > 0) {
        LaunchScope scope(kStChamferSample, st);
        ch_count_kernel<<<grid_blocks(n_faces * 32, kChThreads), kChThreads, 0, st>>>(
            n_faces, n_verts, faces, verts, thresh, (uint32_t*)(w + L.count), (unsigned long long*)info);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

int surfel_chamfer_sample_emit(long long n_verts, long long n_faces, const double* verts, const long long* faces,
                               double thresh, void* workspace, size_t workspace_bytes, long long n_samples,
                               double* out, void* stream) {
    const char* who = "surfel_chamfer_sample_emit";
    if (n_verts < 0 || n_faces < 0 || n_samples < 0 || n_verts + n_samples > kChMaxPoints ||
        n_faces > kChMaxPoints) {
        surfel_set_error("%s: %lld vertices and %lld samples; at most %lld points in all are supported", who, n_verts,
                         n_samples, kChMaxPoints);
        return 1;
    }
    if (n_faces == 0 || n_samples == 0) return 0;
    if (!verts || !faces || !out) { surfel_set_error("%s: NULL vertices, faces or output", who); return 1; }
    const SampleLayout L = sample_layout(n_faces);
    if (!workspace_ok(who, workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.ctrl, 0, 64, st));
    const unsigned nb = grid_blocks(n_faces, kChThreads);
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status, 0, (size_t)nb * 8, st));
    LaunchScope scope(kStChamferSample, st);
    ch_emit_kernel<<<nb, kChThreads, 0, st>>>(n_faces, n_verts, faces, verts, thresh, (const uint32_t*)(w + L.count),
                                              (uint32_t*)(w + L.ctrl), (unsigned long long*)(w + L.status), out);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

size_t surfel_chamfer_workspace_bytes(long long n_points, long long n_stl) {
    if (n_points < 0 || n_stl < 0 || n_points > kChMaxPoints || n_stl > kChMaxPoints) return 0;
    return eval_layout(n_points, n_stl).total;
}

int surfel_chamfer_downsample(long long n_points, long long n_stl, const double* pcd, double thresh,
                              void* workspace, size_t workspace_bytes, int* rounds, void* stream) {
    const char* who = "surfel_chamfer_downsample";
    if (!eval_sizes_ok(who, n_points, n_stl)) return 1;
    if (!pcd || !rounds) { surfel_set_error("%s: NULL cloud or rounds", who); return 1; }
    const EvalLayout L = eval_layout(n_points, n_stl);
    if (!workspace_ok(who, workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    EvalBufs B{(char*)workspace, &L, st};
    const uint32_t n = (uint32_t)n_points;
    uint8_t* state = (uint8_t*)(B.w + L.state);
    uint32_t* undecided = (uint32_t*)(B.w + L.rounds);
    Tree t;
    if (build_tree(B, n, pcd, (double4*)(B.w + L.pts_a), (double4*)(B.w + L.boxes_a), t, kStChamferDownsample)) return 1;
    SURFEL_CUDA_OK(cudaMemsetAsync(state, kUndecided, n, st));
    const double r2 = thresh * thresh;
    *rounds = 0;
    // the one host read that sizes no output: the count of undecided points after each batch of rounds
    for (int done = 0; !done;) {
        SURFEL_CUDA_OK(cudaMemsetAsync(undecided, 0, kRoundBatch * 4, st));
        for (int r = 0; r < kRoundBatch; r++) {
            LaunchScope scope(kStChamferDownsample, st);
            ch_round_kernel<<<grid_blocks((long long)t.cnt[0] * 32, kChThreads), kChThreads, 0, st>>>(t, r2, state,
                                                                                                    undecided, r);
            SURFEL_CUDA_OK(cudaGetLastError());
        }
        uint32_t left[kRoundBatch];
        SURFEL_CUDA_OK(cudaMemcpyAsync(left, undecided, sizeof(left), cudaMemcpyDeviceToHost, st));
        SURFEL_CUDA_OK(cudaStreamSynchronize(st));
        for (int r = 0; r < kRoundBatch && !done; r++) {
            ++*rounds;
            done = left[r] == 0;
        }
    }
    return 0;
}

int surfel_chamfer_select(long long n_points, long long n_stl, const double* pcd, const double* stl,
                          const double* box_lo, const double* box_hi, const double* bb0, double res,
                          const unsigned char* obs_mask, const int* obs_shape, const double* plane, void* workspace,
                          size_t workspace_bytes, double* data_down, double* data_in, double* data_in_obs,
                          unsigned int* obs_down, double* stl_above, unsigned int* above_idx, long long* info,
                          void* stream) {
    const char* who = "surfel_chamfer_select";
    if (!eval_sizes_ok(who, n_points, n_stl)) return 1;
    if (!pcd || !stl || !box_lo || !box_hi || !bb0 || !obs_mask || !obs_shape || !plane || !data_down || !data_in ||
        !data_in_obs || !obs_down || !stl_above || !above_idx || !info) {
        surfel_set_error("%s: NULL argument", who);
        return 1;
    }
    SelectParams sp;
    for (int a = 0; a < 3; a++) {
        if (obs_shape[a] < 1) { surfel_set_error("%s: observation mask of shape with a zero side", who); return 1; }
        sp.lo[a] = box_lo[a];
        sp.hi[a] = box_hi[a];
        sp.bb0[a] = bb0[a];
        sp.shape[a] = obs_shape[a];
    }
    sp.res = res;
    const EvalLayout L = eval_layout(n_points, n_stl);
    if (!workspace_ok(who, workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    uint32_t* ctrl = (uint32_t*)(w + L.ctrl);
    SURFEL_CUDA_OK(cudaMemsetAsync(ctrl, 0, 8, st));
    const unsigned nb_n = grid_blocks(n_points, kChThreads), nb_s = grid_blocks(n_stl, kChThreads);
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status_n, 0, (size_t)3 * nb_n * 8, st));
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status_s, 0, (size_t)nb_s * 8, st));
    {
        LaunchScope scope(kStChamferSelect, st);
        ch_select_kernel<<<nb_n, kChThreads, 0, st>>>(
            (uint32_t)n_points, pcd, (const uint8_t*)(w + L.state), sp, obs_mask, ctrl,
            (unsigned long long*)(w + L.status_n), data_down, data_in, data_in_obs, obs_down, info);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    {
        LaunchScope scope(kStChamferSelect, st);
        ch_plane_kernel<<<nb_s, kChThreads, 0, st>>>((uint32_t)n_stl, stl, plane[0], plane[1], plane[2], plane[3],
                                                     ctrl + 1, (unsigned long long*)(w + L.status_s), stl_above,
                                                     above_idx, info + 3);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

int surfel_chamfer_distances(long long n_points, long long n_stl, const double* stl, long long n_down, long long n_in,
                             const double* data_in, long long n_obs, const double* data_in_obs,
                             const unsigned int* obs_down, long long n_above, const double* stl_above,
                             const unsigned int* above_idx, double max_dist, double vis, void* workspace,
                             size_t workspace_bytes, double* dist_d2s, double* dist_s2d, double* data_color,
                             double* stl_color, double* sums, void* stream) {
    const char* who = "surfel_chamfer_distances";
    if (!eval_sizes_ok(who, n_points, n_stl)) return 1;
    if (n_in < 1 || n_obs < 1 || n_above < 1 || n_down < n_in || n_in < n_obs || n_down > n_points ||
        n_above > n_stl) {
        surfel_set_error("%s: counts %lld kept, %lld inbound, %lld observed, %lld above do not fit %lld points and %lld "
                         "STL points (each set must be non-empty)", who, n_down, n_in, n_obs, n_above, n_points, n_stl);
        return 1;
    }
    if (!stl || !data_in || !data_in_obs || !obs_down || !stl_above || !above_idx || !dist_d2s || !dist_s2d ||
        !data_color || !stl_color || !sums) {
        surfel_set_error("%s: NULL argument", who);
        return 1;
    }
    const EvalLayout L = eval_layout(n_points, n_stl);
    if (!workspace_ok(who, workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    EvalBufs B{(char*)workspace, &L, st};
    double4* q = (double4*)(B.w + L.pts_q);
    double2* partial = (double2*)(B.w + L.partial);
    {
        LaunchScope scope(kStChamferNn, st);
        ch_fill_blue_kernel<<<grid_blocks(n_down, kChThreads), kChThreads, 0, st>>>(n_down, data_color);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    {
        LaunchScope scope(kStChamferNn, st);
        ch_fill_blue_kernel<<<grid_blocks(n_stl, kChThreads), kChThreads, 0, st>>>(n_stl, stl_color);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    // d2s: data_in_obs against all of the STL
    Tree ts, ti;
    if (build_tree(B, (uint32_t)n_stl, stl, (double4*)(B.w + L.pts_b), (double4*)(B.w + L.boxes_b), ts, kStChamferNn))
        return 1;
    if (sort_points(B, (uint32_t)n_obs, data_in_obs, q, kStChamferNn)) return 1;
    {
        LaunchScope scope(kStChamferNn, st);
        ch_nn_kernel<<<grid_blocks(n_obs, kChThreads), kChThreads, 0, st>>>((uint32_t)n_obs, q, ts, max_dist, vis,
                                                                            obs_down, dist_d2s, data_color);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    // s2d: stl_above against data_in
    if (build_tree(B, (uint32_t)n_in, data_in, (double4*)(B.w + L.pts_a), (double4*)(B.w + L.boxes_a), ti, kStChamferNn))
        return 1;
    if (sort_points(B, (uint32_t)n_above, stl_above, q, kStChamferNn)) return 1;
    {
        LaunchScope scope(kStChamferNn, st);
        ch_nn_kernel<<<grid_blocks(n_above, kChThreads), kChThreads, 0, st>>>((uint32_t)n_above, q, ti, max_dist, vis,
                                                                              above_idx, dist_s2d, stl_color);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    const long long ns[2] = {n_obs, n_above};
    const double* ds[2] = {dist_d2s, dist_s2d};
    for (int k = 0; k < 2; k++) {
        const unsigned nb = grid_blocks(ns[k], kChThreads * kSumPer);
        {
            LaunchScope scope(kStChamferNn, st);
            ch_sum_kernel<<<nb, kChThreads, 0, st>>>((uint32_t)ns[k], ds[k], max_dist, partial);
            SURFEL_CUDA_OK(cudaGetLastError());
        }
        {
            LaunchScope scope(kStChamferNn, st);
            ch_sum_final_kernel<<<1, kChThreads, 0, st>>>((int)nb, partial, sums + 2 * k);
            SURFEL_CUDA_OK(cudaGetLastError());
        }
    }
    return 0;
}

}  // extern "C"
