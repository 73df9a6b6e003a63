// mcubes.cu — marching cubes of the reference's unbounded mesh extraction (utils/mcube_utils.py:17-95,
// marching_cubes_with_contraction, `render.py --unbounded`) on the device: per crop a count and an emit pass over the
// crop's grid points, and after all crops one merge (DESIGN.md §7j has the rules; tests/mcubes_ref.py restates them).
//
//  * surfel_mcubes_crop_count: one thread per grid point of the side^3 crop.  A point counts the crossing edges it
//    owns (its three edges towards +x, +y, +z; a point on the crop's upper plane belongs to the next crop, unless
//    this crop is the last along that axis) and, when it is a cube's lower corner, the cube's triangles from the
//    table.  Both counts are scanned across the grid with a single-pass decoupled look-back (scan.cuh);
//    each block keeps its exclusive prefix and the last block writes the crop's two totals, which the caller reads
//    to size the crop's outputs.
//  * surfel_mcubes_crop_emit: the same walk, with the block's prefix from the count pass: each crossing edge writes
//    one record (its vertex key and its contracted position), each cube its triangles as key triples, in cube order
//    (x slowest) then table order.
//  * surfel_mcubes_merge: sorts all records by key with launch_radix_sort_pairs, keeps the first of each key
//    (equal keys carry equal positions) with a second look-back scan, uncontracts and clips the vertices, and maps
//    every triangle key to its rank by binary search.
//
// A vertex's key is (global grid point) * 4 + axis for a vertex inside an edge, and (global grid point) * 4 + 3 for
// a vertex on a grid corner (t exactly 0 or 1).  Positions use fixed, uncontracted float32 arithmetic (the file is
// compiled with -fmad=false): t = va / (va - vb), p = pa + t * (pb - pa) per component.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "../../include/surfel_rasterizer.h"
#include "common.cuh"
#include "contraction.cuh"
#include "kernels.h"
#include "profile.h"
#include "scan.cuh"

namespace surfel {

#include "mcubes_table.inc"

namespace {

constexpr int kMcThreads = 256;
constexpr int kMcMaxCrops = 1024;                 // crops per axis: keys of (511 * 1024 + 1)^3 * 4 fit 64 bits
constexpr float kMcMaxRange = 32.f;               // the reference's max_range

// corner k of a cube is at (k & 1, k >> 1 & 1, k >> 2 & 1); edge e runs from kEdgeLo[e] along axis e / 4
__device__ const unsigned char kEdgeLo[12] = {0, 2, 4, 6, 0, 1, 4, 5, 0, 1, 2, 3};

struct McCrop {
    const float* vol;      // side^3 values, x slowest
    int s;                 // side
    int own_hi[3];         // the crop is the last along axis d, so it owns its upper plane
    long long g0[3];       // global grid index of local index 0
    long long G;           // global grid points per axis
    LinAxis ax[3];
};

// One grid point's share of a crop: its corner values, its owned crossing edges and its cube's case.
struct McPoint {
    int l[3];
    float v[8];            // values at the corners of the cube whose lower corner this point is (those that exist)
    unsigned rec_axes;     // bit d: the owned edge along d crosses
    int ncase, ntri;
};

__device__ __forceinline__ McPoint mc_point(const McCrop& c, long long i) {
    McPoint p;
    const long long s = c.s;
    p.l[0] = (int)(i / (s * s)); p.l[1] = (int)(i / s % s); p.l[2] = (int)(i % s);
    const bool up[3] = {p.l[0] < c.s - 1, p.l[1] < c.s - 1, p.l[2] < c.s - 1};
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int dx = k & 1, dy = k >> 1 & 1, dz = k >> 2 & 1;
        p.v[k] = 0.f;
        if ((!dx || up[0]) && (!dy || up[1]) && (!dz || up[2]))
            p.v[k] = __ldg(c.vol + i + (dx * s + dy) * s + dz);
    }
    p.rec_axes = 0;
    if ((up[0] || c.own_hi[0]) && (up[1] || c.own_hi[1]) && (up[2] || c.own_hi[2])) {
#pragma unroll
        for (int d = 0; d < 3; d++)
            if (up[d] && ((p.v[0] < 0.f) != (p.v[1 << d] < 0.f))) p.rec_axes |= 1u << d;
    }
    p.ncase = 0;
    p.ntri = 0;
    if (up[0] && up[1] && up[2]) {
#pragma unroll
        for (int k = 0; k < 8; k++) p.ncase |= (p.v[k] < 0.f) << k;
        p.ntri = kMcTable[p.ncase][0];
    }
    return p;
}

__device__ __forceinline__ uint32_t mc_packed(const McPoint& p) {
    return (uint32_t)__popc(p.rec_axes) | (uint32_t)p.ntri << 16;     // block sums <= 768 and <= 1280
}

__device__ __forceinline__ float edge_t(float va, float vb) { return __fdiv_rn(va, __fsub_rn(va, vb)); }

__device__ __forceinline__ unsigned long long gpoint(const McCrop& c, int a, int b, int d) {
    return ((unsigned long long)(c.g0[0] + a) * c.G + (unsigned long long)(c.g0[1] + b)) * c.G +
           (unsigned long long)(c.g0[2] + d);
}

// the vertex key of the edge from grid point pa (global index) along axis d, with values va, vb at its ends
__device__ __forceinline__ unsigned long long edge_key(const McCrop& c, unsigned long long pa, int d, float t) {
    const unsigned long long stride = d == 0 ? (unsigned long long)(c.G * c.G) : d == 1 ? (unsigned long long)c.G : 1ull;
    if (t == 0.f) return pa * 4 + 3;
    if (t == 1.f) return (pa + stride) * 4 + 3;
    return pa * 4 + d;
}

struct McCtrl {
    uint32_t* ctrl;                 // [0] ticket, [1] merged vertex count
    unsigned long long* status;     // [C][blocks]
    uint2* prefix;                  // [blocks] exclusive (records, triangles) of each block
};

__global__ void __launch_bounds__(kMcThreads) mc_count_kernel(const __grid_constant__ McCrop c, McCtrl w,
                                                              long long* totals) {
    __shared__ uint32_t s_warp[kMcThreads / 32], s_excl[2];
    const uint32_t bid = block_ticket(&w.ctrl[0]);
    const long long n = (long long)c.s * c.s * c.s;
    const long long i = (long long)bid * kMcThreads + threadIdx.x;
    uint32_t mine = 0;
    if (i < n) mine = mc_packed(mc_point(c, i));
    uint32_t packed_total;
    block_exclusive_scan<kMcThreads>(mine, s_warp, packed_total);
    const uint32_t total[2] = {packed_total & 0xffffu, packed_total >> 16};
    block_lookback<2>(w.status, gridDim.x, bid, total, s_excl);
    if (threadIdx.x == 0) {
        w.prefix[bid] = make_uint2(s_excl[0], s_excl[1]);
        if (bid == gridDim.x - 1) {
            totals[0] = (long long)s_excl[0] + total[0];
            totals[1] = (long long)s_excl[1] + total[1];
        }
    }
}

__global__ void __launch_bounds__(kMcThreads) mc_emit_kernel(const __grid_constant__ McCrop c, const uint2* prefix,
                                                             unsigned long long* __restrict__ vkeys,
                                                             float* __restrict__ vpos,
                                                             unsigned long long* __restrict__ tkeys) {
    __shared__ uint32_t s_warp[kMcThreads / 32];
    const long long n = (long long)c.s * c.s * c.s;
    const long long i = (long long)blockIdx.x * kMcThreads + threadIdx.x;
    McPoint p;
    uint32_t mine = 0;
    if (i < n) {
        p = mc_point(c, i);
        mine = mc_packed(p);
    }
    uint32_t total;
    const uint32_t excl = block_exclusive_scan<kMcThreads>(mine, s_warp, total);
    if (i >= n || mine == 0) return;
    const uint2 pre = prefix[blockIdx.x];
    const unsigned long long P = gpoint(c, p.l[0], p.l[1], p.l[2]);
    float pa[3];
#pragma unroll
    for (int d = 0; d < 3; d++) pa[d] = linspace_at(c.ax[d], p.l[d], c.s);
    long long r = (long long)pre.x + (excl & 0xffffu);
#pragma unroll
    for (int d = 0; d < 3; d++) {
        if (!(p.rec_axes >> d & 1)) continue;
        const float va = p.v[0], vb = p.v[1 << d];
        const float t = edge_t(va, vb);
        float pb[3] = {pa[0], pa[1], pa[2]};
        pb[d] = linspace_at(c.ax[d], p.l[d] + 1, c.s);
        vkeys[r] = edge_key(c, P, d, t);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            float x = __fadd_rn(pa[k], __fmul_rn(t, __fsub_rn(pb[k], pa[k])));
            if (t == 0.f) x = pa[k];
            if (t == 1.f) x = pb[k];
            vpos[3 * r + k] = x;
        }
        r++;
    }
    const long long t0 = (long long)pre.y + (excl >> 16);
    const signed char* row = kMcTable[p.ncase];
    for (int k = 0; k < p.ntri; k++) {
        for (int j = 0; j < 3; j++) {
            const int e = row[1 + 3 * k + j];
            const int lo = kEdgeLo[e], d = e >> 2;
            const unsigned long long pa_g = gpoint(c, p.l[0] + (lo & 1), p.l[1] + (lo >> 1 & 1), p.l[2] + (lo >> 2 & 1));
            tkeys[3 * (t0 + k) + j] = edge_key(c, pa_g, d, edge_t(p.v[lo], p.v[lo | 1 << d]));
        }
    }
}

__global__ void mc_sort_init_kernel(long long n, const unsigned long long* __restrict__ keys,
                                    uint64_t* __restrict__ ka, uint32_t* __restrict__ va) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        ka[i] = keys[i];
        va[i] = (uint32_t)i;
    }
}

// the first record of each key: its rank among the distinct keys, its key, and its vertex uncontracted and clipped
__global__ void __launch_bounds__(kMcThreads) mc_unique_kernel(long long n, const uint64_t* __restrict__ keys,
                                                               const uint32_t* __restrict__ vals,
                                                               const float* __restrict__ pos, McCtrl w, float radius,
                                                               float cx, float cy, float cz,
                                                               unsigned long long* __restrict__ ukeys,
                                                               float* __restrict__ verts, long long* n_verts) {
    const uint32_t bid = block_ticket(&w.ctrl[0]);
    const long long i = (long long)bid * kMcThreads + threadIdx.x;
    const bool first = i < n && (i == 0 || keys[i] != keys[i - 1]);
    const GridScan s = grid_exclusive_scan<kMcThreads>(first ? 1u : 0u, bid, w.status);
    if (s.last && threadIdx.x == 0) {
        w.ctrl[1] = s.base + s.total;
        *n_verts = (long long)s.base + s.total;
    }
    if (!first) return;
    const long long r = s.rank;
    const uint32_t src = vals[i];
    float X = pos[3 * (size_t)src], Y = pos[3 * (size_t)src + 1], Z = pos[3 * (size_t)src + 2];
    inv_contraction(contraction_norm(X, Y, Z), X, Y, Z, radius, cx, cy, cz);
    auto clip = [](float x) { return x < -kMcMaxRange ? -kMcMaxRange : (x > kMcMaxRange ? kMcMaxRange : x); };
    ukeys[r] = keys[i];
    verts[3 * r] = clip(X);
    verts[3 * r + 1] = clip(Y);
    verts[3 * r + 2] = clip(Z);
}

__global__ void mc_faces_kernel(long long n, const unsigned long long* __restrict__ tkeys,
                                const unsigned long long* __restrict__ ukeys, const uint32_t* ctrl,
                                long long* __restrict__ faces) {
    const long long U = ctrl[1];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const unsigned long long k = tkeys[i];
        long long lo = 0, hi = U;          // first index whose key is >= k; every triangle key is a vertex key
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (ukeys[mid] < k) lo = mid + 1; else hi = mid;
        }
        faces[i] = lo;
    }
}

struct CropLayout {
    size_t ctrl, status, prefix, total;
    unsigned blocks;
};

CropLayout crop_layout(int side) {
    CropLayout L;
    L.blocks = grid_blocks((long long)side * side * side, kMcThreads);
    size_t o = 0;
    L.ctrl = o;   o = align_up(o + 64, 256);
    L.status = o; o = align_up(o + (size_t)2 * L.blocks * 8, 256);
    L.prefix = o; o = align_up(o + (size_t)L.blocks * 8, 256);
    L.total = o;
    return L;
}

struct MergeLayout {
    size_t ctrl, status, sort, ukeys, total;
    unsigned blocks;
};

MergeLayout merge_layout(long long n) {
    MergeLayout L;
    const size_t m = n > 0 ? (size_t)n : 1;
    L.blocks = grid_blocks(n, kMcThreads);
    size_t o = 0;
    L.ctrl = o;   o = align_up(o + 64, 256);
    L.status = o; o = align_up(o + (size_t)L.blocks * 8, 256);
    L.sort = o;   o = align_up(o + radix_sort_workspace_bytes(m), 256);
    L.ukeys = o;  o = align_up(o + m * 8, 256);
    L.total = o;
    return L;
}

bool side_ok(int side) { return side >= 2 && side <= kMcMaxSide; }

// the crop's part of the global grid; returns false (error set) on a bad crop
bool make_crop(const char* who, int side, const float* volume, const int* crop, int crops, McCrop& c) {
    if (!side_ok(side)) { surfel_set_error("%s: side %d outside [2, %d]", who, side, kMcMaxSide); return false; }
    if (crops < 1 || crops > kMcMaxCrops) {
        surfel_set_error("%s: %d crops per axis outside [1, %d]", who, crops, kMcMaxCrops);
        return false;
    }
    if (!crop) { surfel_set_error("%s: NULL crop index", who); return false; }
    for (int d = 0; d < 3; d++)
        if (crop[d] < 0 || crop[d] >= crops) {
            surfel_set_error("%s: crop index %d outside [0, %d)", who, crop[d], crops);
            return false;
        }
    if (!volume) { surfel_set_error("%s: NULL volume", who); return false; }
    c.vol = volume;
    c.s = side;
    c.G = (long long)(side - 1) * crops + 1;
    for (int d = 0; d < 3; d++) {
        c.own_hi[d] = crop[d] == crops - 1;
        c.g0[d] = (long long)crop[d] * (side - 1);
        c.ax[d] = LinAxis{0.f, 0.f, 0.f};
    }
    return true;
}

}  // namespace
}  // namespace surfel

using namespace surfel;

extern "C" {

size_t surfel_mcubes_crop_workspace_bytes(int side) {
    if (!side_ok(side)) return 0;
    return crop_layout(side).total;
}

int surfel_mcubes_crop_count(int side, const float* volume, const int* crop, int crops_per_axis, void* workspace,
                             size_t workspace_bytes, long long* totals, void* stream) {
    McCrop c;
    if (!make_crop("surfel_mcubes_crop_count", side, volume, crop, crops_per_axis, c)) return 1;
    if (!totals) { surfel_set_error("surfel_mcubes_crop_count: NULL totals"); return 1; }
    const CropLayout L = crop_layout(side);
    if (!workspace_ok("surfel_mcubes_crop_count", workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.ctrl, 0, 64, st));
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status, 0, (size_t)2 * L.blocks * 8, st));
    McCtrl m{(uint32_t*)(w + L.ctrl), (unsigned long long*)(w + L.status), (uint2*)(w + L.prefix)};
    LaunchScope scope(kStMcubesCrop, st);
    mc_count_kernel<<<L.blocks, kMcThreads, 0, st>>>(c, m, totals);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_mcubes_crop_emit(int side, const float* volume, const double* bounds, const int* crop, int crops_per_axis,
                            const void* workspace, size_t workspace_bytes, long long n_records, long long n_tris,
                            unsigned long long* vert_keys, float* vert_pos, unsigned long long* tri_keys,
                            void* stream) {
    McCrop c;
    if (!make_crop("surfel_mcubes_crop_emit", side, volume, crop, crops_per_axis, c)) return 1;
    if (!bounds) { surfel_set_error("surfel_mcubes_crop_emit: NULL bounds"); return 1; }
    if (n_records < 0 || n_tris < 0) { surfel_set_error("surfel_mcubes_crop_emit: negative count"); return 1; }
    if ((n_records > 0 && (!vert_keys || !vert_pos)) || (n_tris > 0 && !tri_keys)) {
        surfel_set_error("surfel_mcubes_crop_emit: NULL output");
        return 1;
    }
    const CropLayout L = crop_layout(side);
    if (!workspace_ok("surfel_mcubes_crop_emit", workspace, workspace_bytes, L.total)) return 1;
    if (n_records == 0 && n_tris == 0) return 0;
    for (int d = 0; d < 3; d++) c.ax[d] = make_lin_axis(bounds[2 * d], bounds[2 * d + 1], side);
    cudaStream_t st = (cudaStream_t)stream;
    LaunchScope scope(kStMcubesCrop, st);
    mc_emit_kernel<<<L.blocks, kMcThreads, 0, st>>>(c, (const uint2*)((const char*)workspace + L.prefix), vert_keys,
                                                     vert_pos, tri_keys);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

size_t surfel_mcubes_merge_workspace_bytes(long long n_records) {
    if (n_records < 0 || n_records > kRadixSortMaxPairs) return 0;
    return merge_layout(n_records).total;
}

int surfel_mcubes_merge(long long n_records, const unsigned long long* vert_keys, const float* vert_pos,
                        long long n_tris, const unsigned long long* tri_keys, int key_bits, const float* center,
                        double radius, void* workspace, size_t workspace_bytes, float* verts, long long* faces,
                        long long* n_verts, void* stream) {
    if (n_records < 0 || n_tris < 0) { surfel_set_error("surfel_mcubes_merge: negative count"); return 1; }
    if (n_records > kRadixSortMaxPairs) {
        surfel_set_error("surfel_mcubes_merge: %lld vertex records exceed the radix sort's limit of 2^30", n_records);
        return 1;
    }
    if (n_tris > 0 && n_records == 0) {
        surfel_set_error("surfel_mcubes_merge: %lld triangles without vertices", n_tris);
        return 1;
    }
    if (n_tris > (1ll << 40)) { surfel_set_error("surfel_mcubes_merge: %lld triangles", n_tris); return 1; }
    if (key_bits < 1 || key_bits > 64) { surfel_set_error("surfel_mcubes_merge: key_bits %d", key_bits); return 1; }
    if (!center || !n_verts) { surfel_set_error("surfel_mcubes_merge: NULL center or vertex count"); return 1; }
    if ((n_records > 0 && (!vert_keys || !vert_pos || !verts)) || (n_tris > 0 && (!tri_keys || !faces))) {
        surfel_set_error("surfel_mcubes_merge: NULL input or output");
        return 1;
    }
    const MergeLayout L = merge_layout(n_records);
    if (!workspace_ok("surfel_mcubes_merge", workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.ctrl, 0, 64, st));
    if (n_records == 0) {
        SURFEL_CUDA_OK(cudaMemsetAsync(n_verts, 0, sizeof(long long), st));
        return 0;
    }
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status, 0, (size_t)L.blocks * 8, st));
    const RadixSortWs sort = radix_sort_ws(w + L.sort, (size_t)n_records, key_bits);
    const int grid = (int)std::min<long long>((n_records + 255) / 256, (long long)current_device_sm_count() * 8);
    {
        LaunchScope scope(kStMcubesMerge, st);
        mc_sort_init_kernel<<<grid, 256, 0, st>>>(n_records, vert_keys, sort.in.keys, sort.in.vals);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    if (launch_radix_sort_pairs(sort, (size_t)n_records, st)) return 1;
    McCtrl m{(uint32_t*)(w + L.ctrl), (unsigned long long*)(w + L.status), nullptr};
    unsigned long long* ukeys = (unsigned long long*)(w + L.ukeys);
    {
        LaunchScope scope(kStMcubesMerge, st);
        mc_unique_kernel<<<L.blocks, kMcThreads, 0, st>>>(n_records, sort.out.keys, sort.out.vals, vert_pos, m,
                                                           (float)radius, center[0], center[1], center[2], ukeys,
                                                           verts, n_verts);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    if (n_tris > 0) {
        const long long nk = 3 * n_tris;
        const int fgrid = (int)std::min<long long>((nk + 255) / 256, (long long)current_device_sm_count() * 16);
        LaunchScope scope(kStMcubesMerge, st);
        mc_faces_kernel<<<fgrid, 256, 0, st>>>(nk, tri_keys, ukeys, m.ctrl, faces);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

}  // extern "C"
