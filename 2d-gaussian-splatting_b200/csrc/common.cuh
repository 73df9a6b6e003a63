// common.cuh — constants, HBM record layouts and small device helpers shared by all kernels.
//
// Algorithm constants follow SURVEY.md Appendix A (the un-vendored upstream rasterizer
// hbb1/diff-surfel-rasterization @ e0ed0207; its config lives in files absent from
// /root/reference) and are kept in this one header, as SURVEY §7 asks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace surfel {

constexpr int kBlockX = 16;
constexpr int kBlockY = 16;
constexpr int kTilePixels = kBlockX * kBlockY;
constexpr float kNear = 0.2f;
constexpr float kFar = 100.0f;
constexpr float kFilterSize = 0.707106f;
constexpr float kFilterInvSquare = 2.0f;
constexpr float kCutoff = 3.0f;
constexpr float kAlphaMax = 0.99f;
constexpr float kAlphaMin = 1.0f / 255.0f;
constexpr float kTMin = 0.0001f;

// out_others channel order (reference gaussian_renderer/__init__.py:118-135)
constexpr int kChDepth = 0, kChAlpha = 1, kChNormal = 2, kChMidDepth = 5, kChDistortion = 6;

// ---------------------------------------------------------------------------------------------
// HBM layout of the per-splat state written by preprocess and gathered by render (fwd and bwd).
//
// RENDER RECORD: 128 bytes = one full cache line, read with 128-bit loads.  The ray-splat
// intersection of upstream's renderCUDA (k = px*Tw - Tu, l = py*Tw - Tv, p = cross(k, l), SURVEY A.3)
// is AFFINE in the pixel:  p(px,py) = Tu x Tv + px (Tv x Tw) + py (Tw x Tu)  — the adjugate of the
// splat->pixel homography applied to (px, py, 1).  Preprocess therefore emits the three vectors once
// per splat, expanded about the splat's own screen position c = xy (the AABB centre of A.1 step 5):
//      p = Pc + (px - c.x) P1 + (py - c.y) P2,   P1 = Tv' x Tw,  P2 = Tw x Tu',  Pc = Tu' x Tv',
//      Tu' = Tu - c.x Tw,  Tv' = Tv - c.y Tw
// computed in double and rounded once (in absolute pixel coordinates the float32 terms cancel to a few
// units in 1e5).  The render kernels spend 6 FMA per (pixel, splat) on p instead of 6 FMA + 3 MUL +
// 3 FMA for k, l and their cross product, and the result is closer to the exact value of upstream's
// formula than upstream's own float32 evaluation.  The ray-splat depth s.x*Tw.x + s.y*Tw.y + Tw.z equals
// det(T) / p.z exactly (w of the intersection point), which is how the forward evaluates it.
//   q0 = (P1.x, P1.y, P1.z, c.x)        q1 = (P2.x, P2.y, P2.z, c.y)
//   q2 = (Pc.x, Pc.y, Pc.z, +-opacity)  q3 = (n.x, n.y, n.z, Tw.z)          n = view-space normal
//        (opacity < 0: the splat may reach in front of the near plane -> per-pixel `depth < near` test needed)
//   q4 = (r, g, b, det T)               q5 = (Tw.x, Tw.y, splat index bits, view depth)
//   q6 = conservative screen AABB (x0, y0, x1, y1) of the region where alpha can reach 1/255
//   q7 = extents of the same region along the diagonals (min x+y, max x+y, min x-y, max x-y)
// q6/q7 are only read while a tile's list is staged (each staging thread classifies its splat against
// the eight 8x4 warp footprints of the tile); q0..q5 (q0..q4 in the forward) go to shared memory.
// ---------------------------------------------------------------------------------------------
constexpr int kRecQuads = 8;
constexpr int kRecBytes = kRecQuads * 16;
constexpr int kRecQuadsFwd = 5;     // quads the forward stages in shared memory
constexpr int kRecQuadsBwd = 6;     // quads the backward stages

// TRANSFORM RECORD: 48 bytes per splat, upstream's geometry-state fields that the render kernels do
// not need but preprocess backward, the binning kernels and the parity tests do:
//   t0 = (Tu.x, Tu.y, Tu.z, Tv.x)   t1 = (Tv.y, Tv.z, Tw.x, Tw.y)   t2 = (Tw.z, xy.x, xy.y, view depth)
constexpr int kTmQuads = 3;

// Per-splat gradient record accumulated by render backward (float atomics), 24 floats = 96 B.
// dL_dtransMat is NOT accumulated directly.  With a = dL/dp per (pixel,splat) (p = Pc + dx P1 + dy P2, the
// affine form above, (dx,dy) = pixel - c) the sums  A = sum a,  Bx = sum dx*a,  By = sum dy*a  ARE the
// gradients of (Pc, P1, P2); the ray-splat depth det T / p.z contributes -dL_dz*depth/p.z to a.z and
// Zd = sum dL_dz / p.z  (the gradient of det T); the low-pass branch contributes Zl = sum dL_dz*(s.x, s.y, 1)
// to dL_dTw (upstream's "Propagate the gradients of depth"; (0, 0, dL_dz) with the exact derivative).
// Preprocess backward turns them into dL_dT once per splat (three cross products + det's gradient) instead
// of every lane doing two cross products per pair:
//   dTu' = Tv' x A + By x Tw,  dTv' = A x Tu' + Tw x Bx,  dTw = Bx x Tv' + Tu' x By - c.x dTu' - c.y dTv'
//   (+ Zd * (Tv x Tw, Tw x Tu, Tu x Tv) + Zl on Tw)
//   [0..2] A  [3..5] Bx  [6..8] By  [9] Zd  [10..12] Zl  [13..14] dL_dmean2D.xy  [15] dL_dopacity
//   [16..18] dL_dnormal  [19..21] dL_dcolor  [22..23] pad
constexpr int kGradFloats = 24;
constexpr int kGradUsed = 22;

struct GeomLayout {
    size_t rec, tmat, tiles_touched, offsets, clamped, scan_status, counters, total;
};
struct ImageLayout {
    size_t accum, n_contrib, tile_count, total;  // accum: final_T, M1, M2; n_contrib: last, median; per-tile instance counts
};
struct BinningLayout {
    size_t pairs, ranges, temp, total;   // the radix sort's buffers, tile ranges, scratch of either sort
};

__host__ __device__ inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

constexpr int kPreBlock = 128;   // preprocess threads per block (and scan tile)

inline GeomLayout geom_layout(int P) {
    GeomLayout L;
    size_t o = 0;
    size_t p = (size_t)(P > 0 ? P : 1);
    L.rec = o;            o = align_up(o + p * kRecBytes, 256);
    L.tmat = o;           o = align_up(o + p * kTmQuads * 16, 256);
    L.tiles_touched = o;  o = align_up(o + p * 4, 256);
    L.offsets = o;        o = align_up(o + p * 4, 256);
    L.clamped = o;        o = align_up(o + p, 256);
    L.scan_status = o;    o = align_up(o + ((p + kPreBlock - 1) / kPreBlock + 1) * 8, 256);
    L.counters = o;       o = align_up(o + 64, 256);   // [0] ticket, [1] num_rendered
    L.total = o;
    return L;
}
inline ImageLayout image_layout(int W, int H) {
    ImageLayout L;
    size_t n = (size_t)W * (size_t)H;
    size_t o = 0;
    L.accum = o;      o = align_up(o + n * 3 * 4, 256);
    L.n_contrib = o;  o = align_up(o + n * 2 * 4, 256);
    const size_t tiles = (size_t)((W + kBlockX - 1) / kBlockX) * (size_t)((H + kBlockY - 1) / kBlockY);
    L.tile_count = o; o = align_up(o + tiles * 4, 256);
    L.total = o;
    return L;
}

// float -> int32, truncate toward zero, saturating, NaN -> 0 (PTX cvt.rzi.s32.f32; the oracle's
// f2i_sat() restates exactly this).
__device__ __forceinline__ int f2i_sat(float x) { return __float2int_rz(x); }

__device__ __forceinline__ void get_rect(float cx, float cy, int radius, int gx, int gy, int row0,
                                         int row1, int& x0, int& y0, int& x1, int& y1) {
    const float r = (float)radius;
    x0 = min(gx, max(0, f2i_sat((cx - r) / (float)kBlockX)));
    y0 = min(gy, max(0, f2i_sat((cy - r) / (float)kBlockY)));
    x1 = min(gx, max(0, f2i_sat(((cx + r) + (float)(kBlockX - 1)) / (float)kBlockX)));
    y1 = min(gy, max(0, f2i_sat(((cy + r) + (float)(kBlockY - 1)) / (float)kBlockY)));
    y0 = min(row1, max(row0, y0));
    y1 = min(row1, max(row0, y1));
}

__device__ __forceinline__ float4 ld_nc_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}

// 16-byte global -> shared copy that bypasses registers and L1 (LDGSTS), to a shared-window address
// (__cvta_generic_to_shared), and the wait for all of this thread's copies.
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

// Fixed-order block sum of K double terms, called by every thread of a kThreads block (tid: its linear index): a
// warp butterfly, then the warps' sums in warp order.  Thread k < K hands term k's sum to store(k, sum), so each
// caller keeps its own partials layout; the order depends on the block shape alone, so the sums are bit-identical
// across calls.
template <int K, int kThreads, class Store>
__device__ __forceinline__ void block_sum(const double (&acc)[K], int tid, Store store) {
    __shared__ double s_red[kThreads / 32][K];
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int k = 0; k < K; k++) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) s_red[warp][k] = v;
    }
    __syncthreads();
    if (tid < K) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kThreads / 32; w++) s += s_red[w][tid];
        store(tid, s);
    }
}

}  // namespace surfel

// Error plumbing shared by the C-ABI translation units.
void surfel_set_error(const char* fmt, ...);

// Whether `ws` is a workspace of at least `need` bytes; if not, sets the error of entry point `who`.
inline bool workspace_ok(const char* who, const void* ws, size_t bytes, size_t need) {
    if (!ws) { surfel_set_error("%s: NULL workspace", who); return false; }
    if (bytes < need) { surfel_set_error("%s: workspace of %zu bytes, %zu needed", who, bytes, need); return false; }
    return true;
}

// Per-device one-time initialisation (function attributes and __constant__ tables live per device, and a
// process may drive several): slot of the current device in a caller-owned `static bool done[kMaxDevices]`,
// or -1 if it cannot be determined (then the caller initialises again; all such initialisations are idempotent).
constexpr int kMaxDevices = 64;
inline int current_device_slot() {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return -1;
    return dev;
}
// SM count of the current device (cached per device), for persistent grid-stride launches.
inline int current_device_sm_count() {
    static int cached[kMaxDevices] = {};
    const int slot = current_device_slot();
    if (slot >= 0 && cached[slot] > 0) return cached[slot];
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
        n = 132;
    if (slot >= 0) cached[slot] = n;
    return n;
}
#define SURFEL_CUDA_OK(expr)                                                              \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            surfel_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),      \
                             __FILE__, __LINE__);                                         \
            return 1;                                                                     \
        }                                                                                 \
    } while (0)
