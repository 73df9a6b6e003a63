// tsdf.cu — the SDF field of the reference's unbounded mesh extraction (utils/mesh_utils.py:184-279,
// compute_unbounded_tsdf / compute_sdf_perframe, `render.py --unbounded`), fused into one pass per sample
// (DESIGN.md §7i has the rules and quirks; tests/tsdf_ref.py emulates this file's arithmetic).
//
// One thread per sample.  It computes the sample's truncation and world position once, then folds every frame in
// list order, carrying the running mean and weight in registers: project, test the mask, sample the depth map
// (and in colour mode the RGB map), fold.  Per-frame constants (the three used columns of the 4x4 matrix, H, W,
// the int64 offset into the map buffer) are staged through shared memory in batches of kTsdfBatch, so every
// thread of a CTA reads the same frame at the same time.  No masks, no host syncs, no per-frame launches.
//
// The arithmetic is fixed and uncontracted (the file is compiled with -fmad=false and every operation below is
// an explicitly rounded intrinsic), so the result is bit-reproducible and a numpy float32 emulation reproduces it:
//  * norm: sqrt((x*x + y*y) + z*z), correctly rounded;  1/x: correctly rounded reciprocal;  y/|y|, pix = xy/w:
//    correctly rounded division;
//  * projection: ((x*M0j + y*M1j) + z*M2j) + M3j for the columns j = 0, 1, 3 of the row-vector product;
//  * grid_sample(bilinear, border, align_corners=True): s = ((p + 1) * 0.5) * (W - 1), clipped to [0, W - 1];
//    x0 = floor(s), w = s - x0, e = 1 - w (likewise n, s for y); weights nw = s*e, ne = s*w, sw = n*e, se = n*w;
//    value = nw*v_nw, then + ne*v_ne, + sw*v_sw, + se*v_se for the taps inside the map, in that order.  Taps are
//    read with ordinary loads: texture filtering would round the weights to 8 bits.
//  * fold: t = (t*w + s) / (w + 1), w = w + 1.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>

#include "../../include/surfel_rasterizer.h"
#include "common.cuh"
#include "contraction.cuh"
#include "profile.h"

namespace surfel {

constexpr int kTsdfThreads = 256;
// frames staged per round: 32 x 64 B = 2 KB of shared memory
constexpr int kTsdfBatch = 32;
constexpr int kTsdfMaxSide = 1 << 24;          // W - 1 and H - 1 must be exact in float32

struct __align__(16) TsdfFrame {
    float m[12];          // (M0j, M1j, M2j, M3j) for j = 0, 1, 3 (x, y and the homogeneous w)
    int H, W;
    long long off;        // element offset of the depth map; the RGB map is at 3 * off
};
static_assert(sizeof(TsdfFrame) == 64, "TsdfFrame is staged as four int4 per frame");

__device__ __forceinline__ float clamp_unit(float v) {   // torch.clamp(v, -1, 1): NaN stays NaN
    return v < -1.f ? -1.f : (v > 1.f ? 1.f : v);
}

__device__ __forceinline__ float proj_col(const float* c, float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, c[0]), __fmul_rn(y, c[1])), __fmul_rn(z, c[2])), c[3]);
}

// Bilinear taps of one frame at the source position (sx, sy), already clipped to the map.
struct Taps {
    long long base;
    float nw, ne, sw, se;
    bool east, south;
};

__device__ __forceinline__ Taps make_taps(float px, float py, int H, int W, long long off) {
    const float wm1 = (float)(W - 1), hm1 = (float)(H - 1);
    float sx = __fmul_rn(__fmul_rn(__fadd_rn(px, 1.f), 0.5f), wm1);
    float sy = __fmul_rn(__fmul_rn(__fadd_rn(py, 1.f), 0.5f), hm1);
    sx = fminf(fmaxf(sx, 0.f), wm1);
    sy = fminf(fmaxf(sy, 0.f), hm1);
    const float x0 = floorf(sx), y0 = floorf(sy);
    const float w = __fsub_rn(sx, x0), e = __fsub_rn(1.f, w);
    const float n = __fsub_rn(sy, y0), s = __fsub_rn(1.f, n);
    const int ix = (int)x0, iy = (int)y0;
    Taps t;
    t.base = off + (long long)iy * W + ix;
    t.nw = __fmul_rn(s, e); t.ne = __fmul_rn(s, w); t.sw = __fmul_rn(n, e); t.se = __fmul_rn(n, w);
    t.east = ix + 1 < W;
    t.south = iy + 1 < H;
    return t;
}

__device__ __forceinline__ float sample(const float* __restrict__ map, const Taps& t, int W) {
    float v = __fmul_rn(__ldg(map + t.base), t.nw);
    if (t.east) v = __fadd_rn(v, __fmul_rn(__ldg(map + t.base + 1), t.ne));
    if (t.south) v = __fadd_rn(v, __fmul_rn(__ldg(map + t.base + W), t.sw));
    if (t.east && t.south) v = __fadd_rn(v, __fmul_rn(__ldg(map + t.base + W + 1), t.se));
    return v;
}

// Where a sample's point comes from: a (N,3) buffer, or (grid mode, DESIGN.md §7j) its index in a side^3 crop of
// three torch.linspace axes laid out as meshgrid(indexing="ij") lays them out, x slowest.
struct PointBuffer {
    const float* pts;
    __device__ __forceinline__ void load(long long i, float& X, float& Y, float& Z) const {
        X = pts[3 * i]; Y = pts[3 * i + 1]; Z = pts[3 * i + 2];
    }
};

struct PointGrid {
    LinAxis ax[3];
    int side;
    __device__ __forceinline__ void load(long long i, float& X, float& Y, float& Z) const {
        const long long s = side;
        X = linspace_at(ax[0], (int)(i / (s * s)), side);
        Y = linspace_at(ax[1], (int)(i / s % s), side);
        Z = linspace_at(ax[2], (int)(i % s), side);
    }
};

template <bool kColour, class Points>
__global__ void __launch_bounds__(kTsdfThreads)
tsdf_kernel(long long N, const Points pts, int V, const TsdfFrame* __restrict__ frames,
            const float* __restrict__ depth, const float* __restrict__ rgb, float cx, float cy, float cz, float radius,
            float trunc0, float* __restrict__ out) {
    __shared__ TsdfFrame sf[kTsdfBatch];
    const long long i = (long long)blockIdx.x * kTsdfThreads + threadIdx.x;
    const bool live = i < N;
    float X = 0.f, Y = 0.f, Z = 0.f, trunc = trunc0;
    if (live) {
        pts.load(i, X, Y, Z);
        if (!kColour) {
            // contracted -> world: adaptive truncation, uncontract, unnormalize
            const float mag = contraction_norm(X, Y, Z);
            if (mag > 1.f) trunc = __fmul_rn(trunc0, __frcp_rn(__fsub_rn(2.f, fminf(mag, 1.9f))));
            inv_contraction(mag, X, Y, Z, radius, cx, cy, cz);
        }
    }
    const float neg_trunc = -trunc;
    float t = kColour ? 0.f : -1.f, r = 0.f, g = 0.f, b = 0.f, wt = 1.f;
    for (int f0 = 0; f0 < V; f0 += kTsdfBatch) {
        const int nb = min(kTsdfBatch, V - f0);
        __syncthreads();                          // the previous batch is no longer read
        for (int k = threadIdx.x; k < nb * 4; k += kTsdfThreads)
            reinterpret_cast<int4*>(sf)[k] = __ldg(reinterpret_cast<const int4*>(frames + f0) + k);
        __syncthreads();
        if (!live) continue;
        for (int k = 0; k < nb; k++) {
            const TsdfFrame& F = sf[k];
            const float hw = proj_col(F.m + 8, X, Y, Z);
            const float px = __fdiv_rn(proj_col(F.m, X, Y, Z), hw);
            const float py = __fdiv_rn(proj_col(F.m + 4, X, Y, Z), hw);
            if (!(px > -1.f && px < 1.f && py > -1.f && py < 1.f && hw > 0.f)) continue;
            const Taps tp = make_taps(px, py, F.H, F.W, F.off);
            const float sdf = __fsub_rn(sample(depth, tp, F.W), hw);
            if (!(sdf > neg_trunc)) continue;
            const float wp = __fadd_rn(wt, 1.f);
            if (kColour) {
                const long long plane = (long long)F.H * F.W;
                Taps tc = tp;
                tc.base = tp.base + 2 * F.off;     // 3 * off + iy * W + ix
                r = __fdiv_rn(__fadd_rn(__fmul_rn(r, wt), sample(rgb, tc, F.W)), wp);
                tc.base += plane;
                g = __fdiv_rn(__fadd_rn(__fmul_rn(g, wt), sample(rgb, tc, F.W)), wp);
                tc.base += plane;
                b = __fdiv_rn(__fadd_rn(__fmul_rn(b, wt), sample(rgb, tc, F.W)), wp);
            } else {
                const float s = clamp_unit(__fdiv_rn(sdf, trunc));
                t = __fdiv_rn(__fadd_rn(__fmul_rn(t, wt), s), wp);
            }
            wt = wp;
        }
    }
    if (!live) return;
    if (kColour) {
        out[3 * i] = r; out[3 * i + 1] = g; out[3 * i + 2] = b;
    } else {
        out[i] = t;
    }
}

// The checks, the frame-table upload and the launch of both entry points; `who` names the entry point in errors.
template <class Points>
static int tsdf_run(const char* who, long long n_points, const Points& pts, bool have_pts, int n_frames,
                    const surfel_tsdf_frame_t* frames, long long map_pixels, const float* depth, const float* rgb,
                    const float* center, double radius, double trunc, float* out, void* stream) {
    if (n_points < 0 || n_frames < 0 || map_pixels < 0) {
        surfel_set_error("%s: negative count (n_points %lld, n_frames %d, map_pixels %lld)", who, n_points, n_frames,
                         map_pixels);
        return 1;
    }
    const long long blocks = (n_points + kTsdfThreads - 1) / kTsdfThreads;
    if (blocks > 0x7fffffffLL) {
        surfel_set_error("%s: %lld points exceed the grid limit", who, n_points);
        return 1;
    }
    if (!center) { surfel_set_error("%s: NULL center", who); return 1; }
    if (n_frames > 0 && !frames) { surfel_set_error("%s: NULL frame table", who); return 1; }
    for (int f = 0; f < n_frames; f++) {
        const surfel_tsdf_frame_t& F = frames[f];
        if (F.height < 1 || F.width < 1 || F.height > kTsdfMaxSide || F.width > kTsdfMaxSide) {
            surfel_set_error("%s: frame %d is %d x %d (each side must be in [1, 2^24])", who, f, F.height, F.width);
            return 1;
        }
        if (F.offset < 0 || F.offset > map_pixels || (long long)F.height * F.width > map_pixels - F.offset) {
            surfel_set_error("%s: frame %d (offset %lld, %d x %d) lies outside the %lld map pixels", who, f,
                             (long long)F.offset, F.height, F.width, map_pixels);
            return 1;
        }
    }
    if (n_points == 0) return 0;
    if (!have_pts || !out) { surfel_set_error("%s: NULL points or output", who); return 1; }
    if (n_frames > 0 && !depth) { surfel_set_error("%s: NULL depth maps", who); return 1; }

    cudaStream_t st = (cudaStream_t)stream;
    TsdfFrame* dframes = nullptr;
    if (n_frames > 0) {
        // The table goes to the device in stream order: a stream-ordered allocation, an asynchronous copy from
        // the host (staged by the driver before this call returns, so the caller's table may go right away)
        // and a stream-ordered free after the kernel.
        const size_t bytes = sizeof(TsdfFrame) * (size_t)n_frames;
        TsdfFrame* host = (TsdfFrame*)malloc(bytes);
        if (!host) { surfel_set_error("%s: out of host memory", who); return 1; }
        for (int f = 0; f < n_frames; f++) {
            const surfel_tsdf_frame_t& F = frames[f];
            const int col[3] = {0, 1, 3};
            for (int j = 0; j < 3; j++)
                for (int row = 0; row < 4; row++) host[f].m[4 * j + row] = F.full_proj_transform[4 * row + col[j]];
            host[f].H = F.height;
            host[f].W = F.width;
            host[f].off = F.offset;
        }
        cudaError_t e = cudaMallocAsync((void**)&dframes, bytes, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dframes, host, bytes, cudaMemcpyHostToDevice, st);
        free(host);
        if (e != cudaSuccess) {
            if (dframes) cudaFreeAsync(dframes, st);
            surfel_set_error("%s: frame table upload failed: %s", who, cudaGetErrorString(e));
            return 1;
        }
    }
    const float cx = center[0], cy = center[1], cz = center[2];
    {
        LaunchScope scope(kStTsdf, st);
        if (rgb)
            tsdf_kernel<true, Points><<<(unsigned)blocks, kTsdfThreads, 0, st>>>(
                n_points, pts, n_frames, dframes, depth, rgb, cx, cy, cz, (float)radius, (float)trunc, out);
        else
            tsdf_kernel<false, Points><<<(unsigned)blocks, kTsdfThreads, 0, st>>>(
                n_points, pts, n_frames, dframes, depth, nullptr, cx, cy, cz, (float)radius, (float)trunc, out);
    }
    const cudaError_t launch = cudaGetLastError();
    if (dframes) SURFEL_CUDA_OK(cudaFreeAsync(dframes, st));
    if (launch != cudaSuccess) {
        surfel_set_error("%s: launch failed: %s", who, cudaGetErrorString(launch));
        return 1;
    }
    return 0;
}

}  // namespace surfel

using namespace surfel;

extern "C" {

int surfel_tsdf_eval(long long n_points, const float* points, int n_frames, const surfel_tsdf_frame_t* frames,
                     long long map_pixels, const float* depth, const float* rgb, const float* center, double radius,
                     double trunc, float* out, void* stream) {
    return tsdf_run("surfel_tsdf_eval", n_points, PointBuffer{points}, points != nullptr, n_frames, frames,
                    map_pixels, depth, rgb, center, radius, trunc, out, stream);
}

int surfel_tsdf_eval_grid(int side, const double* bounds, int n_frames, const surfel_tsdf_frame_t* frames,
                          long long map_pixels, const float* depth, const float* center, double radius, double trunc,
                          float* out, void* stream) {
    if (side < 2 || side > kMcMaxSide) {
        surfel_set_error("surfel_tsdf_eval_grid: side %d outside [2, %d]", side, kMcMaxSide);
        return 1;
    }
    if (!bounds) { surfel_set_error("surfel_tsdf_eval_grid: NULL bounds"); return 1; }
    PointGrid g;
    for (int d = 0; d < 3; d++) g.ax[d] = make_lin_axis(bounds[2 * d], bounds[2 * d + 1], side);
    g.side = side;
    return tsdf_run("surfel_tsdf_eval_grid", (long long)side * side * side, g, true, n_frames, frames, map_pixels,
                    depth, nullptr, center, radius, trunc, out, stream);
}

}  // extern "C"
