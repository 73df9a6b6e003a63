// postprocess.cu — fused caller-side post-process of render() (SURVEY §8(f) row f1, a "next" row).
//
// The reference turns the rasterizer's 7-channel allmap into its regulariser inputs with ~10 PyTorch
// kernels per direction (/root/reference/gaussian_renderer/__init__.py:118-147 and
// /root/reference/utils/point_utils.py:9-37): normal rotation to world space, expected depth =
// D/alpha with nan_to_num, median depth with nan_to_num, surf_depth = lerp(expected, median,
// depth_ratio), pseudo surface normal = normalize(cross of central differences of the back-projected
// depth points) * alpha.detach().  These are pure HBM-streaming stencils; here they are two kernels
// forward and two backward.  OPT-IN: the reference's render() keeps working unchanged on the plain op.
//
//   rays[0..8]  : row-major 3x3 M with ray_dir(x,y) = (x, y, 1) . M      (pixel -> world direction)
//   rays[9..11] : camera centre o;   point(x,y) = depth * ray_dir + o
//   rot[0..8]   : row-major 3x3 Rw with n_world = n_view . Rw             (= world_view[:3,:3]^T)
#include "common.cuh"
#include "kernels.h"
#include "profile.h"

namespace surfel {

// torch.nan_to_num(x, 0, 0): nan -> 0, +inf -> 0, -inf -> lowest finite float (neginf left at its default)
__device__ __forceinline__ float nan_to_zero(float v) {
    if (v != v) return 0.0f;
    if (v > 3.4028235e38f) return 0.0f;
    if (v < -3.4028235e38f) return -3.4028235e38f;
    return v;
}
__device__ __forceinline__ bool is_finite(float v) { return v == v && fabsf(v) <= 3.4028235e38f; }

// surf_depth = nan_to_num(D / alpha) * (1 - depth_ratio) + depth_ratio * nan_to_num(median), at pixel j
__device__ __forceinline__ float surf_depth_at(const float* __restrict__ allmap, int N, int j, float ratio) {
    const float med = nan_to_zero(allmap[5 * N + j]);
    const float ex = nan_to_zero(allmap[j] / allmap[N + j]);
    return ex * (1.0f - ratio) + ratio * med;
}

__global__ void post_fwd_depth_normal_kernel(int W, int H, float ratio, const float* __restrict__ allmap,
                                             const float* __restrict__ rot, float* __restrict__ rend_normal,
                                             float* __restrict__ surf_depth) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int N = W * H;
    if (i >= N) return;
    const float nx = allmap[2 * N + i], ny = allmap[3 * N + i], nz = allmap[4 * N + i];
    surf_depth[i] = surf_depth_at(allmap, N, i, ratio);
#pragma unroll
    for (int c = 0; c < 3; c++) rend_normal[c * N + i] = nx * rot[c] + ny * rot[3 + c] + nz * rot[6 + c];
}

struct P3 { float x, y, z; };
__device__ __forceinline__ P3 point_from(float d, const float* __restrict__ rays, int x, int y) {
    const float fx = (float)x, fy = (float)y;
    P3 p;
    p.x = d * (fx * rays[0] + fy * rays[3] + rays[6]) + rays[9];
    p.y = d * (fx * rays[1] + fy * rays[4] + rays[7]) + rays[10];
    p.z = d * (fx * rays[2] + fy * rays[5] + rays[8]) + rays[11];
    return p;
}
__device__ __forceinline__ P3 point_at(const float* __restrict__ depth, const float* __restrict__ rays, int W, int x, int y) {
    return point_from(depth[y * W + x], rays, x, y);
}

// surf_normal = normalize(cross(P[y+1,x]-P[y-1,x], P[y,x+1]-P[y,x-1])) * alpha ; zero on the border
__global__ void post_fwd_surf_normal_kernel(int W, int H, const float* __restrict__ allmap,
                                            const float* __restrict__ surf_depth, const float* __restrict__ rays,
                                            float* __restrict__ surf_normal) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    const int N = W * H, i = y * W + x;
    float n0 = 0, n1 = 0, n2 = 0;
    if (x > 0 && y > 0 && x < W - 1 && y < H - 1) {
        const P3 a = point_at(surf_depth, rays, W, x, y + 1), b = point_at(surf_depth, rays, W, x, y - 1);
        const P3 c = point_at(surf_depth, rays, W, x + 1, y), d = point_at(surf_depth, rays, W, x - 1, y);
        const float dx0 = a.x - b.x, dx1 = a.y - b.y, dx2 = a.z - b.z;
        const float dy0 = c.x - d.x, dy1 = c.y - d.y, dy2 = c.z - d.z;
        const float v0 = dx1 * dy2 - dx2 * dy1, v1 = dx2 * dy0 - dx0 * dy2, v2 = dx0 * dy1 - dx1 * dy0;
        const float inv = 1.0f / fmaxf(sqrtf(v0 * v0 + v1 * v1 + v2 * v2), 1e-12f);
        const float al = allmap[N + i];
        n0 = v0 * inv * al; n1 = v1 * inv * al; n2 = v2 * inv * al;
    }
    surf_normal[i] = n0; surf_normal[N + i] = n1; surf_normal[2 * N + i] = n2;
}

// vjp of normalize(v), v = dx x dy, for the normal's cotangent g (alpha already folded in): o = d(dx), d(dy)
__device__ __forceinline__ void normal_vjp(const float dx[3], const float dy[3], const float v[3], float len,
                                           const float g[3], float o[6]) {
    float dv[3];
    if (len > 1e-12f) {
        const float inv = 1.0f / len;
        const float n[3] = {v[0] * inv, v[1] * inv, v[2] * inv};
        const float ng = n[0] * g[0] + n[1] * g[1] + n[2] * g[2];
        for (int k = 0; k < 3; k++) dv[k] = (g[k] - n[k] * ng) * inv;
    } else {
        for (int k = 0; k < 3; k++) dv[k] = g[k] * 1e12f;  // v / eps branch of F.normalize
    }
    // v = dx x dy :  d(dx) = dy x dv ,  d(dy) = dv x dx
    o[0] = dy[1] * dv[2] - dy[2] * dv[1]; o[1] = dy[2] * dv[0] - dy[0] * dv[2]; o[2] = dy[0] * dv[1] - dy[1] * dv[0];
    o[3] = dv[1] * dx[2] - dv[2] * dx[1]; o[4] = dv[2] * dx[0] - dv[0] * dx[2]; o[5] = dv[0] * dx[1] - dv[1] * dx[0];
}

// backward 1: per interior pixel, vjp of the normal -> d(dx), d(dy) (6 planes in tmp; zero on the border)
__global__ void post_bwd_normal_vjp_kernel(int W, int H, const float* __restrict__ allmap,
                                           const float* __restrict__ surf_depth, const float* __restrict__ rays,
                                           const float* __restrict__ g_surf_normal, float* __restrict__ tmp) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    const int N = W * H, i = y * W + x;
    float o[6] = {0, 0, 0, 0, 0, 0};
    if (x > 0 && y > 0 && x < W - 1 && y < H - 1) {
        const P3 a = point_at(surf_depth, rays, W, x, y + 1), b = point_at(surf_depth, rays, W, x, y - 1);
        const P3 c = point_at(surf_depth, rays, W, x + 1, y), d = point_at(surf_depth, rays, W, x - 1, y);
        const float dx[3] = {a.x - b.x, a.y - b.y, a.z - b.z}, dy[3] = {c.x - d.x, c.y - d.y, c.z - d.z};
        const float v[3] = {dx[1] * dy[2] - dx[2] * dy[1], dx[2] * dy[0] - dx[0] * dy[2], dx[0] * dy[1] - dx[1] * dy[0]};
        const float len = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        const float al = allmap[N + i];                      // alpha is detached in the reference
        const float g[3] = {g_surf_normal[i] * al, g_surf_normal[N + i] * al, g_surf_normal[2 * N + i] * al};
        normal_vjp(dx, dy, v, len, g, o);
    }
#pragma unroll
    for (int k = 0; k < 6; k++) tmp[k * N + i] = o[k];
}

// gather the point gradients (tmp) of the 4 neighbours, chain them with g_depth (the cotangent of surf_depth) to
// depth and write allmap channels 0, 1 and 5
__device__ __forceinline__ void depth_chain(int W, int H, int x, int y, float ratio, const float* __restrict__ allmap,
                                            const float* __restrict__ rays, const float* __restrict__ tmp,
                                            float g_depth, float* __restrict__ g_allmap) {
    const int N = W * H, i = y * W + x;
    // P[y,x] is "P[y+1]" of pixel (y-1,x), "P[y-1]" of (y+1,x), "P[x+1]" of (y,x-1), "P[x-1]" of (y,x+1)
    float dP[3] = {0, 0, 0};
#pragma unroll
    for (int k = 0; k < 3; k++) {
        if (y > 0) dP[k] += tmp[k * N + i - W];
        if (y < H - 1) dP[k] -= tmp[k * N + i + W];
        if (x > 0) dP[k] += tmp[(3 + k) * N + i - 1];
        if (x < W - 1) dP[k] -= tmp[(3 + k) * N + i + 1];
    }
    const float fx = (float)x, fy = (float)y;
    const float r0 = fx * rays[0] + fy * rays[3] + rays[6], r1 = fx * rays[1] + fy * rays[4] + rays[7],
                r2 = fx * rays[2] + fy * rays[5] + rays[8];
    const float gd = dP[0] * r0 + dP[1] * r1 + dP[2] * r2 + g_depth;
    const float D = allmap[i], A = allmap[N + i], med = allmap[5 * N + i];
    const float ex = D / A;
    // nan_to_num passes no gradient where D/alpha is not finite (a hole, alpha == 0); there the chain rule's
    // 0 / alpha would be 0/0, so the fused backward writes 0 where the reference's autograd yields NaN
    const bool fin = is_finite(ex);
    const float g_ex = fin ? gd * (1.0f - ratio) : 0.0f;
    g_allmap[i] = fin ? g_ex / A : 0.0f;
    g_allmap[N + i] = fin ? -g_ex * D / (A * A) : 0.0f;
    g_allmap[5 * N + i] = is_finite(med) ? gd * ratio : 0.0f;
}

// backward 2: gather the point gradients of the 4 neighbours, chain to depth and to allmap
__global__ void post_bwd_allmap_kernel(int W, int H, float ratio, const float* __restrict__ allmap,
                                       const float* __restrict__ rays, const float* __restrict__ rot,
                                       const float* __restrict__ tmp, const float* __restrict__ g_rend_normal,
                                       const float* __restrict__ g_surf_depth, float* __restrict__ g_allmap) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    const int N = W * H, i = y * W + x;
    depth_chain(W, H, x, y, ratio, allmap, rays, tmp, g_surf_depth ? g_surf_depth[i] : 0.0f, g_allmap);
    g_allmap[6 * N + i] = 0.0f;
    float gn[3] = {0, 0, 0};
    if (g_rend_normal) { gn[0] = g_rend_normal[i]; gn[1] = g_rend_normal[N + i]; gn[2] = g_rend_normal[2 * N + i]; }
#pragma unroll
    for (int k = 0; k < 3; k++) g_allmap[(2 + k) * N + i] = gn[0] * rot[3 * k] + gn[1] * rot[3 * k + 1] + gn[2] * rot[3 * k + 2];
}

// ---- the regularisers of train.py (normal consistency and depth distortion), straight from allmap ----------------
//   normal_loss = lambda_normal * mean(1 - rend_normal . surf_normal),   dist_loss = lambda_dist * mean(rend_dist)
// Neither rend_normal, surf_depth, surf_normal nor a cotangent plane is written: each kernel recomputes the 3x3
// stencil it needs from allmap, and the backward's only scratch is the 6-plane point gradient of the §7b tail.

// dx = P[y+1,x] - P[y-1,x], dy = P[y,x+1] - P[y,x-1] at an interior pixel, the points back-projected from allmap
__device__ __forceinline__ void stencil_from_allmap(int W, int x, int y, float ratio, const float* __restrict__ allmap,
                                                    const float* __restrict__ rays, int N, float dx[3], float dy[3]) {
    const int i = y * W + x;
    const P3 a = point_from(surf_depth_at(allmap, N, i + W, ratio), rays, x, y + 1);
    const P3 b = point_from(surf_depth_at(allmap, N, i - W, ratio), rays, x, y - 1);
    const P3 c = point_from(surf_depth_at(allmap, N, i + 1, ratio), rays, x + 1, y);
    const P3 d = point_from(surf_depth_at(allmap, N, i - 1, ratio), rays, x - 1, y);
    dx[0] = a.x - b.x; dx[1] = a.y - b.y; dx[2] = a.z - b.z;
    dy[0] = c.x - d.x; dy[1] = c.y - d.y; dy[2] = c.z - d.z;
}

__device__ __forceinline__ void rend_normal_at(const float* __restrict__ allmap, const float* __restrict__ rot, int N,
                                               int i, float r[3]) {
    const float nx = allmap[2 * N + i], ny = allmap[3 * N + i], nz = allmap[4 * N + i];
#pragma unroll
    for (int c = 0; c < 3; c++) r[c] = nx * rot[c] + ny * rot[3 + c] + nz * rot[6 + c];
}

constexpr int kRegThreads = 256;    // the 32x8 block of the other stencil kernels

// forward: per pixel 1 - rend_normal . surf_normal and rend_dist, summed in double per block (fixed order: warp
// butterfly, then the 8 warps in turn); partials[2b], partials[2b+1] are block b's two sums
__global__ void __launch_bounds__(kRegThreads)
post_reg_fwd_kernel(int W, int H, float ratio, int with_normal, int with_dist, const float* __restrict__ allmap,
                    const float* __restrict__ rot, const float* __restrict__ rays, double* __restrict__ partials) {
    __shared__ double red[2][kRegThreads / 32];
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    const int tid = threadIdx.y * blockDim.x + threadIdx.x;
    double en = 0.0, ed = 0.0;
    if (x < W && y < H) {
        const int N = W * H, i = y * W + x;
        if (with_normal) {
            float sn[3] = {0, 0, 0}, r[3];
            if (x > 0 && y > 0 && x < W - 1 && y < H - 1) {
                float dx[3], dy[3];
                stencil_from_allmap(W, x, y, ratio, allmap, rays, N, dx, dy);
                const float v0 = dx[1] * dy[2] - dx[2] * dy[1], v1 = dx[2] * dy[0] - dx[0] * dy[2], v2 = dx[0] * dy[1] - dx[1] * dy[0];
                const float inv = 1.0f / fmaxf(sqrtf(v0 * v0 + v1 * v1 + v2 * v2), 1e-12f);
                const float al = allmap[N + i];
                sn[0] = v0 * inv * al; sn[1] = v1 * inv * al; sn[2] = v2 * inv * al;
            }
            rend_normal_at(allmap, rot, N, i, r);
            en = (double)(1.0f - (r[0] * sn[0] + r[1] * sn[1] + r[2] * sn[2]));
        }
        if (with_dist) ed = (double)allmap[6 * N + i];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { en += __shfl_xor_sync(0xffffffffu, en, o); ed += __shfl_xor_sync(0xffffffffu, ed, o); }
    if ((tid & 31) == 0) { red[0][tid >> 5] = en; red[1][tid >> 5] = ed; }
    __syncthreads();
    if (tid == 0) {
        double a = 0.0, b = 0.0;
        for (int w = 0; w < kRegThreads / 32; w++) { a += red[0][w]; b += red[1][w]; }
        const int blk = blockIdx.y * gridDim.x + blockIdx.x;
        partials[2 * blk] = a; partials[2 * blk + 1] = b;
    }
}

// one block: each thread sums a fixed stride of the partials in order, then a fixed tree; the values go out as
// float32, lambda * (sum / N) rounded once
__global__ void __launch_bounds__(kRegThreads)
post_reg_final_kernel(int nblocks, int N, double lambda_normal, double lambda_dist, const double* __restrict__ partials,
                      float* __restrict__ normal_loss, float* __restrict__ dist_loss) {
    __shared__ double sn[kRegThreads], sd[kRegThreads];
    const int t = threadIdx.x;
    double a = 0.0, b = 0.0;
    for (int j = t; j < nblocks; j += kRegThreads) { a += partials[2 * j]; b += partials[2 * j + 1]; }
    sn[t] = a; sd[t] = b;
    __syncthreads();
    for (int s = kRegThreads / 2; s > 0; s >>= 1) {
        if (t < s) { sn[t] += sn[t + s]; sd[t] += sd[t + s]; }
        __syncthreads();
    }
    if (t == 0) {
        *normal_loss = (float)(lambda_normal * (sn[0] / (double)N));
        *dist_loss = (float)(lambda_dist * (sd[0] / (double)N));
    }
}

// backward 1: the normal term's cotangents -s * surf_normal (to rend_normal, local: allmap channels 2-4) and
// -s * rend_normal (to surf_normal, through the stencil: the 6 point-gradient planes in tmp), s = gscale[0]
__global__ void post_reg_bwd_normal_kernel(int W, int H, float ratio, const float* __restrict__ allmap,
                                           const float* __restrict__ rot, const float* __restrict__ rays,
                                           const float* __restrict__ gscale, float* __restrict__ tmp,
                                           float* __restrict__ g_allmap) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    const int N = W * H, i = y * W + x;
    const float s = gscale[0];
    float o[6] = {0, 0, 0, 0, 0, 0}, sn[3] = {0, 0, 0}, r[3];
    rend_normal_at(allmap, rot, N, i, r);
    if (x > 0 && y > 0 && x < W - 1 && y < H - 1) {
        float dx[3], dy[3];
        stencil_from_allmap(W, x, y, ratio, allmap, rays, N, dx, dy);
        const float v[3] = {dx[1] * dy[2] - dx[2] * dy[1], dx[2] * dy[0] - dx[0] * dy[2], dx[0] * dy[1] - dx[1] * dy[0]};
        const float len = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        const float inv = 1.0f / fmaxf(len, 1e-12f);
        const float al = allmap[N + i];                      // alpha is detached in the reference
        sn[0] = v[0] * inv * al; sn[1] = v[1] * inv * al; sn[2] = v[2] * inv * al;
        const float g[3] = {-s * r[0] * al, -s * r[1] * al, -s * r[2] * al};
        normal_vjp(dx, dy, v, len, g, o);
    }
#pragma unroll
    for (int k = 0; k < 6; k++) tmp[k * N + i] = o[k];
    const float gn[3] = {-s * sn[0], -s * sn[1], -s * sn[2]};
#pragma unroll
    for (int k = 0; k < 3; k++) g_allmap[(2 + k) * N + i] = gn[0] * rot[3 * k] + gn[1] * rot[3 * k + 1] + gn[2] * rot[3 * k + 2];
}

// backward 2: channels 0, 1 and 5 through the stencil (tmp; all of 0-5 are 0 without the normal term, tmp NULL) and
// channel 6, the distortion term's constant gscale[1]
__global__ void post_reg_bwd_allmap_kernel(int W, int H, float ratio, const float* __restrict__ allmap,
                                           const float* __restrict__ rays, const float* __restrict__ tmp,
                                           const float* __restrict__ gscale, float* __restrict__ g_allmap) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    const int N = W * H, i = y * W + x;
    if (tmp) {
        depth_chain(W, H, x, y, ratio, allmap, rays, tmp, 0.0f, g_allmap);
    } else {
#pragma unroll
        for (int k = 0; k < 6; k++) g_allmap[k * N + i] = 0.0f;
    }
    g_allmap[6 * N + i] = gscale[1];
}

}  // namespace surfel

using namespace surfel;

// the kernels index the 7 planes of allmap with int, and the 32x8 grid's y extent is limited to 65535
static bool post_size_ok(int W, int H) {
    return W > 0 && H > 0 && 7LL * W * H <= 0x7fffffffLL && (H + 7) / 8 <= 65535;
}

extern "C" {

int surfel_post_forward(int W, int H, float depth_ratio, const float* allmap, const float* rot,
                        const float* rays, float* rend_normal, float* surf_depth, float* surf_normal,
                        void* stream) {
    if (!post_size_ok(W, H)) { surfel_set_error("surfel_post_forward: bad size"); return 1; }
    if (!allmap || !rot || !rays || !rend_normal || !surf_depth || !surf_normal) {
        surfel_set_error("surfel_post_forward: NULL required pointer"); return 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int N = W * H;
    prof_count_launch(); prof_count_launch();
    post_fwd_depth_normal_kernel<<<(N + 255) / 256, 256, 0, st>>>(W, H, depth_ratio, allmap, rot, rend_normal, surf_depth);
    SURFEL_CUDA_OK(cudaGetLastError());
    dim3 blk(32, 8), grd((W + 31) / 32, (H + 7) / 8);
    post_fwd_surf_normal_kernel<<<grd, blk, 0, st>>>(W, H, allmap, surf_depth, rays, surf_normal);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_post_backward(int W, int H, float depth_ratio, const float* allmap, const float* rot,
                         const float* rays, const float* surf_depth, const float* g_rend_normal,
                         const float* g_surf_depth, const float* g_surf_normal, float* tmp6,
                         float* g_allmap, void* stream) {
    if (!post_size_ok(W, H)) { surfel_set_error("surfel_post_backward: bad size"); return 1; }
    if (!allmap || !rot || !rays || !surf_depth || !tmp6 || !g_allmap) {
        surfel_set_error("surfel_post_backward: NULL required pointer"); return 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    dim3 blk(32, 8), grd((W + 31) / 32, (H + 7) / 8);
    prof_count_launch(); prof_count_launch();
    if (g_surf_normal) {
        post_bwd_normal_vjp_kernel<<<grd, blk, 0, st>>>(W, H, allmap, surf_depth, rays, g_surf_normal, tmp6);
    } else {
        SURFEL_CUDA_OK(cudaMemsetAsync(tmp6, 0, (size_t)6 * W * H * 4, st));
    }
    SURFEL_CUDA_OK(cudaGetLastError());
    post_bwd_allmap_kernel<<<grd, blk, 0, st>>>(W, H, depth_ratio, allmap, rays, rot, tmp6, g_rend_normal, g_surf_depth, g_allmap);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

size_t surfel_post_reg_partials_bytes(int W, int H) {
    if (!post_size_ok(W, H)) return 0;
    return (size_t)2 * sizeof(double) * ((W + 31) / 32) * ((H + 7) / 8);
}

int surfel_post_reg_forward(int W, int H, float depth_ratio, double lambda_normal, double lambda_dist,
                            const float* allmap, const float* rot, const float* rays, double* partials,
                            float* normal_loss, float* dist_loss, void* stream) {
    if (!post_size_ok(W, H)) { surfel_set_error("surfel_post_reg_forward: bad size"); return 1; }
    if (!allmap || !rot || !rays || !partials || !normal_loss || !dist_loss) {
        surfel_set_error("surfel_post_reg_forward: NULL required pointer"); return 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (lambda_normal == 0.0 && lambda_dist == 0.0) {        // both terms off: nothing reads allmap
        SURFEL_CUDA_OK(cudaMemsetAsync(normal_loss, 0, sizeof(float), st));
        SURFEL_CUDA_OK(cudaMemsetAsync(dist_loss, 0, sizeof(float), st));
        return 0;
    }
    dim3 blk(32, 8), grd((W + 31) / 32, (H + 7) / 8);
    prof_count_launch(); prof_count_launch();
    post_reg_fwd_kernel<<<grd, blk, 0, st>>>(W, H, depth_ratio, lambda_normal != 0.0, lambda_dist != 0.0, allmap, rot,
                                             rays, partials);
    SURFEL_CUDA_OK(cudaGetLastError());
    post_reg_final_kernel<<<1, kRegThreads, 0, st>>>(grd.x * grd.y, W * H, lambda_normal, lambda_dist, partials,
                                                     normal_loss, dist_loss);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_post_reg_backward(int W, int H, float depth_ratio, double lambda_normal, double lambda_dist,
                             const float* allmap, const float* rot, const float* rays, const float* gscale2,
                             float* tmp6, float* g_allmap, void* stream) {
    if (!post_size_ok(W, H)) { surfel_set_error("surfel_post_reg_backward: bad size"); return 1; }
    const bool with_normal = lambda_normal != 0.0;
    if (!allmap || !rot || !rays || !gscale2 || !g_allmap || (with_normal && !tmp6)) {
        surfel_set_error("surfel_post_reg_backward: NULL required pointer"); return 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (!with_normal && lambda_dist == 0.0) {                 // both terms off: nothing reads allmap
        SURFEL_CUDA_OK(cudaMemsetAsync(g_allmap, 0, (size_t)7 * W * H * sizeof(float), st));
        return 0;
    }
    dim3 blk(32, 8), grd((W + 31) / 32, (H + 7) / 8);
    if (with_normal) {
        prof_count_launch();
        post_reg_bwd_normal_kernel<<<grd, blk, 0, st>>>(W, H, depth_ratio, allmap, rot, rays, gscale2, tmp6, g_allmap);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    prof_count_launch();
    post_reg_bwd_allmap_kernel<<<grd, blk, 0, st>>>(W, H, depth_ratio, allmap, rays, with_normal ? tmp6 : nullptr,
                                                    gscale2, g_allmap);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
