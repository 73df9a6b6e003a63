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

__global__ void post_fwd_depth_normal_kernel(int W, int H, float ratio, const float* __restrict__ allmap,
                                             const float* __restrict__ rot, float* __restrict__ rend_normal,
                                             float* __restrict__ surf_depth) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int N = W * H;
    if (i >= N) return;
    const float D = allmap[i], A = allmap[N + i];
    const float nx = allmap[2 * N + i], ny = allmap[3 * N + i], nz = allmap[4 * N + i];
    const float med = nan_to_zero(allmap[5 * N + i]);
    const float ex = nan_to_zero(D / A);
    surf_depth[i] = ex * (1.0f - ratio) + ratio * med;
#pragma unroll
    for (int c = 0; c < 3; c++) rend_normal[c * N + i] = nx * rot[c] + ny * rot[3 + c] + nz * rot[6 + c];
}

struct P3 { float x, y, z; };
__device__ __forceinline__ P3 point_at(const float* __restrict__ depth, const float* __restrict__ rays, int W, int x, int y) {
    const float d = depth[y * W + x], fx = (float)x, fy = (float)y;
    P3 p;
    p.x = d * (fx * rays[0] + fy * rays[3] + rays[6]) + rays[9];
    p.y = d * (fx * rays[1] + fy * rays[4] + rays[7]) + rays[10];
    p.z = d * (fx * rays[2] + fy * rays[5] + rays[8]) + rays[11];
    return p;
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
#pragma unroll
    for (int k = 0; k < 6; k++) tmp[k * N + i] = o[k];
}

// backward 2: gather the point gradients of the 4 neighbours, chain to depth and to allmap
__global__ void post_bwd_allmap_kernel(int W, int H, float ratio, const float* __restrict__ allmap,
                                       const float* __restrict__ rays, const float* __restrict__ rot,
                                       const float* __restrict__ tmp, const float* __restrict__ g_rend_normal,
                                       const float* __restrict__ g_surf_depth, float* __restrict__ g_allmap) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
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
    const float gd = dP[0] * r0 + dP[1] * r1 + dP[2] * r2 + (g_surf_depth ? g_surf_depth[i] : 0.0f);
    const float D = allmap[i], A = allmap[N + i], med = allmap[5 * N + i];
    const float ex = D / A;
    // nan_to_num passes no gradient where D/alpha is not finite (a hole, alpha == 0); there the chain rule's
    // 0 / alpha would be 0/0, so the fused backward writes 0 where the reference's autograd yields NaN
    const bool fin = is_finite(ex);
    const float g_ex = fin ? gd * (1.0f - ratio) : 0.0f;
    g_allmap[i] = fin ? g_ex / A : 0.0f;
    g_allmap[N + i] = fin ? -g_ex * D / (A * A) : 0.0f;
    g_allmap[5 * N + i] = is_finite(med) ? gd * ratio : 0.0f;
    g_allmap[6 * N + i] = 0.0f;
    float gn[3] = {0, 0, 0};
    if (g_rend_normal) { gn[0] = g_rend_normal[i]; gn[1] = g_rend_normal[N + i]; gn[2] = g_rend_normal[2 * N + i]; }
#pragma unroll
    for (int k = 0; k < 3; k++) g_allmap[(2 + k) * N + i] = gn[0] * rot[3 * k] + gn[1] * rot[3 * k + 1] + gn[2] * rot[3 * k + 2];
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

}  // extern "C"
