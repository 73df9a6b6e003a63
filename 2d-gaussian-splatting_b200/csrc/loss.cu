// loss.cu — fused photometric loss (SURVEY §8(f) row f2):  (1-l)*L1(img,gt) + l*(1 - SSIM(img,gt)).
//
// Restates /root/reference/utils/loss_utils.py:6-7 (l1_loss) and :43-73 (ssim: 11x11 Gaussian window,
// sigma 1.5, zero padding 5, per-channel, C1 = 0.01^2, C2 = 0.03^2, mean over all pixels) as used at
// /root/reference/train.py:73-74.  The reference runs 5 grouped conv2d + ~15 elementwise kernels forward
// and their autograd backward; here the forward is ONE kernel (separable convolution of the five moment
// images in shared memory, SSIM map, L1, block reduction, and the three partial-derivative maps the
// backward needs) and the backward is ONE kernel (separable convolution of those three maps).
#include "common.cuh"
#include "kernels.h"
#include "profile.h"

namespace surfel {

constexpr int kWin = 11, kHalfW = 5, kLT = 16, kHaloW = kLT + 2 * kHalfW;   // 26
__constant__ float c_gauss[kWin];

__global__ void __launch_bounds__(256)
l1_ssim_fwd_kernel(int C, int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                   float* __restrict__ dmu1, float* __restrict__ ds11, float* __restrict__ ds12,
                   double* __restrict__ sums /* [0]=sum |x-y|, [1]=sum ssim */) {
    __shared__ float sx[kHaloW][kHaloW + 1], sy[kHaloW][kHaloW + 1];
    __shared__ float hz[5][kHaloW][kLT + 1];
    __shared__ double red[2][8];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kLT + tx;
    const int x0 = blockIdx.x * kLT, y0 = blockIdx.y * kLT, c = blockIdx.z;
    const float* X = img + (size_t)c * H * W;
    const float* Y = gt + (size_t)c * H * W;
    for (int i = tid; i < kHaloW * kHaloW; i += 256) {
        const int ly = i / kHaloW, lx = i - ly * kHaloW;
        const int gx = x0 + lx - kHalfW, gy = y0 + ly - kHalfW;
        const bool in = gx >= 0 && gx < W && gy >= 0 && gy < H;
        sx[ly][lx] = in ? X[(size_t)gy * W + gx] : 0.0f;
        sy[ly][lx] = in ? Y[(size_t)gy * W + gx] : 0.0f;
    }
    __syncthreads();
    for (int i = tid; i < kHaloW * kLT; i += 256) {          // horizontal pass
        const int ly = i / kLT, lx = i - ly * kLT;
        float a = 0, b = 0, aa = 0, bb = 0, ab = 0;
#pragma unroll
        for (int k = 0; k < kWin; k++) {
            const float g = c_gauss[k], u = sx[ly][lx + k], v = sy[ly][lx + k];
            a += g * u; b += g * v; aa += g * u * u; bb += g * v * v; ab += g * u * v;
        }
        hz[0][ly][lx] = a; hz[1][ly][lx] = b; hz[2][ly][lx] = aa; hz[3][ly][lx] = bb; hz[4][ly][lx] = ab;
    }
    __syncthreads();
    float mu1 = 0, mu2 = 0, s11 = 0, s22 = 0, s12 = 0;
#pragma unroll
    for (int k = 0; k < kWin; k++) {                         // vertical pass
        const float g = c_gauss[k];
        mu1 += g * hz[0][ty + k][tx]; mu2 += g * hz[1][ty + k][tx];
        s11 += g * hz[2][ty + k][tx]; s22 += g * hz[3][ty + k][tx]; s12 += g * hz[4][ty + k][tx];
    }
    const int gx = x0 + tx, gy = y0 + ty;
    double l1 = 0.0, ss = 0.0;
    if (gx < W && gy < H) {
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        const float mu1s = mu1 * mu1, mu2s = mu2 * mu2, m12 = mu1 * mu2;
        const float sg1 = s11 - mu1s, sg2 = s22 - mu2s, sg12 = s12 - m12;
        const float A = 2.0f * m12 + C1, B = 2.0f * sg12 + C2, Cc = mu1s + mu2s + C1, Dd = sg1 + sg2 + C2;
        const float inv = 1.0f / (Cc * Dd);
        const float f = A * B * inv;
        const size_t o = (size_t)c * H * W + (size_t)gy * W + gx;
        // partial derivatives of f w.r.t. the window moments of img (mu1, E[x^2], E[xy])
        dmu1[o] = ((2.0f * mu2 * (B - A)) * Cc * Dd - A * B * (2.0f * mu1 * (Dd - Cc))) * inv * inv;
        ds11[o] = -A * B * inv / Dd;
        ds12[o] = 2.0f * A * inv;
        ss = (double)f;
        l1 = (double)fabsf(sx[ty + kHalfW][tx + kHalfW] - sy[ty + kHalfW][tx + kHalfW]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { l1 += __shfl_xor_sync(0xffffffffu, l1, o); ss += __shfl_xor_sync(0xffffffffu, ss, o); }
    if ((tid & 31) == 0) { red[0][tid >> 5] = l1; red[1][tid >> 5] = ss; }
    __syncthreads();
    if (tid == 0) {
        double a = 0, b = 0;
        for (int w = 0; w < 8; w++) { a += red[0][w]; b += red[1][w]; }
        atomicAdd(sums, a); atomicAdd(sums + 1, b);
    }
}

// dL/dimg = gl1 * sign(x-y) + gss * [ conv(dmu1) + 2x*conv(ds11) + y*conv(ds12) ]
__global__ void __launch_bounds__(256)
l1_ssim_bwd_kernel(int C, int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                   const float* __restrict__ dmu1, const float* __restrict__ ds11, const float* __restrict__ ds12,
                   const float* __restrict__ gscale /* [0]=dL/d(sum l1), [1]=dL/d(sum ssim) */,
                   float* __restrict__ g_img) {
    __shared__ float sm[3][kHaloW][kHaloW + 1];
    __shared__ float hz[3][kHaloW][kLT + 1];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kLT + tx;
    const int x0 = blockIdx.x * kLT, y0 = blockIdx.y * kLT, c = blockIdx.z;
    const size_t plane = (size_t)c * H * W;
    for (int i = tid; i < kHaloW * kHaloW; i += 256) {
        const int ly = i / kHaloW, lx = i - ly * kHaloW;
        const int gx = x0 + lx - kHalfW, gy = y0 + ly - kHalfW;
        const bool in = gx >= 0 && gx < W && gy >= 0 && gy < H;
        const size_t o = plane + (size_t)gy * W + gx;
        sm[0][ly][lx] = in ? dmu1[o] : 0.0f;
        sm[1][ly][lx] = in ? ds11[o] : 0.0f;
        sm[2][ly][lx] = in ? ds12[o] : 0.0f;
    }
    __syncthreads();
    for (int i = tid; i < kHaloW * kLT; i += 256) {
        const int ly = i / kLT, lx = i - ly * kLT;
        float a = 0, b = 0, d = 0;
#pragma unroll
        for (int k = 0; k < kWin; k++) {
            const float g = c_gauss[k];
            a += g * sm[0][ly][lx + k]; b += g * sm[1][ly][lx + k]; d += g * sm[2][ly][lx + k];
        }
        hz[0][ly][lx] = a; hz[1][ly][lx] = b; hz[2][ly][lx] = d;
    }
    __syncthreads();
    float a = 0, b = 0, d = 0;
#pragma unroll
    for (int k = 0; k < kWin; k++) {
        const float g = c_gauss[k];
        a += g * hz[0][ty + k][tx]; b += g * hz[1][ty + k][tx]; d += g * hz[2][ty + k][tx];
    }
    const int gx = x0 + tx, gy = y0 + ty;
    if (gx < W && gy < H) {
        const size_t o = plane + (size_t)gy * W + gx;
        const float x = img[o], y = gt[o];
        const float df = x - y;
        const float sgn = df > 0.0f ? 1.0f : (df < 0.0f ? -1.0f : 0.0f);
        g_img[o] = gscale[0] * sgn + gscale[1] * (a + 2.0f * x * b + y * d);
    }
}

}  // namespace surfel

using namespace surfel;

// one block per 16x16 tile per channel: grid y and z are limited to 65535
static bool loss_shape_ok(int C, int H, int W) {
    return C > 0 && H > 0 && W > 0 && C <= 65535 && (H + kLT - 1) / kLT <= 65535;
}

extern "C" {

int surfel_l1_ssim_forward(int C, int H, int W, const float* img, const float* gt, float* dmu1,
                           float* ds11, float* ds12, double* sums2, void* stream) {
    if (!loss_shape_ok(C, H, W)) { surfel_set_error("surfel_l1_ssim_forward: bad shape"); return 1; }
    if (!img || !gt || !dmu1 || !ds11 || !ds12 || !sums2) {
        surfel_set_error("surfel_l1_ssim_forward: NULL required pointer"); return 1;
    }
    cudaStream_t st = (cudaStream_t)stream;
    static bool init[kMaxDevices] = {};                 // the window lives in __constant__ memory: one copy per device
    const int slot = current_device_slot();
    if (slot < 0 || !init[slot]) {
        // same construction as the reference: exp(-(x-5)^2 / (2*1.5^2)) as float32, normalised in float32
        float g[kWin], s = 0.0f;
        for (int i = 0; i < kWin; i++) { g[i] = (float)exp(-(double)((i - kHalfW) * (i - kHalfW)) / (2.0 * 1.5 * 1.5)); s += g[i]; }
        for (int i = 0; i < kWin; i++) g[i] /= s;
        SURFEL_CUDA_OK(cudaMemcpyToSymbol(c_gauss, g, sizeof(g)));
        if (slot >= 0) init[slot] = true;
    }
    SURFEL_CUDA_OK(cudaMemsetAsync(sums2, 0, 2 * sizeof(double), st));
    dim3 grid((W + kLT - 1) / kLT, (H + kLT - 1) / kLT, C), blk(kLT, kLT);
    prof_count_launch();
    l1_ssim_fwd_kernel<<<grid, blk, 0, st>>>(C, H, W, img, gt, dmu1, ds11, ds12, sums2);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_l1_ssim_backward(int C, int H, int W, const float* img, const float* gt, const float* dmu1,
                            const float* ds11, const float* ds12, const float* gscale2, float* g_img,
                            void* stream) {
    if (!loss_shape_ok(C, H, W)) { surfel_set_error("surfel_l1_ssim_backward: bad shape"); return 1; }
    if (!img || !gt || !dmu1 || !ds11 || !ds12 || !gscale2 || !g_img) {
        surfel_set_error("surfel_l1_ssim_backward: NULL required pointer"); return 1;
    }
    dim3 grid((W + kLT - 1) / kLT, (H + kLT - 1) / kLT, C), blk(kLT, kLT);
    prof_count_launch();
    l1_ssim_bwd_kernel<<<grid, blk, 0, (cudaStream_t)stream>>>(C, H, W, img, gt, dmu1, ds11, ds12, gscale2, g_img);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
