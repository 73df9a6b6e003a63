// camera_bwd.cu — gradients of the camera: dL/dviewmatrix, dL/dprojmatrix and dL/dcampos (DESIGN §7p).
//
// Runs after surfel_backward on the same stream and workspaces, and reads what that call left behind: the
// 24-float gradient record (dL_dnormal, dL_dcolor), the full dL_dT after the AABB-centre fold (dL_dtransMat),
// the stored view-space normal of the render record (its sign is the forward's dual-visible flip) and the clamp
// bits.  preprocess backward itself is untouched.
//
// Per visible splat (row-vector matrices, pr = projmatrix, vm = viewmatrix, 16 contiguous floats each):
//   G_j[r] = gT[3j] L0[r] + gT[3j+1] L1[r] + gT[3j+2] p[r]  (r < 3),   G_j[3] = gT[3j+2]
//            L0 = mod s_u R[:,0], L1 = mod s_v R[:,1]  (the forward's T = [L0; L1; p 1] Pm_j, exact in the modifier)
//   V[r][c] = mult L2[r] gn[c]                               (the stored normal is mult L2 . vm[:3,:3])
//   C       = -(the SH view-direction term of dL_dmeans3D)   (the direction is means3D - campos)
// and the finish maps G to projmatrix through ndc2pix:
//   dpr[4r] = W/2 G_0[r],  dpr[4r+1] = H/2 G_1[r],  dpr[4r+3] = (W-1)/2 G_0[r] + (H-1)/2 G_1[r] + G_2[r],  dpr[4r+2] = 0.
// On the transMat_precomp path T and the normal do not depend on the camera: only C is formed.
//
// Tile-row bands (DESIGN §7r): every pixel belongs to one band, so a band's record holds partial sums and the rules
// above, linear in the record, give the band's share of the whole-frame gradient.  launch_camera_bwd_sums runs the
// same per-splat kernel and hands out the 35 double sums before the final rounding, so that a multi-GPU caller adds
// the bands in float64 and rounds once.
//
// Determinism: splat i belongs to block i / chunk for a chunk that depends on P alone; each thread adds its splats'
// float32 terms into double registers, the block reduces them in a fixed tree into one double partial per term, and
// one block adds the partials in block order and rounds each output once.  No atomics: repeat calls are
// bit-identical, on any stream and any device.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "profile.h"
#include "splat_math.cuh"

namespace surfel {

namespace {

constexpr int kCamTerms = 24;          // 12 G, 9 V, 3 C
constexpr int kCamThreads = 256;
constexpr int kCamMaxBlocks = 1024;

int cam_blocks(int P) { return P <= 0 ? 0 : std::min(kCamMaxBlocks, (P + kCamThreads - 1) / kCamThreads); }

}  // namespace

__global__ void __launch_bounds__(kCamThreads) camera_bwd_kernel(CamBwdParams p, int chunk) {
    double acc[kCamTerms];
#pragma unroll
    for (int k = 0; k < kCamTerms; k++) acc[k] = 0.0;
    const bool geom = p.transMat_precomp == nullptr;
    const bool has_sh = !p.has_colors_precomp && p.shs != nullptr;
    const int begin = blockIdx.x * chunk, end = min(p.P, begin + chunk);
    for (int idx = begin + threadIdx.x; idx < end; idx += kCamThreads) {
        if (p.radii[idx] <= 0) continue;
        float t[kCamTerms];
#pragma unroll
        for (int k = 0; k < kCamTerms; k++) t[k] = 0.0f;
        const float px = p.means3D[3 * (size_t)idx], py = p.means3D[3 * (size_t)idx + 1], pz = p.means3D[3 * (size_t)idx + 2];
        const float4 rg = reinterpret_cast<const float4*>(p.grad_rec + (size_t)idx * kGradFloats)[4];   // gn, gc.x
        const float2 rg2 = reinterpret_cast<const float2*>(p.grad_rec + (size_t)idx * kGradFloats)[10];  // gc.yz
        if (geom) {
            // rsqrtf rounds once; preprocess's 1/sqrtf rounds twice, and where |q|^2 rounds to 1 - 2^-24 that alone moves
            // a diagonal entry of R near 0.15 by 1.3e-6 of its value, beyond the bound of DESIGN §7p's exact test
            const float4 q = reinterpret_cast<const float4*>(p.rotations)[idx];
            const QuatRotation qr = quat_rotation(q, rsqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w));
            const float (&R)[3][3] = qr.R;
            const float2 sc = reinterpret_cast<const float2*>(p.scales)[idx];
            const float su = p.scale_modifier * sc.x, sv = p.scale_modifier * sc.y;
            const float L0[3] = {R[0][0] * su, R[1][0] * su, R[2][0] * su};
            const float L1[3] = {R[0][1] * sv, R[1][1] * sv, R[2][1] * sv};
            const float L2[3] = {R[0][2], R[1][2], R[2][2]};
            const float pp[3] = {px, py, pz};
            const float* gT = p.dL_dtransMat + 9 * (size_t)idx;
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const float a = gT[3 * j], b = gT[3 * j + 1], c = gT[3 * j + 2];
#pragma unroll
                for (int r = 0; r < 3; r++) t[4 * j + r] = a * L0[r] + b * L1[r] + c * pp[r];
                t[4 * j + 3] = c;
            }
            // the forward stored mult * (L2 . vm[:3,:3]); its sign against the recomputed normal is mult
            const float4 n = p.rec[(size_t)idx * kRecQuads + 3];
            const float* vm = p.viewmatrix;
            const float nv0 = vm[0] * L2[0] + vm[4] * L2[1] + vm[8] * L2[2];
            const float nv1 = vm[1] * L2[0] + vm[5] * L2[1] + vm[9] * L2[2];
            const float nv2 = vm[2] * L2[0] + vm[6] * L2[1] + vm[10] * L2[2];
            const float mult = n.x * nv0 + n.y * nv1 + n.z * nv2 > 0.0f ? 1.0f : -1.0f;
            const float gn[3] = {rg.x, rg.y, rg.z};
#pragma unroll
            for (int r = 0; r < 3; r++) {
                const float m = mult * L2[r];
#pragma unroll
                for (int c = 0; c < 3; c++) t[12 + 3 * r + c] = m * gn[c];
            }
        }
        if (has_sh) {
            const uint8_t cb = p.clamped[idx];
            const float dR[3] = {(cb & 1) ? 0.0f : rg.w, (cb & 2) ? 0.0f : rg2.x, (cb & 4) ? 0.0f : rg2.y};
            if (p.D > 0 && (dR[0] != 0.0f || dR[1] != 0.0f || dR[2] != 0.0f)) {
                // the direction is means3D - campos: minus preprocess backward's SH term of dL_dmeans3D
                const float* sh = p.shs + (size_t)idx * 3 * p.M;
                const float dox = px - p.campos[0], doy = py - p.campos[1], doz = pz - p.campos[2];
                const float invl = 1.0f / sqrtf(dox * dox + doy * doy + doz * doz);
                const float3 dd = sh_backward(p.D, dox * invl, doy * invl, doz * invl, dR,
                                              [&](int i, int c) { return __ldg(sh + 3 * i + c); }, [](int, float) {});
                const float3 g = sh_direction_to_mean(dox, doy, doz, invl, dd);
                t[21] = -g.x; t[22] = -g.y; t[23] = -g.z;
            }
        }
#pragma unroll
        for (int k = 0; k < kCamTerms; k++) acc[k] += (double)t[k];
    }

    block_sum<kCamTerms, kCamThreads>(acc, threadIdx.x,
                                      [&](int k, double v) { p.partials[(size_t)blockIdx.x * kCamTerms + k] = v; });
}

// the block partials added in block order; projmatrix through ndc2pix.  Out is float (each output rounded once) or
// double (the sums before rounding, for a caller that adds several tile-row bands first)
template <typename Out>
__device__ __forceinline__ void camera_finish(int nblocks, int W, int H, const double* __restrict__ partials,
                                              Out* __restrict__ dvm, Out* __restrict__ dpr, Out* __restrict__ dcam) {
    __shared__ double s[kCamTerms];
    const int k = threadIdx.x;
    if (k < kCamTerms) {
        double a = 0.0;
        for (int b = 0; b < nblocks; b++) a += partials[(size_t)b * kCamTerms + k];
        s[k] = a;
    }
    __syncthreads();
    if (k < 16) {
        const int r = k >> 2, c = k & 3;
        const double G0 = s[r], G1 = s[4 + r], G2 = s[8 + r];
        double v;
        if (c == 0) v = 0.5 * W * G0;
        else if (c == 1) v = 0.5 * H * G1;
        else if (c == 2) v = 0.0;
        else v = 0.5 * (W - 1) * G0 + 0.5 * (H - 1) * G1 + G2;
        dpr[k] = (Out)v;
        dvm[k] = (r < 3 && c < 3) ? (Out)s[12 + 3 * r + c] : (Out)0;
    } else if (k < 19) {
        dcam[k - 16] = (Out)s[21 + k - 16];
    }
}

__global__ void camera_finish_kernel(int nblocks, int W, int H, const double* __restrict__ partials,
                                     float* __restrict__ dvm, float* __restrict__ dpr, float* __restrict__ dcam) {
    camera_finish<float>(nblocks, W, H, partials, dvm, dpr, dcam);
}

__global__ void camera_sums_finish_kernel(int nblocks, int W, int H, const double* __restrict__ partials,
                                          double* __restrict__ dvm, double* __restrict__ dpr, double* __restrict__ dcam) {
    camera_finish<double>(nblocks, W, H, partials, dvm, dpr, dcam);
}

size_t camera_partials_bytes(int P) { return (size_t)std::max(1, cam_blocks(P)) * kCamTerms * sizeof(double); }

namespace {

// the per-splat kernel into p.partials; returns the number of partials (blocks) it wrote
int launch_camera_partials(const CamBwdParams& p, cudaStream_t stream) {
    const int nb = cam_blocks(p.P);
    if (nb > 0) {
        const int chunk = (p.P + nb - 1) / nb;
        LaunchScope scope(kStCameraBwd, stream);
        camera_bwd_kernel<<<nb, kCamThreads, 0, stream>>>(p, chunk);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return nb;
}

}  // namespace

int launch_camera_bwd(const CamBwdParams& p, cudaStream_t stream) {
    const int nb = launch_camera_partials(p, stream);
    {
        LaunchScope scope(kStCameraFinish, stream);
        camera_finish_kernel<<<1, 32, 0, stream>>>(nb, p.W, p.H, p.partials, p.dL_dviewmatrix, p.dL_dprojmatrix, p.dL_dcampos);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

int launch_camera_bwd_sums(const CamBwdParams& p, double* dvm, double* dpr, double* dcam, cudaStream_t stream) {
    const int nb = launch_camera_partials(p, stream);
    {
        LaunchScope scope(kStCameraFinish, stream);
        camera_sums_finish_kernel<<<1, 32, 0, stream>>>(nb, p.W, p.H, p.partials, dvm, dpr, dcam);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

}  // namespace surfel
