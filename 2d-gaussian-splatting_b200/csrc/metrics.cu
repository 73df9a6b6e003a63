// metrics.cu — the per-view novel-view metrics of the reference's metrics.py on the device: PSNR
// (utils/image_utils.py), and LPIPS with the VGG-16 trunk (lpipsPyTorch).  SSIM reuses the fused loss of loss.cu.
// DESIGN.md §7o has the rules; tests/metrics_ref.py restates them in float64.
//
//  * surfel_metrics_lpips_input: z-scores render and gt ((x - mean) / std, two correctly rounded float32 operations,
//    as the reference's broadcast tensors compute them) into one NHWC batch of two images.
//  * surfel_metrics_pack_conv: [Cout][Cin][3][3] -> [Cout][ky][kx][Cin], the K-major layout the tensor cores read.
//    Layers that run on the tensor cores (Cin a multiple of 32) have their weights rounded to TF32 here, once, to
//    nearest with ties away (cvt.rna.tf32.f32); conv1_1 (Cin = 3) keeps float32 weights.
//  * surfel_metrics_conv3x3: 3x3 convolution, padding 1, + bias, ReLU, over NHWC float32.
//     - Cin = 3 (conv1_1, ~0.5 % of the FLOPs): plain float32 FMA, one thread per output pixel.
//     - Cin % 32 == 0: implicit GEMM on wgmma.mma_async TF32 with float32 accumulation.  M = output pixels of both
//       images, N = Cout, K = 9 Cin, ordered (ky, kx, ci) so a K tile of 32 is one tap's 32 channels: 128
//       contiguous bytes of one NHWC pixel.  One warpgroup owns a 128 x BN tile (two m64 halves per k8 step).
//       Operands sit in a ring of kStages shared-memory stages in the 128-byte swizzled K-major layout; they are
//       fed by cp.async (16 bytes a copy, zero-filled outside the image) kStages - 2 tiles ahead, and each stage is
//       guarded by an mbarrier every thread arrives on once its own copies have landed (and rounded).  Each thread
//       rounds the activations it staged to TF32, to nearest with ties away, before it arrives: the tensor core
//       alone would read the top 19 bits (truncation), a bias toward zero that 13 layers compound.  Both operands
//       are thus TF32 rounded to nearest.  Bias and ReLU run in the epilogue.
//  * surfel_metrics_maxpool: 2 x 2, stride 2, floor (odd sides drop the last row / column).  Exact.
//  * surfel_metrics_lpips_tap: per pixel, the channel norms of both images, f / (sqrt(sum f^2) + 1e-10), the
//    squared difference and its dot product with the lin weights; summed in double per block over a fixed
//    pixel-to-block assignment.  surfel_metrics_lpips_finish sums the blocks in order, so repeat calls agree bit
//    for bit.
//  * surfel_metrics_psnr: sum (a - b)^2 per image in double (the difference and the square of two float32 values
//    are exact in double), in a fixed order, then 20 log10(1 / sqrt(mse)) once in double, rounded to float32.
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/surfel_rasterizer.h"
#include "common.cuh"
#include "kernels.h"
#include "profile.h"

namespace surfel {
namespace {

constexpr int kMinSide = 16;                 // four floor pools before conv5 leave a side of at least 1
constexpr int kMaxSide = 16384;              // 2 H W pixel indices stay below 2^31
constexpr int kRedBlocks = 256;              // fixed blocks of every deterministic reduction
constexpr int kRedThreads = 256;
constexpr int kTaps = 5;

constexpr int kBM = 128, kBK = 32, kStages = 6, kConvThreads = 128;
constexpr int kRowBytes = kBK * 4;           // one swizzle row: 32 float32 of K

__host__ __device__ constexpr int stage_bytes(int bn) { return (kBM + bn) * kRowBytes; }
__host__ __device__ constexpr int conv_smem_bytes(int bn) { return kStages * stage_bytes(bn) + 1024 + 64; }

// ---- PTX helpers ----

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.shared::cta.b64 st, [%0];\n}\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n.reg .pred done;\nWAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 done, [%0], %1;\n"
        "@!done bra WAIT_%=;\n}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }

// Shared-memory matrix descriptor of a K-major operand in the 128-byte swizzle: rows of 128 bytes, 8-row atoms of
// 1024 bytes (the stride byte offset), atoms 1024-byte aligned.  The leading byte offset is unused in this mode.
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr) {
    return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) |
           ((uint64_t)1 << 62);
}

// D (64 x N, float32 fragments) += A (64 x 8, desc) * B (N x 8, desc)^T, TF32 operands, both K-major
__device__ __forceinline__ void wgmma_m64n64k8(float* d, uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_m64n128k8(float* d, uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t da, uint64_t db) {
    if constexpr (BN == 128) wgmma_m64n128k8(d, da, db, 1);
    else wgmma_m64n64k8(d, da, db, 1);
}

__device__ __forceinline__ float to_tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// ---- input stage ----

struct ZParams { float mean[3], std[3]; };

__global__ void __launch_bounds__(256) mt_zscore_kernel(long long hw, const float* __restrict__ x,
                                                        const float* __restrict__ y, ZParams z,
                                                        float* __restrict__ out) {
    const long long n = 2 * hw * 3;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % 3);
        const long long p = i / 3, b = p / hw, q = p - b * hw;
        const float v = (b == 0 ? x : y)[c * hw + q];
        out[i] = __fdiv_rn(__fsub_rn(v, z.mean[c]), z.std[c]);
    }
}

__global__ void __launch_bounds__(256) mt_pack_kernel(int cout, int cin, bool tf32, const float* __restrict__ w,
                                                      float* __restrict__ packed) {
    const long long n = (long long)cout * cin * 9;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int ci = (int)(i % cin);
        const long long r = i / cin;
        const int tap = (int)(r % 9), co = (int)(r / 9);
        const float v = w[((long long)co * cin + ci) * 9 + tap];
        packed[i] = tf32 ? to_tf32_rna(v) : v;
    }
}

// ---- conv1_1: Cin = 3, float32 ----

__global__ void __launch_bounds__(128) mt_conv_c3_kernel(int n_img, int H, int W, const float* __restrict__ in,
                                                         const float* __restrict__ wp /* [64][9][3] */,
                                                         const float* __restrict__ bias, float* __restrict__ out) {
    __shared__ float sw[64 * 27], sb[64];
    for (int i = threadIdx.x; i < 64 * 27; i += blockDim.x) sw[i] = wp[i];
    for (int i = threadIdx.x; i < 64; i += blockDim.x) sb[i] = bias[i];
    __syncthreads();
    const long long M = (long long)n_img * H * W;
    const long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (p >= M) return;
    const int hw = H * W, b = (int)(p / hw), q = (int)(p - (long long)b * hw), oy = q / W, ox = q - oy * W;
    float v[27];
#pragma unroll
    for (int t = 0; t < 9; t++) {
        const int iy = oy + t / 3 - 1, ix = ox + t % 3 - 1;
        const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
        const float* s = in + ((long long)b * hw + (long long)iy * W + ix) * 3;
#pragma unroll
        for (int c = 0; c < 3; c++) v[t * 3 + c] = ok ? s[c] : 0.0f;
    }
    float4* o = (float4*)(out + p * 64);
#pragma unroll 4
    for (int g = 0; g < 16; g++) {
        float a[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const float* wr = sw + (g * 4 + j) * 27;
            float acc = 0.0f;
#pragma unroll
            for (int k = 0; k < 27; k++) acc = fmaf(wr[k], v[k], acc);
            a[j] = fmaxf(acc + sb[g * 4 + j], 0.0f);
        }
        o[g] = make_float4(a[0], a[1], a[2], a[3]);
    }
}

// ---- Cin % 32 == 0: implicit GEMM on wgmma TF32 ----

template <int BN>
__global__ void __launch_bounds__(kConvThreads, 1)
mt_conv_wgmma_kernel(int n_img, int H, int W, int cin, int cout, const float* __restrict__ in,
                     const float* __restrict__ wp /* [cout][9][cin] */, const float* __restrict__ bias,
                     float* __restrict__ out) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* full = (uint64_t*)(smem + kStages * stage_bytes(BN));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int hw = H * W, M = n_img * hw;
    const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
    const int kc = cin / kBK, KT = 9 * kc;
    if (tid == 0) {
        for (int s = 0; s < kStages; s++) mbar_init(full + s, kConvThreads);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    // the rows this thread stages: r = (tid >> 3) + 16 i, chunk tid & 7 (16 bytes) of each
    const int chunk = tid & 7, swz = ((chunk ^ ((tid >> 3) & 7)) << 4);
    int rq[8], ryx[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int m = m0 + (tid >> 3) + 16 * i;
        if (m < M) {
            const int b = m / hw, q = m - b * hw, oy = q / W, ox = q - oy * W;
            rq[i] = m;
            ryx[i] = (oy << 16) | ox;
        } else {
            rq[i] = -1;
            ryx[i] = 0;
        }
    }
    const uint32_t s_base = smem_u32(smem);
    auto load_tile = [&](int slot, int kt) {
        const int tap = kt / kc, c0 = (kt - tap * kc) * kBK, dy = tap / 3 - 1, dx = tap % 3 - 1;
        const uint32_t sa = s_base + slot * stage_bytes(BN), sb = sa + kBM * kRowBytes;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int oy = ryx[i] >> 16, ox = ryx[i] & 0xffff, iy = oy + dy, ix = ox + dx;
            const bool ok = rq[i] >= 0 && iy >= 0 && iy < H && ix >= 0 && ix < W;
            const float* src = ok ? in + (size_t)(rq[i] + dy * W + dx) * cin + c0 + chunk * 4 : in;
            cp_async16(sa + ((tid >> 3) + 16 * i) * kRowBytes + swz, src, ok);
        }
#pragma unroll
        for (int i = 0; i < BN / 16; i++) {
            const int n = (tid >> 3) + 16 * i;
            const float* src = wp + ((size_t)(n0 + n) * 9 + tap) * cin + c0 + chunk * 4;
            cp_async16(sb + n * kRowBytes + swz, src, true);
        }
    };
    __syncthreads();                                   // barriers initialised

    float acc[2][BN / 2];
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
        for (int j = 0; j < BN / 2; j++) acc[h][j] = 0.0f;

#pragma unroll
    for (int s = 0; s < kStages - 2; s++) {
        if (s < KT) load_tile(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < KT; kt++) {
        const int slot = kt % kStages;
        cp_async_wait<kStages - 3>();                  // this thread's copies of tile kt have landed
        {
            // round this thread's activation chunks to TF32 in place, to nearest: truncation would bias every
            // layer's output low, and 13 layers compound it
            const uint32_t sa = s_base + slot * stage_bytes(BN);
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const uint32_t a = sa + ((tid >> 3) + 16 * i) * kRowBytes + swz;
                float4 v;
                asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];\n"
                             : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
                asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"r"(a), "f"(to_tf32_rna(v.x)),
                             "f"(to_tf32_rna(v.y)), "f"(to_tf32_rna(v.z)), "f"(to_tf32_rna(v.w)) : "memory");
            }
        }
        fence_proxy_async();                           // ... and are visible to the tensor core's async proxy
        mbar_arrive(full + slot);
        mbar_wait(full + slot, (uint32_t)((kt / kStages) & 1));
        // every warp has passed wgmma_wait<1> of iteration kt - 1, so the wgmma of tile kt - 2 is done and its slot
        // can be refilled
        const int nt = kt + kStages - 2;
        if (nt < KT) load_tile(nt % kStages, nt);
        cp_async_commit();
        const uint32_t sa = s_base + slot * stage_bytes(BN), sb = sa + kBM * kRowBytes;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kBK / 8; kk++) {
            const uint64_t db = smem_desc(sb + kk * 32);
            wgmma_tile<BN>(acc[0], smem_desc(sa + kk * 32), db);
            wgmma_tile<BN>(acc[1], smem_desc(sa + 64 * kRowBytes + kk * 32), db);
        }
        wgmma_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    cp_async_wait<0>();

    // epilogue: accumulator fragment of m64nBN: rows 16 warp + lane / 4 (+ 8), columns 8 g + 2 (lane % 4) (+ 1)
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int r0 = m0 + h * 64 + 16 * warp + (lane >> 2);
#pragma unroll
        for (int g = 0; g < BN / 8; g++) {
            const int col = n0 + 8 * g + 2 * (lane & 3);
            const float b0 = bias[col], b1 = bias[col + 1];
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int r = r0 + 8 * e;
                if (r < M) {
                    const float2 v = make_float2(fmaxf(acc[h][4 * g + 2 * e] + b0, 0.0f),
                                                 fmaxf(acc[h][4 * g + 2 * e + 1] + b1, 0.0f));
                    *(float2*)(out + (size_t)r * cout + col) = v;
                }
            }
        }
    }
}

// ---- 2 x 2 max-pool, floor ----

__global__ void __launch_bounds__(256) mt_pool_kernel(int n_img, int H, int W, int C, const float* __restrict__ in,
                                                      float* __restrict__ out) {
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    const long long n = (long long)n_img * Ho * Wo * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        const long long p = i / C4;
        const int ox = (int)(p % Wo);
        const long long t = p / Wo;
        const int oy = (int)(t % Ho), b = (int)(t / Ho);
        const float4* s = (const float4*)in + (((long long)b * H + 2 * oy) * W + 2 * ox) * C4 + c;
        const float4 a = s[0], e = s[C4], f = s[(long long)W * C4], g = s[(long long)W * C4 + C4];
        ((float4*)out)[i] = make_float4(fmaxf(fmaxf(a.x, e.x), fmaxf(f.x, g.x)), fmaxf(fmaxf(a.y, e.y), fmaxf(f.y, g.y)),
                                        fmaxf(fmaxf(a.z, e.z), fmaxf(f.z, g.z)), fmaxf(fmaxf(a.w, e.w), fmaxf(f.w, g.w)));
    }
}

// ---- LPIPS tap ----

__global__ void __launch_bounds__(kRedThreads) mt_tap_kernel(int hw, int C, const float* __restrict__ feat,
                                                             const float* __restrict__ lin,
                                                             double* __restrict__ partials) {
    __shared__ double red[kRedThreads / 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = kRedThreads / 32;
    double acc = 0.0;
    for (int p = blockIdx.x * wpb + warp; p < hw; p += kRedBlocks * wpb) {
        const float* fx = feat + (size_t)p * C;
        const float* fy = feat + ((size_t)hw + p) * C;
        float4 a[4], b[4];
        float sx = 0.0f, sy = 0.0f;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int c = 4 * lane + 128 * j;
            if (c < C) {
                a[j] = *(const float4*)(fx + c);
                b[j] = *(const float4*)(fy + c);
                sx += a[j].x * a[j].x + a[j].y * a[j].y + a[j].z * a[j].z + a[j].w * a[j].w;
                sy += b[j].x * b[j].x + b[j].y * b[j].y + b[j].z * b[j].z + b[j].w * b[j].w;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            sx += __shfl_xor_sync(0xffffffffu, sx, o);
            sy += __shfl_xor_sync(0xffffffffu, sy, o);
        }
        const float nx = __fadd_rn(__fsqrt_rn(sx), 1e-10f), ny = __fadd_rn(__fsqrt_rn(sy), 1e-10f);
        float v = 0.0f;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int c = 4 * lane + 128 * j;
            if (c < C) {
                const float4 w = *(const float4*)(lin + c);
                float d;
                d = __fdiv_rn(a[j].x, nx) - __fdiv_rn(b[j].x, ny); v = fmaf(w.x, d * d, v);
                d = __fdiv_rn(a[j].y, nx) - __fdiv_rn(b[j].y, ny); v = fmaf(w.y, d * d, v);
                d = __fdiv_rn(a[j].z, nx) - __fdiv_rn(b[j].z, ny); v = fmaf(w.z, d * d, v);
                d = __fdiv_rn(a[j].w, nx) - __fdiv_rn(b[j].w, ny); v = fmaf(w.w, d * d, v);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        acc += (double)v;
    }
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < wpb; w++) s += red[w];
        partials[blockIdx.x] = s;
    }
}

struct TapCounts { long long hw[kTaps]; };

// one thread per tap: the blocks in order, the mean rounded to float32, then the five taps summed in float32
__global__ void mt_lpips_finish_kernel(TapCounts n, const double* __restrict__ partials, float* __restrict__ out,
                                       float* __restrict__ taps) {
    __shared__ float tv[kTaps];
    if (threadIdx.x < kTaps) {
        double s = 0.0;
        for (int b = 0; b < kRedBlocks; b++) s += partials[threadIdx.x * kRedBlocks + b];
        tv[threadIdx.x] = (float)(s / (double)n.hw[threadIdx.x]);
        if (taps) taps[threadIdx.x] = tv[threadIdx.x];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float r = tv[0];
        for (int t = 1; t < kTaps; t++) r = __fadd_rn(r, tv[t]);
        out[0] = r;
    }
}

// ---- PSNR ----

__global__ void __launch_bounds__(kRedThreads) mt_sqdiff_kernel(long long per_image, const float* __restrict__ a,
                                                                const float* __restrict__ b,
                                                                double* __restrict__ partials) {
    __shared__ double red[kRedThreads];
    const size_t base = (size_t)blockIdx.y * per_image;
    double s = 0.0;
    for (long long i = blockIdx.x * (long long)kRedThreads + threadIdx.x; i < per_image;
         i += (long long)kRedBlocks * kRedThreads) {
        const double d = (double)a[base + i] - (double)b[base + i];
        s += d * d;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = kRedThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) partials[(size_t)blockIdx.y * kRedBlocks + blockIdx.x] = red[0];
}

__global__ void mt_psnr_finish_kernel(int n, long long per_image, const double* __restrict__ partials,
                                      float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int b = 0; b < kRedBlocks; b++) s += partials[(size_t)i * kRedBlocks + b];
    const double mse = s / (double)per_image;
    out[i] = (float)(20.0 * log10(1.0 / sqrt(mse)));
}

int grid_of(long long n, int threads) {
    const long long g = (n + threads - 1) / threads;
    return (int)(g < 1 ? 1 : (g > 4 * 132 * 16 ? 4 * 132 * 16 : g));
}

bool is_device_ptr(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

bool side_ok(int H, int W) { return H >= kMinSide && W >= kMinSide && H <= kMaxSide && W <= kMaxSide; }

}  // namespace
}  // namespace surfel

using namespace surfel;

extern "C" {

int surfel_metrics_min_side(void) { return kMinSide; }
int surfel_metrics_max_side(void) { return kMaxSide; }
size_t surfel_metrics_partials_count(int n_images) {
    return n_images < 1 ? 0 : (size_t)(n_images > kTaps ? n_images : kTaps) * kRedBlocks;
}

int surfel_metrics_lpips_input(int n, int c, int height, int width, const float* x, const float* y, float* out,
                               void* stream) {
    if (n != 1) { surfel_set_error("surfel_metrics_lpips_input: batch of %d images, LPIPS takes one", n); return 1; }
    if (c != 3) { surfel_set_error("surfel_metrics_lpips_input: %d channels, expected 3", c); return 1; }
    if (!side_ok(height, width)) {
        surfel_set_error("surfel_metrics_lpips_input: image %d x %d outside [%d, %d] per side", height, width,
                         kMinSide, kMaxSide);
        return 1;
    }
    if (!x || !y || !out) { surfel_set_error("surfel_metrics_lpips_input: NULL pointer"); return 1; }
    if (!is_device_ptr(x) || !is_device_ptr(y) || !is_device_ptr(out)) {
        surfel_set_error("surfel_metrics_lpips_input: inputs must be device memory");
        return 1;
    }
    // the reference's buffers: torch.Tensor([-.030, -.088, -.188]) and ([.458, .448, .450]), doubles to float32
    ZParams z;
    const double mean[3] = {-.030, -.088, -.188}, sd[3] = {.458, .448, .450};
    for (int i = 0; i < 3; i++) { z.mean[i] = (float)mean[i]; z.std[i] = (float)sd[i]; }
    const long long hw = (long long)height * width;
    prof_count_launch();
    mt_zscore_kernel<<<grid_of(2 * hw * 3, 256), 256, 0, (cudaStream_t)stream>>>(hw, x, y, z, out);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_metrics_pack_conv(int cout, int cin, const float* w, float* packed, void* stream) {
    if (cout < 1 || cout % 64 != 0 || cout > 4096 || !(cin == 3 || (cin > 0 && cin % kBK == 0 && cin <= 4096))) {
        surfel_set_error("surfel_metrics_pack_conv: %d -> %d channels unsupported", cin, cout);
        return 1;
    }
    if (!w || !packed) { surfel_set_error("surfel_metrics_pack_conv: NULL pointer"); return 1; }
    prof_count_launch();
    mt_pack_kernel<<<grid_of((long long)cout * cin * 9, 256), 256, 0, (cudaStream_t)stream>>>(cout, cin, cin != 3, w,
                                                                                            packed);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_metrics_conv3x3(int n, int height, int width, int cin, int cout, const float* in, const float* packed,
                           const float* bias, float* out, void* stream) {
    if (n < 1 || n > 2 || height < 1 || width < 1 || height > kMaxSide || width > kMaxSide) {
        surfel_set_error("surfel_metrics_conv3x3: bad shape %d x %d x %d", n, height, width);
        return 1;
    }
    const bool c3 = cin == 3 && cout == 64;
    const bool tc = cin > 0 && cin % kBK == 0 && cin <= 4096 && cout > 0 && cout % 64 == 0 && cout <= 4096;
    if (!c3 && !tc) { surfel_set_error("surfel_metrics_conv3x3: %d -> %d channels unsupported", cin, cout); return 1; }
    if (!in || !packed || !bias || !out) { surfel_set_error("surfel_metrics_conv3x3: NULL pointer"); return 1; }
    cudaStream_t st = (cudaStream_t)stream;
    const long long M = (long long)n * height * width;
    if (c3) {
        prof_count_launch();
        mt_conv_c3_kernel<<<(unsigned)((M + 127) / 128), 128, 0, st>>>(n, height, width, in, packed, bias, out);
        SURFEL_CUDA_OK(cudaGetLastError());
        return 0;
    }
    static bool init[kMaxDevices] = {};
    const int slot = current_device_slot();
    if (slot < 0 || !init[slot]) {
        SURFEL_CUDA_OK(cudaFuncSetAttribute(mt_conv_wgmma_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            conv_smem_bytes(128)));
        SURFEL_CUDA_OK(cudaFuncSetAttribute(mt_conv_wgmma_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            conv_smem_bytes(64)));
        if (slot >= 0) init[slot] = true;
    }
    const unsigned gm = (unsigned)((M + kBM - 1) / kBM);
    prof_count_launch();
    if (cout % 128 == 0)
        mt_conv_wgmma_kernel<128><<<dim3(gm, cout / 128), kConvThreads, conv_smem_bytes(128), st>>>(
            n, height, width, cin, cout, in, packed, bias, out);
    else
        mt_conv_wgmma_kernel<64><<<dim3(gm, cout / 64), kConvThreads, conv_smem_bytes(64), st>>>(
            n, height, width, cin, cout, in, packed, bias, out);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_metrics_maxpool(int n, int height, int width, int c, const float* in, float* out, void* stream) {
    if (n < 1 || n > 2 || height < 2 || width < 2 || height > kMaxSide || width > kMaxSide || c < 4 || c % 4 != 0 ||
        c > 4096) {
        surfel_set_error("surfel_metrics_maxpool: bad shape %d x %d x %d x %d", n, height, width, c);
        return 1;
    }
    if (!in || !out) { surfel_set_error("surfel_metrics_maxpool: NULL pointer"); return 1; }
    prof_count_launch();
    mt_pool_kernel<<<grid_of((long long)n * (height / 2) * (width / 2) * (c / 4), 256), 256, 0, (cudaStream_t)stream>>>(
        n, height, width, c, in, out);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_metrics_lpips_tap(int tap, int height, int width, int c, const float* feat, const float* lin,
                             double* partials, void* stream) {
    if (tap < 0 || tap >= kTaps) { surfel_set_error("surfel_metrics_lpips_tap: tap %d outside [0, 5)", tap); return 1; }
    if (height < 1 || width < 1 || height > kMaxSide || width > kMaxSide || c < 4 || c % 4 != 0 || c > 512) {
        surfel_set_error("surfel_metrics_lpips_tap: bad shape %d x %d x %d", height, width, c);
        return 1;
    }
    if (!feat || !lin || !partials) { surfel_set_error("surfel_metrics_lpips_tap: NULL pointer"); return 1; }
    prof_count_launch();
    mt_tap_kernel<<<kRedBlocks, kRedThreads, 0, (cudaStream_t)stream>>>(height * width, c, feat, lin,
                                                                         partials + (size_t)tap * kRedBlocks);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_metrics_lpips_finish(const long long* tap_pixels_host, const double* partials, float* out, float* taps,
                                void* stream) {
    if (!tap_pixels_host || !partials || !out) { surfel_set_error("surfel_metrics_lpips_finish: NULL pointer"); return 1; }
    TapCounts n;
    for (int t = 0; t < kTaps; t++) {
        if (tap_pixels_host[t] < 1) { surfel_set_error("surfel_metrics_lpips_finish: empty tap %d", t); return 1; }
        n.hw[t] = tap_pixels_host[t];
    }
    prof_count_launch();
    mt_lpips_finish_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(n, partials, out, taps);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_metrics_psnr(int n, long long per_image, const float* a, const float* b, double* partials, float* out,
                        void* stream) {
    if (n < 1 || n > 65535 || per_image < 1) {
        surfel_set_error("surfel_metrics_psnr: bad shape %d x %lld", n, per_image);
        return 1;
    }
    if (!a || !b || !partials || !out) { surfel_set_error("surfel_metrics_psnr: NULL pointer"); return 1; }
    if (!is_device_ptr(a) || !is_device_ptr(b)) { surfel_set_error("surfel_metrics_psnr: inputs must be device memory"); return 1; }
    cudaStream_t st = (cudaStream_t)stream;
    prof_count_launch();
    mt_sqdiff_kernel<<<dim3(kRedBlocks, n), kRedThreads, 0, st>>>(per_image, a, b, partials);
    SURFEL_CUDA_OK(cudaGetLastError());
    prof_count_launch();
    mt_psnr_finish_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, per_image, partials, out);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
