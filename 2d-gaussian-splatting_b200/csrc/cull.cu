// cull.cu — DTU mask culling of a mesh (cull_scan of the reference's scripts/eval_dtu/evaluate_single_scene.py, the
// step between mesh extraction and eval.py) on the device.  DESIGN.md §7n has the rules; tests/cull_ref.py restates
// them.  The file is compiled with -fmad=false and every operation the rules fix is a __f*_rn / __d*_rn intrinsic.
//
//  * surfel_cull_dilate: binary dilation of each view's mask by disk(r) = {dx^2 + dy^2 <= r^2} with a zero border.
//     - rows: one block per mask row packs the row into bits in shared memory (one ballot per 32 pixels), then each
//       pixel's distance to the nearest set pixel of its row, clamped at r + 1, is found from the words with
//       __ffs / __clz and stored as one byte.
//     - columns: a block owns a 128 x 32 tile and stages the row distances of its rows and an r-row halo in shared
//       memory (rows outside the image read 255, so the border is zero).  A pixel is set iff some |dy| <= r has
//       dist[y + dy][x] <= hw[dy], hw[dy] = isqrt(r^2 - dy^2): the disk's half-width at dy.  A thread tests four
//       pixels per shared word with __vcmpleu4, and eight lanes assemble one 32-pixel output word.
//  * surfel_cull_vertices: one thread per vertex, in mesh order (extracted meshes are spatially coherent, so a warp's
//    samples land near each other), with every view's 3 x 4 projection staged in shared memory.  The float32 test of
//    rule 3 runs view by view and stops at the first view that fails.  The same kernel ranks the kept vertices with
//    the look-back scan of scan.cuh; a second one checks each face's indices (no index addresses memory unless it is
//    in range) and ranks the faces whose three vertices are kept.
//  * surfel_cull_emit: with the two counts read back, writes the kept vertices in world units (two roundings, no FMA),
//    their colour rows byte for byte, and the kept faces renumbered.  Both scans keep order, so the outputs are the
//    reference's whatever the schedule.
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

constexpr int kCuThreads = 256;
constexpr int kCuTileX = 128, kCuTileY = 32;        // column pass: 32 lanes x 4 pixels, 8 warps x 4 rows
constexpr int kCuMaxRadius = 254;                  // row distances clamp at r + 1 and travel in one byte
constexpr int kCuMaxViews = 512;                   // 48 bytes of projection per view in shared memory
constexpr int kCuMaxSide = 1 << 15;
constexpr long long kCuMaxCount = (1ll << 31) - 1; // ranks and counts travel in 32 bits, ~0u marks "dropped"
constexpr uint32_t kDropped = 0xffffffffu;

int blocks_of(long long n) { return (int)std::max<long long>(1, (n + kCuThreads - 1) / kCuThreads); }
__host__ __device__ inline int words_of(int width) { return (width + 31) / 32; }

// ---- dilation ----

// distance from x to the nearest set bit of the row (nw words, bits beyond the width clear), clamped at lim
__device__ __forceinline__ int row_distance(const uint32_t* bits, int nw, int x, int lim) {
    const int w = x >> 5, b = x & 31;
    int d = lim;
    const uint32_t right = bits[w] >> b;                 // bit x at position 0
    if (right) {
        d = min(d, __ffs(right) - 1);
    } else {
        for (int k = w + 1; k < nw && k * 32 - x < d; k++) {
            const uint32_t v = bits[k];
            if (v) { d = min(d, k * 32 + __ffs(v) - 1 - x); break; }
        }
    }
    const uint32_t left = bits[w] << (31 - b);           // bit x at position 31
    if (left) {
        d = min(d, __clz(left));
    } else {
        for (int k = w - 1; k >= 0 && x - (k * 32 + 31) < d; k--) {
            const uint32_t v = bits[k];
            if (v) { d = min(d, x - (k * 32 + 31 - __clz(v))); break; }
        }
    }
    return d;
}

__global__ void __launch_bounds__(kCuThreads) cu_rows_kernel(int width, int radius,
                                                             const unsigned char* __restrict__ masks,
                                                             unsigned char* __restrict__ dist) {
    extern __shared__ uint32_t s_bits[];
    const size_t row = blockIdx.x;
    const int nw = words_of(width), lane = threadIdx.x & 31;
    const unsigned char* m = masks + row * width;
    for (int base = 0; base < nw * 32; base += kCuThreads) {
        const int x = base + threadIdx.x;
        const unsigned word = __ballot_sync(0xffffffffu, x < width && m[x] != 0);
        if (lane == 0 && x < nw * 32) s_bits[x >> 5] = word;
    }
    __syncthreads();
    unsigned char* out = dist + row * width;
    for (int x = threadIdx.x; x < width; x += kCuThreads) out[x] = (unsigned char)row_distance(s_bits, nw, x, radius + 1);
}

__global__ void __launch_bounds__(kCuThreads) cu_columns_kernel(int height, int width, int radius,
                                                                const unsigned char* __restrict__ dist,
                                                                uint32_t* __restrict__ out) {
    extern __shared__ uint32_t s_tile[];                  // (kCuTileY + 2r) rows of kCuTileX bytes, then hw[2r + 1]
    unsigned char* tile = (unsigned char*)s_tile;
    const int rows = kCuTileY + 2 * radius;
    unsigned char* hw = tile + (size_t)rows * kCuTileX;
    const int view = blockIdx.z, x0 = blockIdx.x * kCuTileX, y0 = blockIdx.y * kCuTileY;
    const unsigned char* d = dist + (size_t)view * height * width;
    for (int i = threadIdx.x; i < rows * kCuTileX; i += kCuThreads) {
        const int ty = i / kCuTileX, tx = i % kCuTileX, y = y0 - radius + ty, x = x0 + tx;
        tile[i] = (y >= 0 && y < height && x < width) ? d[(size_t)y * width + x] : (unsigned char)255;
    }
    for (int dy = threadIdx.x; dy <= 2 * radius; dy += kCuThreads) {
        const int e = dy - radius, rem = radius * radius - e * e;
        int h = (int)sqrtf((float)rem);
        while (h * h > rem) h--;
        while ((h + 1) * (h + 1) <= rem) h++;
        hw[dy] = (unsigned char)h;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = words_of(width);
    for (int ty = warp; ty < kCuTileY; ty += kCuThreads / 32) {
        const int y = y0 + ty;
        if (y >= height) break;
        uint32_t set = 0;                                // 0xff per byte (pixel) found
        for (int k = 0; k <= 2 * radius && set != 0xffffffffu; k++) {
            const uint32_t w4 = *(const uint32_t*)(tile + (size_t)(ty + k) * kCuTileX + 4 * lane);
            set |= __vcmpleu4(w4, 0x01010101u * hw[k]);
        }
        uint32_t nib = (set & 1u) | ((set >> 7) & 2u) | ((set >> 14) & 4u) | ((set >> 21) & 8u);
        nib <<= 4 * (lane & 7);
        nib |= __shfl_xor_sync(0xffffffffu, nib, 1);
        nib |= __shfl_xor_sync(0xffffffffu, nib, 2);
        nib |= __shfl_xor_sync(0xffffffffu, nib, 4);
        const int word = x0 / 32 + lane / 8;
        if ((lane & 7) == 0 && word < nw) out[((size_t)view * height + y) * nw + word] = nib;
    }
}

size_t rows_smem(int width) { return (size_t)words_of(width) * 4; }
size_t columns_smem(int radius) { return (size_t)(kCuTileY + 2 * radius) * kCuTileX + align_up(2 * radius + 1, 4); }

// ---- vertices and faces ----

struct CuView {
    float img_w1, img_h1;     // float32(W - 1), float32(H - 1) of image_size
    float mask_w1, mask_h1;   // float32(width - 1), float32(height - 1) of the masks
    int height, width, nw;
};

__device__ __forceinline__ float dot4(const float* a, float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a[0], x), __fmul_rn(a[1], y)), __fmul_rn(a[2], z)), a[3]);
}

// rule 3 for one vertex against every view: false at the first view whose projection lands inside the frame on a
// pixel the dilated mask does not cover
__device__ __forceinline__ bool vertex_kept(float x, float y, float z, int n_views, const float* s_proj,
                                            const CuView& cv, const uint32_t* __restrict__ dilated) {
    for (int k = 0; k < n_views; k++) {
        const float* a = s_proj + 12 * k;
        const float c0 = dot4(a, x, y, z), c1 = dot4(a + 4, x, y, z), c2 = dot4(a + 8, x, y, z);
        const float d = __fadd_rn(c2, 1e-6f);
        const float gx = __fmul_rn(__fsub_rn(__fdiv_rn(__fdiv_rn(c0, d), cv.img_w1), 0.5f), 2.0f);
        const float gy = __fmul_rn(__fsub_rn(__fdiv_rn(__fdiv_rn(c1, d), cv.img_h1), 0.5f), 2.0f);
        if (!(gx > -1.0f && gx < 1.0f && gy > -1.0f && gy < 1.0f)) continue;    // NaN is not valid: the view passes
        const int ix = __float2int_rn(__fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.0f), 2.0f), cv.mask_w1));
        const int iy = __float2int_rn(__fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.0f), 2.0f), cv.mask_h1));
        const bool hit = ix >= 0 && ix < cv.width && iy >= 0 && iy < cv.height &&
                         ((__ldg(dilated + ((size_t)k * cv.height + iy) * cv.nw + (ix >> 5)) >> (ix & 31)) & 1u);
        if (!hit) return false;
    }
    return true;
}

// info: [1] |= 1 on a coordinate that is not finite in float32, [2] = the number of kept vertices
__global__ void __launch_bounds__(kCuThreads) cu_vertices_kernel(long long M, const double* __restrict__ verts,
                                                                 int n_views, const float* __restrict__ proj,
                                                                 CuView cv, const uint32_t* __restrict__ dilated,
                                                                 unsigned char* __restrict__ keep,
                                                                 uint32_t* __restrict__ vnew, uint32_t* ctrl,
                                                                 unsigned long long* status, long long* info) {
    extern __shared__ float s_proj[];
    __shared__ uint32_t s_warp[kCuThreads / 32], s_bid, s_excl[1];
    for (int i = threadIdx.x; i < 12 * n_views; i += kCuThreads) s_proj[i] = proj[i];
    if (threadIdx.x == 0) s_bid = atomicAdd(&ctrl[0], 1u);
    __syncthreads();
    const uint32_t bid = s_bid;
    const long long v = (long long)bid * kCuThreads + threadIdx.x;
    bool kept = false;
    if (v < M) {
        const float x = __double2float_rn(verts[3 * v]), y = __double2float_rn(verts[3 * v + 1]),
                    z = __double2float_rn(verts[3 * v + 2]);
        if (!(isfinite(x) && isfinite(y) && isfinite(z))) atomicOr((unsigned long long*)info + 1, 1ull);
        kept = vertex_kept(x, y, z, n_views, s_proj, cv, dilated);
        keep[v] = kept ? 1 : 0;
    }
    uint32_t total;
    const uint32_t excl = block_exclusive_scan<kCuThreads>(kept ? 1u : 0u, s_warp, total);
    block_lookback<1>(status, gridDim.x, bid, &total, s_excl);
    if (v < M) vnew[v] = kept ? s_excl[0] + excl : kDropped;
    if (bid == gridDim.x - 1 && threadIdx.x == 0) info[2] = (long long)s_excl[0] + total;
}

// info: [0] |= 1 on a face index outside [0, M), [3] = the number of kept faces
__global__ void __launch_bounds__(kCuThreads) cu_faces_kernel(long long F, long long M,
                                                              const long long* __restrict__ faces,
                                                              const uint32_t* __restrict__ vnew,
                                                              uint32_t* __restrict__ frank, uint32_t* ctrl,
                                                              unsigned long long* status, long long* info) {
    __shared__ uint32_t s_warp[kCuThreads / 32], s_bid, s_excl[1];
    if (threadIdx.x == 0) s_bid = atomicAdd(&ctrl[1], 1u);
    __syncthreads();
    const uint32_t bid = s_bid;
    const long long f = (long long)bid * kCuThreads + threadIdx.x;
    bool kept = false;
    if (f < F) {
        bool ok = true;
        kept = true;
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const long long i = faces[3 * f + j];
            const bool in = i >= 0 && i < M;
            ok &= in;
            kept &= in && vnew[in ? i : 0] != kDropped;
        }
        if (!ok) atomicOr((unsigned long long*)info, 1ull);
    }
    uint32_t total;
    const uint32_t excl = block_exclusive_scan<kCuThreads>(kept ? 1u : 0u, s_warp, total);
    block_lookback<1>(status, gridDim.x, bid, &total, s_excl);
    if (f < F) frank[f] = kept ? s_excl[0] + excl : kDropped;
    if (bid == gridDim.x - 1 && threadIdx.x == 0) info[3] = (long long)s_excl[0] + total;
}

struct CuWorld { double s, t[3]; };

__global__ void __launch_bounds__(kCuThreads) cu_emit_vertices_kernel(long long M, const double* __restrict__ verts,
                                                                      const uint32_t* __restrict__ vnew, CuWorld wt,
                                                                      const unsigned char* __restrict__ colors,
                                                                      long long color_bytes,
                                                                      double* __restrict__ out_verts,
                                                                      unsigned char* __restrict__ out_colors) {
    const long long v = (long long)blockIdx.x * kCuThreads + threadIdx.x;
    if (v >= M) return;
    const uint32_t r = vnew[v];
    if (r == kDropped) return;
#pragma unroll
    for (int j = 0; j < 3; j++) out_verts[3 * (size_t)r + j] = __dadd_rn(__dmul_rn(verts[3 * v + j], wt.s), wt.t[j]);
    for (long long b = 0; b < color_bytes; b++) out_colors[(size_t)r * color_bytes + b] = colors[v * color_bytes + b];
}

__global__ void __launch_bounds__(kCuThreads) cu_emit_faces_kernel(long long F, const long long* __restrict__ faces,
                                                                   const uint32_t* __restrict__ vnew,
                                                                   const uint32_t* __restrict__ frank,
                                                                   long long* __restrict__ out_faces) {
    const long long f = (long long)blockIdx.x * kCuThreads + threadIdx.x;
    if (f >= F) return;
    const uint32_t r = frank[f];
    if (r == kDropped) return;
#pragma unroll
    for (int j = 0; j < 3; j++) out_faces[3 * (size_t)r + j] = vnew[faces[3 * f + j]];
}

struct CuLayout {
    size_t ctrl, status_m, status_f, vnew, frank, dist, total;
};

CuLayout cu_layout(long long n_views, int height, int width, long long M, long long F) {
    CuLayout L;
    size_t o = 0;
    L.ctrl = o;     o = align_up(o + 64, 256);
    L.status_m = o; o = align_up(o + (size_t)blocks_of(M) * 8, 256);
    L.status_f = o; o = align_up(o + (size_t)blocks_of(F) * 8, 256);
    L.vnew = o;     o = align_up(o + (size_t)std::max<long long>(M, 1) * 4, 256);
    L.frank = o;    o = align_up(o + (size_t)std::max<long long>(F, 1) * 4, 256);
    L.dist = o;     o = align_up(o + (size_t)n_views * height * width, 256);
    L.total = o;
    return L;
}

bool sizes_ok(const char* who, long long n_views, int height, int width, long long M, long long F) {
    if (n_views < 1 || n_views > kCuMaxViews) {
        surfel_set_error("%s: %lld views; 1 to %d are supported", who, n_views, kCuMaxViews);
        return false;
    }
    if (height < 1 || width < 1 || height > kCuMaxSide || width > kCuMaxSide) {
        surfel_set_error("%s: masks of %d x %d; each side must lie in [1, %d]", who, width, height, kCuMaxSide);
        return false;
    }
    if (M < 0 || F < 0 || M > kCuMaxCount || F > kCuMaxCount) {
        surfel_set_error("%s: %lld vertices, %lld faces; 0 to %lld of each are supported", who, M, F, kCuMaxCount);
        return false;
    }
    return true;
}

bool workspace_ok(const char* who, const void* ws, size_t bytes, size_t need) {
    if (!ws) { surfel_set_error("%s: NULL workspace", who); return false; }
    if (bytes < need) {
        surfel_set_error("%s: workspace of %zu bytes, %zu needed", who, bytes, need);
        return false;
    }
    return true;
}

}  // namespace
}  // namespace surfel

using namespace surfel;

extern "C" {

int surfel_cull_max_views(void) { return kCuMaxViews; }
int surfel_cull_max_radius(void) { return kCuMaxRadius; }

size_t surfel_cull_workspace_bytes(long long n_views, int height, int width, long long n_verts, long long n_faces) {
    if (n_views < 1 || n_views > kCuMaxViews || height < 1 || width < 1 || height > kCuMaxSide ||
        width > kCuMaxSide || n_verts < 0 || n_faces < 0 || n_verts > kCuMaxCount || n_faces > kCuMaxCount)
        return 0;
    return cu_layout(n_views, height, width, n_verts, n_faces).total;
}

int surfel_cull_dilate(int n_views, int height, int width, int radius, const unsigned char* masks, void* workspace,
                       size_t workspace_bytes, unsigned int* dilated, void* stream) {
    const char* who = "surfel_cull_dilate";
    if (!sizes_ok(who, n_views, height, width, 0, 0)) return 1;
    if (radius < 0 || radius > kCuMaxRadius) {
        surfel_set_error("%s: radius %d outside [0, %d]", who, radius, kCuMaxRadius);
        return 1;
    }
    if (!masks || !dilated) {
        surfel_set_error("%s: NULL masks or output", who);
        return 1;
    }
    const CuLayout L = cu_layout(n_views, height, width, 0, 0);
    if (!workspace_ok(who, workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* dist = (unsigned char*)workspace + L.dist;
    {
        LaunchScope scope(kStCullDilate, st);
        cu_rows_kernel<<<n_views * height, kCuThreads, rows_smem(width), st>>>(width, radius, masks, dist);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    const size_t smem = columns_smem(radius);
    SURFEL_CUDA_OK(cudaFuncSetAttribute(cu_columns_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    {
        LaunchScope scope(kStCullDilate, st);
        const dim3 grid((width + kCuTileX - 1) / kCuTileX, (height + kCuTileY - 1) / kCuTileY, n_views);
        cu_columns_kernel<<<grid, kCuThreads, smem, st>>>(height, width, radius, dist, dilated);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

int surfel_cull_vertices(long long n_verts, const double* verts, long long n_faces, const long long* faces,
                         int n_views, const float* proj, int image_width, int image_height, int height, int width,
                         const unsigned int* dilated, void* workspace, size_t workspace_bytes, unsigned char* keep,
                         long long* info, void* stream) {
    const char* who = "surfel_cull_vertices";
    if (!sizes_ok(who, n_views, height, width, n_verts, n_faces)) return 1;
    if (image_width < 1 || image_height < 1) {
        surfel_set_error("%s: image size %d x %d", who, image_width, image_height);
        return 1;
    }
    if (!info || !proj || !dilated || (n_verts > 0 && (!verts || !keep)) || (n_faces > 0 && !faces)) {
        surfel_set_error("%s: NULL vertices, faces, projections, masks, keep flags or info", who);
        return 1;
    }
    const CuLayout L = cu_layout(n_views, height, width, n_verts, n_faces);
    if (!workspace_ok(who, workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    uint32_t* ctrl = (uint32_t*)(w + L.ctrl);
    SURFEL_CUDA_OK(cudaMemsetAsync(info, 0, 4 * sizeof(long long), st));
    SURFEL_CUDA_OK(cudaMemsetAsync(ctrl, 0, 64, st));
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status_m, 0, (size_t)blocks_of(n_verts) * 8, st));
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status_f, 0, (size_t)blocks_of(n_faces) * 8, st));
    CuView cv;
    cv.img_w1 = (float)(image_width - 1);
    cv.img_h1 = (float)(image_height - 1);
    cv.mask_w1 = (float)(width - 1);
    cv.mask_h1 = (float)(height - 1);
    cv.height = height;
    cv.width = width;
    cv.nw = words_of(width);
    {
        LaunchScope scope(kStCullVertices, st);
        cu_vertices_kernel<<<blocks_of(n_verts), kCuThreads, (size_t)n_views * 12 * sizeof(float), st>>>(
            n_verts, verts, n_views, proj, cv, dilated, keep, (uint32_t*)(w + L.vnew), ctrl,
            (unsigned long long*)(w + L.status_m), info);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    {
        LaunchScope scope(kStCullFaces, st);
        cu_faces_kernel<<<blocks_of(n_faces), kCuThreads, 0, st>>>(n_faces, n_verts, faces, (uint32_t*)(w + L.vnew),
                                                                   (uint32_t*)(w + L.frank), ctrl,
                                                                   (unsigned long long*)(w + L.status_f), info);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

int surfel_cull_emit(long long n_verts, const double* verts, long long n_faces, const long long* faces,
                     const double* world, const void* colors, long long color_row_bytes, const void* workspace,
                     size_t workspace_bytes, long long n_kept_verts, long long n_kept_faces, double* out_verts,
                     long long* out_faces, void* out_colors, void* stream) {
    const char* who = "surfel_cull_emit";
    if (n_verts < 0 || n_faces < 0 || n_verts > kCuMaxCount || n_faces > kCuMaxCount) {
        surfel_set_error("%s: %lld vertices, %lld faces; 0 to %lld of each are supported", who, n_verts, n_faces,
                         kCuMaxCount);
        return 1;
    }
    if (n_kept_verts < 0 || n_kept_verts > n_verts || n_kept_faces < 0 || n_kept_faces > n_faces) {
        surfel_set_error("%s: %lld of %lld vertices and %lld of %lld faces kept", who, n_kept_verts, n_verts,
                         n_kept_faces, n_faces);
        return 1;
    }
    if (color_row_bytes < 0 || (color_row_bytes > 0 && n_kept_verts > 0 && (!colors || !out_colors))) {
        surfel_set_error("%s: colour rows of %lld bytes with NULL colours or output", who, color_row_bytes);
        return 1;
    }
    if (!world || (n_kept_verts > 0 && (!verts || !out_verts)) || (n_kept_faces > 0 && (!faces || !out_faces))) {
        surfel_set_error("%s: NULL vertices, faces, world transform or outputs", who);
        return 1;
    }
    // the ranks come before the row distances in the layout, so their offsets do not depend on the masks
    const CuLayout L = cu_layout(0, 1, 1, n_verts, n_faces);
    if (!workspace_ok(who, workspace, workspace_bytes, L.dist)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    const char* w = (const char*)workspace;
    CuWorld wt;
    wt.s = world[0];
    wt.t[0] = world[1];
    wt.t[1] = world[2];
    wt.t[2] = world[3];
    if (n_kept_verts > 0) {
        LaunchScope scope(kStCullEmit, st);
        cu_emit_vertices_kernel<<<blocks_of(n_verts), kCuThreads, 0, st>>>(
            n_verts, verts, (const uint32_t*)(w + L.vnew), wt, (const unsigned char*)colors, color_row_bytes,
            out_verts, (unsigned char*)out_colors);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    if (n_kept_faces > 0) {
        LaunchScope scope(kStCullEmit, st);
        cu_emit_faces_kernel<<<blocks_of(n_faces), kCuThreads, 0, st>>>(
            n_faces, faces, (const uint32_t*)(w + L.vnew), (const uint32_t*)(w + L.frank), out_faces);
        SURFEL_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

}  // extern "C"
