// kernels.h — internal launch interface between the C-ABI (api.cu) and the kernel TUs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

namespace surfel {

struct PreFwdParams {
    int P, D, M, W, H, gx, gy, row0, row1, prefiltered;
    float scale_modifier;
    const float* means3D; const float* scales; const float* rotations; const float* opacities;
    const float* shs; const float* transMat_precomp; const float* colors_precomp;
    const float* viewmatrix; const float* projmatrix; const float* campos;
    int* radii; float4* rec; float4* tmat; uint32_t* tiles_touched; uint32_t* offsets; uint8_t* clamped;
    unsigned long long* scan_status; uint32_t* counters;
    uint32_t* tile_count;   // optional (tiles): per-tile instance counts accumulated here (fused count)
    uint32_t* num_rendered_mapped;   // optional: device-visible alias of the caller's pinned host word for R
};

struct PreBwdParams {
    int P, D, M, W, H;
    float scale_modifier;
    const float* means3D; const float* scales; const float* rotations; const float* shs;
    const float* transMat_precomp; int has_colors_precomp;
    const float* viewmatrix; const float* projmatrix; const float* campos;
    const int* radii; const float4* tmat; const uint8_t* clamped;
    const float* grad_rec;            // (P, kGradFloats) accumulated by render backward
    float* dL_dmeans2D;               // (P,3) out: densification proxy in .xy
    float* dL_dcolors;                // (P,3) out (gradient of colors_precomp)
    float* dL_dopacity;               // (P,1) out
    float* dL_dmeans3D;               // (P,3) out
    float* dL_dtransMat;              // (P,9) out (gradient of cov3D_precomp)
    float* dL_dsh;                    // (P,M,3) out
    float* dL_dscales;                // (P,2) out
    float* dL_drots;                  // (P,4) out
    int defer_sh;                     // 1: dL_dsh is NOT written; dL_dcolors receives the clamp-masked colour gradient
};

// camera gradients (camera_bwd.cu): runs after surfel_backward on its record, dL_dT and workspaces
struct CamBwdParams {
    int P, D, M, W, H;
    float scale_modifier;
    const float* means3D; const float* scales; const float* rotations; const float* shs;
    const float* transMat_precomp; int has_colors_precomp;
    const float* viewmatrix; const float* campos;
    const int* radii; const float4* rec; const uint8_t* clamped;
    const float* grad_rec;            // (P, kGradFloats) left by surfel_backward
    const float* dL_dtransMat;        // (P,9) full dL_dT written by preprocess backward (scales+rotations path)
    double* partials;                 // camera_partials_bytes(P)
    float* dL_dviewmatrix; float* dL_dprojmatrix; float* dL_dcampos;   // (16), (16), (3) out
};

struct RenderParams {
    int W, H, gx, gy, row0, row1;
    const uint2* ranges; const uint32_t* point_list; const float4* rec;
    const float* bg;   // device (3)
    // forward outputs / backward inputs
    float* out_color; float* out_others; float* accum; uint32_t* n_contrib;
    // backward
    const float* dL_dpix; const float* dL_dothers; float* grad_rec; int lowpass_quirk;
    size_t out_plane, grad_plane;   // floats between planes of the outputs / of the cotangents (default H*W)
    // forward: replicated output frames (peer mappings or one multicast address), see surfel_settings
    int rep_count; unsigned long long rep_base[8];
};

int launch_preprocess_fwd(const PreFwdParams& p, cudaStream_t stream);
int launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                        cudaStream_t stream);
int launch_preprocess_bwd(const PreBwdParams& p, cudaStream_t stream);
// dL_dsh (P,M,3) = SH basis(direction of the splat) (x) dL_dcolors (P,3): the rank-1 expansion that
// preprocess_bwd skips in defer_sh mode (so that a multi-GPU caller can reduce 3 floats per splat instead of 3M)
int launch_sh_grad_expand(int P, int M, int D, const float* means3D, const float* campos,
                          const float* dL_dcolors, float* dL_dsh, cudaStream_t stream);

size_t camera_partials_bytes(int P);
int launch_camera_bwd(const CamBwdParams& p, cudaStream_t stream);
// the same step with the 35 sums written as double before rounding (p.dL_d* unused): a tile-row band's share
int launch_camera_bwd_sums(const CamBwdParams& p, double* dvm, double* dpr, double* dcam, cudaStream_t stream);

// binning
int launch_duplicate_with_keys(int P, int gx, int gy, int row0, int row1, const float4* tmat,
                               const int* radii, const uint32_t* offsets, uint64_t* keys,
                               uint32_t* vals, cudaStream_t stream);
int launch_identify_tile_ranges(size_t R, int tiles, const uint64_t* keys_sorted, uint2* ranges,
                                cudaStream_t stream);

// CUB-free stable LSD radix sort of (u64 key, u32 value) pairs on key bits [0, end_bit).  The pairs ping-pong
// between two buffers, one 8-bit digit per pass; radix_sort_ws() tells the caller which buffer to fill (in) and
// which one holds the result (out), so no caller needs the pass count.
constexpr long long kRadixSortMaxPairs = (1ll << 30) - 1;
struct SortPairs { uint64_t* keys; uint32_t* vals; };
struct RadixSortWs { SortPairs in, out, spare; void* temp; int end_bit; };   // spare: the buffer that is not out
int radix_key_bits(unsigned long long max_key);   // least end_bit that orders every key in [0, max_key]
size_t radix_sort_temp_bytes(size_t n);
size_t radix_sort_pairs_bytes(size_t capacity);       // both buffers for up to `capacity` pairs
size_t radix_sort_workspace_bytes(size_t capacity);   // both buffers, then the pass scratch
// Over radix_sort_workspace_bytes(capacity) at base, or over radix_sort_pairs_bytes(capacity) at base when the
// caller keeps the pass scratch at `temp`; or over buffers A and B that the caller placed itself.
RadixSortWs radix_sort_ws(void* base, size_t capacity, int end_bit, void* temp = nullptr);
RadixSortWs radix_sort_ws(SortPairs a, SortPairs b, void* temp, int end_bit);
int launch_radix_sort_pairs(const RadixSortWs& ws, size_t n, cudaStream_t stream);   // ws.in[0, n) -> ws.out

// Tile-bucketed binning (bucket_sort.cu): counting scatter by tile + per-tile shared-memory sort.
// Produces ranges + point_list (+ keys_sorted if non-NULL) identical to duplicate -> stable radix
// sort -> identifyTileRanges.  `pairs` is an R x u64 scratch buffer (the radix sort's spare keys).
size_t bucket_temp_bytes(int tiles);
int launch_bucket_binning(int P, size_t R, int gx, int gy, int row0, int row1, const float4* tmat,
                          const int* radii, const uint32_t* offsets, unsigned long long* pairs,
                          uint32_t* point_list, unsigned long long* keys_sorted, uint2* ranges,
                          void* temp, const uint32_t* tile_count_ready, cudaStream_t stream);

int launch_render_fwd(const RenderParams& p, cudaStream_t stream);
int launch_render_bwd(const RenderParams& p, cudaStream_t stream);

}  // namespace surfel
