/*
 * surfel_rasterizer.h — C ABI of the H100-native differentiable 2D-surfel rasterizer
 * (libsurfel_b200.so, built from 2d-gaussian-splatting_b200/csrc by nvcc for sm_90a).
 *
 * This is the drop-in boundary for the native module of hbb1/diff-surfel-rasterization
 * (pinned by /root/reference/.SUBMODULES.json:10-14; its C++/CUDA sources are NOT vendored in
 * /root/reference, so the citations below are to the reference's own call sites and to
 * SURVEY.md §8(b), which records the upstream pybind11 signatures being replaced):
 *
 *   upstream _C.rasterize_gaussians(bg, means3D, colors, opacity, scales, rotations,
 *       scale_modifier, transMat_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, H, W, sh,
 *       degree, campos, prefiltered, debug) -> (num_rendered, color, others, radii, geomBuffer,
 *       binningBuffer, imgBuffer)
 *     == surfel_forward_preprocess()  [preprocess + tile-count scan -> num_rendered]
 *      + surfel_forward_render()      [duplicateWithKeys, radix sort, tile ranges, blend]
 *     reference call site: /root/reference/gaussian_renderer/__init__.py:37-53, :97-106
 *   upstream _C.rasterize_gaussians_backward(...) -> 8 gradient tensors
 *     == surfel_backward()
 *     reference consumers: /root/reference/train.py:90, :127-128,
 *                          /root/reference/scene/gaussian_model.py:405-407
 *   upstream _C.mark_visible(means3D, viewmatrix, projmatrix) -> bool tensor
 *     == surfel_mark_visible()
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name ends in _host;
 *   - all tensors are contiguous float32 unless stated; "absent" optional inputs are NULL
 *     (upstream passes empty tensors);
 *   - ownership: the caller (PyTorch on the Python side) owns every buffer, including the three
 *     opaque workspaces (geometry / binning / image state) whose sizes the *_bytes() functions
 *     return; forward fills them, backward reads them, nothing is retained across calls;
 *   - every launch is ordered on the cudaStream_t passed as `stream` (void*); no call synchronises
 *     the device; nothing about a CALL is retained.  Process-global state, all of it optional tooling:
 *     the last-error string (thread-local), the binning-variant switch (surfel_set_variant /
 *     SURFEL_SORT), the launch counter and the per-stage profiling switch (surfel_profile_*), and
 *     the per-device "function attribute set" flags of kernels that opt into large shared memory;
 *   - return value: 0 on success, non-zero on failure with surfel_last_error() describing it
 *     (the Python wrapper raises RuntimeError, like upstream's AT_ERROR path).
 */
#ifndef SURFEL_RASTERIZER_H_
#define SURFEL_RASTERIZER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SURFEL_ABI_VERSION 3
#define SURFEL_MAX_OUT_REPLICAS 8

/* Mirrors GaussianRasterizationSettings (fields constructed at
 * /root/reference/gaussian_renderer/__init__.py:37-51) plus the tile-row band used by the
 * multi-GPU tile-band partition (SURVEY §8e).  tile_row_begin == tile_row_end == 0 => full frame. */
typedef struct surfel_settings {
    int32_t image_height;
    int32_t image_width;
    float tanfovx;
    float tanfovy;
    float scale_modifier;
    int32_t sh_degree;
    int32_t prefiltered;
    int32_t debug;
    int32_t tile_row_begin;
    int32_t tile_row_end;
    const float* bg;          /* (3)    device */
    const float* viewmatrix;  /* (4,4)  device, row-vector convention (scene/cameras.py:56) */
    const float* projmatrix;  /* (4,4)  device, viewmatrix @ P^T      (scene/cameras.py:57-58) */
    const float* campos;      /* (3)    device                        (scene/cameras.py:59) */
    /* Distance, in floats, between consecutive planes of out_color / out_others (forward) and of
     * dL_dout_color / dL_dout_others (backward); 0 = image_height * image_width (contiguous (C,H,W), what
     * upstream allocates).  A larger stride lets the tile-band mode render straight into a frame padded to
     * equal bands, which an in-place all-gather then completes (SURVEY §8e) — no staging or stitch copies. */
    int64_t out_plane_stride;
    int64_t grad_plane_stride;
    /* Forward outputs written to REPLICATED frames (multi-GPU tile-band mode, SURVEY §8e): when
     * out_replica_count > 0 the render kernel stores every output value of its band to each address
     * out_replica_base[r] + 4 * (plane * out_plane_stride + y * W + x), plane = 0..2 for out_color and 3..9 for
     * out_others, INSTEAD of to out_color / out_others (which must still be valid pointers laid out the same way:
     * out_others == out_color + 3 * out_plane_stride).  The addresses are device pointers valid in this process:
     * peer mappings of the other GPUs' frames and this GPU's own frame (symmetric memory over NVLink), or ONE
     * NVSwitch multicast address that fans a single store out to all of them.  The exchange of the band outputs
     * is thereby done by the stores of the kernel that produces them; the caller only has to run a cross-GPU
     * barrier before any rank reads rows outside its own band.  0 = off (default). */
    int32_t out_replica_count;
    /* Backward, SH inputs only.  1 = surfel_backward() does NOT write dL_dsh; instead dL_dcolors (P,3, required)
     * receives the gradient of the splat's SH colour with the forward's clamp mask applied — the 3 numbers the
     * (P,M,3) SH gradient is a rank-1 expansion of.  A multi-GPU caller sums those 3 floats per splat across
     * ranks (16 floats per splat in all instead of 61) and then calls surfel_sh_grad_expand() once.  0 = off. */
    int32_t sh_grad_deferred;
    uint64_t out_replica_base[SURFEL_MAX_OUT_REPLICAS];
} surfel_settings_t;

int surfel_abi_version(void);
const char* surfel_last_error(void);

/* Selects between the two binning implementations (both sm_90a, bit-identical output, see DESIGN.md):
 * "sort" = "bucket" (default: tile buckets + per-tile sort) | "radix" (device-wide CUB-free onesweep).
 * Environment default: SURFEL_SORT.  Process-global; do not change it between a forward and its backward. */
int surfel_set_variant(const char* name, const char* value);
/* 1 iff R passed to surfel_forward_render / surfel_backward may be an upper bound ("capacity") of the
 * true instance count, which lets the caller launch stage 2 before it has read R back. */
int surfel_accepts_capacity(void);

/* Workspace sizes (bytes).  R = number of (splat, tile) instances ("num_rendered"). */
size_t surfel_geom_bytes(int P);
size_t surfel_image_bytes(int W, int H);
size_t surfel_binning_bytes(size_t R, int W, int H);

/* Byte offsets of the sub-arrays inside the workspaces, for tests and debugging.
 *   geom   : out[0]=render records (P x 128 B: adjugate of T about the splat's screen position, opacity,
 *            normal, rgb, det T, Tw, culling boxes), [1]=tiles_touched u32, [2]=offsets u32 (inclusive),
 *            [3]=clamped u8 (bit c = channel c clamped), [4]=counters u32 ([1] = R),
 *            [5]=transform records (P x 48 B: transMat[9], xy[2], view depth)
 *   binning: out[0]=keys_unsorted u64, [1]=vals_unsorted u32, [2]=keys_sorted u64,
 *            [3]=vals_sorted u32 (the per-tile point list), [4]=ranges uint2 per tile
 *            (unsorted and sorted regions coincide when the sort runs an even number of passes)
 *   image  : out[0]=accum f32 (final_T, M1, M2 planes), [1]=n_contrib u32 (last, median planes) */
int surfel_geom_offsets(int P, size_t* out6);
int surfel_binning_offsets(size_t R, int W, int H, size_t* out5);
int surfel_image_offsets(int W, int H, size_t* out2);

/* Forward, stage 1: preprocess every splat and scan tiles_touched.  Writes radii (P) int32 and the
 * geometry workspace.  If image_ws != NULL the per-tile instance counts are accumulated there in the
 * same launch (fused count for the tile-bucketed binning; pass tile_counts_ready = 1 downstream).  The instance count R is left in the workspace and, if
 * num_rendered_host != NULL, delivered there in stream order: for pinned, device-mapped host memory
 * (cudaHostAlloc / torch pin_memory) the kernel stores it directly (no copy-engine transfer that
 * could queue behind a bulk download on another stream); otherwise by a 4-byte cudaMemcpyAsync.  The
 * caller synchronises the stream (or an event) before reading it to size the binning workspace. */
int surfel_forward_preprocess(const surfel_settings_t* s, int P, int M, const float* means3D,
                              const float* opacities, const float* scales, const float* rotations,
                              const float* transMat_precomp, const float* shs,
                              const float* colors_precomp, int32_t* radii, void* geom_ws, void* image_ws,
                              uint32_t* num_rendered_host, void* stream);

/* Forward, stage 2: emit keys, sort, find tile ranges, blend.  out_color (3,H,W), out_others
 * (7,H,W): 0 = sum w*depth, 1 = alpha, 2-4 = view-space normal, 5 = median depth, 6 = distortion
 * (channel order consumed at /root/reference/gaussian_renderer/__init__.py:118-135). */
int surfel_forward_render(const surfel_settings_t* s, int P, uint32_t R, const int32_t* radii,
                          const void* geom_ws, void* binning_ws, void* image_ws, int tile_counts_ready,
                          float* out_color, float* out_others, void* stream);

/* The two halves of stage 2, exposed separately for parity tests. */
int surfel_bin_duplicate(const surfel_settings_t* s, int P, uint32_t R, const void* geom_ws,
                         const int32_t* radii, void* binning_ws, void* stream);
int surfel_bin_sort(const surfel_settings_t* s, uint32_t R, void* binning_ws, void* stream);
/* Production binning used by surfel_forward_render: counting scatter of (depth|idx) pairs into tile
 * buckets + per-tile shared-memory sort; fills ranges and the point list (vals_sorted), and the
 * sorted keys too when write_keys != 0.  Result is identical to surfel_bin_duplicate + surfel_bin_sort
 * (the CUB-free device-wide radix sort), which stays selectable with SURFEL_SORT=radix. */
int surfel_bin_bucket(const surfel_settings_t* s, int P, uint32_t R, const void* geom_ws,
                      const int32_t* radii, void* binning_ws, const void* image_ws_with_counts,
                      int write_keys, void* stream);
int surfel_render_forward(const surfel_settings_t* s, uint32_t R, const void* geom_ws,
                          const void* binning_ws, void* image_ws, float* out_color,
                          float* out_others, void* stream);

/* Backward.  dL_dout_color (3,H,W), dL_dout_others (7,H,W).  grad_scratch: P *
 * surfel_grad_scratch_floats() floats (zeroed here).  Outputs are written for every splat (zeros where culled), so they may be uninitialised:
 *   dL_dmeans2D (P,3) [densification proxy in .xy, SURVEY A.5], dL_dcolors (P,3),
 *   dL_dopacity (P,1), dL_dmeans3D (P,3), dL_dtransMat (P,9), dL_dsh (P,M,3),
 *   dL_dscales (P,2), dL_drotations (P,4).  Optional outputs may be NULL when the matching input
 *   is absent.  lowpass_depth_quirk: 1 = the published upstream kernel's depth gradient in the low-pass
 *   branch, dL_dTw += (s.x, s.y, 1) * dL_dz (what callers should pass: the reference trains on it);
 *   0 = the exact derivative of the forward there, (0, 0, 1) * dL_dz.  See DESIGN.md. */
int surfel_grad_scratch_floats(void);
int surfel_backward(const surfel_settings_t* s, int P, int M, uint32_t R, const float* means3D,
                    const float* scales, const float* rotations, const float* transMat_precomp,
                    const float* shs, int has_colors_precomp, const int32_t* radii,
                    const void* geom_ws, const void* binning_ws, const void* image_ws,
                    const float* dL_dout_color, const float* dL_dout_others, float* grad_scratch,
                    float* dL_dmeans2D, float* dL_dcolors, float* dL_dopacity, float* dL_dmeans3D,
                    float* dL_dtransMat, float* dL_dsh, float* dL_dscales, float* dL_drotations,
                    int lowpass_depth_quirk, void* stream);

/* dL_dsh (P,M,3) = basis_k(normalize(means3D - campos)) * dL_dcolors[c] for k < (sh_degree+1)^2, zero beyond:
 * the expansion surfel_backward() skips when surfel_settings.sh_grad_deferred = 1.  Rows of splats whose
 * colour gradient is exactly zero are zero. */
int surfel_sh_grad_expand(int P, int M, int sh_degree, const float* means3D, const float* campos,
                          const float* dL_dcolors, float* dL_dsh, void* stream);

/* GaussianRasterizer.markVisible: near-plane test (present: P bytes, 0/1). */
int surfel_mark_visible(int P, const float* means3D, const float* viewmatrix,
                        const float* projmatrix, uint8_t* present, void* stream);

/* Stand-alone CUB-free stable radix sort of (u64 key, u32 value) pairs on key bits [0,end_bit).
 * Data starts in A; *result_in_b tells where the sorted pairs are (buffers ping-pong per pass). */
size_t surfel_sort_temp_bytes(size_t n);
int surfel_sort_pairs(uint64_t* keys_a, uint32_t* vals_a, uint64_t* keys_b, uint32_t* vals_b,
                      size_t n, int end_bit, void* temp, int* result_in_b, void* stream);

/* OPT-IN fused post-process of the op's allmap (SURVEY §8f row f1): what the reference's render() does
 * with ~10 PyTorch kernels per direction at /root/reference/gaussian_renderer/__init__.py:118-147 and
 * /root/reference/utils/point_utils.py:9-37.  rot (9): n_world = n_view . rot (= world_view[:3,:3]^T);
 * rays (12): 3x3 pixel->world ray matrix (row-major, dir = (x,y,1).M) followed by the camera centre.
 * Outputs: rend_normal (3,H,W), surf_depth (1,H,W), surf_normal (3,H,W).  Backward: cotangents of the
 * three outputs (any may be NULL), tmp6 = (6,H,W) scratch, g_allmap (7,H,W) fully written. */
int surfel_post_forward(int W, int H, float depth_ratio, const float* allmap, const float* rot,
                        const float* rays, float* rend_normal, float* surf_depth, float* surf_normal,
                        void* stream);
int surfel_post_backward(int W, int H, float depth_ratio, const float* allmap, const float* rot,
                         const float* rays, const float* surf_depth, const float* g_rend_normal,
                         const float* g_surf_depth, const float* g_surf_normal, float* tmp6,
                         float* g_allmap, void* stream);

/* OPT-IN fused 2DGS regularisers (SURVEY §8f row f2), straight from allmap with no intermediate plane:
 *   normal_loss = lambda_normal * mean(1 - sum_c rend_normal_c * surf_normal_c)
 *   dist_loss   = lambda_dist * mean(rend_dist)
 * with rend_normal, surf_normal (alpha detached, zero on the border) as surfel_post_forward computes them and
 * rot / rays as there.  Forward: partials is device scratch of surfel_post_reg_partials_bytes(W, H) bytes
 * (0 for a bad size); normal_loss and dist_loss are one device float each.  The sums are reduced in double in
 * a fixed order, so the values are bit-identical from run to run and on any stream.  Backward: gscale2
 * (device, 2 floats) = (dL/dnormal_loss * lambda_normal / N, dL/ddist_loss * lambda_dist / N), N = W * H;
 * tmp6 = (6,H,W) scratch, required only when lambda_normal != 0; g_allmap (7,H,W) fully written.  Where
 * D / alpha is not finite its term contributes 0 to channels 0 and 1.  lambda_normal == 0 skips the stencil
 * (normal_loss and channels 0-5 exactly 0); with both lambdas 0 nothing reads allmap. */
size_t surfel_post_reg_partials_bytes(int W, int H);
int surfel_post_reg_forward(int W, int H, float depth_ratio, double lambda_normal, double lambda_dist,
                            const float* allmap, const float* rot, const float* rays, double* partials,
                            float* normal_loss, float* dist_loss, void* stream);
int surfel_post_reg_backward(int W, int H, float depth_ratio, double lambda_normal, double lambda_dist,
                             const float* allmap, const float* rot, const float* rays, const float* gscale2,
                             float* tmp6, float* g_allmap, void* stream);

/* OPT-IN fused photometric loss (SURVEY §8f row f2): (1-l)*L1 + l*(1-SSIM) of
 * /root/reference/train.py:73-74 with /root/reference/utils/loss_utils.py:6-7, :43-73 (11x11 Gaussian
 * window, sigma 1.5, zero padding, per channel).  forward: sums2[0] = sum |img-gt|, sums2[1] = sum of
 * the SSIM map (doubles, device) and the three (C,H,W) derivative maps the backward consumes.
 * backward: gscale2 (device, 2 floats) = dL/d(sums2); g_img (C,H,W) fully written. */
int surfel_l1_ssim_forward(int C, int H, int W, const float* img, const float* gt, float* dmu1,
                           float* ds11, float* ds12, double* sums2, void* stream);
int surfel_l1_ssim_backward(int C, int H, int W, const float* img, const float* gt, const float* dmu1,
                            const float* ds11, const float* ds12, const float* gscale2, float* g_img,
                            void* stream);

/* ---- SURVEY §8(f) row f3: the parameter update after the backward -------------------------------
 * surfel_adam_step replaces torch.optim.Adam(l, lr=0.0, eps=1e-15).step() of the reference
 * (/root/reference/scene/gaussian_model.py:148-166, /root/reference/train.py:138-140): ONE launch
 * updates every parameter group in place (param, exp_avg, exp_avg_sq), arithmetic as torch's
 * single-tensor Adam (no weight decay, no amsgrad).  The host folds the step count into
 *   step_size = lr / (1 - beta1^step),   bias2_sqrt = sqrt(1 - beta2^step)
 * (in double, as torch does); betas and eps are doubles so that 1 - beta is rounded once.
 * surfel_densify_stats replaces /root/reference/train.py:125-128 (max_radii2D update) and
 * /root/reference/scene/gaussian_model.py:405-407 (add_densification_stats): where radii > 0,
 *   max_radii2D = max(max_radii2D, radii); xyz_gradient_accum += |means2D_grad (3)|; denom += 1.
 * max_radii2D may be NULL. */
#define SURFEL_ADAM_MAX_GROUPS 8
typedef struct surfel_adam_group {
    float* param;            /* n floats, updated in place */
    const float* grad;       /* n floats */
    float* exp_avg;          /* n floats, updated in place */
    float* exp_avg_sq;       /* n floats, updated in place */
    long long n;
    float step_size;
    float bias2_sqrt;
    int aligned16;           /* filled in by the library */
} surfel_adam_group_t;
int surfel_adam_step(int n_groups, const surfel_adam_group_t* groups, double beta1, double beta2, double eps,
                     void* stream);
int surfel_densify_stats(int P, const int32_t* radii, const float* means2D_grad, float* xyz_gradient_accum,
                         float* denom, float* max_radii2D, void* stream);

/* ---- SURVEY §8(f) row f4: the model's on-disk format either side of the path ------------------
 * The reference saves / loads a trained model as a binary little-endian PLY with one row of 61
 * float32 per splat, pre-activation, SH channel-major (/root/reference/scene/gaussian_model.py:176-209
 * save_ply, :215-255 load_ply):  x y z nx ny nz f_dc_0..2 f_rest_0..44 opacity scale_0..1 rot_0..3.
 * surfel_ply_unpack turns raw rows (device memory, `row_floats` floats each, any property order)
 * into the rasterizer's inputs in one pass.  columns[58] gives, for every target float, its column
 * in the row; target order: 0..2 xyz | 3..50 shs[k][c] (coefficient-major (16,3): k = 0 is f_dc_c,
 * k >= 1 is f_rest_{c*15 + k-1}) | 51 opacity | 52..53 scale | 54..57 rot (w,x,y,z).
 * activate = 1 applies what the reference's getters apply before the op (gaussian_model.py:35-41,
 * :95-115): opacity = sigmoid, scale = exp, rot = q / max(|q|, 1e-12); activate = 0 leaves the
 * stored parameters.  surfel_ply_pack is the inverse of save_ply's gather: parameters
 * (xyz (P,3), features_dc (P,1,3), features_rest (P,15,3), opacity (P,1), scaling (P,2),
 * rotation (P,4)) -> rows in the reference's column order with zero normals. */
#define SURFEL_PLY_ROW_FLOATS 61
#define SURFEL_PLY_TARGETS 58
#define SURFEL_PLY_MAX_ROW_FLOATS 127
int surfel_ply_unpack(int P, int row_floats, const float* rows, const int32_t* columns, int activate,
                      float* means3D, float* shs, float* opacities, float* scales, float* rotations, void* stream);
int surfel_ply_pack(int P, const float* xyz, const float* features_dc, const float* features_rest,
                    const float* opacity, const float* scaling, const float* rotation, float* rows, void* stream);

/* ---- Model initialisation: simple_knn.distCUDA2 of /root/reference/scene/gaussian_model.py:20, :134 ----
 * out[i] = mean of the squared distances from point i to its three nearest OTHER points (rules: DESIGN.md
 * §7g, csrc/knn.cu).  Exact; d2 = (dx*dx + dy*dy) + dz*dz in float32 without FMA, result ((a+b)+c)/3.0f
 * over the three smallest, so it is bit-reproducible.  Fewer than three finite other points: the mean over
 * those that exist (0 if none).  A row with a NaN / inf coordinate is nobody's neighbour and gets NaN.
 * xyz: (P,3) contiguous float32; out: (P) float32; workspace: surfel_knn_workspace_bytes(P) bytes
 * (uninitialised is fine), its size passed as workspace_bytes.  P = 0 launches nothing; P must be below
 * 2^30 (surfel_knn_workspace_bytes returns 0 for a P out of range). */
size_t surfel_knn_workspace_bytes(int P);
int surfel_knn_mean_sq_dist(int P, const float* xyz, float* out, void* workspace, size_t workspace_bytes,
                            void* stream);

/* ---- Densification: GaussianModel.densify_and_prune of the reference trainer ----------------------
 * (scene/gaussian_model.py:348-403, train.py:132; rules in DESIGN.md §7h, csrc/densify.cu).  Clone, split
 * and the final prune of every parameter group and its Adam moments, as one compaction:
 *  surfel_densify_plan decides every row from (xyz_gradient_accum (P,1), denom (P,1), scaling (P,2),
 *   opacity (P,1)) and writes totals[4] (device int32) = { kept originals, kept clones, split rows S, P' }.
 *   The thresholds are the doubles Python forms (max_grad, min_opacity, percent_dense * extent,
 *   0.1 * extent, max_screen_size), each rounded once to float32 as torch does when it compares; the
 *   screen-size and world-size prune apply only when use_max_screen_size is non-zero.
 *  surfel_densify_apply then writes the P' output rows of every group: kept originals (moments kept) |
 *   kept clones | kept split copies A | kept split copies B (zero moments).  P_out and n_split are
 *   totals[3] and totals[2] as read back by the caller; z is the (2 n_split, 3) standard normal draw (rows
 *   [0, S) for copies A, [S, 2S) for copies B, in split-row order).  A group with NULL moments has no
 *   optimizer state and is gathered without it.  At most one group each of kind XYZ (3 floats per row),
 *   SCALING (2) and ROTATION (4), and a table with the XYZ group needs the other two (split copies' xyz reads
 *   them); the others are COPY.  The groups of one plan may be split over several apply calls (the Python
 *   wrapper applies f_rest first and frees its old tensors before it allocates the other groups' new ones).
 * All float arrays are contiguous float32; the workspace is surfel_densify_workspace_bytes(P) bytes
 * (uninitialised is fine) and must be the same between the plan and the apply of one call.  P must be
 * below 2^30 (surfel_densify_workspace_bytes returns 0 for a P out of range). */
#define SURFEL_DENSIFY_MAX_GROUPS 8
enum { SURFEL_DENSIFY_COPY = 0, SURFEL_DENSIFY_XYZ = 1, SURFEL_DENSIFY_SCALING = 2, SURFEL_DENSIFY_ROTATION = 3 };
typedef struct surfel_densify_group {
    const float* param;        /* P rows of row_floats */
    const float* exp_avg;      /* P rows, or NULL (no state) */
    const float* exp_avg_sq;   /* P rows, or NULL (no state) */
    float* out_param;          /* P' rows */
    float* out_exp_avg;        /* P' rows; NULL iff exp_avg is NULL */
    float* out_exp_avg_sq;     /* P' rows; NULL iff exp_avg_sq is NULL */
    int row_floats;
    int kind;                  /* SURFEL_DENSIFY_* */
} surfel_densify_group_t;
size_t surfel_densify_workspace_bytes(int P);
int surfel_densify_plan(int P, const float* xyz_gradient_accum, const float* denom, const float* scaling,
                        const float* opacity, double max_grad, double min_opacity, double clone_max_scale,
                        double prune_max_scale, int use_max_screen_size, double max_screen_size, void* workspace,
                        size_t workspace_bytes, int32_t* totals, void* stream);
int surfel_densify_apply(int P, int P_out, int n_split, int n_groups, const surfel_densify_group_t* groups,
                         const float* z, const void* workspace, size_t workspace_bytes, void* stream);

/* ---- Mesh extraction: the SDF field of GaussianExtractor.extract_mesh_unbounded ------------------
 * (utils/mesh_utils.py:184-279 of the reference, `render.py --unbounded`; rules and quirks in DESIGN.md §7i,
 * csrc/tsdf.cu).  Folds every frame, in table order, into each of n_points samples in one pass:
 *  field mode (rgb == NULL): points are in contracted space.  Each gets the adaptive truncation
 *   trunc * 1/(2 - min(|y|, 1.9)) where |y| > 1, is uncontracted and unnormalized (x * radius + center), and
 *   out[i] (n_points floats) is the running TSDF mean, starting at -1 with weight 1.
 *  colour mode (rgb != NULL): points are world points, the truncation is the scalar, and out (n_points x 3
 *   floats) is the running mean of the sampled RGB, starting at 0 with weight 1.
 * A frame counts for a sample when the projected pix = xy / w lies strictly inside (-1, 1)^2, w > 0 and
 * depth - w > -trunc, with depth (and RGB) sampled as grid_sample(bilinear, border, align_corners=True).
 * points: (n_points, 3) contiguous float32 on the device.  frames: a HOST table of n_frames entries, copied to
 * the device in stream order by the call.  depth: the frames' (H, W) maps concatenated, map_pixels floats, frame
 * f at frames[f].offset; rgb: their (3, H, W) maps concatenated in the same order (frame f at 3 * offset).
 * center: 3 host floats; radius and trunc are the doubles the caller forms, each rounded once to float32.
 * Each side of a frame must be in [1, 2^24] and the frame inside map_pixels.  Runs on `stream`, needs no
 * workspace and does not synchronise; the result is bit-reproducible (fixed, uncontracted float32 arithmetic). */
typedef struct surfel_tsdf_frame {
    float full_proj_transform[16];   /* row-major 4x4: the homogeneous point is the row vector [x y z 1] times it */
    int32_t height, width;
    int64_t offset;                  /* element offset of the frame's depth map in `depth` */
} surfel_tsdf_frame_t;
int surfel_tsdf_eval(long long n_points, const float* points, int n_frames, const surfel_tsdf_frame_t* frames,
                     long long map_pixels, const float* depth, const float* rgb, const float* center, double radius,
                     double trunc, float* out, void* stream);
/* Grid mode of the field (DESIGN.md §7j): the side^3 points of one crop, torch.linspace(bounds[2d], bounds[2d+1], side)
 * on each axis d (bounds: 6 host doubles x0, x1, y0, y1, z0, z1, each rounded once to float32) laid out as
 * meshgrid(indexing="ij") lays them out, x slowest.  out (side^3 floats) is what surfel_tsdf_eval in field mode
 * returns for those points, without a points buffer.  side in [2, 512]. */
int surfel_tsdf_eval_grid(int side, const double* bounds, int n_frames, const surfel_tsdf_frame_t* frames,
                          long long map_pixels, const float* depth, const float* center, double radius, double trunc,
                          float* out, void* stream);

/* ---- Mesh extraction: marching cubes over contracted crops (marching_cubes_with_contraction of the reference's
 * utils/mcube_utils.py; rules in DESIGN.md §7j, csrc/mcubes.cu).  The grid is crops_per_axis^3 crops of side^3
 * points, crop (i, j, k) covering global points [i, j, k] * (side - 1) + [0, side); neighbouring crops share
 * their boundary plane, which must hold the same values in both.  A corner is inside iff its value is < 0.
 *  surfel_mcubes_crop_count: counts the crop's vertex records (the crossing edges it owns) and triangles into
 *   totals[0] and totals[1] (device int64), and keeps per-block offsets in the workspace
 *   (surfel_mcubes_crop_workspace_bytes(side) bytes, uninitialised is fine).
 *  surfel_mcubes_crop_emit: with the same arguments and workspace, and the crop's bounds (as in
 *   surfel_tsdf_eval_grid) and totals, writes n_records vertex keys (uint64) and contracted positions (3 floats
 *   each), and n_tris triangles as key triples (uint64), in cube order (x slowest) then table order.
 *  surfel_mcubes_merge: over the records and triangles of all crops, in crop order: writes the distinct keys'
 *   vertices in ascending key order, uncontracted (DESIGN.md §7i rule 3), scaled by radius, moved by the 3 host
 *   floats of center and clipped to [-32, 32], to verts (at least n_records rows of 3 floats), their number to
 *   n_verts (device int64), and each triangle's vertex indices to faces (n_tris rows of 3 int64).  key_bits: the
 *   bits of the largest key, 4 * G^3 - 1 with G = (side - 1) * crops_per_axis + 1.  n_records must be below 2^30;
 *   the workspace is surfel_mcubes_merge_workspace_bytes(n_records) bytes (0 when out of range).
 * All three run on `stream` and do not synchronise; the caller reads the totals to size the outputs. */
size_t surfel_mcubes_crop_workspace_bytes(int side);
int surfel_mcubes_crop_count(int side, const float* volume, const int* crop, int crops_per_axis, void* workspace,
                             size_t workspace_bytes, long long* totals, void* stream);
int surfel_mcubes_crop_emit(int side, const float* volume, const double* bounds, const int* crop, int crops_per_axis,
                            const void* workspace, size_t workspace_bytes, long long n_records, long long n_tris,
                            unsigned long long* vert_keys, float* vert_pos, unsigned long long* tri_keys,
                            void* stream);
size_t surfel_mcubes_merge_workspace_bytes(long long n_records);
int surfel_mcubes_merge(long long n_records, const unsigned long long* vert_keys, const float* vert_pos,
                        long long n_tris, const unsigned long long* tri_keys, int key_bits, const float* center,
                        double radius, void* workspace, size_t workspace_bytes, float* verts, long long* faces,
                        long long* n_verts, void* stream);

/* ---- Mesh cluster filtering (post_process_mesh of the reference's utils/mesh_utils.py; rules in DESIGN.md §7k,
 * csrc/meshpost.cu).  A mesh of n_verts vertices and n_faces faces (rows of 3 int64 vertex indices) on the device;
 * n_verts below 2^31 and 3 * n_faces below 2^30.  Both calls use a workspace of
 * surfel_meshpost_workspace_bytes(n_verts, n_faces) bytes (0 when out of range; uninitialised is fine), run on
 * `stream` and do not synchronise.
 *  surfel_meshpost_clusters: the faces' connected components over shared edges (unordered vertex-index pairs),
 *   numbered by the rank of each component's smallest face: each face's cluster id to face_cluster (n_faces int32),
 *   each cluster's face count to cluster_count[0, C) (n_faces int32 are written), C to info[0] and 1 to info[1] if
 *   any face index lies outside [0, n_verts), else 0 (info: 2 device int64).  Only when info[1] is 0 do the ids
 *   and counts mean anything.
 *  surfel_meshpost_compact: with those ids and counts, C = n_clusters and index in [0, C): keeps the faces whose
 *   cluster has at least max(the index-th smallest count, 50) faces; writes the old index of each vertex that a kept
 *   face references, in order, to vert_map (n_verts int64), the kept faces that are not degenerate (three distinct
 *   indices), in order and renumbered, to out_faces (n_faces rows of 3 int64), and the number of each to info[0]
 *   and info[1]. */
size_t surfel_meshpost_workspace_bytes(long long n_verts, long long n_faces);
int surfel_meshpost_clusters(long long n_verts, long long n_faces, const long long* faces, void* workspace,
                             size_t workspace_bytes, int* face_cluster, int* cluster_count, long long* info,
                             void* stream);
int surfel_meshpost_compact(long long n_verts, long long n_faces, const long long* faces, const int* face_cluster,
                            const int* cluster_count, long long n_clusters, long long index, void* workspace,
                            size_t workspace_bytes, long long* out_faces, long long* vert_map, long long* info,
                            void* stream);

/* ---- DTU Chamfer evaluation (scripts/eval_dtu/eval.py of the reference; rules in DESIGN.md §7m, csrc/chamfer.cu).
 * Everything is float64 rows of 3 on the device; every call runs on `stream`.  Point sets hold at most
 * surfel_chamfer_max_points() points (the radix sort's limit).
 *  surfel_chamfer_sample_count: per triangle of the mesh (faces: n_faces rows of 3 int64), the number of points
 *   the reference's sampling emits at density `thresh`; info (4 device int64): [0] their sum (a triangle beyond the
 *   limit counts 2^31), [1] 1 if a face index lies outside [0, n_verts), [2] 1 if a vertex coordinate is not finite,
 *   [3] the number of triangles of positive area.  The workspace is surfel_chamfer_sample_workspace_bytes(n_faces).
 *  surfel_chamfer_sample_emit: with the same workspace and n_samples = info[0], writes the samples, in triangle and
 *   row-major order, to rows n_verts .. n_verts + n_samples - 1 of out (rows 0 .. n_verts - 1 are the caller's).
 *  The next three share one workspace of surfel_chamfer_workspace_bytes(n_points, n_stl) bytes, in this order:
 *  surfel_chamfer_downsample: the greedy radius-`thresh` downsampling of the (already shuffled) cloud, kept in the
 *   workspace; synchronises the stream once per eight rounds and returns the number of rounds in *rounds.
 *  surfel_chamfer_select: the kept points to data_down, those inside [box_lo, box_hi) to data_in, those of data_in
 *   whose cell rint((x - bb0) / res) of the X*Y*Z mask obs_mask (uint8, C order) is set to data_in_obs with their
 *   data_down row in obs_down, and the STL points above `plane` to stl_above with their STL row in above_idx
 *   (every output sized for all points); the four counts to info (4 device int64).
 *  surfel_chamfer_distances: with those counts (each set non-empty), the distance of each data_in_obs row to the
 *   STL and of each stl_above row to data_in (+inf at or beyond max_dist) to dist_d2s / dist_s2d, the colours of
 *   data_down (n_down rows) and of the STL (n_stl rows), and (sum, count) of the distances below max_dist of each
 *   pass to sums[0..1] and sums[2..3]. */
long long surfel_chamfer_max_points(void);
size_t surfel_chamfer_sample_workspace_bytes(long long n_faces);
int surfel_chamfer_sample_count(long long n_verts, long long n_faces, const double* verts, const long long* faces,
                                double thresh, void* workspace, size_t workspace_bytes, long long* info,
                                void* stream);
int surfel_chamfer_sample_emit(long long n_verts, long long n_faces, const double* verts, const long long* faces,
                               double thresh, void* workspace, size_t workspace_bytes, long long n_samples,
                               double* out, void* stream);
size_t surfel_chamfer_workspace_bytes(long long n_points, long long n_stl);
int surfel_chamfer_downsample(long long n_points, long long n_stl, const double* pcd, double thresh,
                              void* workspace, size_t workspace_bytes, int* rounds, void* stream);
int surfel_chamfer_select(long long n_points, long long n_stl, const double* pcd, const double* stl,
                          const double* box_lo, const double* box_hi, const double* bb0, double res,
                          const unsigned char* obs_mask, const int* obs_shape, const double* plane, void* workspace,
                          size_t workspace_bytes, double* data_down, double* data_in, double* data_in_obs,
                          unsigned int* obs_down, double* stl_above, unsigned int* above_idx, long long* info,
                          void* stream);
int surfel_chamfer_distances(long long n_points, long long n_stl, const double* stl, long long n_down, long long n_in,
                             const double* data_in, long long n_obs, const double* data_in_obs,
                             const unsigned int* obs_down, long long n_above, const double* stl_above,
                             const unsigned int* above_idx, double max_dist, double vis, void* workspace,
                             size_t workspace_bytes, double* dist_d2s, double* dist_s2d, double* data_color,
                             double* stl_color, double* sums, void* stream);

/* ---- DTU mask culling (cull_scan of the reference's scripts/eval_dtu/evaluate_single_scene.py; rules in DESIGN.md
 * §7n, csrc/cull.cu).  n_views masks of height x width bytes (C order, nonzero = set), 1 <= n_views <=
 * surfel_cull_max_views(), each side in [1, 32768]; meshes of at most 2^31 - 1 vertices and faces.  One workspace of
 * surfel_cull_workspace_bytes(n_views, height, width, n_verts, n_faces) bytes (0 when out of range; uninitialised is
 * fine) serves the three calls, in this order; each runs on `stream` and does not synchronise.
 *  surfel_cull_dilate: each mask dilated by disk(radius) with a zero border, 0 <= radius <= surfel_cull_max_radius(),
 *   bit-packed to dilated: n_views * height rows of ceil(width / 32) words, pixel x of a row in bit x % 32 of word
 *   x / 32, bits beyond the width clear.
 *  surfel_cull_vertices: verts (n_verts rows of 3 float64) against the dilated masks through proj (n_views rows of
 *   3 x 4 float32, device) with the image size image_width x image_height: 1 or 0 per vertex to keep (n_verts bytes);
 *   info (4 device int64): [0] 1 if a face index (faces: n_faces rows of 3 int64) lies outside [0, n_verts), [1] 1 if
 *   a vertex coordinate is not finite in float32, [2] the kept vertices, [3] the kept faces (all three vertices kept).
 *  surfel_cull_emit: with the same workspace and n_kept_verts = info[2], n_kept_faces = info[3], the kept vertices
 *   in order as v * world[0] + world[1..3] (float64, world: 4 host doubles) to out_verts (n_kept_verts rows of 3),
 *   their colour rows (color_row_bytes each, 0 for none) to out_colors, and the kept faces in order, renumbered, to
 *   out_faces (n_kept_faces rows of 3 int64).  Outputs with nothing to hold may be NULL. */
int surfel_cull_max_views(void);
int surfel_cull_max_radius(void);
size_t surfel_cull_workspace_bytes(long long n_views, int height, int width, long long n_verts, long long n_faces);
int surfel_cull_dilate(int n_views, int height, int width, int radius, const unsigned char* masks, void* workspace,
                       size_t workspace_bytes, unsigned int* dilated, void* stream);
int surfel_cull_vertices(long long n_verts, const double* verts, long long n_faces, const long long* faces,
                         int n_views, const float* proj, int image_width, int image_height, int height, int width,
                         const unsigned int* dilated, void* workspace, size_t workspace_bytes, unsigned char* keep,
                         long long* info, void* stream);
int surfel_cull_emit(long long n_verts, const double* verts, long long n_faces, const long long* faces,
                     const double* world, const void* colors, long long color_row_bytes, const void* workspace,
                     size_t workspace_bytes, long long n_kept_verts, long long n_kept_faces, double* out_verts,
                     long long* out_faces, void* out_colors, void* stream);

/* ---- Novel-view metrics (metrics.py of the reference: PSNR of utils/image_utils.py and LPIPS-VGG of lpipsPyTorch;
 * rules in DESIGN.md §7o, csrc/metrics.cu).  SSIM is surfel_l1_ssim_forward's sums[1] / (C H W).  Activations are
 * NHWC float32 batches of n images (n = 2 for LPIPS: render then gt).  Each call runs on `stream` and does not
 * synchronise.
 *  surfel_metrics_lpips_input: x, y (3 x H x W each, device) z-scored into out (2 x H x W x 3).  Rejects n != 1,
 *   c != 3, a side outside [surfel_metrics_min_side(), surfel_metrics_max_side()] and host memory.
 *  surfel_metrics_pack_conv: a conv weight [cout][cin][3][3] to packed [cout][3][3][cin] (rounded to TF32, to
 *   nearest, when cin % 32 == 0; cin 3 is copied).  cout a multiple of 64.
 *  surfel_metrics_conv3x3: relu(conv3x3(in, packed, padding 1) + bias), in n x H x W x cin, out n x H x W x cout.
 *   cin 3 with cout 64 runs in float32; cin % 32 == 0 runs on the TF32 tensor cores (wgmma).
 *  surfel_metrics_maxpool: 2 x 2 stride-2 max-pool with floor, n x H x W x c to n x (H/2) x (W/2) x c, c % 4 == 0.
 *  surfel_metrics_lpips_tap: tap (0..4) of the 2 x H x W x c features: the sum over pixels of
 *   lin . (fx / (|fx| + 1e-10) - fy / (|fy| + 1e-10))^2, as fixed per-block partials in partials (double, at least
 *   surfel_metrics_partials_count(1) entries).
 *  surfel_metrics_lpips_finish: out[0] = sum over taps of float32(partial sum / tap_pixels_host[t]); taps (5 floats,
 *   may be NULL) gets each tap's mean.
 *  surfel_metrics_psnr: out[i] = float32(20 log10(1 / sqrt(mse_i))), mse of the i-th per_image floats of a and b
 *   summed in double; partials holds surfel_metrics_partials_count(n) doubles. */
int surfel_metrics_min_side(void);
int surfel_metrics_max_side(void);
size_t surfel_metrics_partials_count(int n_images);
int surfel_metrics_lpips_input(int n, int c, int height, int width, const float* x, const float* y, float* out,
                               void* stream);
int surfel_metrics_pack_conv(int cout, int cin, const float* w, float* packed, void* stream);
int surfel_metrics_conv3x3(int n, int height, int width, int cin, int cout, const float* in, const float* packed,
                           const float* bias, float* out, void* stream);
int surfel_metrics_maxpool(int n, int height, int width, int c, const float* in, float* out, void* stream);
int surfel_metrics_lpips_tap(int tap, int height, int width, int c, const float* feat, const float* lin,
                             double* partials, void* stream);
int surfel_metrics_lpips_finish(const long long* tap_pixels_host, const double* partials, float* out, float* taps,
                                void* stream);
int surfel_metrics_psnr(int n, long long per_image, const float* a, const float* b, double* partials, float* out,
                        void* stream);

/* Instrumentation used by bench.py: number of kernels this library has launched in this process,
 * and optional per-stage CUDA-event timing (events recorded on the launching stream around each
 * kernel while enabled; surfel_profile_read() waits for them and returns summed ms / launch counts
 * per stage since the previous read). */
unsigned long long surfel_launch_count(void);
void surfel_profile_enable(int on);
int surfel_profile_num_stages(void);
const char* surfel_profile_stage_name(int stage);
int surfel_profile_read(double* ms_out, int* count_out);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_RASTERIZER_H_ */
