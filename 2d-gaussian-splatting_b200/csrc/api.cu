// api.cu — the C-ABI entry points declared in include/surfel_rasterizer.h.
// Thin: argument checks, workspace carving, kernel launches on the caller's stream.  No torch.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <algorithm>

#include "../../include/surfel_rasterizer.h"
#include "common.cuh"
#include "kernels.h"

using namespace surfel;

static thread_local char g_err[512] = "";

void surfel_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

namespace {

// Kernel variants (same architecture, alternative implementations kept for A/B measurement).
// Defaults come from the environment once; surfel_set_variant() changes them at run time (tests).
struct Variants { int sort_radix; };
Variants& variants() {
    static Variants v = [] {
        auto is = [](const char* name, const char* val) { const char* e = getenv(name); return e && !strcmp(e, val) ? 1 : 0; };
        return Variants{is("SURFEL_SORT", "radix")};
    }();
    return v;
}

struct Frame { int W, H, gx, gy, row0, row1, tiles; };

bool frame_of(const surfel_settings_t* s, Frame& f) {
    if (!s) { surfel_set_error("settings is NULL"); return false; }
    f.W = s->image_width; f.H = s->image_height;
    if (f.W <= 0 || f.H <= 0) { surfel_set_error("bad image size %dx%d", f.W, f.H); return false; }
    f.gx = (f.W + kBlockX - 1) / kBlockX; f.gy = (f.H + kBlockY - 1) / kBlockY;
    f.tiles = f.gx * f.gy;
    f.row0 = s->tile_row_begin; f.row1 = s->tile_row_end;
    if (f.row0 == 0 && f.row1 == 0) f.row1 = f.gy;
    if (f.row0 < 0 || f.row1 > f.gy || f.row0 > f.row1) {
        surfel_set_error("bad tile row band [%d,%d) for %d tile rows", f.row0, f.row1, f.gy);
        return false;
    }
    return true;
}

// keys are tile << 32 | depth bits; the width covers tile indices up to `tiles` itself
int tile_key_bits(int tiles) { return radix_key_bits((unsigned long long)(unsigned)tiles << 32 | 0xffffffffull); }

size_t binning_pairs(size_t R) { return R > 0 ? R : 1; }

BinningLayout binning_layout(size_t R, int tiles) {
    BinningLayout L;
    const size_t r = binning_pairs(R);
    size_t o = 0;
    L.pairs = o;  o = align_up(o + radix_sort_pairs_bytes(r), 256);
    L.ranges = o; o = align_up(o + (size_t)tiles * 8, 256);
    L.temp = o;   o = align_up(o + std::max(radix_sort_temp_bytes(r), bucket_temp_bytes(tiles)), 256);
    L.total = o;
    return L;
}

// sort.in: duplicated keys and values; sort.out: the sorted ones, whichever sort bins them
struct BinView { RadixSortWs sort; uint2* ranges; };

BinView bin_view(void* ws, size_t R, int tiles) {
    const BinningLayout L = binning_layout(R, tiles);
    char* c = (char*)ws;
    return BinView{radix_sort_ws(c + L.pairs, binning_pairs(R), tile_key_bits(tiles), c + L.temp),
                   (uint2*)(c + L.ranges)};
}

// Device-visible alias of a pinned (cudaHostAlloc / cudaHostRegister, mapped) host word, or nullptr
// for pageable memory.  Queried on every call (about a microsecond): a cached answer could outlive
// the allocation it described.
uint32_t* mapped_alias(uint32_t* host) {
    if (!host) return nullptr;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, host) == cudaSuccess && a.type == cudaMemoryTypeHost && a.devicePointer)
        return (uint32_t*)a.devicePointer;
    (void)cudaGetLastError();
    return nullptr;
}

// SH degree D is supported (0..3) and its (D + 1)^2 coefficients fit in a row of M
bool sh_degree_ok(int D, int M) { return D >= 0 && D <= 3 && (D + 1) * (D + 1) <= M; }

// the checks and parameters both camera entry points share; `name` prefixes the error messages
bool camera_params(const char* name, const surfel_settings_t* s, int P, int M, const float* means3D,
                   const float* scales, const float* rotations, const float* transMat_precomp, const float* shs,
                   int has_colors_precomp, const int32_t* radii, const void* geom_ws, const float* grad_scratch,
                   const float* dL_dtransMat, double* partials, bool band_ok, const void* out0, const void* out1,
                   const void* out2, Frame& f, CamBwdParams& p) {
    if (!frame_of(s, f)) return false;
    if (P < 0) { surfel_set_error("P < 0"); return false; }
    if (!band_ok && (f.row0 != 0 || f.row1 != f.gy)) { surfel_set_error("%s: a tile-row band has no camera gradient", name); return false; }
    if (!partials || !out0 || !out1 || !out2) { surfel_set_error("%s: NULL output or partials", name); return false; }
    if (P > 0 && (!means3D || !radii || !geom_ws || !grad_scratch)) { surfel_set_error("%s: NULL required input", name); return false; }
    if (P > 0 && !transMat_precomp && (!scales || !rotations || !dL_dtransMat)) {
        surfel_set_error("%s: need scales, rotations and dL_dtransMat, or transMat_precomp", name);
        return false;
    }
    const bool sh = !has_colors_precomp && shs != nullptr;
    if (sh && !sh_degree_ok(s->sh_degree, M)) {
        surfel_set_error("%s: sh_degree %d unsupported for M=%d", name, s->sh_degree, M);
        return false;
    }
    GeomLayout L = geom_layout(P);
    const char* g = (const char*)geom_ws;
    memset(&p, 0, sizeof(p));
    p.P = P; p.D = s->sh_degree; p.M = M; p.W = f.W; p.H = f.H; p.scale_modifier = s->scale_modifier;
    p.means3D = means3D; p.scales = scales; p.rotations = rotations; p.shs = shs;
    p.transMat_precomp = transMat_precomp; p.has_colors_precomp = has_colors_precomp;
    p.viewmatrix = s->viewmatrix; p.campos = s->campos;
    p.radii = radii; p.rec = (const float4*)(g + L.rec); p.clamped = (const uint8_t*)(g + L.clamped);
    p.grad_rec = grad_scratch; p.dL_dtransMat = dL_dtransMat; p.partials = partials;
    return true;
}

}  // namespace

extern "C" {

int surfel_abi_version(void) { return SURFEL_ABI_VERSION; }

int surfel_set_variant(const char* name, const char* value) {
    if (!name || !value) { surfel_set_error("surfel_set_variant: NULL argument"); return 1; }
    Variants& v = variants();
    if (!strcmp(name, "sort")) {
        if (!strcmp(value, "bucket")) v.sort_radix = 0; else if (!strcmp(value, "radix")) v.sort_radix = 1; else goto bad;
    } else goto bad;
    return 0;
bad:
    surfel_set_error("surfel_set_variant: unknown variant %s=%s", name, value);
    return 1;
}
const char* surfel_last_error(void) { return g_err; }

// 1 iff surfel_forward_render accepts an UPPER BOUND of the instance count as R (speculative launch):
// true for the tile-bucketed binning, false for the device-wide radix sort (it sorts exactly R pairs).
int surfel_accepts_capacity(void) { return variants().sort_radix ? 0 : 1; }

size_t surfel_geom_bytes(int P) { return geom_layout(P).total; }
size_t surfel_image_bytes(int W, int H) { return image_layout(W, H).total; }
size_t surfel_binning_bytes(size_t R, int W, int H) {
    const int tiles = ((W + kBlockX - 1) / kBlockX) * ((H + kBlockY - 1) / kBlockY);
    return binning_layout(R, tiles).total;
}

int surfel_geom_offsets(int P, size_t* out) {
    GeomLayout L = geom_layout(P);
    out[0] = L.rec; out[1] = L.tiles_touched; out[2] = L.offsets; out[3] = L.clamped; out[4] = L.counters;
    out[5] = L.tmat;
    return 0;
}
int surfel_binning_offsets(size_t R, int W, int H, size_t* out) {
    const int tiles = ((W + kBlockX - 1) / kBlockX) * ((H + kBlockY - 1) / kBlockY);
    const BinView v = bin_view(nullptr, R, tiles);   // at base 0 every address is an offset
    out[0] = (size_t)v.sort.in.keys; out[1] = (size_t)v.sort.in.vals;
    out[2] = (size_t)v.sort.out.keys; out[3] = (size_t)v.sort.out.vals;
    out[4] = (size_t)v.ranges;
    return 0;
}
int surfel_image_offsets(int W, int H, size_t* out) {
    ImageLayout L = image_layout(W, H);
    out[0] = L.accum; out[1] = L.n_contrib;
    return 0;
}

int surfel_forward_preprocess(const surfel_settings_t* s, int P, int M, const float* means3D,
                              const float* opacities, const float* scales, const float* rotations,
                              const float* transMat_precomp, const float* shs,
                              const float* colors_precomp, int32_t* radii, void* geom_ws, void* image_ws,
                              uint32_t* num_rendered_host, void* stream) {
    Frame f;
    if (!frame_of(s, f)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    if (P < 0) { surfel_set_error("P < 0"); return 1; }
    if (P > 0 && (!means3D || !opacities || !radii || !geom_ws)) { surfel_set_error("NULL required pointer"); return 1; }
    if (P > 0 && !transMat_precomp && (!scales || !rotations)) { surfel_set_error("need scales+rotations or transMat_precomp"); return 1; }
    if (P > 0 && !colors_precomp && !shs) { surfel_set_error("need shs or colors_precomp"); return 1; }
    if (!colors_precomp && !sh_degree_ok(s->sh_degree, M)) {
        surfel_set_error("sh_degree %d unsupported for M=%d coefficients (max degree 3)", s->sh_degree, M);
        return 1;
    }
    GeomLayout L = geom_layout(P);
    char* g = (char*)geom_ws;
    if (P == 0) {
        if (num_rendered_host) *num_rendered_host = 0;
        return 0;
    }
    PreFwdParams p;
    p.P = P; p.D = s->sh_degree; p.M = M; p.W = f.W; p.H = f.H; p.gx = f.gx; p.gy = f.gy;
    p.row0 = f.row0; p.row1 = f.row1; p.prefiltered = s->prefiltered; p.scale_modifier = s->scale_modifier;
    p.means3D = means3D; p.scales = scales; p.rotations = rotations; p.opacities = opacities;
    p.shs = shs; p.transMat_precomp = transMat_precomp; p.colors_precomp = colors_precomp;
    p.viewmatrix = s->viewmatrix; p.projmatrix = s->projmatrix; p.campos = s->campos;
    p.radii = radii; p.rec = (float4*)(g + L.rec); p.tmat = (float4*)(g + L.tmat); p.tiles_touched = (uint32_t*)(g + L.tiles_touched);
    p.offsets = (uint32_t*)(g + L.offsets); p.clamped = (uint8_t*)(g + L.clamped);
    p.scan_status = (unsigned long long*)(g + L.scan_status); p.counters = (uint32_t*)(g + L.counters);
    p.tile_count = image_ws ? (uint32_t*)((char*)image_ws + image_layout(f.W, f.H).tile_count) : nullptr;
    p.num_rendered_mapped = mapped_alias(num_rendered_host);
    if (launch_preprocess_fwd(p, st)) return 1;
    if (num_rendered_host && !p.num_rendered_mapped)     // pageable / unmapped destination: copy engine
        SURFEL_CUDA_OK(cudaMemcpyAsync(num_rendered_host, p.counters + 1, 4, cudaMemcpyDeviceToHost, st));
    return 0;
}

int surfel_bin_duplicate(const surfel_settings_t* s, int P, uint32_t R, const void* geom_ws,
                         const int32_t* radii, void* binning_ws, void* stream) {
    Frame f;
    if (!frame_of(s, f)) return 1;
    if (R == 0 || P == 0) return 0;
    GeomLayout L = geom_layout(P);
    const char* g = (const char*)geom_ws;
    BinView v = bin_view(binning_ws, R, f.tiles);
    return launch_duplicate_with_keys(P, f.gx, f.gy, f.row0, f.row1, (const float4*)(g + L.tmat), radii,
                                      (const uint32_t*)(g + L.offsets), v.sort.in.keys, v.sort.in.vals,
                                      (cudaStream_t)stream);
}

int surfel_bin_sort(const surfel_settings_t* s, uint32_t R, void* binning_ws, void* stream) {
    Frame f;
    if (!frame_of(s, f)) return 1;
    BinView v = bin_view(binning_ws, R, f.tiles);
    if (launch_radix_sort_pairs(v.sort, R, (cudaStream_t)stream)) return 1;
    return launch_identify_tile_ranges(R, f.tiles, v.sort.out.keys, v.ranges, (cudaStream_t)stream);
}

int surfel_render_forward(const surfel_settings_t* s, uint32_t R, const void* geom_ws,
                          const void* binning_ws, void* image_ws, float* out_color,
                          float* out_others, void* stream) {
    Frame f;
    if (!frame_of(s, f)) return 1;
    BinView v = bin_view(const_cast<void*>(binning_ws), R, f.tiles);
    ImageLayout I = image_layout(f.W, f.H);
    RenderParams p;
    memset(&p, 0, sizeof(p));
    p.W = f.W; p.H = f.H; p.gx = f.gx; p.gy = f.gy; p.row0 = f.row0; p.row1 = f.row1;
    p.ranges = v.ranges; p.point_list = v.sort.out.vals;
    p.rec = (const float4*)((const char*)geom_ws + 0);   // records sit at offset 0 of the geometry workspace
    p.bg = s->bg;
    p.out_color = out_color; p.out_others = out_others;
    p.out_plane = s->out_plane_stride > 0 ? (size_t)s->out_plane_stride : (size_t)f.W * f.H;
    if (p.out_plane < (size_t)f.W * f.H) { surfel_set_error("out_plane_stride smaller than the image"); return 1; }
    p.rep_count = s->out_replica_count;
    if (p.rep_count < 0 || p.rep_count > SURFEL_MAX_OUT_REPLICAS) { surfel_set_error("out_replica_count out of range"); return 1; }
    if (p.rep_count > 0 && out_others != out_color + 3 * p.out_plane) {
        surfel_set_error("out_replica_base needs out_others == out_color + 3 * out_plane_stride (one 10-plane frame)");
        return 1;
    }
    for (int r = 0; r < SURFEL_MAX_OUT_REPLICAS; r++) {
        p.rep_base[r] = r < p.rep_count ? (unsigned long long)s->out_replica_base[r] : 0ull;
        if (r < p.rep_count && (p.rep_base[r] == 0 || (p.rep_base[r] & 3ull))) { surfel_set_error("out_replica_base: null or misaligned address"); return 1; }
    }
    p.accum = (float*)((char*)image_ws + I.accum); p.n_contrib = (uint32_t*)((char*)image_ws + I.n_contrib);
    return launch_render_fwd(p, (cudaStream_t)stream);
}

int surfel_bin_bucket(const surfel_settings_t* s, int P, uint32_t R, const void* geom_ws,
                      const int32_t* radii, void* binning_ws, const void* image_ws_with_counts,
                      int write_keys, void* stream) {
    Frame f;
    if (!frame_of(s, f)) return 1;
    GeomLayout L = geom_layout(P);
    const char* g = (const char*)geom_ws;
    BinView v = bin_view(binning_ws, R, f.tiles);
    // the same result buffers as the radix sort's; its spare keys hold the scratch pairs
    return launch_bucket_binning(P, R, f.gx, f.gy, f.row0, f.row1, (const float4*)(g + L.tmat), radii,
                                 (const uint32_t*)(g + L.offsets), (unsigned long long*)v.sort.spare.keys,
                                 v.sort.out.vals, write_keys ? (unsigned long long*)v.sort.out.keys : nullptr,
                                 v.ranges, v.sort.temp,
                                 image_ws_with_counts ? (const uint32_t*)((const char*)image_ws_with_counts +
                                                                          image_layout(f.W, f.H).tile_count) : nullptr,
                                 (cudaStream_t)stream);
}

int surfel_forward_render(const surfel_settings_t* s, int P, uint32_t R, const int32_t* radii,
                          const void* geom_ws, void* binning_ws, void* image_ws, int tile_counts_ready,
                          float* out_color, float* out_others, void* stream) {
    // SURFEL_SORT=radix selects the device-wide onesweep radix sort instead of the tile-bucketed path
    const bool use_radix = variants().sort_radix != 0;
    if (!use_radix) {
        if (surfel_bin_bucket(s, P, R, geom_ws, radii, binning_ws, tile_counts_ready ? image_ws : nullptr, 0, stream)) return 1;
        return surfel_render_forward(s, R, geom_ws, binning_ws, image_ws, out_color, out_others, stream);
    }
    if (surfel_bin_duplicate(s, P, R, geom_ws, radii, binning_ws, stream)) return 1;
    if (surfel_bin_sort(s, R, binning_ws, stream)) return 1;
    return surfel_render_forward(s, R, geom_ws, binning_ws, image_ws, out_color, out_others, stream);
}

int surfel_backward(const surfel_settings_t* s, int P, int M, uint32_t R, const float* means3D,
                    const float* scales, const float* rotations, const float* transMat_precomp,
                    const float* shs, int has_colors_precomp, const int32_t* radii,
                    const void* geom_ws, const void* binning_ws, const void* image_ws,
                    const float* dL_dout_color, const float* dL_dout_others, float* grad_scratch,
                    float* dL_dmeans2D, float* dL_dcolors, float* dL_dopacity, float* dL_dmeans3D,
                    float* dL_dtransMat, float* dL_dsh, float* dL_dscales, float* dL_drotations,
                    int lowpass_depth_quirk, void* stream) {
    Frame f;
    if (!frame_of(s, f)) return 1;
    if (P <= 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (!grad_scratch || !dL_dmeans2D || !dL_dopacity || !dL_dmeans3D) { surfel_set_error("NULL required gradient buffer"); return 1; }
    GeomLayout L = geom_layout(P);
    const char* g = (const char*)geom_ws;
    SURFEL_CUDA_OK(cudaMemsetAsync(grad_scratch, 0, (size_t)P * kGradFloats * 4, st));
    if (R > 0) {
        BinView v = bin_view(const_cast<void*>(binning_ws), R, f.tiles);
        ImageLayout I = image_layout(f.W, f.H);
        RenderParams p;
        memset(&p, 0, sizeof(p));
        p.W = f.W; p.H = f.H; p.gx = f.gx; p.gy = f.gy; p.row0 = f.row0; p.row1 = f.row1;
        p.ranges = v.ranges; p.point_list = v.sort.out.vals; p.rec = (const float4*)(g + L.rec); p.bg = s->bg;
        p.accum = (float*)((char*)image_ws + I.accum); p.n_contrib = (uint32_t*)((char*)image_ws + I.n_contrib);
        p.dL_dpix = dL_dout_color; p.dL_dothers = dL_dout_others; p.grad_rec = grad_scratch;
        p.grad_plane = s->grad_plane_stride > 0 ? (size_t)s->grad_plane_stride : (size_t)f.W * f.H;
        if (p.grad_plane < (size_t)f.W * f.H) { surfel_set_error("grad_plane_stride smaller than the image"); return 1; }
        p.lowpass_quirk = lowpass_depth_quirk;
        if (launch_render_bwd(p, st)) return 1;
    }
    PreBwdParams q;
    memset(&q, 0, sizeof(q));
    q.P = P; q.D = s->sh_degree; q.M = M; q.W = f.W; q.H = f.H; q.scale_modifier = s->scale_modifier;
    q.means3D = means3D; q.scales = scales; q.rotations = rotations; q.shs = shs;
    q.transMat_precomp = transMat_precomp; q.has_colors_precomp = has_colors_precomp;
    q.viewmatrix = s->viewmatrix; q.projmatrix = s->projmatrix; q.campos = s->campos;
    q.radii = radii; q.tmat = (const float4*)(g + L.tmat); q.clamped = (const uint8_t*)(g + L.clamped);
    q.grad_rec = grad_scratch;
    q.dL_dmeans2D = dL_dmeans2D; q.dL_dcolors = dL_dcolors; q.dL_dopacity = dL_dopacity;
    q.dL_dmeans3D = dL_dmeans3D; q.dL_dtransMat = dL_dtransMat; q.dL_dsh = dL_dsh;
    q.dL_dscales = dL_dscales; q.dL_drots = dL_drotations;
    q.defer_sh = (s->sh_grad_deferred && shs != nullptr && !has_colors_precomp) ? 1 : 0;
    if (q.defer_sh && !dL_dcolors) { surfel_set_error("sh_grad_deferred needs dL_dcolors"); return 1; }
    return launch_preprocess_bwd(q, st);
}

size_t surfel_camera_partials_bytes(int P) { return camera_partials_bytes(P); }

int surfel_camera_backward(const surfel_settings_t* s, int P, int M, const float* means3D, const float* scales,
                           const float* rotations, const float* transMat_precomp, const float* shs,
                           int has_colors_precomp, const int32_t* radii, const void* geom_ws,
                           const float* grad_scratch, const float* dL_dtransMat, double* partials,
                           float* dL_dviewmatrix, float* dL_dprojmatrix, float* dL_dcampos, void* stream) {
    Frame f;
    CamBwdParams p;
    if (!camera_params("surfel_camera_backward", s, P, M, means3D, scales, rotations, transMat_precomp, shs,
                       has_colors_precomp, radii, geom_ws, grad_scratch, dL_dtransMat, partials, false,
                       dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, f, p))
        return 1;
    p.dL_dviewmatrix = dL_dviewmatrix; p.dL_dprojmatrix = dL_dprojmatrix; p.dL_dcampos = dL_dcampos;
    return launch_camera_bwd(p, (cudaStream_t)stream);
}

int surfel_camera_backward_sums(const surfel_settings_t* s, int P, int M, const float* means3D, const float* scales,
                                const float* rotations, const float* transMat_precomp, const float* shs,
                                int has_colors_precomp, const int32_t* radii, const void* geom_ws,
                                const float* grad_scratch, const float* dL_dtransMat, double* partials,
                                double* dL_dviewmatrix, double* dL_dprojmatrix, double* dL_dcampos, void* stream) {
    Frame f;
    CamBwdParams p;
    if (!camera_params("surfel_camera_backward_sums", s, P, M, means3D, scales, rotations, transMat_precomp, shs,
                       has_colors_precomp, radii, geom_ws, grad_scratch, dL_dtransMat, partials, true,
                       dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, f, p))
        return 1;
    return launch_camera_bwd_sums(p, dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, (cudaStream_t)stream);
}

int surfel_sh_grad_expand(int P, int M, int sh_degree, const float* means3D, const float* campos,
                          const float* dL_dcolors, float* dL_dsh, void* stream) {
    if (P <= 0 || M <= 0) return 0;
    if (!means3D || !campos || !dL_dcolors || !dL_dsh) { surfel_set_error("surfel_sh_grad_expand: NULL argument"); return 1; }
    if (!sh_degree_ok(sh_degree, M)) { surfel_set_error("surfel_sh_grad_expand: degree / M mismatch"); return 1; }
    return launch_sh_grad_expand(P, M, sh_degree, means3D, campos, dL_dcolors, dL_dsh, (cudaStream_t)stream);
}

int surfel_mark_visible(int P, const float* means3D, const float* viewmatrix,
                        const float* projmatrix, uint8_t* present, void* stream) {
    (void)projmatrix;
    return launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream);
}

size_t surfel_sort_temp_bytes(size_t n) { return radix_sort_temp_bytes(n); }
int surfel_grad_scratch_floats(void) { return kGradFloats; }

int surfel_sort_pairs(uint64_t* keys_a, uint32_t* vals_a, uint64_t* keys_b, uint32_t* vals_b,
                      size_t n, int end_bit, void* temp, int* result_in_b, void* stream) {
    const RadixSortWs ws = radix_sort_ws(SortPairs{keys_a, vals_a}, SortPairs{keys_b, vals_b}, temp, end_bit);
    if (result_in_b) *result_in_b = ws.out.keys != keys_a;
    return launch_radix_sort_pairs(ws, n, (cudaStream_t)stream);
}

}  // extern "C"
