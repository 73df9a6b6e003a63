// preprocess_fwd.cu — per-splat forward preprocess FUSED with the tile-count prefix scan.
//
// Replaces upstream preprocessCUDA (forward) + cub::DeviceScan::InclusiveSum (SURVEY §8a rows
// a6, a7; algorithm: SURVEY Appendix A.1/A.2).  One thread per splat:
//   near cull -> splat->pixel homography T (in-tree restatement:
//   /root/reference/gaussian_renderer/__init__.py:64-75) -> view-space normal + dual-visible flip
//   -> AABB centre/extent -> radius -> tile rect -> SH->RGB (/root/reference/utils/sh_utils.py:57-112)
// then a block scan of tiles_touched chained across blocks with a decoupled look-back (scan.cuh), so the
// inclusive offsets and the instance count R come out of the same launch (no separate scan
// kernel, no second pass over tiles_touched).
//
// Notes: SH rows (192 B/splat, AoS) are the dominant HBM stream; with the vectorised layout they are
// prefetched by cp.async (LDGSTS) while the geometry is computed.  Only rows of splats that
// survive culling are fetched, warp-cooperatively with 128-bit loads into padded shared memory
// (conflict-free 13-quad stride), instead of upstream's per-thread stride-192 scalar reads.
//
// PARITY: this TU is compiled with -fmad=false and evaluates every expression in the order the
// oracle (oracle/surfel_oracle.c) documents, so radii / rects / tiles_touched / depth bits are
// bit-identical to the CPU restatement.
#include "common.cuh"
#include "kernels.h"
#include "profile.h"
#include "scan.cuh"
#include "splat_math.cuh"

namespace surfel {

// colour channel c of the SH row sh (3 floats per coefficient) in the unit direction (x, y, z): the basis values
// times the coefficients, added in basis order
__device__ __forceinline__ float sh_eval_channel(const float* sh, int c, int D, float x, float y, float z) {
    float r;
    sh_basis(D, x, y, z, [&](int i, float b) { r = i == 0 ? b * sh[c] : r + b * sh[3 * i + c]; });
    return r;
}

constexpr int kShRowQuads = 13;                 // 12 data quads + 1 pad: conflict-free LDS.128
constexpr int kShRowFloatsScalar = 49;          // scalar path stride (odd: conflict-free LDS.32)

#ifndef SURFEL_PRE_BLOCKS
#define SURFEL_PRE_BLOCKS 7      // 73 registers, spills gone from the record math: 0.124 ms vs 0.137 ms at 8 (64 registers), 0.134 at 6
#endif
template <bool kVec4>
__global__ void __launch_bounds__(kPreBlock, SURFEL_PRE_BLOCKS) preprocess_fwd_kernel(PreFwdParams p) {
    __shared__ float4 s_sh[(kPreBlock / 32) * 32 * kShRowQuads];
    __shared__ int s_rows[kPreBlock];            // per warp: compacted list of visible lanes
    __shared__ uint32_t s_warp_sum[kPreBlock / 32];
    __shared__ uint32_t s_bid, s_excl;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_bid = atomicAdd(&p.counters[0], 1u);   // ticket => forward progress of look-back
    __syncthreads();
    const uint32_t bid = s_bid;
    const int idx = (int)(bid * kPreBlock) + tid;

    bool visible = false;
    uint32_t tt = 0;
    int rx0 = 0, ry0 = 0, rw = 1;
    float tm[9], nrm[3] = {0, 0, 0}, cx = 0, cy = 0, pvz = 0, opa = 0;
    int radius_i = 0;
    float px = 0, py = 0, pz = 0, pvx = 0, pvy = 0, opa_in = 0;
    float4 rot_in = make_float4(1.0f, 0.0f, 0.0f, 0.0f);
    float2 scale_in = make_float2(0.0f, 0.0f);
    const float* vm = p.viewmatrix;

    if (idx < p.P) {
        px = p.means3D[3 * (size_t)idx + 0];
        py = p.means3D[3 * (size_t)idx + 1];
        pz = p.means3D[3 * (size_t)idx + 2];
        // every per-splat input is requested in the same round trip as the position (a culled splat
        // wastes 28 bytes; a visible one saves two dependent trips to HBM)
        if (p.transMat_precomp == nullptr) {
            rot_in = reinterpret_cast<const float4*>(p.rotations)[idx];
            scale_in = reinterpret_cast<const float2*>(p.scales)[idx];
        }
        opa_in = p.opacities[idx];
        pvx = ((vm[0] * px + vm[4] * py) + vm[8] * pz) + vm[12];
        pvy = ((vm[1] * px + vm[5] * py) + vm[9] * pz) + vm[13];
        pvz = ((vm[2] * px + vm[6] * py) + vm[10] * pz) + vm[14];
    }
    // ---- SH prefetch (vectorised layout only).  The rows of splats that pass the near plane and whose
    // centre projects within 1.5x the screen are requested NOW with cp.async and land in the warp's
    // panel while T / AABB / tile counts / the scan are computed; whatever turns out visible without
    // having been requested (huge off-screen splats) is fetched later by the plain path.  Only the
    // data movement changes: the arithmetic below is untouched. ----
    unsigned prefetched = 0;
    if (kVec4) {
        bool cand = false;
        if (idx < p.P && pvz > kNear) {
            const float* pr = p.projmatrix;
            const float hx = ((pr[0] * px + pr[4] * py) + pr[8] * pz) + pr[12];
            const float hy = ((pr[1] * px + pr[5] * py) + pr[9] * pz) + pr[13];
            const float hw4 = ((pr[3] * px + pr[7] * py) + pr[11] * pz) + pr[15];
            const float lim = 1.5f * fabsf(hw4);
            cand = fabsf(hx) <= lim && fabsf(hy) <= lim;
        }
        prefetched = __ballot_sync(0xffffffffu, cand);
        if (prefetched) {
            const int warp_base = (int)(bid * kPreBlock) + warp * 32;
            float4* dst = s_sh + warp * 32 * kShRowQuads;
            const float4* src = reinterpret_cast<const float4*>(p.shs) + (size_t)warp_base * 12;
#pragma unroll
            for (int it = 0; it < 12; it++) {
                const int f = it * 32 + lane;              // quad f of the warp's contiguous 6 KB of SH
                const int row = f / 12, q = f - row * 12;
                if ((prefetched >> row) & 1u) cp_async16(__cvta_generic_to_shared(dst + row * kShRowQuads + q), src + f);
            }
        }
    }
    if (idx < p.P) {
        if (pvz > kNear) {
            // per-view Pm = projmatrix * ndc2pix (columns x*w, y*w, w)
            const float hw = (float)p.W / 2.0f, hh = (float)p.H / 2.0f;
            const float cw = (float)(p.W - 1) / 2.0f, ch = (float)(p.H - 1) / 2.0f;
            if (p.transMat_precomp == nullptr) {
                const float2 sc = scale_in;
                const QuatRotation qr = quat_rotation(rot_in);
                const float (&R)[3][3] = qr.R;
                const float su = p.scale_modifier * sc.x, sv = p.scale_modifier * sc.y;
                const float L0[3] = {R[0][0] * su, R[1][0] * su, R[2][0] * su};
                const float L1[3] = {R[0][1] * sv, R[1][1] * sv, R[2][1] * sv};
                const float L2[3] = {R[0][2], R[1][2], R[2][2]};
#pragma unroll
                for (int j = 0; j < 3; j++) {
                    float Pm0, Pm1, Pm2, Pm3;
                    const float* pr = p.projmatrix;
                    if (j == 0) {
                        Pm0 = pr[0] * hw + pr[3] * cw; Pm1 = pr[4] * hw + pr[7] * cw;
                        Pm2 = pr[8] * hw + pr[11] * cw; Pm3 = pr[12] * hw + pr[15] * cw;
                    } else if (j == 1) {
                        Pm0 = pr[1] * hh + pr[3] * ch; Pm1 = pr[5] * hh + pr[7] * ch;
                        Pm2 = pr[9] * hh + pr[11] * ch; Pm3 = pr[13] * hh + pr[15] * ch;
                    } else {
                        Pm0 = pr[3]; Pm1 = pr[7]; Pm2 = pr[11]; Pm3 = pr[15];
                    }
                    tm[3 * j + 0] = (L0[0] * Pm0 + L0[1] * Pm1) + L0[2] * Pm2;
                    tm[3 * j + 1] = (L1[0] * Pm0 + L1[1] * Pm1) + L1[2] * Pm2;
                    tm[3 * j + 2] = ((px * Pm0 + py * Pm1) + pz * Pm2) + Pm3;
                }
                nrm[0] = (vm[0] * L2[0] + vm[4] * L2[1]) + vm[8] * L2[2];
                nrm[1] = (vm[1] * L2[0] + vm[5] * L2[1]) + vm[9] * L2[2];
                nrm[2] = (vm[2] * L2[0] + vm[6] * L2[1]) + vm[10] * L2[2];
            } else {
#pragma unroll
                for (int k = 0; k < 9; k++) tm[k] = p.transMat_precomp[9 * (size_t)idx + k];
                nrm[0] = 0.0f; nrm[1] = 0.0f; nrm[2] = 1.0f;
            }
            const float c = -((pvx * nrm[0] + pvy * nrm[1]) + pvz * nrm[2]);
            if (c != 0.0f) {
                const float mult = c > 0.0f ? 1.0f : -1.0f;
                nrm[0] *= mult; nrm[1] *= mult; nrm[2] *= mult;
                const float t0 = kCutoff * kCutoff, t1 = kCutoff * kCutoff, t2 = -1.0f;
                const float d = (t0 * (tm[6] * tm[6]) + t1 * (tm[7] * tm[7])) + t2 * (tm[8] * tm[8]);
                if (d != 0.0f) {
                    const float f0 = t0 / d, f1 = t1 / d, f2 = t2 / d;
                    cx = (f0 * (tm[0] * tm[6]) + f1 * (tm[1] * tm[7])) + f2 * (tm[2] * tm[8]);
                    cy = (f0 * (tm[3] * tm[6]) + f1 * (tm[4] * tm[7])) + f2 * (tm[5] * tm[8]);
                    const float ex = (f0 * (tm[0] * tm[0]) + f1 * (tm[1] * tm[1])) + f2 * (tm[2] * tm[2]);
                    const float ey = (f0 * (tm[3] * tm[3]) + f1 * (tm[4] * tm[4])) + f2 * (tm[5] * tm[5]);
                    const float hx = sqrtf(fmaxf(1e-4f, cx * cx - ex));
                    const float hy = sqrtf(fmaxf(1e-4f, cy * cy - ey));
                    const float radius = ceilf(fmaxf(fmaxf(hx, hy), kCutoff * kFilterSize));
                    if (radius == radius && cx == cx && cy == cy) {
                        radius_i = f2i_sat(radius);
                        int x0, y0, x1, y1;
                        get_rect(cx, cy, radius_i, p.gx, p.gy, p.row0, p.row1, x0, y0, x1, y1);
                        tt = (uint32_t)((x1 - x0) * (y1 - y0));
                        visible = tt != 0;
                        rx0 = x0; ry0 = y0; rw = max(1, x1 - x0);
                    }
                }
            }
        }
        if (visible) opa = opa_in;
    }

    // ---- fused per-tile instance count for the tile-bucketed binning (bucket_sort.cu): small rects
    // are counted by their own thread, large ones are spread over the warp ----
    if (p.tile_count != nullptr) {
        if (visible && tt <= 8u) {
            for (uint32_t i = 0; i < tt; i++) {
                const uint32_t ry = i / (uint32_t)rw, rx = i - ry * (uint32_t)rw;
                atomicAdd(p.tile_count + (uint32_t)(ry0 + (int)ry) * (uint32_t)p.gx + (uint32_t)(rx0 + (int)rx), 1u);
            }
        }
        unsigned big = __ballot_sync(0xffffffffu, visible && tt > 8u);
        while (big) {
            const int src = __ffs(big) - 1;
            big &= big - 1;
            const int bx0 = __shfl_sync(0xffffffffu, rx0, src), by0 = __shfl_sync(0xffffffffu, ry0, src);
            const uint32_t bw = (uint32_t)__shfl_sync(0xffffffffu, rw, src), bt = __shfl_sync(0xffffffffu, tt, src);
            for (uint32_t i = lane; i < bt; i += 32) {
                const uint32_t ry = i / bw, rx = i - ry * bw;
                atomicAdd(p.tile_count + (uint32_t)(by0 + (int)ry) * (uint32_t)p.gx + (uint32_t)(bx0 + (int)rx), 1u);
            }
        }
    }

    // ---- block inclusive scan of tiles_touched; the block aggregate is published NOW, before the
    // SH work, so that by the time successor blocks look back (at their very end) it is long there ----
    uint32_t incl = tt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s_warp_sum[warp] = incl;
    __syncthreads();
    uint32_t warp_excl = 0, block_total = 0;
#pragma unroll
    for (int w = 0; w < kPreBlock / 32; w++) {
        const uint32_t s = s_warp_sum[w];
        if (w < warp) warp_excl += s;
        block_total += s;
    }
    if (tid == 0) publish_aggregate(p.scan_status, bid, block_total);

    // ---- SH -> RGB for surviving splats (rows staged warp-cooperatively) ----
    float rgb[3] = {0, 0, 0};
    unsigned clamp_bits = 0;
    const unsigned vis_mask = __ballot_sync(0xffffffffu, visible);
    if (kVec4) cp_async_wait_all();      // this lane's prefetched quads have landed (made visible to the warp below)
    if (p.colors_precomp == nullptr) {
        if (vis_mask) {
            int* rows = s_rows + warp * 32;
            const int nvis = __popc(vis_mask);
            if (visible) rows[__popc(vis_mask & ((1u << lane) - 1u))] = lane;
            __syncwarp();
            const int warp_base = (int)(bid * kPreBlock) + warp * 32;
            float sh[48];
            if (kVec4) {
                float4* dst = s_sh + warp * 32 * kShRowQuads;
                const float4* src = reinterpret_cast<const float4*>(p.shs);
                unsigned missing = vis_mask & ~prefetched;     // visible but not requested up front (rare)
                while (missing) {
                    const int row = __ffs(missing) - 1;
                    missing &= missing - 1;
                    if (lane < 12) dst[row * kShRowQuads + lane] = ld_nc_f4(src + (size_t)(warp_base + row) * 12 + lane);
                }
                __syncwarp();
                if (visible) {
#pragma unroll
                    for (int q = 0; q < 12; q++) {
                        const float4 v = dst[lane * kShRowQuads + q];
                        sh[4 * q + 0] = v.x; sh[4 * q + 1] = v.y; sh[4 * q + 2] = v.z; sh[4 * q + 3] = v.w;
                    }
                }
            } else {
                float* dst = reinterpret_cast<float*>(s_sh) + warp * 32 * 52;
                const int ncoef = 3 * (p.D + 1) * (p.D + 1);
                const size_t row_stride = (size_t)3 * p.M;
                for (int f = lane; f < nvis * ncoef; f += 32) {
                    const int slot = f / ncoef, q = f - slot * ncoef;
                    const int row = rows[slot];
                    dst[row * kShRowFloatsScalar + q] = p.shs[(size_t)(warp_base + row) * row_stride + q];
                }
                __syncwarp();
                if (visible) {
#pragma unroll
                    for (int q = 0; q < 48; q++) sh[q] = q < ncoef ? dst[lane * kShRowFloatsScalar + q] : 0.0f;
                }
            }
            if (visible) {
                float dx = px - p.campos[0], dy = py - p.campos[1], dz = pz - p.campos[2];
                const float len = sqrtf((dx * dx + dy * dy) + dz * dz);
                dx = dx / len; dy = dy / len; dz = dz / len;
#pragma unroll
                for (int ch = 0; ch < 3; ch++) {
                    const float v = sh_eval_channel(sh, ch, p.D, dx, dy, dz) + 0.5f;
                    if (v < 0.0f) clamp_bits |= 1u << ch;
                    rgb[ch] = fmaxf(v, 0.0f);
                }
            }
        }
    } else if (visible) {
        rgb[0] = p.colors_precomp[3 * (size_t)idx + 0];
        rgb[1] = p.colors_precomp[3 * (size_t)idx + 1];
        rgb[2] = p.colors_precomp[3 * (size_t)idx + 2];
    }

    // ---- write per-splat state ----
    __syncwarp();   // every lane has consumed its SH row: the panel is reused for the records
    if (idx < p.P) {
        p.radii[idx] = visible ? radius_i : 0;
        p.tiles_touched[idx] = tt;
        p.clamped[idx] = (uint8_t)clamp_bits;
        if (visible) {
            // ---- render record (common.cuh).  Everything below is evaluated about the splat's own
            // screen position c = (cx, cy), in double: in absolute pixel coordinates the adjugate and
            // the conic extents subtract float32 terms of order |pixel|^2 (ADVICE r1: at 4K the loss
            // exceeded the culling margin). ----
            // records go to the warp's shared-memory panel (11-quad stride: conflict-free) as soon as their
            // values exist, so that the double-precision temporaries die early
            float4* r = s_sh + warp * 32 * kShRowQuads + lane * 11;
            float tu[3], tv[3];          // rows of T about c, rounded once
            {
                const double Twx = tm[6], Twy = tm[7], Twz = tm[8];
                const double Tux = (double)tm[0] - (double)cx * Twx, Tuy = (double)tm[1] - (double)cx * Twy, Tuz = (double)tm[2] - (double)cx * Twz;
                const double Tvx = (double)tm[3] - (double)cy * Twx, Tvy = (double)tm[4] - (double)cy * Twy, Tvz = (double)tm[5] - (double)cy * Twz;
                // P1 = Tv' x Tw, P2 = Tw x Tu', Pc = Tu' x Tv', det T = Tu' . P1 (invariant under the shift)
                const double P1x = Tvy * Twz - Tvz * Twy, P1y = Tvz * Twx - Tvx * Twz, P1z = Tvx * Twy - Tvy * Twx;
                r[0] = make_float4((float)P1x, (float)P1y, (float)P1z, cx);
                r[4] = make_float4(rgb[0], rgb[1], rgb[2], (float)(Tux * P1x + Tuy * P1y + Tuz * P1z));
                r[1] = make_float4((float)(Twy * Tuz - Twz * Tuy), (float)(Twz * Tux - Twx * Tuz), (float)(Twx * Tuy - Twy * Tux), cy);
                // The sign of the stored opacity is a per-splat flag: negative = some point of the splat within the
                // reach of alpha >= 1/255 may lie in front of the near plane, so the render kernels must apply
                // A.3's per-pixel `depth < near` skip; positive (practically every splat) = the ray-splat depth
                // w = Tw . (u, v, 1) stays >= near on the whole disc u^2 + v^2 <= tau (and Tw.z, the low-pass
                // depth, does too), so they can leave the test out.  min over the disc = Tw.z - sqrt(tau |Tw.xy|^2).
                const float tau_n = 2.0f * logf(fmaxf(255.0f * opa, 1.0f)) + 0.01f;
                const float wmin = tm[8] - sqrtf(tau_n * (tm[6] * tm[6] + tm[7] * tm[7]));
                const bool near_safe = wmin >= kNear * 1.001f;
                r[2] = make_float4((float)(Tuy * Tvz - Tuz * Tvy), (float)(Tuz * Tvx - Tux * Tvz), (float)(Tux * Tvy - Tuy * Tvx),
                                   near_safe ? opa : -opa);
                tu[0] = (float)Tux; tu[1] = (float)Tuy; tu[2] = (float)Tuz;
                tv[0] = (float)Tvx; tv[1] = (float)Tvy; tv[2] = (float)Tvz;
            }

            // conservative region of {alpha >= 1/255} = low-pass disk  U  projected ellipse rho3d <= tau,
            // as extents along x, y, x+y and x-y relative to c (see DESIGN.md, render culling); float32 is
            // enough here: the rows are already centred
            float ext[8];     // lo/hi along x, y, u = x+y, v = x-y
            const float a255 = 255.0f * opa;
            if (a255 < 0.999f) {
#pragma unroll
                for (int k = 0; k < 4; k++) { ext[2 * k] = 3.0e38f; ext[2 * k + 1] = -3.0e38f; }   // can never reach 1/255: empty
            } else {
                const float tau = 2.0f * logf(a255) + 0.01f;
                const float r2 = sqrtf(0.5f * tau) + 0.05f;
                const float r2d = r2 * 1.41421366f;
                ext[0] = -r2; ext[1] = r2; ext[2] = -r2; ext[3] = r2; ext[4] = -r2d; ext[5] = r2d; ext[6] = -r2d; ext[7] = r2d;
                const float wxy = tm[6] * tm[6] + tm[7] * tm[7], wz2 = tm[8] * tm[8];
                bool bounded = tm[8] > 0.0f && wz2 > 1.05f * tau * wxy;
                if (bounded) {
                    const float d = tau * wxy - wz2;
                    const float f0 = tau / d, f2 = -1.0f / d;
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        // direction n: T_n = n.x Tu' + n.y Tv'
                        const float nx = k == 1 ? 0.0f : 1.0f, ny = k == 0 ? 0.0f : (k == 3 ? -1.0f : 1.0f);
                        const float ax = nx * tu[0] + ny * tv[0], ay = nx * tu[1] + ny * tv[1], az = nx * tu[2] + ny * tv[2];
                        const float ec = f0 * (ax * tm[6] + ay * tm[7]) + f2 * (az * tm[8]);
                        const float ee = f0 * (ax * ax + ay * ay) + f2 * (az * az);
                        const float eh = sqrtf(fmaxf(0.0f, ec * ec - ee));
                        const float mg = 0.05f + 1e-4f * (fabsf(ec) + eh);
                        if (!(ec == ec) || !(eh == eh)) bounded = false;
                        ext[2 * k] = fminf(ext[2 * k], ec - eh - mg);
                        ext[2 * k + 1] = fmaxf(ext[2 * k + 1], ec + eh + mg);
                    }
                }
                if (!bounded) {
#pragma unroll
                    for (int k = 0; k < 4; k++) { ext[2 * k] = -3.0e38f; ext[2 * k + 1] = 3.0e38f; }   // unbounded conic: never culled
                }
            }
            const float cu = cx + cy, cv = cx - cy;
            // the warp then streams its 32 render records (4 KB contiguous) and 32 transform records
            // (1.5 KB) to HBM with fully coalesced 128-bit stores
            r[3] = make_float4(nrm[0], nrm[1], nrm[2], tm[8]);
            r[5] = make_float4(tm[6], tm[7], __uint_as_float((uint32_t)idx), pvz);
            r[6] = make_float4(cx + ext[0], cy + ext[2], cx + ext[1], cy + ext[3]);
            r[7] = make_float4(cu + ext[4], cu + ext[5], cv + ext[6], cv + ext[7]);
            r[8] = make_float4(tm[0], tm[1], tm[2], tm[3]);
            r[9] = make_float4(tm[4], tm[5], tm[6], tm[7]);
            r[10] = make_float4(tm[8], cx, cy, pvz);
        }
    }
    {
        __syncwarp();
        const int warp_first = (int)(bid * kPreBlock) + warp * 32;
        const int nrows = min(32, p.P - warp_first);
        const float4* src = s_sh + warp * 32 * kShRowQuads;
        float4* dst = p.rec + (size_t)warp_first * kRecQuads;
        for (int f = lane; f < nrows * kRecQuads; f += 32) {
            const int row = f >> 3, q = f & 7;
            if ((vis_mask >> row) & 1u) dst[f] = src[row * 11 + q];
        }
        float4* dst2 = p.tmat + (size_t)warp_first * kTmQuads;
        for (int f = lane; f < nrows * kTmQuads; f += 32) {
            const int row = f / kTmQuads, q = f - row * kTmQuads;
            if ((vis_mask >> row) & 1u) dst2[f] = src[row * 11 + 8 + q];
        }
    }

    // ---- decoupled look-back across blocks (predecessor aggregates were published early) ----
    if (warp == 0) {
        const uint32_t excl = warp_lookback(p.scan_status, bid, block_total);
        if (lane == 0) {
            s_excl = excl;
            if (bid == gridDim.x - 1) {
                p.counters[1] = excl + block_total;   // R = num_rendered
                // R also goes straight into the caller's pinned host word (zero-copy store): a 4-byte
                // cudaMemcpyAsync would queue on the D2H copy engine BEHIND any bulk download another
                // stream has in flight (measured: +6.7 ms per step in the host-buffer pipeline).
                if (p.num_rendered_mapped) {
                    *(volatile uint32_t*)p.num_rendered_mapped = excl + block_total;
                    __threadfence_system();
                }
            }
        }
    }
    __syncthreads();
    if (idx < p.P) p.offsets[idx] = s_excl + warp_excl + incl;
}

// markVisible: near-plane test only (SURVEY §2.2 checkFrustum).
__global__ void mark_visible_kernel(int P, const float* __restrict__ means3D,
                                    const float* __restrict__ vm, uint8_t* __restrict__ present) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float px = means3D[3 * (size_t)idx], py = means3D[3 * (size_t)idx + 1], pz = means3D[3 * (size_t)idx + 2];
    const float pvz = ((vm[2] * px + vm[6] * py) + vm[10] * pz) + vm[14];
    present[idx] = (uint8_t)(pvz > kNear);
}

int launch_preprocess_fwd(const PreFwdParams& p, cudaStream_t stream) {
    if (p.P <= 0) return 0;
    const int blocks = (p.P + kPreBlock - 1) / kPreBlock;
    SURFEL_CUDA_OK(cudaMemsetAsync(p.scan_status, 0, (size_t)(blocks + 1) * 8, stream));
    SURFEL_CUDA_OK(cudaMemsetAsync(p.counters, 0, 64, stream));
    if (p.tile_count) SURFEL_CUDA_OK(cudaMemsetAsync(p.tile_count, 0, (size_t)p.gx * p.gy * 4, stream));
    const bool vec4 = p.colors_precomp == nullptr && p.D <= 3 && p.M == 16 &&
                      (reinterpret_cast<uintptr_t>(p.shs) % 16 == 0);
    LaunchScope scope(kStPreFwd, stream);
    if (vec4) preprocess_fwd_kernel<true><<<blocks, kPreBlock, 0, stream>>>(p);
    else      preprocess_fwd_kernel<false><<<blocks, kPreBlock, 0, stream>>>(p);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                        cudaStream_t stream) {
    if (P <= 0) return 0;
    LaunchScope scope(kStMarkVisible, stream);
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, viewmatrix, present);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace surfel
