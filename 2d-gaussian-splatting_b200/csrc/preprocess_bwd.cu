// preprocess_bwd.cu — per-splat backward of the preprocess.
//
// Replaces upstream preprocessCUDA backward with its helpers compute_transmat_aabb vjp,
// quat_to_rotmat_vjp and SH backward (SURVEY §8a row a13; algorithm SURVEY Appendix A.5):
//   1. fold dL_dmean2D (low-pass branch) into dL_dT through the AABB-centre formula,
//   2. dL_dT -> dL_dmean3D, dL_dscale, dL_dq (unit quaternion) and the normal's vjp,
//   3. SH backward (dL_dsh, and dL_dmean3D through the view direction),
//   4. overwrite dL_dmean2D with the densification proxy dL_dT[2|5] * depth * 0.5 * (W|H)
//      (dL_dT before step 1 on the scales+rotations path, after it on the transMat_precomp path, as upstream).
// The kernel writes EVERY output row (zeros for culled splats), so the caller can hand in
// uninitialised tensors: no separate zero-fill pass over the 59 floats/splat of gradients.
// Kept quirk (SURVEY A.5): like upstream, the backward takes L = R diag(s) with scale_modifier fixed to 1, so
// dL_dscale and the scale-weighted columns 0 and 1 of dL_dR ignore the modifier (only the viewer uses modifier != 1).
#include "common.cuh"
#include "kernels.h"
#include "profile.h"
#include "splat_math.cuh"

namespace surfel {

constexpr int kRowQuads = 13;   // 12 data quads + 1 pad: conflict-free 128-bit row access

// kStaged: SH rows (in) and dL_dsh rows (out) travel through shared memory so that every global
// access is a fully coalesced 128-bit transaction (M == 16, degree 3, 16-byte aligned tensors);
// otherwise each thread addresses its own rows directly (any M / degree).
template <bool kStaged>
__global__ void __launch_bounds__(128, 6) preprocess_bwd_kernel(PreBwdParams p) {
    __shared__ float4 s_rows[kStaged ? 4 * 32 * kRowQuads : 1];
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool in_range = idx < p.P;
    if (!kStaged && !in_range) return;
    const bool visible = in_range && p.radii[idx] > 0;
    const bool geom = p.transMat_precomp == nullptr;
    const bool has_sh = !p.has_colors_precomp && p.shs != nullptr;

    float gT[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    float gm2x = 0, gm2y = 0, gopa = 0, gn[3] = {0, 0, 0}, gc[3] = {0, 0, 0};
    float tm[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    float g3[3] = {0, 0, 0}, gs[2] = {0, 0}, gq[4] = {0, 0, 0, 0};
    float px = 0, py = 0, pz = 0, proxy2 = 0, proxy5 = 0;
    float dR_out[3] = {0, 0, 0};      // clamp-masked colour gradient (what the SH expansion multiplies)
    const bool emit_sh = !p.defer_sh;

    // Every input of the splat is requested in the first round trip to HBM: the SH rows by cp.async
    // (LDGSTS) straight into the warp's panel, position / rotation / scale into registers, while the
    // gradient record and the forward record are fetched and the homography vjp is computed.
    const unsigned vis_mask = kStaged ? __ballot_sync(0xffffffffu, visible) : 0u;
    if (kStaged && has_sh && vis_mask) {
        const float4* src = reinterpret_cast<const float4*>(p.shs) + (size_t)(blockIdx.x * blockDim.x + warp * 32) * 12;
        float4* dst = s_rows + warp * 32 * kRowQuads;
#pragma unroll
        for (int it = 0; it < 12; it++) {
            const int f = it * 32 + lane;
            const int row = f / 12, q = f - row * 12;
            if ((vis_mask >> row) & 1u) cp_async16(__cvta_generic_to_shared(dst + row * kRowQuads + q), src + f);
        }
    }
    float4 rot_in = make_float4(1.0f, 0.0f, 0.0f, 0.0f);
    float2 scale_in = make_float2(0.0f, 0.0f);
    if (visible) {
        px = p.means3D[3 * (size_t)idx]; py = p.means3D[3 * (size_t)idx + 1]; pz = p.means3D[3 * (size_t)idx + 2];
        if (geom) {
            rot_in = reinterpret_cast<const float4*>(p.rotations)[idx];
            scale_in = reinterpret_cast<const float2*>(p.scales)[idx];
        }
    }

    if (visible) {
        const float4* gr = reinterpret_cast<const float4*>(p.grad_rec + (size_t)idx * kGradFloats);
        const float4 a = gr[0], b = gr[1], c = gr[2], d = gr[3], e = gr[4], f5 = gr[5];
        const float4* r = p.tmat + (size_t)idx * kTmQuads;      // (Tu, Tv.x) (Tv.yz, Tw.xy) (Tw.z, xy, depth)
        const float4 q0 = r[0], q1 = r[1], q2 = r[2];
        tm[0] = q0.x; tm[1] = q0.y; tm[2] = q0.z; tm[3] = q0.w; tm[4] = q1.x; tm[5] = q1.y;
        tm[6] = q1.z; tm[7] = q1.w; tm[8] = q2.x;
        gm2x = d.y; gm2y = d.z; gopa = d.w;
        gn[0] = e.x; gn[1] = e.y; gn[2] = e.z; gc[0] = e.w; gc[1] = f5.x; gc[2] = f5.y;
        {
            // dL_dT from the accumulated sums A, Bx, By, Zd, Zl (record layout: common.cuh)
            const float A[3] = {a.x, a.y, a.z}, Bx[3] = {a.w, b.x, b.y}, By[3] = {b.z, b.w, c.x};
            const float Zd = c.y, Zl[3] = {c.z, c.w, d.x};
            const float cx = q2.y, cy = q2.z;
            // -Tu' = cx Tw - Tu and -Tv' in double: cx*Tw.z and Tu.z agree to a few units in 1e5
            const float kc[3] = {(float)((double)cx * tm[6] - (double)tm[0]), (float)((double)cx * tm[7] - (double)tm[1]), (float)((double)cx * tm[8] - (double)tm[2])};
            const float lc[3] = {(float)((double)cy * tm[6] - (double)tm[3]), (float)((double)cy * tm[7] - (double)tm[4]), (float)((double)cy * tm[8] - (double)tm[5])};
            const float* Tu = tm; const float* Tv = tm + 3; const float* Tw = tm + 6;
#define CROSS(o, u, v) do { o[0] = u[1] * v[2] - u[2] * v[1]; o[1] = u[2] * v[0] - u[0] * v[2]; o[2] = u[0] * v[1] - u[1] * v[0]; } while (0)
            float t1[3], t2[3], t3[3], t4[3];
            CROSS(t1, lc, A); CROSS(t2, Tw, By);          // dTu' = -(lc x A) - (Tw x By) = Tv' x A + By x Tw
            CROSS(t3, A, kc); CROSS(t4, Bx, Tw);          // dTv' = -(A x kc) - (Bx x Tw) = A x Tu' + Tw x Bx
            float u1[3], u2[3];
            CROSS(u1, lc, Bx); CROSS(u2, By, kc);         // Bx x Tv' + Tu' x By
            float d1[3], d2[3], d3[3];                    // gradient of det T: (Tv x Tw, Tw x Tu, Tu x Tv)
            CROSS(d1, Tv, Tw); CROSS(d2, Tw, Tu); CROSS(d3, Tu, Tv);
#undef CROSS
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const float gu = -t1[k] - t2[k], gv = -t3[k] - t4[k];
                gT[k] = gu + Zd * d1[k];
                gT[3 + k] = gv + Zd * d2[k];
                gT[6 + k] = -cx * gu - cy * gv + u1[k] + u2[k] + Zd * d3[k] + Zl[k];
            }
        }

        // Densification proxy source (step 4).  Upstream folds dL_dmean2D into a LOCAL copy of dL_dT and
        // writes it back only on the transMat_precomp path, so on the scales+rotations (training) path the
        // proxy reads the RAW render-backward dL_dtransMat[2|5] — without the low-pass filter's gradient
        // (/root/reference/README.md:118); on the precomp path it reads the folded one.
        proxy2 = gT[2]; proxy5 = gT[5];
        // 1. AABB-centre vjp
        if (gm2x != 0.0f || gm2y != 0.0f) {
            const float t[3] = {kCutoff * kCutoff, kCutoff * kCutoff, -1.0f};
            const float dd = t[0] * tm[6] * tm[6] + t[1] * tm[7] * tm[7] + t[2] * tm[8] * tm[8];
            float f[3], dT3[3], dot = 0.0f;
#pragma unroll
            for (int k = 0; k < 3; k++) {
                f[k] = t[k] / dd;
                gT[k] += gm2x * f[k] * tm[6 + k];
                gT[3 + k] += gm2y * f[k] * tm[6 + k];
                dT3[k] = gm2x * f[k] * tm[k] + gm2y * f[k] * tm[3 + k];
                dot += (gm2x * tm[k] * tm[6 + k] + gm2y * tm[3 + k] * tm[6 + k]) * f[k];
            }
            const float dL_dd = dot * (-1.0f / dd);
#pragma unroll
            for (int k = 0; k < 3; k++) gT[6 + k] += dT3[k] + dL_dd * (t[k] * tm[6 + k] * 2.0f);
        }
        if (!geom) { proxy2 = gT[2]; proxy5 = gT[5]; }

        if (geom) {
            const float* vm = p.viewmatrix;
            const float* pr = p.projmatrix;
            const float hw = (float)p.W / 2.0f, hh = (float)p.H / 2.0f;
            const float cw = (float)(p.W - 1) / 2.0f, ch = (float)(p.H - 1) / 2.0f;
            const float2 sc = scale_in;
            const QuatRotation qr = quat_rotation(rot_in);
            const float w = qr.w, x = qr.x, y = qr.y, z = qr.z;
            const float (&R)[3][3] = qr.R;
            // dRows[i][k] = sum_j gT[3j+i] * Pm[k][j]
            float dRows[3][3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const float Pm0 = pr[4 * k + 0] * hw + pr[4 * k + 3] * cw;
                const float Pm1 = pr[4 * k + 1] * hh + pr[4 * k + 3] * ch;
                const float Pm2 = pr[4 * k + 3];
#pragma unroll
                for (int i = 0; i < 3; i++) dRows[i][k] = gT[i] * Pm0 + gT[3 + i] * Pm1 + gT[6 + i] * Pm2;
            }
            float dtn[3];
#pragma unroll
            for (int r2 = 0; r2 < 3; r2++) dtn[r2] = vm[4 * r2 + 0] * gn[0] + vm[4 * r2 + 1] * gn[1] + vm[4 * r2 + 2] * gn[2];
            // dual-visible sign, recomputed as in the forward
            const float L2[3] = {R[0][2], R[1][2], R[2][2]};
            const float nv0 = vm[0] * L2[0] + vm[4] * L2[1] + vm[8] * L2[2];
            const float nv1 = vm[1] * L2[0] + vm[5] * L2[1] + vm[9] * L2[2];
            const float nv2 = vm[2] * L2[0] + vm[6] * L2[1] + vm[10] * L2[2];
            const float pvx = vm[0] * px + vm[4] * py + vm[8] * pz + vm[12];
            const float pvy = vm[1] * px + vm[5] * py + vm[9] * pz + vm[13];
            const float pvz = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
            const float cs = -(pvx * nv0 + pvy * nv1 + pvz * nv2);
            const float mult = cs > 0.0f ? 1.0f : -1.0f;
            float v[3][3];   // v[c][r] = dL/dR[r][c]
#pragma unroll
            for (int r2 = 0; r2 < 3; r2++) {
                v[0][r2] = dRows[0][r2] * sc.x; v[1][r2] = dRows[1][r2] * sc.y; v[2][r2] = dtn[r2] * mult;
            }
            gs[0] = dRows[0][0] * R[0][0] + dRows[0][1] * R[1][0] + dRows[0][2] * R[2][0];
            gs[1] = dRows[1][0] * R[0][1] + dRows[1][1] * R[1][1] + dRows[1][2] * R[2][1];
            gq[0] = 2.0f * (x * (v[1][2] - v[2][1]) + y * (v[2][0] - v[0][2]) + z * (v[0][1] - v[1][0]));
            gq[1] = 2.0f * (-2.0f * x * (v[1][1] + v[2][2]) + y * (v[0][1] + v[1][0]) + z * (v[0][2] + v[2][0]) + w * (v[1][2] - v[2][1]));
            gq[2] = 2.0f * (x * (v[0][1] + v[1][0]) - 2.0f * y * (v[0][0] + v[2][2]) + z * (v[1][2] + v[2][1]) + w * (v[2][0] - v[0][2]));
            gq[3] = 2.0f * (x * (v[0][2] + v[2][0]) + y * (v[1][2] + v[2][1]) - 2.0f * z * (v[0][0] + v[1][1]) + w * (v[0][1] - v[1][0]));
            g3[0] = dRows[2][0]; g3[1] = dRows[2][1]; g3[2] = dRows[2][2];
        }
    }

    // 3. SH backward (writes the full dL_dsh row; zeros when culled / beyond the active degree)
    if (has_sh) {
        float v[48];                       // staged path: sh row in, dL_dsh row out (in place)
        float4* wrow = s_rows + (kStaged ? (warp * 32 + lane) * kRowQuads : 0);
        const int warp_first = blockIdx.x * blockDim.x + warp * 32;
        if (kStaged) {
            // the warp's SH rows (only rows of visible splats) were requested at the top of the kernel
            cp_async_wait_all();
            __syncwarp();
            if (visible) {
#pragma unroll
                for (int q = 0; q < 12; q++) {
                    const float4 t = wrow[q];
                    v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
                }
            }
        }
        float* gsh = kStaged ? nullptr : p.dL_dsh + (size_t)idx * 3 * p.M;
        const float* shg = kStaged ? nullptr : p.shs + (size_t)idx * 3 * p.M;
        const int ncoef_active = visible ? (p.D + 1) * (p.D + 1) : 0;
        if (visible) {
            const uint8_t cb = p.clamped[idx];
            const float dR[3] = {(cb & 1) ? 0.0f : gc[0], (cb & 2) ? 0.0f : gc[1], (cb & 4) ? 0.0f : gc[2]};
            dR_out[0] = dR[0]; dR_out[1] = dR[1]; dR_out[2] = dR[2];
            const float dox = px - p.campos[0], doy = py - p.campos[1], doz = pz - p.campos[2];
            const float sq = dox * dox + doy * doy + doz * doz;
            const float invl = 1.0f / sqrtf(sq);
            const float x = dox * invl, y = doy * invl, z = doz * invl;
            // the staged row is overwritten in place: sh_backward reads a band's coefficients before handing out its basis
            auto shv = [&](int i, int c) { return kStaged ? v[3 * i + c] : shg[3 * i + c]; };
            auto gs = [&](int i, float b) {
                if (kStaged) { v[3 * i] = b * dR[0]; v[3 * i + 1] = b * dR[1]; v[3 * i + 2] = b * dR[2]; }
                else if (emit_sh) { gsh[3 * i] = b * dR[0]; gsh[3 * i + 1] = b * dR[1]; gsh[3 * i + 2] = b * dR[2]; }
            };
            const float3 gm = sh_direction_to_mean(dox, doy, doz, invl, sh_backward(p.D, x, y, z, dR, shv, gs));
            g3[0] += gm.x; g3[1] += gm.y; g3[2] += gm.z;
        }
        if (!emit_sh) {
            // deferred: the caller expands basis (x) colour gradient itself (surfel_sh_grad_expand), typically
            // after summing the 3-float colour gradients of several GPUs
        } else if (kStaged) {
            // row back to shared memory (zeros for culled splats and for coefficients beyond the
            // active degree), then one coalesced sweep to HBM
#pragma unroll
            for (int i = 0; i < 48; i++) if (i >= 3 * ncoef_active) v[i] = 0.0f;
#pragma unroll
            for (int q = 0; q < 12; q++)
                wrow[q] = visible ? make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
            __syncwarp();
            const int nrows = min(32, p.P - warp_first);
            float4* dstg = reinterpret_cast<float4*>(p.dL_dsh) + (size_t)warp_first * 12;
            const float4* srcw = s_rows + warp * 32 * kRowQuads;
            for (int f = lane; f < nrows * 12; f += 32) {
                const int row = f / 12, q = f - row * 12;
                dstg[f] = srcw[row * kRowQuads + q];
            }
        } else {
            for (int i = 3 * ncoef_active; i < 3 * p.M; i++) gsh[i] = 0.0f;
        }
    }
    if (!in_range) return;

    // 4. outputs (every row written)
    float* o;
    o = p.dL_dmeans2D + 3 * (size_t)idx;
    o[0] = visible ? proxy2 * tm[8] * 0.5f * (float)p.W : 0.0f;
    o[1] = visible ? proxy5 * tm[8] * 0.5f * (float)p.H : 0.0f;
    o[2] = 0.0f;
    p.dL_dopacity[idx] = gopa;
    o = p.dL_dmeans3D + 3 * (size_t)idx; o[0] = g3[0]; o[1] = g3[1]; o[2] = g3[2];
    if (p.dL_dcolors) {
        o = p.dL_dcolors + 3 * (size_t)idx;
        if (p.defer_sh) { o[0] = dR_out[0]; o[1] = dR_out[1]; o[2] = dR_out[2]; }
        else            { o[0] = gc[0]; o[1] = gc[1]; o[2] = gc[2]; }
    }
    if (p.dL_dtransMat) {
        o = p.dL_dtransMat + 9 * (size_t)idx;
#pragma unroll
        for (int k = 0; k < 9; k++) o[k] = gT[k];
    }
    if (p.dL_dscales) { o = p.dL_dscales + 2 * (size_t)idx; o[0] = gs[0]; o[1] = gs[1]; }
    if (p.dL_drots) { o = p.dL_drots + 4 * (size_t)idx; o[0] = gq[0]; o[1] = gq[1]; o[2] = gq[2]; o[3] = gq[3]; }
}

// One warp per 32 splats: every lane evaluates the real SH basis of its own splat's view direction into shared
// memory (sh_basis: the basis preprocess backward multiplies), then the warp writes the 32 rows of 3M floats with
// coalesced stores, each value = basis[k] * dL_dcolor[c].  Splats whose colour gradient is exactly zero (culled
// everywhere) get zero rows without touching their direction.
__global__ void __launch_bounds__(128) sh_grad_expand_kernel(int P, int M, int D, const float* __restrict__ means3D,
                                                             const float* __restrict__ campos,
                                                             const float* __restrict__ dcol, float* __restrict__ dsh) {
    __shared__ float s_b[4][32][21];            // 16 basis values + 3 colour gradients per splat; odd stride: conflict-free
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int first = (blockIdx.x * 4 + warp) * 32;
    if (first >= P) return;
    const int idx = first + lane;
    float b[16];
#pragma unroll
    for (int k = 0; k < 16; k++) b[k] = 0.0f;
    float c0 = 0, c1 = 0, c2 = 0;
    if (idx < P) { c0 = dcol[3 * (size_t)idx]; c1 = dcol[3 * (size_t)idx + 1]; c2 = dcol[3 * (size_t)idx + 2]; }
    if (c0 != 0.0f || c1 != 0.0f || c2 != 0.0f) {
        const float dox = means3D[3 * (size_t)idx] - campos[0], doy = means3D[3 * (size_t)idx + 1] - campos[1],
                    doz = means3D[3 * (size_t)idx + 2] - campos[2];
        const float invl = 1.0f / sqrtf(dox * dox + doy * doy + doz * doz);
        sh_basis(D, dox * invl, doy * invl, doz * invl, [&](int i, float v) { b[i] = v; });
    }
#pragma unroll
    for (int k = 0; k < 16; k++) s_b[warp][lane][k] = b[k];
    s_b[warp][lane][16] = c0; s_b[warp][lane][17] = c1; s_b[warp][lane][18] = c2;
    __syncwarp();
    const int rows = min(32, P - first), row_len = 3 * M;
    float* out = dsh + (size_t)first * row_len;
    for (int f = lane; f < rows * row_len; f += 32) {
        const int row = f / row_len, j = f - row * row_len;
        const int k = j / 3, c = j - 3 * k;
        out[f] = k < 16 ? s_b[warp][row][k] * s_b[warp][row][16 + c] : 0.0f;
    }
}

int launch_sh_grad_expand(int P, int M, int D, const float* means3D, const float* campos,
                          const float* dL_dcolors, float* dL_dsh, cudaStream_t stream) {
    if (P <= 0 || M <= 0) return 0;
    sh_grad_expand_kernel<<<(P + 127) / 128, 128, 0, stream>>>(P, M, D, means3D, campos, dL_dcolors, dL_dsh);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_preprocess_bwd(const PreBwdParams& p, cudaStream_t stream) {
    if (p.P <= 0) return 0;
    LaunchScope scope(kStPreBwd, stream);
    const bool staged = !p.has_colors_precomp && p.shs != nullptr && p.D <= 3 && p.M == 16 &&
                        reinterpret_cast<uintptr_t>(p.shs) % 16 == 0 &&
                        (p.defer_sh || reinterpret_cast<uintptr_t>(p.dL_dsh) % 16 == 0);
    if (staged) preprocess_bwd_kernel<true><<<(p.P + 127) / 128, 128, 0, stream>>>(p);
    else        preprocess_bwd_kernel<false><<<(p.P + 127) / 128, 128, 0, stream>>>(p);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace surfel
