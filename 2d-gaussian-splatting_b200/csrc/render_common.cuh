// render_common.cuh — per-(pixel,splat) ray–splat evaluation shared by render forward/backward.
//
// Follows SURVEY.md Appendix A.3 (upstream renderCUDA; source not in /root/reference).  The
// arithmetic up to `alpha` is written with explicit round-to-nearest intrinsics so that forward and
// backward (separate translation units) take bit-identical skip/contribute decisions for a pair —
// the backward replay of transmittance depends on that.
#pragma once
#include "common.cuh"

namespace surfel {

struct PairEval {
    float dx, dy;                   // pixel - splat screen position c (note: upstream's d = c - pixel)
    float pz, inv_pz;               // cross(k,l).z and its reciprocal
    float sx, sy;                   // splat-space intersection
    float rho3d, rho2d;             // ray-splat and low-pass squared distances
    float G, alpha;
};

__device__ __forceinline__ float fast_rcp(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_ex2(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// Per-(pixel, splat) evaluation up to alpha, from the affine form of the ray-splat intersection
// (record layout: common.cuh):  p = Pc + dx P1 + dy P2,  s = p.xy / p.z,  rho3d = |s|^2,
// rho2d = 2 |d|^2,  alpha = min(0.99, opacity * exp(-0.5 min(rho3d, rho2d))).
//   q0 = (P1.x, P1.y, P1.z, c.x)   q1 = (P2.x, P2.y, P2.z, c.y)   q2 = (Pc.x, Pc.y, Pc.z, opacity)
// Returns false when the pair is skipped by A.3's `p.z == 0` or `alpha < 1/255` tests.  The remaining
// A.3 `continue` tests: `power > 0` cannot fire (rho >= 0 or NaN, and NaN compares false upstream as
// well); `depth < near` is applied by the callers once the depth is known, and only for splats that
// preprocess flagged (negative stored opacity) as able to reach in front of the near plane.
// Every operation is an explicit round-to-nearest intrinsic so that forward and backward (separate
// translation units) take bit-identical decisions for a pair.
__device__ __forceinline__ bool eval_pair(float pxf, float pyf, const float4& q0, const float4& q1,
                                          const float4& q2, PairEval& e) {
    e.dx = __fsub_rn(pxf, q0.w); e.dy = __fsub_rn(pyf, q1.w);
    const float ppx = __fmaf_rn(e.dy, q1.x, __fmaf_rn(e.dx, q0.x, q2.x));
    const float ppy = __fmaf_rn(e.dy, q1.y, __fmaf_rn(e.dx, q0.y, q2.y));
    e.pz = __fmaf_rn(e.dy, q1.z, __fmaf_rn(e.dx, q0.z, q2.z));
    e.inv_pz = fast_rcp(e.pz);
    e.sx = __fmul_rn(ppx, e.inv_pz); e.sy = __fmul_rn(ppy, e.inv_pz);
    e.rho3d = __fmaf_rn(e.sx, e.sx, __fmul_rn(e.sy, e.sy));
    const float h = __fmaf_rn(e.dx, e.dx, __fmul_rn(e.dy, e.dy));
    e.rho2d = __fadd_rn(h, h);                                   // FilterInvSquare = 2
    const float rho = fminf(e.rho3d, e.rho2d);
    e.G = fast_ex2(__fmul_rn(rho, -0.72134752044448170368f));    // exp(-0.5 rho)
    e.alpha = fminf(kAlphaMax, __fmul_rn(fabsf(q2.w), e.G));     // |.|: the sign of the stored opacity is the near-plane flag
    return !(e.alpha < kAlphaMin) && e.pz != 0.0f;
}

// Classification of one splat against the eight 8x4 warp footprints of a 16x16 tile, done by the thread
// that stages the splat's record (it has the record in registers): bit w of the result = the region
// where the splat can reach alpha >= 1/255 (screen AABB q6 and diagonal extents q7, both conservative)
// overlaps the footprint of warp w.  A miss is exact, not approximate: no pixel of that footprint can
// pass A.3's alpha test, so the warp never evaluates the pair.  (ox, oy) = the tile's first pixel.
__device__ __forceinline__ uint32_t classify_footprints(const float4& bb, const float4& dg, float ox, float oy) {
    // relative to the tile origin every bound is a small constant
    const float x0 = bb.x - ox, x1 = bb.z - ox, y0 = bb.y - oy, y1 = bb.w - oy;
    const float ou = ox + oy, ov = ox - oy;
    const float u0 = dg.x - ou, u1 = dg.y - ou, v0 = dg.z - ov, v1 = dg.w - ov;
    uint32_t m = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) {
        const float fx0 = (float)((w & 1) << 3), fx1 = fx0 + 7.0f;
        const float fy0 = (float)((w >> 1) << 2), fy1 = fy0 + 3.0f;
        const bool hit = x0 <= fx1 && x1 >= fx0 && y0 <= fy1 && y1 >= fy0 &&
                         u0 <= fx1 + fy1 && u1 >= fx0 + fy0 && v0 <= fx1 - fy0 && v1 >= fx0 - fy1;
        m |= hit ? (1u << w) : 0u;
    }
    return m;
}

// Position of the highest set bit (FLO) and the mask of the bits below a position (BMSK): the hit
// loops of the render kernels peel ballot bits with exactly these two instructions.
__device__ __forceinline__ uint32_t high_bit(uint32_t m) {
    uint32_t r;
    asm("bfind.u32 %0, %1;" : "=r"(r) : "r"(m));
    return r;
}
__device__ __forceinline__ uint32_t low_mask(uint32_t width) {
    uint32_t r;
    asm("bmsk.clamp.b32 %0, 0, %1;" : "=r"(r) : "r"(width));
    return r;
}

// Explicit shared-window addressing: one cvta per kernel instead of a generic->shared conversion
// (S2UR CgaCtaId + ULEA) re-materialised in every inner-loop iteration.
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ float2 lds64(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4& v) {
    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void sts64(uint32_t addr, float a, float b) {
    asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t addr, float a) {
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(a) : "memory");
}
__device__ __forceinline__ float lds32(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds32u(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

// Warp footprint inside a 16x16 tile: 8 (x) by 4 (y) pixels; warp w sits at (w&1, w>>1).
__device__ __forceinline__ void warp_pixel(int warp, int lane, int& lx, int& ly) {
    lx = ((warp & 1) << 3) + (lane & 7);
    ly = ((warp >> 1) << 2) + (lane >> 3);
}

}  // namespace surfel
