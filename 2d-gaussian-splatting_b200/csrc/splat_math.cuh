// splat_math.cuh — the per-splat SH and rotation math shared by preprocess forward, preprocess backward (and its
// SH expansion) and the camera backward, so that each is written once and every caller evaluates the same
// expressions (SURVEY Appendix A.1 / A.5).
#pragma once
#include "common.cuh"

namespace surfel {

// Each translation unit keeps its own copy of the tables (internal linkage: no host-symbol clash, and each
// kernel's constant-bank layout stays its own).
namespace {
__constant__ float kShC2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
__constant__ float kShC3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                               0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                               -0.5900435899266435f};
constexpr float kShC0 = 0.28209479177387814f;
constexpr float kShC1 = 0.4886025119029199f;
}  // namespace

// SH basis of the unit view direction (x, y, z) up to degree D, and the gradient of dR . colour with respect to
// that direction, returned as (ddx, ddy, ddz).  sh(i, c) reads coefficient i of channel c; basis(i, value) receives
// basis value i.  Within each degree band every dot product with dR is read before any of that band's basis
// values is handed out, so a caller may overwrite coefficient i in place from basis(i, .).  Passing a zero dR and
// an sh() that returns 0 leaves only the basis (the direction terms are then dead code).  D is read through the
// reference at each band's test: preprocess backward passes its kernel parameter, and with a by-value copy the
// compiler merges the band tests, which changes which products the unstaged kernel fuses into FMAs (its rounding).
// Basis values 1 and 3 are written -(C1 y), -(C1 x), equal to (-C1) y, (-C1) x, so that the forward's colour sum
// compiles to r - C1 y sh, the form the oracle states.
template <class Sh, class Basis>
__device__ __forceinline__ float3 sh_backward(const int& D, float x, float y, float z, const float dR[3], Sh sh, Basis basis) {
    auto dot = [&](int i) { return dR[0] * sh(i, 0) + dR[1] * sh(i, 1) + dR[2] * sh(i, 2); };
    float ddx = 0, ddy = 0, ddz = 0;
    basis(0, kShC0);
    if (D > 0) {
        const float d1 = dot(1), d2 = dot(2), d3 = dot(3);
        basis(1, -(kShC1 * y)); basis(2, kShC1 * z); basis(3, -(kShC1 * x));
        ddx += -kShC1 * d3; ddy += -kShC1 * d1; ddz += kShC1 * d2;
        if (D > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            const float d4 = dot(4), d5 = dot(5), d6 = dot(6), d7 = dot(7), d8 = dot(8);
            basis(4, kShC2[0] * xy); basis(5, kShC2[1] * yz); basis(6, kShC2[2] * (2.0f * zz - xx - yy));
            basis(7, kShC2[3] * xz); basis(8, kShC2[4] * (xx - yy));
            ddx += kShC2[0] * y * d4 + kShC2[2] * 2.0f * -x * d6 + kShC2[3] * z * d7 + kShC2[4] * 2.0f * x * d8;
            ddy += kShC2[0] * x * d4 + kShC2[1] * z * d5 + kShC2[2] * 2.0f * -y * d6 + kShC2[4] * 2.0f * -y * d8;
            ddz += kShC2[1] * y * d5 + kShC2[2] * 4.0f * z * d6 + kShC2[3] * x * d7;
            if (D > 2) {
                const float d9 = dot(9), d10 = dot(10), d11 = dot(11), d12 = dot(12), d13 = dot(13), d14 = dot(14), d15 = dot(15);
                basis(9, kShC3[0] * y * (3.0f * xx - yy)); basis(10, kShC3[1] * xy * z);
                basis(11, kShC3[2] * y * (4.0f * zz - xx - yy));
                basis(12, kShC3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy));
                basis(13, kShC3[4] * x * (4.0f * zz - xx - yy)); basis(14, kShC3[5] * z * (xx - yy));
                basis(15, kShC3[6] * x * (xx - 3.0f * yy));
                ddx += kShC3[0] * d9 * 6.0f * xy + kShC3[1] * d10 * yz + kShC3[2] * d11 * -2.0f * xy +
                       kShC3[3] * d12 * -6.0f * xz + kShC3[4] * d13 * (-3.0f * xx + 4.0f * zz - yy) +
                       kShC3[5] * d14 * 2.0f * xz + kShC3[6] * d15 * 3.0f * (xx - yy);
                ddy += kShC3[0] * d9 * 3.0f * (xx - yy) + kShC3[1] * d10 * xz +
                       kShC3[2] * d11 * (-3.0f * yy + 4.0f * zz - xx) + kShC3[3] * d12 * -6.0f * yz +
                       kShC3[4] * d13 * -2.0f * xy + kShC3[5] * d14 * -2.0f * yz + kShC3[6] * d15 * -6.0f * xy;
                ddz += kShC3[1] * d10 * xy + kShC3[2] * d11 * 8.0f * yz +
                       kShC3[3] * d12 * 3.0f * (2.0f * zz - xx - yy) + kShC3[4] * d13 * 8.0f * xz +
                       kShC3[5] * d14 * (xx - yy);
            }
        }
    }
    return make_float3(ddx, ddy, ddz);
}

// The SH basis alone: sh_backward with no colour gradient.
template <class Basis>
__device__ __forceinline__ void sh_basis(int D, float x, float y, float z, Basis basis) {
    const float none[3] = {0.0f, 0.0f, 0.0f};
    sh_backward(D, x, y, z, none, [](int, int) { return 0.0f; }, basis);
}

// The direction gradient dd of sh_backward carried through the normalisation u = d |d|^-1 of the unnormalised
// direction d = mean - campos (invl = 1 / |d|): the SH part of dL_dmeans3D.
__device__ __forceinline__ float3 sh_direction_to_mean(float dox, float doy, float doz, float invl, float3 dd) {
    const float inv3 = invl * invl * invl;
    return make_float3(((doy * doy + doz * doz) * dd.x - doy * dox * dd.y - doz * dox * dd.z) * inv3,
                       (-dox * doy * dd.x + (dox * dox + doz * doz) * dd.y - doz * doy * dd.z) * inv3,
                       (-dox * doz * dd.x - doy * doz * dd.y + (dox * dox + doy * doy) * dd.z) * inv3);
}

// q = (w, x, y, z) stored in a float4, times inv = 1 / |q|: the unit quaternion and its rotation matrix R.
struct QuatRotation {
    float w, x, y, z;
    float R[3][3];
};
__device__ __forceinline__ QuatRotation quat_rotation(float4 q, float inv) {
    QuatRotation r;
    const float w = q.x * inv, x = q.y * inv, y = q.z * inv, z = q.w * inv;
    r.w = w; r.x = x; r.y = y; r.z = z;
    r.R[0][0] = 1.0f - 2.0f * (y * y + z * z); r.R[0][1] = 2.0f * (x * y - w * z); r.R[0][2] = 2.0f * (x * z + w * y);
    r.R[1][0] = 2.0f * (x * y + w * z); r.R[1][1] = 1.0f - 2.0f * (x * x + z * z); r.R[1][2] = 2.0f * (y * z - w * x);
    r.R[2][0] = 2.0f * (x * z - w * y); r.R[2][1] = 2.0f * (y * z + w * x); r.R[2][2] = 1.0f - 2.0f * (x * x + y * y);
    return r;
}

// q normalised as preprocess forward and backward do.
__device__ __forceinline__ QuatRotation quat_rotation(float4 q) {
    return quat_rotation(q, 1.0f / sqrtf(((q.x * q.x + q.y * q.y) + q.z * q.z) + q.w * q.w));
}

}  // namespace surfel
