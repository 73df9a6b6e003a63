// contraction.cuh — the contracted grid of the reference's unbounded mesh extraction, shared by tsdf.cu and mcubes.cu
// (DESIGN.md §7i rule 3, §7j rule 1).  Both files are compiled with -fmad=false and use explicitly rounded intrinsics
// only, so a numpy float32 emulation reproduces these bit for bit.
#pragma once
#include <cuda_runtime.h>

namespace surfel {

// |y| = sqrt((x*x + y*y) + z*z), correctly rounded
__device__ __forceinline__ float contraction_norm(float X, float Y, float Z) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(X, X), __fmul_rn(Y, Y)), __fmul_rn(Z, Z)));
}

// contracted -> world, given mag = contraction_norm(X, Y, Z): where !(mag < 1), y = 1/(2 - mag) * (y / mag) (inf or
// NaN at mag = 2, the far side of the centre beyond it), then y * radius + center
__device__ __forceinline__ void inv_contraction(float mag, float& X, float& Y, float& Z, float radius, float cx,
                                                float cy, float cz) {
    if (!(mag < 1.f)) {
        const float r = __frcp_rn(__fsub_rn(2.f, mag));
        X = __fmul_rn(r, __fdiv_rn(X, mag));
        Y = __fmul_rn(r, __fdiv_rn(Y, mag));
        Z = __fmul_rn(r, __fdiv_rn(Z, mag));
    }
    X = __fadd_rn(__fmul_rn(X, radius), cx);
    Y = __fadd_rn(__fmul_rn(Y, radius), cy);
    Z = __fadd_rn(__fmul_rn(Z, radius), cz);
}

// One axis of a crop: torch.linspace(start, end, steps) as torch's CUDA kernel computes it in float32.  start and end
// are the float32 roundings of the caller's doubles, step = (end - start) / (steps - 1) rounded once on the host; the
// first steps / 2 points are start + step * i, the rest end - step * (steps - 1 - i), each contracted to one FMA
// (kLinspaceFma; tests/test_mcubes_gpu.py checks this against torch.linspace itself).
constexpr bool kLinspaceFma = true;
// the largest crop side of the grid-mode field and of marching cubes: a crop's vertex records (<= 3 side^3) and
// triangles (<= 5 (side - 1)^3) are scanned in 32 bits
constexpr int kMcMaxSide = 512;

struct LinAxis {
    float start, end, step;
};

__device__ __forceinline__ float linspace_at(const LinAxis& a, int i, int steps) {
    if (i < steps / 2)
        return kLinspaceFma ? __fmaf_rn(a.step, (float)i, a.start) : __fadd_rn(a.start, __fmul_rn(a.step, (float)i));
    const float k = (float)(steps - 1 - i);
    return kLinspaceFma ? __fmaf_rn(-a.step, k, a.end) : __fsub_rn(a.end, __fmul_rn(a.step, k));
}

// the host side: torch rounds the Python floats once to float32 and divides in float32
inline LinAxis make_lin_axis(double start, double end, int steps) {
    LinAxis a;
    a.start = (float)start;
    a.end = (float)end;
    a.step = steps > 1 ? (a.end - a.start) / (float)(steps - 1) : 0.f;
    return a;
}

}  // namespace surfel
