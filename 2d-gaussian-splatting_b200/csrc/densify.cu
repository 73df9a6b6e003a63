// densify.cu — GaussianModel.densify_and_prune of the reference trainer (scene/gaussian_model.py:348-403,
// called at train.py:132): clone, split and the final prune of all six parameter groups and their Adam moments in
// one compaction, a plan and an apply (DESIGN.md §7h has the rules; tests/densify_ref.py restates them).
//
//  * surfel_densify_plan: one pass over the P rows.  Each row's fate depends on that row alone (rules 2, 3
//    and 7 of §7h never look at the random draw), so the pass decides, per row, whether the original
//    survives, whether it is cloned and the clone survives, whether it is split and its two copies survive,
//    and scans four counters across the grid with a single-pass decoupled look-back (scan.cuh): kept
//    originals, kept clones, split rows (all of them: they index the random draw) and kept split
//    rows.  It stores one int4 per row (the row's rank in each segment, -1 where it has none) and the
//    four totals; the caller reads the totals with one device-to-host copy.
//  * surfel_densify_apply: one launch writes every output row of every group in its table exactly once, params
//    and both moments, from a by-value table of the groups (like surfel_adam_step); a caller may give the groups
//    of one plan to several apply calls, to free old tensors in between.  The output order is the
//    reference's: kept originals | kept clones | kept split copies A | kept split copies B.  Split copies
//    get xyz + R(q) (z*s) and log(exp(scaling) / 1.6); every new row gets zero moments.
//
// Float operations follow torch's CUDA kernels one for one, so decisions and values are bit for bit those
// of the eager reference on the GPU: g = accum / denom (IEEE division, NaN -> 0), exp / log / sigmoid as
// expf / logf / 1 / (1 + expf(-x)), norm of a length-1 row as sqrt(g*g), and `tensor / 1.6` as torch does
// it for a CPU scalar: a multiply by the float reciprocal 1.0f / 1.6f.  The file is compiled with
// -fmad=false so that no product is contracted into a neighbouring sum.  Only the split rows' xyz may differ
// from the reference in the last bits: the reference sums R (z*s) in a cuBLAS bmm of unspecified order.
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/surfel_rasterizer.h"
#include "common.cuh"
#include "profile.h"
#include "scan.cuh"

namespace surfel {

constexpr int kPlanThreads = 256;                 // rows per plan block; block-local counts fit in 16 bits
constexpr int kApplyThreads = 256;
// elements a thread loads before it stores any: the plan and one apply over all groups took 0.695 ms at 1 M rows
// with 4, 0.756 ms with 8 (H100 80GB HBM3, 700 W)
constexpr int kApplyPerThread = 4;
constexpr int kApplyTile = kApplyThreads * kApplyPerThread;   // floats of one group per apply block
constexpr int kDensifyMaxP = (1 << 30) - 1;       // P' <= 2P must fit an int32 row index

struct DensifyLayout {
    size_t ctrl, status, rec, total;
    unsigned blocks;
};

static DensifyLayout densify_layout(int P) {
    DensifyLayout L;
    L.blocks = grid_blocks(P, kPlanThreads);
    size_t o = 0;
    L.ctrl = o;   o = align_up(o + 64, 256);                          // [0] ticket, [4..7] KO, KC, S, KS
    L.status = o; o = align_up(o + (size_t)4 * L.blocks * 8, 256);    // one look-back word per counter per block
    L.rec = o;    o = align_up(o + (size_t)(P > 0 ? P : 1) * 16, 256);
    L.total = o;
    return L;
}

// torch.max over a dim propagates NaN; fmaxf would drop it
__device__ __forceinline__ float max_nan(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }

struct PlanParams {
    int P;
    const float *accum, *denom, *scaling, *opacity;
    float max_grad, min_opacity, clone_max, prune_max, screen, inv_div;
    int use_screen;
    uint32_t* ctrl;
    unsigned long long* status;   // [4][blocks]
    int4* rec;
    int32_t* totals;
};

__global__ void __launch_bounds__(kPlanThreads) densify_plan_kernel(const __grid_constant__ PlanParams p) {
    __shared__ unsigned long long s_warp[kPlanThreads / 32];
    __shared__ uint32_t s_excl[4];
    const int tid = threadIdx.x;
    const uint32_t bid = block_ticket(&p.ctrl[0]);
    const int i = (int)(bid * kPlanThreads) + tid;

    bool keep_orig = false, keep_clone = false, split = false, keep_split = false;
    if (i < p.P) {
        float g = __fdiv_rn(p.accum[i], p.denom[i]);                  // xyz_gradient_accum / denom
        if (g != g) g = 0.0f;                                        // grads[grads.isnan()] = 0
        const float s0 = expf(p.scaling[2 * (size_t)i]), s1 = expf(p.scaling[2 * (size_t)i + 1]);
        const float smax = max_nan(s0, s1);
        const float gnorm = __fsqrt_rn(__fmul_rn(g, g));             // torch.norm over a length-1 dim
        const bool clone = gnorm >= p.max_grad && smax <= p.clone_max;
        split = g >= p.max_grad && smax > p.clone_max;               // a clone's padded gradient is 0
        const float op = p.opacity[i];
        const float sig = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-op)));
        // a clone has its source's opacity and scale, and max_radii2D is all zeros when the prune reads it
        const bool base = sig < p.min_opacity || (p.use_screen && 0.0f > p.screen);
        if (split) {
            const float n0 = expf(logf(__fmul_rn(s0, p.inv_div))), n1 = expf(logf(__fmul_rn(s1, p.inv_div)));
            keep_split = !(base || (p.use_screen && max_nan(n0, n1) > p.prune_max));
        } else {
            keep_orig = !(base || (p.use_screen && smax > p.prune_max));
            keep_clone = clone && keep_orig;
        }
    }
    // four 0/1 counters packed in 16-bit fields (block-local sums <= 256)
    const unsigned long long mine = (unsigned long long)keep_orig | (unsigned long long)keep_clone << 16 |
                                    (unsigned long long)split << 32 | (unsigned long long)keep_split << 48;
    unsigned long long block_total;
    const unsigned long long excl_local = block_exclusive_scan<kPlanThreads>(mine, s_warp, block_total);
    auto field = [](unsigned long long x, int c) { return (uint32_t)(x >> (16 * c)) & 0xffffu; };
    const uint32_t total[4] = {field(block_total, 0), field(block_total, 1), field(block_total, 2),
                               field(block_total, 3)};
    block_lookback<4>(p.status, gridDim.x, bid, total, s_excl);
    if (bid == gridDim.x - 1 && tid == 0) {
        const uint32_t ko = s_excl[0] + total[0], kc = s_excl[1] + total[1], s = s_excl[2] + total[2],
                       ks = s_excl[3] + total[3];
        p.ctrl[4] = ko; p.ctrl[5] = kc; p.ctrl[6] = s; p.ctrl[7] = ks;
        p.totals[0] = (int)ko; p.totals[1] = (int)kc; p.totals[2] = (int)s; p.totals[3] = (int)(ko + kc + 2 * ks);
    }
    if (i < p.P) {
        int4 r;
        r.x = keep_orig ? (int)(s_excl[0] + field(excl_local, 0)) : -1;
        r.y = keep_clone ? (int)(s_excl[1] + field(excl_local, 1)) : -1;
        r.z = keep_split ? (int)(s_excl[3] + field(excl_local, 3)) : -1;
        r.w = split ? (int)(s_excl[2] + field(excl_local, 2)) : -1;
        p.rec[i] = r;
    }
}

struct ApplyGroup {
    const float *p, *m, *v;
    float *op, *om, *ov;
    int D, kind;
};

struct ApplyTable {
    ApplyGroup g[SURFEL_DENSIFY_MAX_GROUPS];
    long long first_block[SURFEL_DENSIFY_MAX_GROUPS + 1];
    int n, P, rot, scale;
    float inv_div;
    const float* z;          // (2S, 3) standard normal draws
    const int4* rec;
    const uint32_t* ctrl;    // [4..7] KO, KC, S, KS
};

// xyz of both copies of split row `row`, component c: xyz + R(q) @ (z0*s0, z1*s1, z2*0), with R built as
// build_rotation does (utils/general_utils.py:78-99) and normal(mean=0, std) = z*std + 0
__device__ __forceinline__ void split_xyz(const ApplyTable& t, long long row, int c, float x, long long zk, long long S,
                                          float& a_out, float& b_out) {
    const float* q = t.g[t.rot].p + 4 * row;
    const float q0 = q[0], q1 = q[1], q2 = q[2], q3 = q[3];
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q0, q0), __fmul_rn(q1, q1)), __fmul_rn(q2, q2)),
                                           __fmul_rn(q3, q3)));
    const float r = __fdiv_rn(q0, nrm), qx = __fdiv_rn(q1, nrm), qy = __fdiv_rn(q2, nrm), qz = __fdiv_rn(q3, nrm);
    auto one_minus = [](float a, float b) { return __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(a, b))); };
    auto two_sub = [](float a, float b) { return __fmul_rn(2.0f, __fsub_rn(a, b)); };
    auto two_add = [](float a, float b) { return __fmul_rn(2.0f, __fadd_rn(a, b)); };
    float R0, R1, R2;
    if (c == 0) {
        R0 = one_minus(__fmul_rn(qy, qy), __fmul_rn(qz, qz));
        R1 = two_sub(__fmul_rn(qx, qy), __fmul_rn(r, qz));
        R2 = two_add(__fmul_rn(qx, qz), __fmul_rn(r, qy));
    } else if (c == 1) {
        R0 = two_add(__fmul_rn(qx, qy), __fmul_rn(r, qz));
        R1 = one_minus(__fmul_rn(qx, qx), __fmul_rn(qz, qz));
        R2 = two_sub(__fmul_rn(qy, qz), __fmul_rn(r, qx));
    } else {
        R0 = two_sub(__fmul_rn(qx, qz), __fmul_rn(r, qy));
        R1 = two_add(__fmul_rn(qy, qz), __fmul_rn(r, qx));
        R2 = one_minus(__fmul_rn(qx, qx), __fmul_rn(qy, qy));
    }
    const float* sc = t.g[t.scale].p + 2 * row;
    const float s0 = expf(sc[0]), s1 = expf(sc[1]);
    auto offset = [&](long long zr) {
        const float* zz = t.z + 3 * zr;
        const float a0 = __fadd_rn(__fmul_rn(zz[0], s0), 0.0f), a1 = __fadd_rn(__fmul_rn(zz[1], s1), 0.0f),
                    a2 = __fadd_rn(__fmul_rn(zz[2], 0.0f), 0.0f);
        return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R0, a0), __fmul_rn(R1, a1)), __fmul_rn(R2, a2)), x);
    };
    a_out = offset(zk);
    b_out = offset(S + zk);
}

__global__ void __launch_bounds__(kApplyThreads) densify_apply_kernel(const __grid_constant__ ApplyTable t) {
    int gi = 0;
    const long long b = blockIdx.x;
#pragma unroll
    for (int k = 1; k < SURFEL_DENSIFY_MAX_GROUPS; k++)
        if (k < t.n && b >= t.first_block[k]) gi = k;
    const ApplyGroup& G = t.g[gi];
    const int D = G.D;
    const long long n_el = (long long)t.P * D;
    const long long base = (b - t.first_block[gi]) * kApplyTile;
    const long long row0 = base / D;
    const int off0 = (int)(base - row0 * D);
    const long long KO = t.ctrl[4], KC = t.ctrl[5], S = t.ctrl[6], KS = t.ctrl[7];
    const bool state = G.m != nullptr;

    // loads of all of this thread's elements first, then the stores: kApplyPerThread independent loads in flight
    float pv[kApplyPerThread], mv[kApplyPerThread], vv[kApplyPerThread];
    int4 rc[kApplyPerThread];
#pragma unroll
    for (int k = 0; k < kApplyPerThread; k++) {
        const int l = off0 + k * kApplyThreads + (int)threadIdx.x;
        const long long e = base + k * kApplyThreads + threadIdx.x;
        rc[k] = make_int4(-1, -1, -1, -1);
        pv[k] = mv[k] = vv[k] = 0.0f;
        if (e < n_el) {
            rc[k] = __ldg(t.rec + row0 + l / D);
            pv[k] = __ldg(G.p + e);
            if (state && rc[k].x >= 0) { mv[k] = __ldg(G.m + e); vv[k] = __ldg(G.v + e); }
        }
    }
#pragma unroll
    for (int k = 0; k < kApplyPerThread; k++) {
        const int l = off0 + k * kApplyThreads + (int)threadIdx.x;
        const int r = l / D, c = l - r * D;
        const int4 q = rc[k];
        if (q.x >= 0) {                                          // surviving original: param and moments kept
            const long long o = (long long)q.x * D + c;
            G.op[o] = pv[k];
            if (state) { G.om[o] = mv[k]; G.ov[o] = vv[k]; }
        }
        if (q.y >= 0) {                                          // clone: a copy with zero moments
            const long long o = (KO + q.y) * D + c;
            G.op[o] = pv[k];
            if (state) { G.om[o] = 0.0f; G.ov[o] = 0.0f; }
        }
        if (q.z >= 0) {                                          // both copies of a split row
            const long long oa = (KO + KC + q.z) * D + c, ob = oa + KS * D;
            float va = pv[k], vb = pv[k];
            if (G.kind == SURFEL_DENSIFY_SCALING) {
                va = vb = logf(__fmul_rn(expf(pv[k]), t.inv_div));   // log(exp(s) / (0.8 * 2))
            } else if (G.kind == SURFEL_DENSIFY_XYZ) {
                split_xyz(t, row0 + r, c, pv[k], q.w, S, va, vb);
            }
            G.op[oa] = va;
            G.op[ob] = vb;
            if (state) { G.om[oa] = 0.0f; G.ov[oa] = 0.0f; G.om[ob] = 0.0f; G.ov[ob] = 0.0f; }
        }
    }
}

}  // namespace surfel

using namespace surfel;

extern "C" {

size_t surfel_densify_workspace_bytes(int P) {
    if (P < 0 || P > kDensifyMaxP) return 0;
    return densify_layout(P).total;
}

int surfel_densify_plan(int P, const float* xyz_gradient_accum, const float* denom, const float* scaling,
                        const float* opacity, double max_grad, double min_opacity, double clone_max_scale,
                        double prune_max_scale, int use_max_screen_size, double max_screen_size, void* workspace,
                        size_t workspace_bytes, int32_t* totals, void* stream) {
    if (P < 0) { surfel_set_error("surfel_densify_plan: P < 0"); return 1; }
    if (P > kDensifyMaxP) { surfel_set_error("surfel_densify_plan: P = %d exceeds %d", P, kDensifyMaxP); return 1; }
    if (!totals) { surfel_set_error("surfel_densify_plan: NULL totals"); return 1; }
    if (P > 0 && (!xyz_gradient_accum || !denom || !scaling || !opacity)) {
        surfel_set_error("surfel_densify_plan: NULL input pointer");
        return 1;
    }
    const DensifyLayout L = densify_layout(P);
    if (!workspace_ok("surfel_densify_plan", workspace, workspace_bytes, L.total)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    char* w = (char*)workspace;
    uint32_t* ctrl = (uint32_t*)(w + L.ctrl);
    SURFEL_CUDA_OK(cudaMemsetAsync(ctrl, 0, 64, st));
    if (P == 0) {
        SURFEL_CUDA_OK(cudaMemsetAsync(totals, 0, 4 * sizeof(int32_t), st));
        return 0;
    }
    SURFEL_CUDA_OK(cudaMemsetAsync(w + L.status, 0, (size_t)4 * L.blocks * 8, st));
    PlanParams p;
    p.P = P;
    p.accum = xyz_gradient_accum; p.denom = denom; p.scaling = scaling; p.opacity = opacity;
    // Python forms the thresholds in double; torch rounds each once to float32 when it compares
    p.max_grad = (float)max_grad; p.min_opacity = (float)min_opacity;
    p.clone_max = (float)clone_max_scale; p.prune_max = (float)prune_max_scale;
    p.use_screen = use_max_screen_size != 0; p.screen = (float)max_screen_size;
    const float div = (float)(0.8 * 2);
    p.inv_div = 1.0f / div;
    p.ctrl = ctrl;
    p.status = (unsigned long long*)(w + L.status);
    p.rec = (int4*)(w + L.rec);
    p.totals = totals;
    LaunchScope scope(kStDensify, st);
    densify_plan_kernel<<<L.blocks, kPlanThreads, 0, st>>>(p);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

int surfel_densify_apply(int P, int P_out, int n_split, int n_groups, const surfel_densify_group_t* groups,
                         const float* z, const void* workspace, size_t workspace_bytes, void* stream) {
    if (P < 0) { surfel_set_error("surfel_densify_apply: P < 0"); return 1; }
    if (P > kDensifyMaxP) { surfel_set_error("surfel_densify_apply: P = %d exceeds %d", P, kDensifyMaxP); return 1; }
    if (P_out < 0 || P_out > 2 * P || n_split < 0 || n_split > P) {
        surfel_set_error("surfel_densify_apply: P_out = %d, n_split = %d inconsistent with P = %d", P_out, n_split, P);
        return 1;
    }
    if (n_groups < 1 || n_groups > SURFEL_DENSIFY_MAX_GROUPS) {
        surfel_set_error("surfel_densify_apply: n_groups %d outside [1, %d]", n_groups, SURFEL_DENSIFY_MAX_GROUPS);
        return 1;
    }
    if (!groups) { surfel_set_error("surfel_densify_apply: NULL groups"); return 1; }
    if (n_split > 0 && !z) { surfel_set_error("surfel_densify_apply: NULL z with %d split rows", n_split); return 1; }
    const DensifyLayout L = densify_layout(P);
    if (!workspace_ok("surfel_densify_apply", workspace, workspace_bytes, L.total)) return 1;
    ApplyTable t;
    t.n = 0; t.P = P; t.rot = t.scale = -1;
    int xyz = -1;
    long long blocks = 0;
    for (int i = 0; i < n_groups; i++) {
        const surfel_densify_group_t& g = groups[i];
        const int need = g.kind == SURFEL_DENSIFY_XYZ ? 3 : g.kind == SURFEL_DENSIFY_SCALING ? 2
                       : g.kind == SURFEL_DENSIFY_ROTATION ? 4 : -1;
        if (g.kind < SURFEL_DENSIFY_COPY || g.kind > SURFEL_DENSIFY_ROTATION) {
            surfel_set_error("surfel_densify_apply: group %d has unknown kind %d", i, g.kind);
            return 1;
        }
        if (g.row_floats < 0 || (need > 0 && g.row_floats != need)) {
            surfel_set_error("surfel_densify_apply: group %d has %d floats per row", i, g.row_floats);
            return 1;
        }
        int* slot = g.kind == SURFEL_DENSIFY_XYZ ? &xyz : g.kind == SURFEL_DENSIFY_SCALING ? &t.scale
                  : g.kind == SURFEL_DENSIFY_ROTATION ? &t.rot : nullptr;
        if (slot) {
            if (*slot >= 0) { surfel_set_error("surfel_densify_apply: two groups of kind %d", g.kind); return 1; }
            *slot = i;
        }
        if (!g.exp_avg != !g.exp_avg_sq || !g.out_exp_avg != !g.out_exp_avg_sq) {
            surfel_set_error("surfel_densify_apply: group %d has only one of its two moments", i);
            return 1;
        }
        const bool in_rows = P > 0 && g.row_floats > 0, out_rows = P_out > 0 && g.row_floats > 0;
        if ((in_rows && !g.param) || (out_rows && !g.out_param)) {
            surfel_set_error("surfel_densify_apply: group %d has a NULL parameter", i);
            return 1;
        }
        if ((in_rows && out_rows && !g.exp_avg != !g.out_exp_avg) || (!in_rows && out_rows)) {
            surfel_set_error("surfel_densify_apply: group %d: moments in and out disagree", i);
            return 1;
        }
    }
    if (xyz >= 0 && (t.scale < 0 || t.rot < 0)) {   // split copies' xyz reads the source rotation and scaling
        surfel_set_error("surfel_densify_apply: a table with the xyz group needs the scaling and rotation groups");
        return 1;
    }
    for (int i = 0; i < n_groups; i++) {
        const surfel_densify_group_t& g = groups[i];
        ApplyGroup& a = t.g[i];
        a.p = g.param; a.m = g.exp_avg; a.v = g.exp_avg_sq;
        a.op = g.out_param; a.om = g.out_exp_avg; a.ov = g.out_exp_avg_sq;
        if (!a.om) a.m = a.v = nullptr;          // no state: gathered without moments
        a.D = g.row_floats; a.kind = g.kind;
        t.first_block[i] = blocks;
        blocks += ((long long)P * g.row_floats + kApplyTile - 1) / kApplyTile;
        t.n++;
    }
    t.first_block[t.n] = blocks;
    if (blocks == 0) return 0;
    if (blocks > 0x7fffffffLL) { surfel_set_error("surfel_densify_apply: too many elements"); return 1; }
    const char* w = (const char*)workspace;
    t.inv_div = 1.0f / (float)(0.8 * 2);
    t.z = z;
    t.rec = (const int4*)(w + L.rec);
    t.ctrl = (const uint32_t*)(w + L.ctrl);
    cudaStream_t st = (cudaStream_t)stream;
    LaunchScope scope(kStDensify, st);
    densify_apply_kernel<<<(unsigned)blocks, kApplyThreads, 0, st>>>(t);
    SURFEL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
