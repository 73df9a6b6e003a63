"""The render kernels held to the exact (float64) evaluation, entry by entry, on certified scenes built around their
batch, warp and edge boundaries (tests/hitloop_scenes.py).

No budget: on a certified scene no pair sits within 1e-4 (relative) of a discontinuity, far above the CUDA path's
few 1e-7 from exact, so every output entry, every n_contrib entry and every gradient row must agree.
  * forward: all 10 output planes and accum within FWD_TOL * max(1, |ref|); both n_contrib planes EQUAL;
  * backward, render level (the per-splat sums the render backward accumulates): within GRAD_TOL times the sum over
    pairs of each contribution evaluated on the absolute values of its terms (oracle render_bwd_f64's dL_dabs), so a
    sum that cancels, across pairs or inside one, is judged at the scale its float32 terms round at;
  * backward, leaf level: the same bound carried through preprocess backward (its per-splat Jacobian, in absolute
    value, applied to those sums).
Each scene runs under one random all-channel cotangent and one per channel group, so the term of one channel
cannot hide behind the others, and against the main library and every batch-size variant of build.py.
"""
import importlib.util
import os

import numpy as np
import pytest

import hitloop_scenes as HS
from parity_bars import record_stats

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location(
    "surfel_b200_build", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                      "2d-gaussian-splatting_b200", "build.py"))
_build = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_build)

# Tolerances, cut from the worst values observed on an H100 80GB HBM3 (400 W power limit) over every scene, cotangent
# and library below, with about 4x headroom.  Each bound is met by every entry: there is no budget.
FWD_TOL = 1e-5          # outputs and accum, |got - ref| / max(1, |ref|); worst observed 2.6e-6 (count1100, allmap)
GRAD_TOL = 1e-5         # render-level sums, |got - ref| / magnitude sum; worst observed 2.9e-6 (ragged41x1, dL_dcolors)
# leaf gradients, |got - ref| / (|J| magnitude sum + ROW_FLOOR * the splat's largest leaf bound)
LEAF_TOL = dict(dL_dtransMat=1e-5,     # worst observed 2.1e-6
                dL_dmeans2D=3e-6,      # 6.0e-7
                dL_dmeans3D=1e-5,      # 2.1e-6
                dL_drotations=1e-5,    # 2.4e-6
                dL_dshs=8e-5,          # 2.0e-5
                dL_dscales=4e-4)       # 8.9e-5 (count33: fronto-parallel splats, where dL_dTu / dL_dTv cancel)
ROW_FLOOR = 1e-3        # x the largest leaf bound of the splat

LIBS = ("main",) + tuple(_build.VARIANTS)
SCENES = tuple(f"count{k}" for k in HS.COUNTS) + (
    "warps_apart", "all_saturate", "median_boundaries", "near_plane", "low_pass", "tile_band") + \
    tuple(f"ragged{W}x{H}" for W, H in HS.RAGGED)
LEAF_KEYS = ("dL_dtransMat", "dL_dmeans2D", "dL_dmeans3D", "dL_dscales", "dL_drotations", "dL_dshs")


def scene(O, name):
    if name.startswith("count"):
        return HS.count_sweep(O, int(name[5:]))
    if name.startswith("ragged"):
        W, H = map(int, name[6:].split("x"))
        return HS.ragged(O, W, H)
    return getattr(HS, name)(O)


_handles = {}


def lib_handle(cuda_lib, name):
    if name == "main":
        return cuda_lib
    if name not in _handles:
        from diff_surfel_rasterization import _cabi
        _handles[name] = _cabi.load_handle(_build.variant_path(name))
    return _handles[name]


_jac = {}


def leaf_jacobian_abs(O, name, s):
    """|d leaf / d render-level sum| per splat, one column per render-level entry (preprocess backward is per splat
    and linear in its inputs): {leaf key: (18, P, ...)} in the order of oracle.ABS_LAYOUT."""
    if name in _jac:
        return _jac[name]
    pre, sc, cam = s["pre"], s["scene"], s["cam"]
    P = pre["radii"].shape[0]
    cols = {k: [] for k in LEAF_KEYS}
    for key, a, b in O.ABS_LAYOUT:
        for j in range(b - a):
            rb = dict(dL_dtransMat=np.zeros((P, 9)), dL_dmean2D=np.zeros((P, 2)), dL_dopacity=np.zeros(P),
                      dL_dnormal=np.zeros((P, 3)), dL_dcolors=np.zeros((P, 3)))
            rb[key].reshape(P, -1)[:, j] = 1.0
            out = O.preprocess_bwd(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], pre, rb, cam["viewmatrix"],
                                   cam["projmatrix"], cam["campos"], cam["W"], cam["H"])
            for k in LEAF_KEYS:
                cols[k].append(np.abs(out[k].astype(np.float64)))
    _jac[name] = {k: np.stack(v) for k, v in cols.items()}
    return _jac[name]


def leaf_bound(O, jac, absum):
    a = np.concatenate([absum[k].reshape(absum[k].shape[0], -1) for k, _, _ in O.ABS_LAYOUT], 1)     # (P, 18)
    return {k: np.einsum("cp...,pc->p...", J, a) for k, J in jac.items()}


def worst_ratio(err, bound):
    """max of err / bound, where bound > 0; and whether an entry with bound 0 has a non-zero error."""
    pos = bound > 0
    r = float((err[pos] / bound[pos]).max()) if pos.any() else 0.0
    return r, bool((err[~pos] > 0).any())


@pytest.mark.parametrize("lib", LIBS)
@pytest.mark.parametrize("name", SCENES)
def test_hitloop_matches_exact_evaluation(oracle, cuda_lib, lib, name):
    from cuda_stages import CudaPipeline
    s = scene(oracle, name)
    HS.assert_certified(s)
    sc, cam, pre, binned, img = s["scene"], s["cam"], s["pre"], s["binned"], s["img"]
    W, H = cam["W"], cam["H"]
    rows = s["rows"]
    pipe = CudaPipeline(sc, cam, HS.BG, tile_rows=rows or (0, 0), lib=lib_handle(cuda_lib, lib))
    gp = pipe.preprocess()
    np.testing.assert_array_equal(gp["radii"], pre["radii"])
    bk = pipe.bucket()
    np.testing.assert_array_equal(bk["ranges"], binned["ranges"])
    np.testing.assert_array_equal(bk["vals_sorted"], binned["vals_sorted"])
    gi = pipe.render()
    ys = slice(0, H) if rows is None else slice(rows[0] * 16, min(H, rows[1] * 16))
    failures = []

    # ---- forward: every entry, no budget
    np.testing.assert_array_equal(gi["n_contrib"][:, ys], img["n_contrib"][:, ys], err_msg="n_contrib (last, median)")
    for key, got, ref in (("color", gi["color"], img["color"]), ("others", gi["others"], img["others"]),
                          ("accum", gi["accum"], img["accum"])):
        g, r = got[:, ys].astype(np.float64), ref[:, ys].astype(np.float64)
        err = np.abs(g - r) / np.maximum(1.0, np.abs(r))
        st = record_stats(f"hitloop fwd {key}", err, dict(tol=FWD_TOL, scene=name, lib=lib))
        if not (np.isfinite(g).all() and st["max"] <= FWD_TOL):
            failures.append(f"forward {key}: max rel error {st['max']:.3e} > {FWD_TOL}")

    # ---- backward, per cotangent
    jac = leaf_jacobian_abs(oracle, name, s)
    img_gpu = dict(accum=img["accum"].copy(), n_contrib=img["n_contrib"].copy())
    img_gpu["accum"][:, ys], img_gpu["n_contrib"][:, ys] = gi["accum"][:, ys], gi["n_contrib"][:, ys]   # a band leaves the other rows unwritten
    for gi_, group in enumerate(HS.CHANNEL_GROUPS):
        gc, go = HS.cotangent(W, H, group, seed=gi_)
        if rows is not None:                               # pixels outside the band have no tile list
            gc[:, :ys.start] = 0; go[:, :ys.start] = 0
        rb = oracle.render_bwd(pre, binned, img_gpu, HS.BG, gc, go, W, H, f64=True)
        ref = oracle.preprocess_bwd(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], pre, rb, cam["viewmatrix"],
                                    cam["projmatrix"], cam["campos"], W, H)
        got = pipe.backward(gc, go)
        rec = got["grad_rec"].astype(np.float64)
        render_level = (("dL_dmean2D", rec[:, 13:15]), ("dL_dopacity", rec[:, 15]), ("dL_dnormal", rec[:, 16:19]),
                        ("dL_dcolors", rec[:, 19:22]))
        for key, g in render_level:
            err = np.abs(g - rb[key])
            r, nz = worst_ratio(err, rb["abs"][key])
            record_stats(f"hitloop bwd {key} / abs-sum", np.array([r]), dict(tol=GRAD_TOL, scene=name, lib=lib, cot=group, nz=nz))
            if r > GRAD_TOL or nz or not np.isfinite(g).all():
                failures.append(f"{group}: render-level {key}: worst error / abs-sum {r:.3e} (nonzero where 0: {nz})")
        bound = leaf_bound(oracle, jac, rb["abs"])
        # preprocess backward forms a splat's leaf gradients from shared sums (the homography gradient from A, Bx, By,
        # Z; the SH row from one colour gradient): an entry's rounding follows the splat's largest term, even where its
        # own exact value is 0
        splat_scale = np.max([bound[k].reshape(bound[k].shape[0], -1).max(1) for k in LEAF_KEYS], 0)
        for key in LEAF_KEYS:
            g = got[key].astype(np.float64).reshape(ref[key].shape)
            if key == "dL_dmeans2D":
                g, rk, bk_ = g[:, :2], ref[key][:, :2], bound[key][:, :2]
            else:
                rk, bk_ = ref[key], bound[key]
            err = np.abs(g - rk)
            bk_ = bk_ + ROW_FLOOR * splat_scale.reshape((-1,) + (1,) * (bk_.ndim - 1))
            r, nz = worst_ratio(err, bk_)
            record_stats(f"hitloop leaf {key} / bound", np.array([r]), dict(tol=LEAF_TOL[key], scene=name, lib=lib, cot=group, nz=nz))
            if r > LEAF_TOL[key] or nz or not np.isfinite(g).all():
                failures.append(f"{group}: leaf {key}: worst error / bound {r:.3e} (nonzero where 0: {nz})")
    assert not failures, f"{name} [{lib}]:\n" + "\n".join(failures)
