"""The float64 restatement of the tail's camera gradients (tests/tail_camera_exact.py, DESIGN §7q), checked on the
CPU before the GPU tests of surface_outputs and surface_regularizers lean on it:
  * its 21 sums, chained through the camera algebra by float64 autograd, equal float64 autograd of the reference's
    tail to 1e-12 of their magnitude, on holes, NaN medians, a far camera and odd frame sizes;
  * they reproduce the reference's own float32 camera gradients (ref_tail_camera.npz) within float32 rounding of
    that magnitude;
  * lambda_normal == 0 gives exactly zero;
  * the C ABI refuses bad sizes and NULL buffers without a device."""
import ctypes
import os

import numpy as np
import pytest
import torch

import tail_camera_exact as C
import tail_loss_scenes as TS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_tail_camera.npz")
KEYS = ("rend_alpha", "rend_normal", "rend_dist", "surf_depth", "surf_normal")
PAIRS = ((0.05, 0.0), (0.05, 100.0), (0.05, 1000.0), (0.0, 100.0), (0.0, 0.0))
EXACT = 1e-12      # float64 against float64: relative to the chained magnitude of the sums
CASES = [("golden", 0.0), ("golden", 1.0), ("holes", 0.3), ("nan_medians", 1.0), ("zero_alpha_depth", 0.0),
         ("far_camera", 0.3), ("f3x3", 0.3), ("f2x2", 0.3), ("f1x64", 0.3), ("f31x7", 0.3), ("f33x9", 0.3)]


def _camera(s):
    H, W = s["allmap"].shape[1:]
    rot, rays = C.view_matrices(torch.from_numpy(s["view"]), torch.from_numpy(s["proj"]), W, H)
    return W, H, rot, rays


def _check(G, B, s, ref, scale):
    """max |chain(G) - ref| / (scale * chained B) over both matrices (0/0 counts as 0, x/0 as inf)."""
    W, H = s["allmap"].shape[2], s["allmap"].shape[1]
    got, bounds = C.chain(G, s["view"], s["proj"], W, H), C.chain_bound(B, s["view"], s["proj"], W, H)
    worst = 0.0
    for g, r, b in zip(got, ref, bounds):
        r = torch.as_tensor(np.asarray(r)).double()
        allowed = scale * (b + g.abs())
        err = (g - r).abs()
        assert bool(((err == 0) | (allowed > 0)).all()), (g, r)
        worst = max(worst, float((err / allowed.clamp_min(1e-300)).max()))
    return worst


@pytest.mark.parametrize("name,ratio", CASES)
def test_restatement_equals_float64_autograd_of_the_outputs_tail(name, ratio):
    s = TS.ALLMAPS[name][0]()
    W, H, rot, rays = _camera(s)
    for kind in ("all", "rend_normal", "surf_normal"):
        cot = TS.cotangents(H, W, "random")
        if kind != "all":
            cot = {k: (v if k == kind else np.zeros_like(v)) for k, v in cot.items()}
        G, B = C.outputs_sums(s["allmap"], rot, rays, ratio, cot)
        ref = C.reference_camera_grads(s["allmap"], s["view"], s["proj"], ratio, C.outputs_loss(cot))
        assert _check(G, B, s, ref, EXACT) <= 1.0, kind
        if kind == "rend_normal":                 # no surf_normal cotangent: no point gradient, no ray term
            assert bool((G[9:] == 0).all())
        if kind == "surf_normal":
            assert bool((G[:9] == 0).all())


@pytest.mark.parametrize("name,ratio", CASES)
def test_restatement_equals_float64_autograd_of_the_regularisers(name, ratio):
    s = TS.ALLMAPS[name][0]()
    W, H, rot, rays = _camera(s)
    for ln, ld, gn in ((0.05, 100.0, 1.0), (0.05, 0.0, -2.5)):
        G, B = C.reg_sums(s["allmap"], rot, rays, ratio, ln, gn)
        loss = C.reg_loss(ln, ld)
        ref = C.reference_camera_grads(s["allmap"], s["view"], s["proj"], ratio, lambda out: gn * loss(out))
        assert _check(G, B, s, ref, EXACT) <= 1.0, (ln, ld, gn)
    G, _ = C.reg_sums(s["allmap"], rot, rays, ratio, 0.0)
    assert bool((G == 0).all())


def test_golden_is_the_tail_golden_scene():
    g = np.load(GOLDEN)
    s = TS.golden()
    assert np.array_equal(g["allmap"], s["allmap"]) and np.array_equal(g["viewmatrix"], s["view"])
    assert np.array_equal(g["projmatrix"], s["proj"])


@pytest.mark.parametrize("ratio", (0.0, 1.0))
def test_restatement_reproduces_the_reference(ratio):
    """The reference ran in float32: its camera gradients sit within u of the sums' chained magnitude (the worst
    ratio on the golden is 0.21; the magnitudes are large there because normalize's eps branch, at holes, scales a
    cotangent by 1e12, and those terms cancel)."""
    g = np.load(GOLDEN)
    s = TS.golden()
    W, H, rot, rays = _camera(s)
    cot = {k: g["cot_" + k] for k in KEYS}
    G, B = C.outputs_sums(s["allmap"], rot, rays, ratio, cot)
    t = f"r{ratio:g}_outputs"
    assert _check(G, B, s, (g[t + "_grad_view"], g[t + "_grad_proj"]), C.U) <= 1.0
    for ln, ld in PAIRS:
        t = f"r{ratio:g}_n{ln:g}_d{ld:g}".replace(".", "p")
        G, B = C.reg_sums(s["allmap"], rot, rays, ratio, ln)
        ref = (g[t + "_grad_view"], g[t + "_grad_proj"])
        if ln == 0.0:
            assert not ref[0].any() and not ref[1].any() and bool((G == 0).all())
        else:
            assert _check(G, B, s, ref, C.U) <= 1.0, t


def test_c_abi_rejects_bad_arguments_without_a_device():
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    err = lambda: lib.surfel_last_error().decode()
    buf = (ctypes.c_double * 16)()
    p = ctypes.addressof(buf)
    for W, H in ((0, 4), (4, -1), (60000, 60000), (1, 600000)):
        assert lib.surfel_post_camera_partials_bytes(W, H) == 0
        assert lib.surfel_post_camera_backward(W, H, 0.0, *([p] * 11), None) != 0 and "bad size" in err()
        assert lib.surfel_post_reg_camera_backward(W, H, 0.0, 0.05, 100.0, *([p] * 8), None) != 0 and "bad size" in err()
    # a 32 x 64 pixel tile per block, 21 double partials each
    assert lib.surfel_post_camera_partials_bytes(33, 65) == 21 * 8 * 2 * 2
    assert lib.surfel_post_camera_partials_bytes(1920, 1080) == 21 * 8 * 60 * 17
    # the three cotangents (arguments 4-6) may be NULL; everything else is required
    for k in (0, 1, 2, 3, 7, 8, 9, 10):
        args = [p] * 11
        args[k] = None
        assert lib.surfel_post_camera_backward(4, 4, 0.0, *args, None) != 0 and "NULL required" in err(), k
    for k in range(8):
        args = [p] * 8
        args[k] = None
        assert lib.surfel_post_reg_camera_backward(4, 4, 0.0, 0.05, 100.0, *args, None) != 0 \
            and "NULL required" in err(), k
