"""The float64 evaluation of train.py's regularisers (tests/surface_reg_exact.py), checked on the CPU before the
GPU tests of postprocess.surface_regularizers lean on it:
  * it reproduces the reference's own values and gradients (ref_surface_reg.npz) within their bounds, with NaN
    exactly where the reference's gradient is NaN, and the D/alpha rule gives 0 there;
  * it agrees with float64 autograd of the restated tail and train.py's lines;
  * a float32 emulation of the fused kernels' algorithm stays inside the bounds on every scene, and each planted
    mistake breaks them;
  * the C ABI refuses bad sizes and NULL buffers without a device."""
import ctypes
import os

import numpy as np
import pytest
import torch

import surface_reg_exact as R
import tail_loss_scenes as TS
from test_postprocess_gpu import reference_tail

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_surface_reg.npz")
RATIOS = (0.0, 1.0)
PAIRS = ((0.05, 0.0), (0.05, 100.0), (0.05, 1000.0), (0.0, 100.0), (0.0, 0.0))


def _tag(ratio, ln, ld):
    return f"r{ratio:g}_n{ln:g}_d{ld:g}".replace(".", "p")


def test_golden_is_the_tail_golden_scene():
    g = np.load(GOLDEN)
    s = TS.golden()
    assert np.array_equal(g["allmap"], s["allmap"]) and np.array_equal(g["viewmatrix"], s["view"])
    assert np.array_equal(g["projmatrix"], s["proj"])
    assert int((s["allmap"][1] == 0).sum()) == 200


@pytest.mark.parametrize("ratio", RATIOS)
@pytest.mark.parametrize("ln,ld", PAIRS)
def test_float64_evaluation_reproduces_the_reference(ratio, ln, ld):
    g = np.load(GOLDEN)
    s = TS.golden()
    t = _tag(ratio, ln, ld)
    ex = R.reg_f64(s["allmap"], s["view"], s["proj"], ratio, ln, ld)
    ref_grad = torch.from_numpy(g[t + "_grad_allmap"])
    worst, _ = R.worst_ratios((g[t + "_normal_loss"], g[t + "_dist_loss"]), ref_grad, ex, "nan")
    assert max(worst.values()) <= 1.0, worst
    # the reference's gradient is NaN in channels 0 and 1 at every hole, whatever the lambdas; the rule gives 0
    nan = torch.isnan(ex[1])
    assert int(nan[:2].sum()) == 400 and not nan[2:].any()
    assert bool((ex[4][nan] == 0).all())
    if ln == 0.0:
        assert float(g[t + "_normal_loss"]) == 0.0 and ex[0][0] == 0.0
        assert bool((ex[1][:6][~nan[:6]] == 0).all()) and bool((ex[3][:6] == 0).all())


@pytest.mark.parametrize("name,ratio", [("golden", 0.3), ("holes", 0.0), ("nan_medians", 1.0), ("far_camera", 0.3),
                                        ("f3x3", 0.3)])
def test_float64_evaluation_matches_autograd_of_the_restatement(name, ratio):
    s = TS.ALLMAPS[name][0]()
    ln, ld = 0.05, 100.0
    a = torch.from_numpy(s["allmap"]).double().requires_grad_(True)
    out = reference_tail(a, R.view_of(s, dtype=torch.float64), ratio)
    normal_error = (1 - (out["rend_normal"] * out["surf_normal"]).sum(dim=0))[None]
    normal_loss, dist_loss = ln * normal_error.mean(), ld * out["rend_dist"].mean()
    (normal_loss + dist_loss).backward()
    normal_loss, dist_loss = normal_loss.detach(), dist_loss.detach()
    (vn, vd), grad, *_ = R.reg_f64(s["allmap"], s["view"], s["proj"], ratio, ln, ld)
    assert abs(float(normal_loss) - vn) <= 1e-12 * max(1.0, abs(vn)) and abs(float(dist_loss) - vd) <= 1e-12 * abs(vd)
    torch.testing.assert_close(a.grad, grad, rtol=1e-10, atol=1e-10 * float(grad.nan_to_num().abs().max()), equal_nan=True)


CPU_CASES = [(n, r) for n, r in TS.ALLMAP_CASES if n != "f1920x1080"]


@pytest.mark.parametrize("ln,ld", [(0.05, 1000.0), (0.05, 0.0), (0.0, 100.0)])
@pytest.mark.parametrize("name,ratio", CPU_CASES)
def test_float32_emulation_stays_inside_the_bounds(name, ratio, ln, ld):
    s = TS.ALLMAPS[name][0]()
    ex = R.reg_f64(s["allmap"], s["view"], s["proj"], ratio, ln, ld)
    values, grad = R.reg_f32_emulation(s["allmap"], s["view"], s["proj"], ratio, ln, ld)
    worst, _ = R.worst_ratios(values, grad, ex, "hole")
    assert max(worst.values()) <= 1.0, worst


def test_bounds_are_not_vacuous():
    """The emulation uses a visible share of the gradient and distortion bounds (measured 0.26 and 0.34 on the
    holes scene and the golden)."""
    for name, ratio in (("holes", 0.3), ("golden", 0.0)):
        s = TS.ALLMAPS[name][0]()
        ex = R.reg_f64(s["allmap"], s["view"], s["proj"], ratio, 0.05, 1000.0)
        worst, _ = R.worst_ratios(*R.reg_f32_emulation(s["allmap"], s["view"], s["proj"], ratio, 0.05, 1000.0), ex, "hole")
        assert worst["grad"] > 0.02 and worst["dist"] > 0.02, worst


@pytest.mark.parametrize("mistake", R.MISTAKES)
def test_bounds_reject_each_planted_mistake(mistake):
    s = TS.golden()
    ex = R.reg_f64(s["allmap"], s["view"], s["proj"], 1.0, 0.05, 100.0)
    values, grad = R.reg_f32_emulation(s["allmap"], s["view"], s["proj"], 1.0, 0.05, 100.0, mistake)
    worst, _ = R.worst_ratios(values, grad, ex, "hole")
    assert max(worst.values()) > 10.0, (mistake, worst)


def test_c_abi_rejects_bad_arguments_without_a_device():
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    err = lambda: lib.surfel_last_error().decode()
    buf = (ctypes.c_double * 16)()
    p = ctypes.addressof(buf)
    for W, H in ((0, 4), (4, -1), (60000, 60000), (1, 600000)):
        assert lib.surfel_post_reg_partials_bytes(W, H) == 0
        assert lib.surfel_post_reg_forward(W, H, 0.0, 0.05, 100.0, p, p, p, p, p, p, None) != 0 and "bad size" in err()
        assert lib.surfel_post_reg_backward(W, H, 0.0, 0.05, 100.0, p, p, p, p, p, p, None) != 0 and "bad size" in err()
    assert lib.surfel_post_reg_partials_bytes(33, 9) == 2 * 8 * 2 * 2
    fwd = [p] * 6
    for k in range(6):
        args = fwd[:k] + [None] + fwd[k + 1:]
        assert lib.surfel_post_reg_forward(4, 4, 0.0, 0.05, 100.0, *args, None) != 0 and "NULL required" in err()
    for k in range(6):
        args = fwd[:k] + [None] + fwd[k + 1:]
        assert lib.surfel_post_reg_backward(4, 4, 0.0, 0.05, 100.0, *args, None) != 0 and "NULL required" in err()
