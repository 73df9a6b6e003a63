"""CPU side of the hit-loop suite (tests/hitloop_scenes.py, tests/test_hitloop_gpu.py):

  * every generator's scene is certified (no evaluated pair within DELTA of a discontinuity) and has the structure it
    claims (the generators assert it; running them here keeps that checked without a GPU);
  * the yardstick itself: on the smallest certified scenes the float64 oracle (oracle_render_fwd_f64 /
    oracle_render_bwd_f64, including its abs-sum output) agrees with dense_torch's float64 autograd, at the new
    edges (lists of 256 and more, near-plane pairs, low-pass pairs, medians at group boundaries).
"""
import numpy as np
import pytest
import torch

import hitloop_scenes as HS
import test_hitloop_gpu as G


@pytest.mark.parametrize("name", G.SCENES)
def test_scene_is_certified_and_structured(oracle, name):
    s = G.scene(oracle, name)          # the generator asserts its structure
    HS.assert_certified(s)
    assert s["worst"] >= HS.DELTA


def test_certificate_sees_a_pair_on_a_threshold(oracle):
    """The certificate is not vacuous: a splat whose alpha is exactly 1/255 at the pixel under its centre, and one
    whose centre sits exactly on a pixel (rho3d = rho2d = 0 there), are reported with zero margin."""
    layer = HS.Layer(16, 16, seed=1)
    layer.add(7.0, 7.0, 3.0, 400.0, 400.0, 0.5)
    layer.add(3.3, 3.4, 4.0, 400.0, 400.0, 1.0 / 255.0)
    scene, _ = layer.scene()
    pre, binned = HS.run_oracle(oracle, scene, layer.cam)
    m, per_splat = oracle.decision_margins(pre, binned, 16, 16)
    assert m["rho_branch"][7, 7] == 0.0
    assert m["alpha_min"].min() < 1e-6
    assert (per_splat < HS.DELTA).all()


def _dense_pre(oracle, s):
    """dense_torch's `pre` from the oracle's float32 preprocess output, as float64 leaves."""
    pre, W, H = s["pre"], s["cam"]["W"], s["cam"]["H"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    r0, r1 = (0, gy) if s["rows"] is None else s["rows"]
    r = pre["radii"].astype(np.float32)
    c = pre["xy"]
    trunc = lambda v: np.trunc(v / np.float32(16)).astype(np.int64)
    rect = np.stack([np.clip(trunc(c[:, 0] - r), 0, gx), np.clip(np.clip(trunc(c[:, 1] - r), 0, gy), r0, r1),
                     np.clip(trunc((c[:, 0] + r) + np.float32(15)), 0, gx),
                     np.clip(np.clip(trunc((c[:, 1] + r) + np.float32(15)), 0, gy), r0, r1)], 1)
    leaf = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    return dict(T=leaf(pre["transMat"]), xy=leaf(pre["xy"]), depth=torch.tensor(pre["depths"], dtype=torch.float64),
                normal=leaf(pre["normal_opacity"][:, :3]), rgb=leaf(pre["rgb"]), opacity=leaf(pre["normal_opacity"][:, 3]),
                rect=torch.tensor(rect), visible=torch.tensor(pre["radii"] > 0))


@pytest.mark.parametrize("name", ["count1", "count33", "count257", "all_saturate", "median_boundaries", "near_plane",
                                  "low_pass"])
def test_float64_oracle_matches_dense_autograd(oracle, name):
    from oracle import dense_torch as DT
    s = G.scene(oracle, name)
    W, H = s["cam"]["W"], s["cam"]["H"]
    img = s["img"]
    for group in ("all", "median"):
        dp = _dense_pre(oracle, s)
        color, others, n_contrib, final_T = DT.rasterize(dp, torch.tensor(HS.BG, dtype=torch.float64), W, H,
                                                        pixel_chunk=256, upstream_lowpass_depth=True)
        if group == "all":
            np.testing.assert_array_equal(n_contrib.numpy(), img["n_contrib"][0])
            np.testing.assert_allclose(color.detach().numpy(), img["color"], rtol=1e-6, atol=1e-6)
            np.testing.assert_allclose(others.detach().numpy(), img["others"], rtol=1e-6, atol=1e-6)
            np.testing.assert_allclose(final_T.numpy(), img["accum"][0], rtol=1e-6, atol=1e-9)
        gc, go = HS.cotangent(W, H, group, seed=3)
        ((color * torch.tensor(gc, dtype=torch.float64)).sum()
         + (others * torch.tensor(go, dtype=torch.float64)).sum()).backward()
        rb = oracle.render_bwd(s["pre"], s["binned"], img, HS.BG, gc, go, W, H, f64=True)
        for key, t in (("dL_dtransMat", dp["T"]), ("dL_dmean2D", dp["xy"]), ("dL_dopacity", dp["opacity"]),
                       ("dL_dnormal", dp["normal"]), ("dL_dcolors", dp["rgb"])):
            ref, absum = rb[key], rb["abs"][key]
            assert (absum >= np.abs(ref) * (1 - 1e-12)).all(), f"{key}: abs-sum below |sum|"
            g = t.grad.numpy() if t.grad is not None else np.zeros_like(ref)
            err = np.abs(g.reshape(ref.shape) - ref)
            # the float32 round trip of the forward state (accum) is the only difference between the two
            assert (err <= 1e-5 * absum + 1e-12).all(), \
                f"{name} [{group}] {key}: worst {float((err / (absum + 1e-30)).max()):.3e} of the abs-sum"
