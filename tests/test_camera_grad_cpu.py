"""The camera-gradient restatement (tests/camera_exact.py) against float64 autograd of oracle/dense_torch.preprocess in
viewmatrix, projmatrix and campos, on every certified scene of tests/preprocess_scenes.py, at SH degrees 0-3, with
colors_precomp, with transMat_precomp (with and without SH) and at scale_modifier 1 and 1.7.  Runs anywhere: the
records are random, not rendered.  Also the pose-refinement loop of the GPU user-story test, rehearsed in float64 on
the dense renderer, and the rule that decides which autograd node the op uses."""
import numpy as np
import pytest
import torch

import camera_exact as CE
import camera_pose as CP
import preprocess_scenes as PS
from oracle import dense_torch as DT

F64 = torch.float64
REL = 1e-12
CASES = [("shs", D) for D in range(4)] + [("colors", 3), ("transmat", 3), ("transmat_sh", 3)]


def case_scene(name, path, mod):
    s = PS.get(name)
    scene, cam = s["scene"], s["cam"]
    if path == "shs":
        return PS.with_sh(scene, 16), cam
    if path == "colors":
        return PS.colors_precomp(scene), cam
    fwd = dense_forward(PS.with_sh(scene, 16), cam, 3, mod)
    out = PS.transmat_precomp(scene, fwd["transMat"].astype(np.float32), fwd["radii"])
    if path == "transmat_sh":
        del out["colors_precomp"]
        out["shs"] = np.ascontiguousarray(scene["shs"][:, :16])
    return out, cam


def dense_forward(scene, cam, D, mod):
    """The forward record PE.Reference needs (radii, T, screen centre, clamp bits), from dense_torch in float64."""
    t = lambda x: None if x is None else torch.tensor(np.asarray(x, np.float64))
    P = scene["means3D"].shape[0]
    pre = DT.preprocess(t(scene["means3D"]), t(scene.get("scales")), t(scene.get("rotations")), torch.zeros(P, 1, dtype=F64),
                        t(scene.get("shs")), t(cam["viewmatrix"]), t(cam["projmatrix"]), t(cam["campos"]), cam["W"], cam["H"],
                        D, mod, t(scene.get("transMat_precomp")), t(scene.get("colors_precomp")))
    return dict(radii=pre["radii"].numpy(), transMat=pre["T"].numpy(), xy=pre["xy"].numpy(),
                clamped=pre["clamped"].numpy().astype(np.uint8))


def random_record(P, seed):
    rec = np.random.default_rng(seed).normal(size=(P, 24))
    rec[:, 22:] = 0.0
    return rec


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-D{c[1]}")
@pytest.mark.parametrize("name", PS.SCENES)
def test_restatement_matches_dense_autograd(name, case):
    path, D = case
    for mod in (1.0, 1.7):
        scene, cam = case_scene(name, path, mod)
        fwd = dense_forward(scene, cam, D, mod)
        assert (fwd["radii"] > 0).any()
        ref = CE.CameraReference(scene, cam, fwd, D, mod)
        rec = random_record(ref.P, 7)
        gT = ref.evaluate(rec)["dL_dtransMat"]
        got = ref._assemble(*ref.terms(rec, gT))
        want = CE.autograd_camera(ref, rec, gT)
        for key in CE.KEYS:
            scale = np.abs(want[key]).max()
            err = np.abs(got[key] - want[key]).max()
            assert err <= REL * scale, f"{name} {case} scale_modifier={mod} {key}: {err:.3e} vs scale {scale:.3e}"
        vm, pr, cp = got["viewmatrix"].reshape(4, 4), got["projmatrix"].reshape(4, 4), got["campos"]
        assert (vm[3] == 0).all() and (vm[:, 3] == 0).all() and (pr[:, 2] == 0).all()
        if path.startswith("transmat"):
            assert (vm == 0).all() and (pr == 0).all(), "rule 4: T and the normal do not depend on the camera"
        else:
            assert np.abs(pr).max() > 0 and np.abs(vm).max() > 0
        if path in ("colors", "transmat") or D == 0:
            assert (cp == 0).all()
        else:
            assert np.abs(cp).max() > 0


def test_sh_direction_term_is_the_sh_part_of_dmeans3D():
    """Rule 3 through preprocess_exact: dL_dmeans3D on the colors_precomp path plus the SH term is dL_dmeans3D with SH."""
    scene, cam = case_scene("orient", "shs", 1.0)
    fwd = dense_forward(scene, cam, 3, 1.0)
    rec = random_record(scene["means3D"].shape[0], 3)
    with_sh = CE.CameraReference(scene, cam, fwd, 3)
    colors = CE.CameraReference(PS.colors_precomp(scene), cam, fwd, 3)
    dR = torch.where(with_sh.clamped, 0.0, torch.as_tensor(rec[:, 19:22]))
    dR[~with_sh.vis] = 0.0
    total = with_sh.evaluate(rec)["dL_dmeans3D"].numpy()
    geom = colors.evaluate(rec)["dL_dmeans3D"].numpy()
    sh = with_sh.sh_direction_term(dR).numpy()
    np.testing.assert_allclose(geom + sh, total, rtol=0, atol=1e-12 * np.abs(total).max())


def test_bound_covers_the_terms():
    """The bound is at least the magnitude of the sum it bounds, entry by entry, and zero exactly where the rules
    give a structural zero."""
    scene, cam = case_scene("layout1000", "shs", 1.7)
    fwd = dense_forward(scene, cam, 3, 1.7)
    ref = CE.CameraReference(scene, cam, fwd, 3, 1.7)
    rec = random_record(ref.P, 1)
    ev, bd = ref.camera(rec), ref.camera_bound(rec)
    for key in CE.KEYS:
        assert (bd[key] >= np.abs(ev[key]) * (1 - 1e-12)).all(), key
        assert ((bd[key] == 0) == (ev[key] == 0)).all(), key


def test_pose_refinement_rehearsal():
    """The GPU user-story loop (tests/camera_pose.py) on the dense float64 renderer at a smaller size: 200 Adam steps
    on a 6-dof pose increment bring both errors below 25 % of their initial value."""
    res = CP.refine(CP.dense_renderer(), P=CP.SMALL_P, W=CP.SMALL_W, H=CP.SMALL_H, steps=CP.STEPS)
    assert res["rot_err"][-1] < 0.25 * res["rot_err"][0], res
    assert res["trans_err"][-1] < 0.25 * res["trans_err"][0], res


def test_banded_dense_gradient_equals_the_full_frame():
    """The banded evaluation the GPU end-to-end test uses for its float64 reference (camera_exact.dense_camera_grad)
    gives the camera gradient of the whole frame rendered at once."""
    import surfel_scenes as S
    P, W, H = 120, 48, 40
    cam = S.to_numpy(S.make_camera(W, H, R=S.look_at_rotation(12, -7), t=[0.15, -0.1, 0.4]))
    scene = S.to_numpy(S.make_scene(P, W, H, 5, depth_complexity=20))
    m = np.concatenate([scene["means3D"], np.ones((P, 1), np.float32)], 1) @ np.linalg.inv(cam["viewmatrix"])
    scene["means3D"] = np.ascontiguousarray(m[:, :3], np.float32)
    bg = np.array([0.1, 0.2, 0.3], np.float32)
    gc, go = (x.double() for x in S.make_cotangents(W, H, 4))
    full = CE.dense_camera_grad(scene, cam, bg, gc, go, F64, band_rows=64)
    banded = CE.dense_camera_grad(scene, cam, bg, gc, go, F64, band_rows=16)
    for a, b in zip(full, banded):
        assert np.abs(a).max() > 0
        np.testing.assert_allclose(b, a, rtol=0, atol=1e-10 * np.abs(a).max())


def test_camera_node_is_chosen_only_when_the_camera_requires_grad():
    from diff_surfel_rasterization import GaussianRasterizationSettings, _wants_camera_grad
    cam = {k: torch.eye(4) for k in ("viewmatrix", "projmatrix")}
    base = GaussianRasterizationSettings(16, 16, 1.0, 1.0, torch.zeros(3), 1.0, cam["viewmatrix"], cam["projmatrix"], 0,
                                         torch.zeros(3), False, False)
    assert not _wants_camera_grad(base)
    for key in ("viewmatrix", "projmatrix", "campos"):
        rs = base._replace(**{key: getattr(base, key).clone().requires_grad_(True)})
        assert _wants_camera_grad(rs), key
        with torch.no_grad():
            assert not _wants_camera_grad(rs), key
