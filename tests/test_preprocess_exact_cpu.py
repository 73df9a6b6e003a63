"""The float64 preprocess-backward reference (tests/preprocess_exact.py) against finite differences, the C oracle
against that reference on every certified scene (tests/preprocess_scenes.py) and path, and the scenes' own
certificates.  Runs anywhere: the records are random, not rendered.

The oracle is fed the reference's record-level gradients (dL_dT before the fold, dL_dmean2D, the normal and colour
gradients), so the comparison covers exactly A.5: the fold, the dual-visible sign, the quaternion and scale vjp's,
the clamp mask, the SH backward at every degree and M, the densification proxy and the scale_modifier convention.
"""
import numpy as np
import pytest
import torch

import preprocess_exact as PE
import preprocess_scenes as PS
from oracle import dense_torch as DT

F64 = torch.float64
# oracle (float32) vs the float64 reference, |got - ref| <= TOL * (|J|.|rec| + ROW_FLOOR * the splat's largest
# bound), over every scene, path, SH case and scale_modifier below
ORACLE_TOL = dict(dL_dtransMat=2e-5, dL_dmeans2D=2e-5, dL_dmeans3D=2e-5, dL_drotations=2e-5, dL_dshs=2e-5,
                  # dL_dscale is a dot product of dRows = dL_dT Pm^T with a unit column of R: Pm's columns are of pixel
                  # scale (W / 2), so the float32 products cancel by more than |J| sees; worst observed 2.5e-5
                  dL_dscales=1e-4)
ROW_FLOOR = 1e-3
FD_TOL = 1e-6           # central differences in float64 (step 1e-5 relative), same bound
SH_CASES = ((0, 16), (1, 16), (2, 16), (3, 16), (0, 1), (1, 4), (2, 9), (3, 25))
FD_SPLATS = 20


def random_record(P, seed):
    rng = np.random.default_rng(seed)
    rec = rng.normal(size=(P, 24))
    rec[:, 22:] = 0.0
    return rec


def oracle_fwd(O, scene, cam, D, mod):
    return O.preprocess_fwd(scene["means3D"], scene.get("scales"), scene.get("rotations"), scene["opacities"],
                            scene.get("shs"), cam["viewmatrix"], cam["projmatrix"], cam["campos"], cam["W"], cam["H"],
                            D, mod, scene.get("transMat_precomp"), scene.get("colors_precomp"))


def case_scene(O, name, path, M, mod):
    s = PS.get(name)
    scene, cam = s["scene"], s["cam"]
    if path == "shs":
        return PS.with_sh(scene, M), cam
    if path == "colors":
        return PS.colors_precomp(scene), cam
    pre = oracle_fwd(O, PS.with_sh(scene, 16), cam, 3, mod)
    return PS.transmat_precomp(scene, pre["transMat"], pre["radii"]), cam


def bounded_ratio(got, ref, bound, key):
    g, r, b = np.asarray(got, np.float64).reshape(ref.shape), ref, bound
    if key == "dL_dmeans2D":
        g, r, b = g[:, :2], r[:, :2], b[:, :2]
    return g, r, b


def splat_scale(bound, keys):
    return np.max([bound[k].reshape(bound[k].shape[0], -1).max(1) for k in keys], 0)


def check_against(got, ev, bd, keys, tol, label):
    scale = splat_scale(bd, keys)
    worst = {}
    for key in keys:
        g, r, b = bounded_ratio(got[key], ev[key], bd[key], key)
        b = b + ROW_FLOOR * scale.reshape((-1,) + (1,) * (b.ndim - 1))
        err = np.abs(g - r)
        assert np.isfinite(g).all(), f"{label} {key}: non-finite"
        assert not (err[b == 0] > 0).any(), f"{label} {key}: non-zero error where the bound is 0"
        pos = b > 0
        worst[key] = float((err[pos] / b[pos]).max()) if pos.any() else 0.0
    bad = {k: v for k, v in worst.items() if v > (tol[k] if isinstance(tol, dict) else tol)}
    assert not bad, f"{label}: worst error / bound above {tol}: {bad}"
    return worst


# ---------------------------------------------------------------------------------------------- scenes
@pytest.mark.parametrize("name", PS.SCENES)
def test_scene_is_certified_and_has_its_feature(name):
    s = PS.get(name)
    scene, cam, f = s["scene"], s["cam"], s["features"]
    assert PS.sign_margin(scene, cam).min() >= PS.SIGN_MARGIN
    assert cam["W"] != cam["H"] and np.abs(np.asarray(cam["viewmatrix"])[3, :3]).max() > 0
    assert not np.allclose(np.asarray(cam["viewmatrix"])[:3, :3], np.eye(3))
    P = scene["means3D"].shape[0]
    if name == "orient":
        assert f["front"] == f["back"] == P // 2 and f["max_aniso"] > 250
    elif name == "grazing":
        assert f["min_angle_deg"] >= 2.0 - 0.1 and f["max_angle_deg"] <= 10.0 + 0.1 and min(f["front"], f["back"]) > P // 4
    elif name == "unnormalised":
        assert f["min_qnorm"] < 2e-2 and f["max_qnorm"] > 50
    elif name == "clamp":
        assert f["splats_per_pattern"] >= 8
        for D in range(4):
            pat, raw = PS.clamp_patterns(scene, cam, D)
            assert np.abs(raw).min() >= PS.RGB_MARGIN and np.bincount(pat, minlength=8).min() >= 8
    elif name == "low_pass":
        assert f["sub_pixel"] >= 200
    elif name == "near":
        assert f["near_crossing"] >= 10
    elif name == "distance":
        assert f["min_dist"] < 0.26 and f["max_dist"] > 89
    else:
        assert f["behind"] == P // 3 and (PS.view_geometry(scene, cam)[0][:, 2] <= 0.2).sum() == P // 3


# ---------------------------------------------------------------------------------------------- finite differences
def _record_scalar(T, c, rec, xy):
    """Per splat: the scalar the record defines, written in upstream's pixel form k = px Tw - Tu, l = py Tw - Tv at
    the fixed screen centre c (p = Pc + dx P1 + dy P2), plus the low-pass centre term."""
    Tu, Tv, Tw = T[:, 0:3], T[:, 3:6], T[:, 6:9]
    k, l = c[:, 0:1] * Tw - Tu, c[:, 1:2] * Tw - Tv
    Pc, P1, P2 = torch.cross(k, l, dim=1), torch.cross(Tw, l, dim=1), torch.cross(k, Tw, dim=1)
    det = torch.linalg.det(T.reshape(-1, 3, 3))
    return ((rec[:, 0:3] * Pc).sum(1) + (rec[:, 3:6] * P1).sum(1) + (rec[:, 6:9] * P2).sum(1) + rec[:, 9] * det
            + (rec[:, 10:13] * Tw).sum(1) + (rec[:, 13:15] * xy).sum(1))


@pytest.mark.parametrize("path", ("shs", "transmat"))
@pytest.mark.parametrize("name", PS.SCENES[:7] + ("layout129",))
def test_reference_matches_finite_differences(oracle, name, path):
    """The reference's every output against central differences of the per-splat scalar the record defines, with the
    whole chain linearised at T(inputs) (so the forward record is the float64 forward of the same inputs)."""
    D, M = (2, 9) if name == "clamp" else (3, 16)
    mod = 1.7
    scene, cam = case_scene(oracle, name, path, M, mod)
    pre32 = oracle_fwd(oracle, scene, cam, D, mod)
    idx = np.nonzero(pre32["radii"] > 0)[0][:FD_SPLATS]
    sub = {k: np.ascontiguousarray(v[idx]) for k, v in scene.items()}
    n = idx.size
    t = lambda x: None if x is None else torch.tensor(np.asarray(x, np.float64))
    vm, pm, campos = t(cam["viewmatrix"]), t(cam["projmatrix"]), t(cam["campos"])
    W, H = cam["W"], cam["H"]
    geom = path != "transmat"
    q0 = t(sub.get("rotations"))
    leaves = dict(means=t(sub["means3D"]))
    if geom:
        leaves.update(scales=t(sub["scales"]), q=q0 / q0.norm(dim=1, keepdim=True))
    else:
        leaves["T"] = t(sub["transMat_precomp"])
    if "shs" in sub:
        leaves["shs"] = t(sub["shs"])
    opa = torch.zeros(n, 1, dtype=F64)

    def forward(lv):
        pre = DT.preprocess(lv["means"], lv.get("scales"), lv.get("q"), opa, None, vm, pm, campos, W, H, D, mod,
                            lv.get("T"), torch.zeros(n, 3, dtype=F64), normalize_quat=False)
        if "shs" in lv:
            d = lv["means"] - campos[None]
            pre["raw"] = DT.eval_sh(D, lv["shs"], d / d.norm(dim=1, keepdim=True)) + 0.5
        return pre

    base = forward(leaves)
    rec = t(random_record(n, 11))
    clamped = (base["raw"] < 0) if "raw" in base else torch.zeros(n, 3, dtype=torch.bool)
    c0 = base["xy"].clone()
    fwd = dict(radii=np.ones(n, np.int32), transMat=base["T"].numpy(), xy=c0.numpy(), clamped=clamped.numpy())
    ev, bd = PE.preprocess_bwd_exact(sub, cam, fwd, rec.numpy(), D, mod, quirk=False)

    def scalar(lv):
        pre = forward(lv)
        s = _record_scalar(pre["T"], c0, rec, pre["xy"]) + (rec[:, 16:19] * pre["normal"]).sum(1)
        if "raw" in pre:
            s = s + (torch.where(clamped, 0.0, rec[:, 19:22]) * pre["raw"]).sum(1)
        return s

    def fd(fn, lv, key):
        x = lv[key]
        g = torch.zeros_like(x)
        flat = x.reshape(n, -1)
        for j in range(flat.shape[1]):
            h = 1e-5 * torch.clamp_min(flat[:, j].abs(), 0.1)
            for sgn in (1.0, -1.0):
                y = flat.clone()
                y[:, j] = y[:, j] + sgn * h
                lv2 = dict(lv)
                lv2[key] = y.reshape(x.shape)
                g.reshape(n, -1)[:, j] += sgn * fn(lv2) / (2 * h)
        return g.numpy()

    got = {"dL_dmeans3D": fd(scalar, leaves, "means")}
    if geom:
        got["dL_dscales"] = fd(scalar, leaves, "scales")
        got["dL_drotations"] = fd(scalar, leaves, "q")
    if "shs" in leaves:
        got["dL_dshs"] = fd(scalar, leaves, "shs")
    # dL_dT itself, folded and raw, by differences in T at the stored point
    Tl = dict(T=base["T"].clone())
    got["dL_dtransMat"] = fd(lambda lv: _record_scalar(lv["T"], c0, rec, PE.aabb_centre(lv["T"], leaves["means"], dict(
        vm=vm, pm=pm, campos=campos, W=W, H=H))), Tl, "T")
    rec_nofold = rec.clone()
    rec_nofold[:, 13:15] = 0.0
    raw = fd(lambda lv: _record_scalar(lv["T"], c0, rec_nofold, torch.zeros(n, 2, dtype=F64)), Tl, "T")
    src = raw if geom else got["dL_dtransMat"]
    got["dL_dmeans2D"] = np.concatenate([DT.densification_proxy(base["T"], torch.tensor(src), W, H).numpy(),
                                         np.zeros((n, 1))], 1)
    keys = tuple(got)
    check_against(got, ev, bd, keys, FD_TOL, f"{name} {path}")
    check_against(dict(dL_dtransMat=raw), dict(dL_dtransMat=ev["dL_dtransMat_raw"]),
                  dict(dL_dtransMat=bd["dL_dtransMat_raw"]), ("dL_dtransMat",), FD_TOL, f"{name} {path} raw dL_dT")


# ---------------------------------------------------------------------------------------------- oracle vs reference
def run_oracle_bwd(O, scene, cam, pre, ev, rec, D, mod):
    rb = dict(dL_dtransMat=ev["dL_dtransMat_raw"], dL_dmean2D=rec[:, 13:15], dL_dopacity=rec[:, 15],
              dL_dnormal=rec[:, 16:19], dL_dcolors=rec[:, 19:22])
    return O.preprocess_bwd(scene["means3D"], scene.get("scales"), scene.get("rotations"), scene.get("shs"), pre, rb,
                            cam["viewmatrix"], cam["projmatrix"], cam["campos"], cam["W"], cam["H"], D, mod,
                            scene.get("transMat_precomp"), scene.get("colors_precomp"))


ORACLE_CASES = [("shs", D, M) for D, M in SH_CASES] + [("colors", 3, 0), ("transmat", 3, 0)]


@pytest.mark.parametrize("case", ORACLE_CASES, ids=lambda c: f"{c[0]}-D{c[1]}-M{c[2]}")
@pytest.mark.parametrize("name", PS.SCENES)
def test_oracle_matches_reference(oracle, name, case):
    path, D, M = case
    P = PS.get(name)["scene"]["means3D"].shape[0]
    if P > 1000 and case not in (("shs", 3, 16), ("shs", 2, 9), ("transmat", 3, 0)):
        pytest.skip("the largest layouts run the staged, one unstaged and the transMat_precomp case")
    for mod in (1.0, 1.7):
        scene, cam = case_scene(oracle, name, path, M, mod)
        pre = oracle_fwd(oracle, scene, cam, D, mod)
        rec = random_record(P, 5)
        rec[pre["radii"] == 0] = 0.0           # render backward leaves the records of culled splats at zero
        ev, bd = PE.preprocess_bwd_exact(scene, cam, pre, rec, D, mod)
        got = run_oracle_bwd(oracle, scene, cam, pre, ev, rec, D, mod)
        keys = [k for k in PE.BOUNDED_KEYS if k in ev and not (k == "dL_dshs" and path != "shs")]
        if path == "shs":
            assert (got["dL_dshs"][:, (D + 1) ** 2:] == 0).all()
        check_against(got, ev, bd, keys, ORACLE_TOL, f"{name} {case} scale_modifier={mod}")


# ---------------------------------------------------------------------------------------------- scale_modifier
@pytest.mark.parametrize("name", ("orient", "grazing"))
def test_scale_modifier_convention_is_pinned(oracle, name):
    """At scale_modifier = 1.7 upstream's convention (scale_modifier_quirk: dL_dscale and the L0/L1 part of dL_dR
    without the modifier) and the exact derivative differ by more than 1e-2 of the gradient's scale on these scenes,
    and the oracle follows the convention."""
    D, M, mod = 3, 16, 1.7
    scene, cam = case_scene(oracle, name, "shs", M, mod)
    pre = oracle_fwd(oracle, scene, cam, D, mod)
    rec = random_record(scene["means3D"].shape[0], 3)
    rec[pre["radii"] == 0] = 0.0
    ref = PE.Reference(scene, cam, pre, D, mod)
    ev = {k: v.numpy() for k, v in ref.evaluate(rec).items()}
    for key in ("dL_dscales", "dL_drotations"):
        ex, qk = ev["exact_" + key], ev["quirk_" + key]
        assert np.abs(qk - ex).max() > 1e-2 * np.abs(ex).max(), key
    got = run_oracle_bwd(oracle, scene, cam, pre, ev, rec, D, mod)
    for key in ("dL_dscales", "dL_drotations"):
        scale = np.abs(ev["quirk_" + key]).max()
        assert np.abs(got[key] - ev["quirk_" + key]).max() < 1e-4 * scale, key
        assert np.abs(got[key] - ev["exact_" + key]).max() > 1e-2 * scale, key
    # at scale_modifier = 1 the convention is the exact derivative
    ref1 = PE.Reference(scene, cam, oracle_fwd(oracle, scene, cam, D, 1.0), D, 1.0)
    ev1 = ref1.evaluate(rec)
    for key in ("dL_dscales", "dL_drotations"):
        assert torch.equal(ev1["exact_" + key], ev1["quirk_" + key]), key
