"""DTU mask culling without a device (DESIGN.md §7n): the restatement tests/cull_ref.py against what the reference's
own cull_scan recorded (tests/golden/ref_cull.npz): the dilated masks bit for bit, every decision and output bit for
bit in the exact (dyadic and structural) cases, and elsewhere every differing decision within rule 3's bound; the
projections against the recorded ones and against cv2; and the C ABI's argument checks."""
import ctypes
import os

import numpy as np
import pytest

import cull_ref as CR

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_cull.npz")
IMAGE = (1600, 1200)


def golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("ref_cull.npz not generated")
    return np.load(GOLDEN)


def case_names(g):
    return sorted({k.split(".")[0] for k in g.files})


def case(g, n):
    return {k.split(".", 1)[1]: g[k] for k in g.files if k.split(".")[0] == n}


def ref_dilated(c):
    N, H, W = c["masks"].shape
    return np.unpackbits(c["dilated_bits"], axis=-1, count=W).astype(bool)


def ref_keep(c):
    """The reference's decision from its recorded grids and samples: (sample + (1 - valid) > 0).all over views."""
    g = c["grid"]
    valid = ((g > -1) & (g < 1)).all(-1)
    return ((c["sample"] + (1.0 - valid)) > 0).all(0)


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b)


def same64(a, b):
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


NAMES = case_names(np.load(GOLDEN)) if os.path.exists(GOLDEN) else []


@pytest.mark.parametrize("name", NAMES)
def test_restatement_matches_reference(name):
    c = case(golden(), name)
    A = c["A"][:, :3]
    r = CR.cull(c["verts"], c["faces"], c["masks"], A, c["scale_mats"], c.get("colors"), IMAGE, int(c["radius"]))
    assert np.array_equal(r["dilated"], ref_dilated(c)), "dilated masks"
    keep = ref_keep(c)
    if str(c["kind"]) == "exact":
        gx, gy = CR.project(c["verts"], A, IMAGE)
        assert same(np.stack([gx, gy], -1), c["grid"]), "grids"
        assert np.array_equal(r["keep"], keep), "decisions"
        assert same64(r["verts"], c["out_verts"]) and same(r["faces"], c["out_faces"])
        if "colors" in c:
            assert same(r["colors"], c["out_colors"])
        return
    differ = np.flatnonzero(r["keep"] != keep)
    tie = CR.near_tie(c["verts"][differ], A, IMAGE, c["masks"].shape[1:])
    assert tie.any(0).all(), f"{int((~tie.any(0)).sum())} of {len(differ)} differing decisions are not near a tie"
    print(f"{name}: {len(differ)} of {len(keep)} decisions differ, all within rule 3's bound")
    if len(differ) == 0:
        assert same64(r["verts"], c["out_verts"]) and same(r["faces"], c["out_faces"])
        if "colors" in c:
            assert same(r["colors"], c["out_colors"])


def test_golden_covers_the_cases():
    g = golden()
    names = case_names(g)
    kinds = {n: str(g[f"{n}.kind"]) for n in names}
    assert sum(k == "exact" for k in kinds.values()) >= 8 and sum(k == "bound" for k in kinds.values()) == 2
    c = case(g, "dyadic")
    grid = c["grid"]
    Wm = c["masks"].shape[2]
    f = (grid[..., 0].astype(np.float64) + 1) / 2 * (Wm - 1)
    assert (f - np.floor(f) == 0.5).sum() > 50, "half-pixel ties"
    assert (np.abs(grid) == 1).sum() > 50, "grid at exactly +-1"
    assert (c["out_verts"].shape[0] < c["verts"].shape[0]) and (c["out_faces"].shape[0] < c["faces"].shape[0])
    assert case(g, "none_kept")["out_verts"].shape[0] == 0
    assert case(g, "all_kept")["out_verts"].shape[0] == 600
    assert int(case(g, "r0")["radius"]) == 0 and int(case(g, "dtu_size")["radius"]) == 24
    assert case(g, "dtu_size")["masks"].shape[1:] == (1200, 1600)
    assert case(g, "mismatch")["masks"].shape[1:] != (1200, 1600)
    # the dyadic cases put vertices behind the camera
    assert (c["verts"][:, 2] + 64 < 0).any()


@pytest.mark.parametrize("name", NAMES)
def test_projections_match_reference(name):
    c = case(golden(), name)
    A = CR.projections(c["world_mats"], c["scale_mats"]).astype(np.float64)
    R = c["A"][:, :3].astype(np.float64)
    assert (np.abs(A - R) <= 1e-6 * np.abs(R) + 1e-30).all()
    if str(c["kind"]) == "exact":
        assert np.array_equal(A, R)


def test_projections_match_cv2():
    cv2 = pytest.importorskip("cv2")
    import torch
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(7)
    worst, loose = 0.0, 0
    for i in range(400):
        K = np.array([[rng.uniform(500, 4000), rng.uniform(-2, 2), rng.uniform(200, 1400)],
                      [0, rng.uniform(500, 4000), rng.uniform(200, 1000)], [0, 0, 1.0]])
        R = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix()
        c = rng.normal(size=3)
        c *= rng.uniform(1, 5) / np.linalg.norm(c)          # DTU's normalised cameras sit 2-3 units out
        Wm = np.eye(4)
        Wm[:3, :4] = (1 if i % 2 else -1) * rng.uniform(0.01, 100) * K @ np.hstack([R, -R @ c[:, None]])
        S = np.eye(4)
        S[:3, :3] *= rng.uniform(0.1, 500)
        S[:3, 3] = rng.normal(size=3) * 100
        P = (Wm.astype(np.float32) @ S.astype(np.float32))[:3, :4]
        Kd, Rd, t = cv2.decomposeProjectionMatrix(P)[:3]
        intr = np.eye(4)
        intr[:3, :3] = Kd / Kd[2, 2]
        pose = np.eye(4, dtype=np.float32)
        pose[:3, :3] = Rd.transpose()
        pose[:3, 3] = (t[:3] / t[3])[:, 0]
        ref = (torch.from_numpy(intr).float() @ torch.inverse(torch.from_numpy(pose))).numpy()[:3].astype(np.float64)
        mine = CR.projections(Wm[None], S[None])[0].astype(np.float64)
        # the reference's A carries the float32 rounding of pose and of its inverse, so an entry formed by
        # cancellation (the fourth column) is only good to its row's scale: the bar is 1e-6 of the row's largest entry
        row = np.abs(ref).max(1, keepdims=True)
        rel = np.abs(mine - ref) / row
        worst = max(worst, float(rel.max()))
        loose += int((np.abs(mine - ref) > 1e-6 * np.abs(ref)).sum())
        assert (rel <= 1e-6).all(), (i, rel.max())
    print(f"400 cameras: worst difference {worst:.2e} of the row's largest entry; {loose} of 4800 entries differ by "
          f"more than 1e-6 of themselves")


def test_dilation_matches_scipy():
    import scipy.ndimage as ndi
    rng = np.random.default_rng(3)
    for r, shape, p in ((0, (17, 40), 0.1), (1, (5, 3), 0.3), (3, (31, 70), 0.02), (7, (64, 33), 0.005),
                        (24, (120, 200), 0.0005)):
        m = rng.random(shape) < p
        m[0, -1] = True
        assert np.array_equal(CR.dilate(m, r), ndi.binary_dilation(m, structure=CR.disk(r), border_value=0)), r


def test_package_projections_match_restatement():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                    "2d-gaussian-splatting_b200"))
    from diff_surfel_rasterization import chamfer
    g = golden()
    for n in case_names(g):
        c = case(g, n)
        assert same(chamfer.dtu_projections(c["world_mats"], c["scale_mats"]),
                    CR.projections(c["world_mats"], c["scale_mats"]))
    with pytest.raises(ValueError):
        chamfer.dtu_projections(np.zeros((2, 4, 4)), np.zeros((2, 4, 4)))
    with pytest.raises(ValueError):
        chamfer.dtu_projections(np.eye(4)[None], np.eye(4)[None].repeat(2, 0))


def _lib():
    from diff_surfel_rasterization import _cabi
    try:
        return _cabi.load()
    except ImportError as ex:
        pytest.skip(f"library not built: {ex}")


def test_c_abi_rejects_bad_arguments():
    lib = _lib()
    lib.surfel_last_error()
    p = ctypes.c_void_p(16)
    assert lib.surfel_cull_max_views() >= 64 and lib.surfel_cull_max_radius() >= 24
    assert lib.surfel_cull_workspace_bytes(0, 10, 10, 5, 5) == 0
    assert lib.surfel_cull_workspace_bytes(3, 0, 10, 5, 5) == 0
    assert lib.surfel_cull_workspace_bytes(3, 10, 10, -1, 5) == 0
    assert lib.surfel_cull_workspace_bytes(3, 10, 10, 1 << 31, 5) == 0
    ws = lib.surfel_cull_workspace_bytes(3, 10, 10, 5, 5)
    assert ws > 300
    assert lib.surfel_cull_dilate(3, 10, 10, -1, p, p, ws, p, None) != 0
    assert b"radius" in lib.surfel_last_error()
    assert lib.surfel_cull_dilate(3, 10, 10, 255, p, p, ws, p, None) != 0
    assert lib.surfel_cull_dilate(0, 10, 10, 2, p, p, ws, p, None) != 0
    assert b"views" in lib.surfel_last_error()
    assert lib.surfel_cull_dilate(3, 10, 10, 2, None, p, ws, p, None) != 0
    assert b"NULL" in lib.surfel_last_error()
    assert lib.surfel_cull_dilate(3, 10, 10, 2, p, p, 1, p, None) != 0
    assert b"workspace" in lib.surfel_last_error()
    assert lib.surfel_cull_vertices(5, p, 5, p, 3, p, 1600, 1200, 10, 10, p, p, ws, p, None, None) != 0
    assert b"NULL" in lib.surfel_last_error()
    assert lib.surfel_cull_vertices(5, p, 5, p, 3, p, 0, 1200, 10, 10, p, p, ws, p, p, None) != 0
    assert b"image size" in lib.surfel_last_error()
    assert lib.surfel_cull_vertices(-5, p, 5, p, 3, p, 1600, 1200, 10, 10, p, p, ws, p, p, None) != 0
    assert lib.surfel_cull_vertices(5, p, 5, p, 3, p, 1600, 1200, 10, 10, p, None, ws, p, p, None) != 0
    assert b"workspace" in lib.surfel_last_error()
    world = (ctypes.c_double * 4)()
    assert lib.surfel_cull_emit(5, p, 5, p, world, None, 3, p, ws, 2, 1, p, p, p, None) != 0
    assert b"colour" in lib.surfel_last_error()
    assert lib.surfel_cull_emit(5, p, 5, p, None, None, 0, p, ws, 2, 1, p, p, None, None) != 0
    assert lib.surfel_cull_emit(5, p, -1, p, world, None, 0, p, ws, 0, 0, p, p, None, None) != 0
    assert lib.surfel_cull_emit(5, p, 5, p, world, None, 0, p, 1, 2, 1, p, p, None, None) != 0
    assert b"workspace" in lib.surfel_last_error()
    assert lib.surfel_cull_emit(5, p, 5, p, world, None, 0, p, ws, 6, 1, p, p, None, None) != 0
    assert b"kept" in lib.surfel_last_error()
