"""Camera gradients of the tile-band frame (DESIGN.md §7r) without a GPU.

  1. linearity: on the CPU oracle's band records (forward and render backward with row0 / row1), the camera
     restatement of tests/camera_exact.py summed over the bands of a partition equals its value on the whole frame's
     records, to 1e-12 of the chained magnitude (the same sums taken over |terms|).  Partitions: tile_row_band and
     equal_band at N = 1..4, one band per tile row, and a partition with a band no splat reaches; SH degrees 0-3,
     colors_precomp, transMat_precomp with and without SH;
  2. the reduction (surfel_parallel.reduce_camera_sums) in a gloo world of 2: a float64 sum and one cast, partials
     that add up under grad_reduce="none", and the same bits on both ranks.
"""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import camera_exact as CE
import surfel_parallel as SP
import surfel_scenes as S

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
F64 = torch.float64
REL = 1e-12
CASES = [("shs", D) for D in range(4)] + [("colors", 3), ("transmat", 3), ("transmat_sh", 3)]
BG = np.array([0.1, 0.2, 0.3], np.float32)
W, H, P = 96, 120, 400           # 8 tile rows


def base_scene():
    cam = S.to_numpy(S.make_camera(W, H, R=S.look_at_rotation(15, -8), t=[0.2, -0.1, 0.3]))
    scene = S.to_numpy(S.make_scene(P, W, H, 17, depth_complexity=20))
    m = np.concatenate([scene["means3D"], np.ones((P, 1), np.float32)], 1) @ np.linalg.inv(cam["viewmatrix"])
    scene["means3D"] = np.ascontiguousarray(m[:, :3], np.float32)
    return scene, cam


def case_scene(O, scene, cam, path):
    if path == "shs":
        return scene
    if path == "colors":
        out = {k: v for k, v in scene.items() if k != "shs"}
        out["colors_precomp"] = np.random.default_rng(2).uniform(0, 1, (P, 3)).astype(np.float32)
        return out
    pre = O.preprocess_fwd(scene["means3D"], scene["scales"], scene["rotations"], scene["opacities"], scene["shs"],
                           cam["viewmatrix"], cam["projmatrix"], cam["campos"], W, H, 3, 1.0)
    out = {k: scene[k] for k in ("means3D", "opacities")}
    out["transMat_precomp"] = pre["transMat"]
    if path == "transmat_sh":
        out["shs"] = scene["shs"]
    else:
        out["colors_precomp"] = np.random.default_rng(3).uniform(0, 1, (P, 3)).astype(np.float32)
    return out


def band_camera(O, scene, cam, D, band, gc, go):
    """(exact camera gradient, chained magnitude) of one band, both dicts of float64 arrays, from the oracle's band
    records: the render backward in float64 gives the band's partial dL_dT, dL_dmean2D, dL_dnormal and dL_dcolor."""
    pre, binned, img = O.forward(scene, cam, BG, D, 1.0, band[0], band[1])
    rb = O.render_bwd(pre, binned, img, BG, gc, go, W, H, f64=True)
    fwd = dict(radii=pre["radii"], transMat=pre["transMat"], xy=pre["xy"], clamped=pre["clamped"])
    ref = CE.CameraReference(scene, cam, fwd, D)
    rec = np.zeros((ref.P, 24))
    rec[:, 13:15] = rb["dL_dmean2D"]
    rec[:, 15] = rb["dL_dopacity"]
    rec[:, 16:19] = rb["dL_dnormal"]
    rec[:, 19:22] = rb["dL_dcolors"]
    # dL_dT: the raw render-backward gradient plus the AABB-centre fold of dL_dmean2D (the record's 13:15)
    gT = ref.evaluate(rec)["dL_dtransMat"] + torch.as_tensor(rb["dL_dtransMat"], dtype=F64) * ref.vis[:, None]
    G, V, C = ref.terms(rec, gT)
    return ref._assemble(G, V, C), ref._assemble(G.abs(), V.abs(), C.abs()), int((pre["radii"] > 0).sum())


def partitions():
    gy = SP.tile_rows(H)
    out = [(f"{f.__name__}/{n}", [f(H, r, n) for r in range(n)]) for f in (SP.tile_row_band, SP.equal_band)
           for n in (1, 2, 3, 4)]
    out.append(("rows", [(r, r + 1) for r in range(gy)]))
    return out


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-D{c[1]}")
def test_band_sums_add_up_to_the_whole_frame(oracle, case):
    path, D = case
    scene, cam = base_scene()
    scene = case_scene(oracle, scene, cam, path)
    gc, go = (x.numpy() for x in S.make_cotangents(W, H, 5))
    whole, mag, nvis = band_camera(oracle, scene, cam, D, (0, SP.tile_rows(H)), gc, go)
    assert nvis > 0
    cache = {}
    for label, bands in partitions():
        total = {k: np.zeros_like(v) for k, v in whole.items()}
        for band in bands:
            if band not in cache:
                cache[band] = band_camera(oracle, scene, cam, D, band, gc, go)[0]
            for k in CE.KEYS:
                total[k] = total[k] + cache[band][k]
        for k in CE.KEYS:
            err = np.abs(total[k] - whole[k]).max()
            assert err <= REL * mag[k].max(), f"{path}-D{D} {label} {k}: {err:.3e} vs {mag[k].max():.3e}"
    if path.startswith("transmat"):
        assert all(np.abs(whole[k]).max() == 0 for k in ("viewmatrix", "projmatrix"))
    else:
        assert np.abs(whole["projmatrix"]).max() > 0 and np.abs(whole["viewmatrix"]).max() > 0


def test_band_without_a_visible_splat_adds_nothing(oracle):
    """Splats kept to the upper half of the frame: the lower bands see none of them, give exactly zero, and the
    partition still adds up to the whole frame."""
    scene, cam = base_scene()
    pre = oracle.preprocess_fwd(scene["means3D"], scene["scales"], scene["rotations"], scene["opacities"], scene["shs"],
                                cam["viewmatrix"], cam["projmatrix"], cam["campos"], W, H, 3, 1.0)
    keep = (pre["radii"] > 0) & (pre["xy"][:, 1] + pre["radii"] < 48)
    assert keep.sum() > 10
    scene = {k: np.ascontiguousarray(v[keep]) for k, v in scene.items()}
    gc, go = (x.numpy() for x in S.make_cotangents(W, H, 6))
    whole, mag, _ = band_camera(oracle, scene, cam, 3, (0, SP.tile_rows(H)), gc, go)
    bands = [SP.equal_band(H, r, 2) for r in range(2)]
    parts = [band_camera(oracle, scene, cam, 3, b, gc, go) for b in bands]
    assert parts[1][2] == 0, "the lower band should see no splat"
    for k in CE.KEYS:
        assert (parts[1][0][k] == 0).all(), k
        err = np.abs(parts[0][0][k] + parts[1][0][k] - whole[k]).max()
        assert err <= REL * mag[k].max(), k


# ---------------------------------------------------------------------------------------------- 2. the reduction
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _sums(rank):
    """Restated band sums: values whose float64 total differs from the float32 total of the rounded parts."""
    rng = np.random.default_rng(100 + rank)
    return torch.as_tensor(rng.normal(size=35) * 10.0 ** rng.integers(-3, 4, 35), dtype=F64)


def _worker(rank, world, port, out):
    for p in (ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import surfel_parallel as SPW
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = {}
        for mode in ("all_reduce", "defer", "none"):
            s = _sums(rank)
            res[mode] = SPW.reduce_camera_sums(s, world, grad_reduce=mode)
        torch.save(res, f"{out}.r{rank}")
    finally:
        dist.destroy_process_group()


def test_reduce_camera_sums_world2(tmp_path):
    out = str(tmp_path / "cam")
    mp.spawn(_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    r = [torch.load(f"{out}.r{k}") for k in range(2)]
    s0, s1 = _sums(0), _sums(1)
    once = (s0 + s1).to(torch.float32)
    for mode in ("all_reduce", "defer"):
        for k in range(2):
            assert r[k][mode].dtype == torch.float32
            assert torch.equal(r[k][mode].view(torch.int32), once.view(torch.int32)), (mode, k)
    twice = s0.to(torch.float32) + s1.to(torch.float32)
    assert not torch.equal(twice, once), "the test sums should tell one rounding from two"
    assert torch.equal(r[0]["none"], s0.to(torch.float32)) and torch.equal(r[1]["none"], s1.to(torch.float32))
    # the two partials add up to the sum, each within its own rounding
    err = (r[0]["none"].double() + r[1]["none"].double() - (s0 + s1)).abs()
    assert (err <= 2.0 ** -24 * (s0.abs() + s1.abs())).all()


def test_reduce_camera_sums_without_a_group_rounds_the_partial():
    s = _sums(3)
    assert torch.equal(SP.reduce_camera_sums(s.clone(), 4), s.to(torch.float32))
    assert torch.equal(SP.reduce_camera_sums(s.clone(), 1, grad_reduce="all_reduce"), s.to(torch.float32))
