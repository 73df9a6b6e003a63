"""Camera gradients of the tile-band frame (surfel_camera_backward_sums, surfel_parallel.rasterize_tile_band,
DESIGN.md §7r) on one GPU.

  1. exact, no budget: on each band's own forward and gradient records, each of the 35 double sums is within
     TOL x (sum over the band's splats of |J| |rec|) of the float64 restatement (tests/camera_exact.py), with the
     structural zeros exactly zero; the total over the bands, rounded once, is within the sum of the band bounds plus
     one rounding of the exact total.  Six certified scenes (EXACT_SCENES), every path of test_camera_grad_gpu, both
     scale_modifiers and both low-pass settings, each (scene, path) on one of five partitions;
  2. one code path: on the whole frame, the double sums rounded to float32 are surfel_camera_backward's outputs, bit
     for bit;
  3. the public path: rasterize_tile_band(rank=r, world=N) called for every r in one process (no process group)
     accumulates the whole-frame camera gradient of GaussianRasterizer, on the parity scenes, an uneven last band and
     a config-5 frame; frames are bit-identical with and without camera gradients, splat gradients agree to the
     render backward's run-to-run spread, and without camera gradients the launch count is the old one;
  4. repeatable: repeat calls and a side stream give bit-identical sums.
"""
import ctypes

import numpy as np
import pytest
import torch

import camera_exact as CE
import hitloop_scenes as HS
import preprocess_scenes as PS
import surfel_scenes as S
from parity_bars import record_stats
from test_camera_grad_gpu import CASES, CAST, TOL, camera_call, case_scene, parity_cases, parity_scene, settings

pytestmark = pytest.mark.gpu

# partitions of the frame's tile rows: (helper, number of bands); "rows" = one band per tile row
PARTITIONS = [("tile_row_band", 2), ("equal_band", 3), ("tile_row_band", 4), ("rows", 0), ("equal_band", 2)]
# the certified scenes of test 1: orientation, clamp, low-pass and near-plane features, one splat and a full layout
EXACT_SCENES = ("orient", "clamp", "low_pass", "near", "layout1", "layout4097")


def bands_of(kind, n, H):
    import surfel_parallel as SP
    if kind == "rows":
        return [(r, r + 1) for r in range(SP.tile_rows(H))]
    f = SP.tile_row_band if kind == "tile_row_band" else SP.equal_band
    return [f(H, r, n) for r in range(n)]


def sums_call(pipe, scratch, dtm, stream=None):
    """surfel_camera_backward_sums on a CudaPipeline's forward state; returns the (35,) float64 sums as numpy."""
    from diff_surfel_rasterization import _cabi
    lib = pipe.lib
    st = torch.cuda.current_stream() if stream is None else stream
    partials = torch.full((lib.surfel_camera_partials_bytes(pipe.P) // 8,), float("nan"), dtype=torch.float64, device="cuda")
    out = torch.full((35,), float("nan"), dtype=torch.float64, device="cuda")
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        _p = lambda t: None if t is None else t.data_ptr()
        _cabi.check(lib.surfel_camera_backward_sums(
            ctypes.byref(pipe.cs), pipe.P, pipe.M, _p(pipe.means3D), _p(pipe.scales), _p(pipe.rotations),
            _p(pipe.transMat_precomp), _p(pipe.shs), int(pipe.colors_precomp is not None), pipe.radii.data_ptr(),
            pipe.geom.data_ptr(), scratch.data_ptr(), _p(dtm), partials.data_ptr(), out[0:16].data_ptr(),
            out[16:32].data_ptr(), out[32:35].data_ptr(), st.cuda_stream), lib)
    st.synchronize()
    return out.cpu().numpy()


def split(v):
    return dict(viewmatrix=v[0:16], projmatrix=v[16:32], campos=v[32:35])


def band_run(scene, cam, D, mod, band, gc, go, lq):
    """Forward and backward of one band through the stages; returns (pipe, forward record, backward outputs)."""
    from cuda_stages import CudaPipeline
    pipe = CudaPipeline(scene, cam, HS.BG, D, mod, tile_rows=band)
    fwd = pipe.preprocess()
    pipe.bucket()
    pipe.render()
    got = pipe.backward(gc, go, lowpass_quirk=lq)
    return pipe, fwd, got


# ---------------------------------------------------------------------------------------------- 1. exact
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-D{c[1]}")
@pytest.mark.parametrize("name", EXACT_SCENES)
def test_band_sums_match_exact(oracle, cuda_lib, name, case):
    from cuda_stages import CudaPipeline
    path, D = case
    kind, n = PARTITIONS[(EXACT_SCENES.index(name) + CASES.index(case)) % len(PARTITIONS)]
    failures, worst = [], {}
    for mod in (1.0, 1.7):
        scene, cam = case_scene(oracle, name, path, mod)
        whole = CudaPipeline(scene, cam, HS.BG, D, mod)
        ref = CE.CameraReference(scene, cam, whole.preprocess(), D, mod)     # its Jacobian is shared by the bands
        gc, go = HS.cotangent(cam["W"], cam["H"], "all", seed=3)
        bands = bands_of(kind, n, int(cam["H"]))
        for lq in (True, False):
            total = np.zeros(35)
            exact = {k: 0.0 for k in CE.KEYS}
            bound = {k: 0.0 for k in CE.KEYS}
            for band in bands:
                pipe, fwd, got = band_run(scene, cam, D, mod, band, gc, go, lq)
                rec = got["grad_rec"].astype(np.float64)
                rec[fwd["radii"] <= 0] = 0.0           # what the band culled has no record (the kernel skips it)
                scratch = torch.tensor(got["grad_rec"], device="cuda")
                dtm = torch.tensor(got["dL_dtransMat"], device="cuda")
                dev = sums_call(pipe, scratch, dtm)
                total += dev
                ev, bd = ref.camera(rec), ref.camera_bound(rec)
                for key, g in split(dev).items():
                    r, b = ev[key], bd[key]
                    exact[key] = exact[key] + r
                    bound[key] = bound[key] + b
                    err = np.abs(g - r)
                    tag = f"scale_modifier={mod} lowpass_quirk={lq} {kind}/{n} band {band} {key}"
                    if not np.isfinite(g).all():
                        failures.append(f"{tag}: non-finite")
                        continue
                    if (g[b == 0] != 0).any():
                        failures.append(f"{tag}: non-zero where the rules give 0: {g[b == 0]}")
                    pos = b > 0
                    ratio = float((err[pos] / b[pos]).max()) if pos.any() else 0.0
                    worst[key] = max(worst.get(key, 0.0), ratio)
                    if (err > TOL * b).any():
                        failures.append(f"{tag}: worst error / bound {ratio:.3e} > {TOL}")
            for key, g in split(total.astype(np.float32).astype(np.float64)).items():
                err = np.abs(g - exact[key])
                if (err > TOL * bound[key] + CAST * np.abs(exact[key])).any():
                    failures.append(f"scale_modifier={mod} lowpass_quirk={lq} {kind}/{n} total {key}: "
                                    f"{err.max():.3e} over the band bounds plus one cast")
    for key, r in worst.items():
        record_stats(f"camera_bwd band sums exact {key} / bound", np.array([r]),
                     dict(tol=TOL, scene=name, case=f"{path}-D{D}", partition=f"{kind}/{n}"))
    assert not failures, f"{name} [{path}-D{D}]:\n" + "\n".join(failures[:20])


# ---------------------------------------------------------------------------------------------- 2. one code path
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-D{c[1]}")
def test_whole_frame_sums_round_to_camera_backward(oracle, cuda_lib, case):
    from cuda_stages import CudaPipeline
    path, D = case
    for name in ("layout4097", "clamp", "orient"):
        scene, cam = case_scene(oracle, name, path, 1.7)
        pipe = CudaPipeline(scene, cam, HS.BG, D, 1.7)
        pipe.preprocess(); pipe.bucket(); pipe.render()
        got = pipe.backward(*HS.cotangent(cam["W"], cam["H"], "all", seed=4))
        scratch = torch.tensor(got["grad_rec"], device="cuda")
        dtm = torch.tensor(got["dL_dtransMat"], device="cuda")
        f32 = camera_call(pipe, scratch, dtm)
        sums = split(sums_call(pipe, scratch, dtm))
        for key in CE.KEYS:
            assert np.array_equal(sums[key].astype(np.float32).view(np.uint32), f32[key].view(np.uint32)), (name, key)


def test_sums_entry_accepts_a_band_and_the_float_entry_still_rejects_it(oracle, cuda_lib):
    from cuda_stages import CudaPipeline
    from diff_surfel_rasterization import _cabi
    scene, cam = case_scene(oracle, "layout1000", "shs", 1.0)
    pipe, fwd, got = band_run(scene, cam, 3, 1.0, (2, 5), *HS.cotangent(cam["W"], cam["H"], "all", seed=5), True)
    scratch = torch.tensor(got["grad_rec"], device="cuda")
    dtm = torch.tensor(got["dL_dtransMat"], device="cuda")
    assert np.isfinite(sums_call(pipe, scratch, dtm)).all()
    with pytest.raises(RuntimeError, match="tile-row band"):
        camera_call(pipe, scratch, dtm)


# ---------------------------------------------------------------------------------------------- 3. public path
def band_op(scene, cam, world, gc, go, camera_grad=True, lib=None):
    """rasterize_tile_band for rank 0..world-1 in turn (no process group), one backward each, the camera leaves shared.
    Returns the band rows of the frames, the splat gradients summed over the bands, the camera gradients and the
    launches per band call."""
    import surfel_parallel as SP
    from diff_surfel_rasterization import GaussianRasterizer
    dev = torch.device("cuda")
    rs = settings(cam, dev, camera_grad=camera_grad)
    leaf = {k: torch.as_tensor(np.asarray(v)).to(dev).requires_grad_(True) for k, v in scene.items()}
    m2d = torch.zeros(leaf["means3D"].shape[0], 3, device=dev, requires_grad=True)
    H = int(cam["H"])
    frames, launches = [], []
    for r in range(world):
        n0 = lib.surfel_launch_count() if lib is not None else 0
        res = SP.rasterize_tile_band(GaussianRasterizer, rs, r, world, means3D=leaf["means3D"], means2D=m2d,
                                     shs=leaf["shs"], opacities=leaf["opacities"], scales=leaf["scales"],
                                     rotations=leaf["rotations"])
        s, e = SP.band_pixel_rows(H, res["band"])
        # without a process group the rows outside the band are not this call's: only the band's rows carry a loss
        ((res["render"][:, s:e] * gc[:, s:e].to(dev)).sum() + (res["allmap"][:, s:e] * go[:, s:e].to(dev)).sum()).backward()
        torch.cuda.synchronize()
        if lib is not None:
            launches.append(lib.surfel_launch_count() - n0)
        frames.append((res["render"][:, s:e].detach().cpu().numpy(), res["allmap"][:, s:e].detach().cpu().numpy()))
    grads = {k: v.grad.cpu().numpy() for k, v in leaf.items()}
    grads["means2D"] = m2d.grad.cpu().numpy()
    cg = {k: getattr(rs, k).grad.cpu().numpy().reshape(-1) for k in CE.KEYS if getattr(rs, k).grad is not None}
    return dict(frames=frames, grads=grads, camera=cg, launches=launches)


def check_public(scene, cam, world, seed, lib):
    from test_camera_grad_gpu import run_op
    gc, go = S.make_cotangents(cam["W"], cam["H"], seed)
    a, b = run_op(scene, cam, gc, go), run_op(scene, cam, gc, go)
    band_op(scene, cam, world, gc, go, camera_grad=False)            # warm-up: instance capacities are known
    plain = band_op(scene, cam, world, gc, go, camera_grad=False, lib=lib)
    plain2 = band_op(scene, cam, world, gc, go, camera_grad=False, lib=lib)
    withcam = band_op(scene, cam, world, gc, go, camera_grad=True, lib=lib)
    assert plain["camera"] == {} and set(withcam["camera"]) == set(CE.KEYS)
    assert plain["launches"] == plain2["launches"], "launch count of a plain band step is not stable"
    assert withcam["launches"] == [n + 2 for n in plain["launches"]], "camera gradients add the camera kernel and finish"
    for (c0, m0), (c1, m1) in zip(plain["frames"], withcam["frames"]):
        assert np.array_equal(c0.view(np.uint32), c1.view(np.uint32)) and np.array_equal(m0.view(np.uint32), m1.view(np.uint32))
    for k in plain["grads"]:
        p, p2, c = plain["grads"][k].astype(np.float64), plain2["grads"][k], withcam["grads"][k]
        spread, diff = np.abs(p2 - p).max(), np.abs(c - p).max()
        assert diff <= max(2.0 * spread, 4e-6 * np.abs(p).max()), f"splat gradient {k}: {diff:.3e} (spread {spread:.3e})"
    for key in CE.KEYS:
        ref, ref2, got = a["camera"][key].astype(np.float64), b["camera"][key], withcam["camera"][key].astype(np.float64)
        scale = np.abs(ref).max()
        spread, diff = np.abs(ref2 - ref).max(), np.abs(got - ref).max()
        # the bands' render backward adds its float atomics in another order than the whole frame's does: the bar is
        # the whole frame's own run-to-run spread (x2), floored at 1e-5 of the scale, plus one cast per band.  Worst
        # observed on an H100 80GB HBM3 (700 W): 3.5e-6 of the scale (projmatrix, 64x48 in 3 bands; spread 1.4e-6)
        bar = max(2.0 * spread, 1e-5 * scale) + world * CAST * scale
        record_stats(f"band camera grad {key}: max|bands - whole| / scale", np.array([diff / scale]),
                     dict(world=world, spread=float(spread / scale), W=int(cam["W"]), H=int(cam["H"])))
        assert scale > 0, key
        assert diff <= bar, f"{key}: max|bands - whole frame| {diff:.3e} > {bar:.3e} (whole-frame run-to-run {spread:.3e})"


@pytest.mark.parametrize("ci", range(3))
def test_public_band_path_sums_to_the_whole_frame(cuda_lib, ci):
    scene, cam = parity_scene(parity_cases()[ci])
    check_public(scene, cam, 2 if ci < 2 else 3, 20 + ci, cuda_lib)


def test_public_band_path_uneven_last_band(cuda_lib):
    import surfel_parallel as SP
    scene, cam = parity_scene(parity_cases()[1])          # 171 rows: 11 tile rows, equal bands of 4, 4 and 3
    bands = [SP.equal_band(int(cam["H"]), r, 3) for r in range(3)]
    assert bands[-1][1] - bands[-1][0] < bands[0][1] - bands[0][0]
    check_public(scene, cam, 3, 30, cuda_lib)


def test_public_band_path_config5(cuda_lib):
    scene, cam = S.named("config5")                       # 2 M splats, 7680 x 4320
    check_public(S.to_numpy(scene), S.to_numpy(cam), 2, 40, cuda_lib)


# ---------------------------------------------------------------------------------------------- 4. repeatable
def test_band_sums_repeat_and_side_stream_bit_identical(oracle, cuda_lib):
    scene, cam = case_scene(oracle, "layout4097", "shs", 1.7)
    pipe, fwd, got = band_run(scene, cam, 3, 1.7, (3, 8), *HS.cotangent(cam["W"], cam["H"], "all", seed=6), True)
    scratch = torch.tensor(got["grad_rec"], device="cuda")
    dtm = torch.tensor(got["dL_dtransMat"], device="cuda")
    first = sums_call(pipe, scratch, dtm)
    assert np.abs(first).max() > 0
    side = torch.cuda.Stream()
    for stream in (None, None, side, side):
        assert np.array_equal(first.view(np.uint64), sums_call(pipe, scratch, dtm, stream).view(np.uint64))
