"""The fused TSDF field on the GPU (csrc/tsdf.cu, DESIGN.md §7i): the reference's stored outputs, bit-for-bit
equality with the float32 emulation of tests/tsdf_ref.py in both modes (rendered depth maps, one 256^3 call, empty
and degenerate inputs, frame counts around the shared-memory batch, NaN and inf, int64 map offsets), and the
wrapper's streams, devices and argument checks."""
import types

import numpy as np
import pytest
import torch

import tsdf_ref as TR
import tsdf_scenes as TS
from test_tsdf_cpu import golden

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _field(views, center, radius, voxel_size, dev="cuda"):
    from diff_surfel_rasterization.tsdf import UnboundedTSDF
    return UnboundedTSDF([d for _, d, _ in views], [c for _, _, c in views], [v for v, _, _ in views],
                         torch.as_tensor(np.asarray(center, F)).to(dev), radius, voxel_size)


def _same(got, want):
    """Bit for bit, except that a NaN's payload is not compared (the GPU writes the canonical NaN, numpy keeps the
    payload of the NaN or inf it came from)."""
    got = got.detach().cpu().numpy()
    assert got.shape == want.shape and got.dtype == want.dtype
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"NaN at {int((np.isnan(got) != nan).sum())} other places"
    g, w = got[~nan].view(np.uint32), want[~nan].view(np.uint32)
    assert np.array_equal(g, w), f"{int((g != w).sum())} of {g.size} values differ"


def _check_both_modes(views, center, radius, voxel_size, pts_field, pts_colour):
    field = _field(views, center, radius, voxel_size)
    frames = TS.frames_of(views)
    _same(field(torch.from_numpy(pts_field).cuda()), TR.emulate(pts_field, frames, center, radius, 5 * voxel_size))
    _same(field.colors(torch.from_numpy(pts_colour).cuda()),
          TR.emulate(pts_colour, frames, center, radius, 5 * voxel_size, colour=True))
    return field


def test_golden_replay():
    g, frames, (center, radius, trunc) = golden()
    views = [(types.SimpleNamespace(full_proj_transform=torch.from_numpy(M)), torch.from_numpy(d[None].copy()),
              torch.from_numpy(c)) for M, d, c in frames]
    field = _field(views, center, radius, float(g["voxel_size"]))
    for colour, pts, ref in ((False, g["points"], g["ref_tsdf"]), (True, g["colour_points"], g["ref_rgb"])):
        x = torch.from_numpy(pts).cuda()
        got = (field.colors(x) if colour else field(x)).cpu().numpy()
        _same(torch.from_numpy(got), TR.emulate(pts, frames, center, radius, trunc, colour))
        value, bound, flagged = TR.evaluate64(pts, frames, center, radius, trunc, colour)
        assert len(TR.check_within(got, value, bound, flagged, factor=1.0)) == 0
        # GPU and reference each within the bound: within twice of each other; the same unobserved samples
        assert len(TR.check_within(got, ref.astype(np.float64), bound, flagged, factor=2.0)) == 0
        if not colour:
            assert np.array_equal(got[~flagged] == -1, ref[~flagged] == -1)


def _rendered_views(n, W, H, P=30000, seed=3):
    """Depth maps of this project's rasterizer (surf_depth of surface_outputs, depth_ratio 0) of one synthetic
    scene from n cameras around it; RGB is the rendered colour."""
    import surfel_scenes as S
    from diff_surfel_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from diff_surfel_rasterization.postprocess import surface_outputs
    scene = {k: v.cuda() for k, v in S.make_scene(P, W, H, seed=seed).items()}
    views = []
    for k in range(n):
        R = S.look_at_rotation(-12 + 24 * k / n, 6 * np.sin(k))
        t = np.array([0.4 * np.cos(k), 0.2 * np.sin(2 * k), 0.3 * np.sin(k)])
        cam = S.make_camera(W, H, R=R, t=t)
        rs = GaussianRasterizationSettings(
            image_height=H, image_width=W, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=torch.zeros(3).cuda(),
            scale_modifier=1.0, viewmatrix=cam["viewmatrix"].cuda(), projmatrix=cam["projmatrix"].cuda(),
            sh_degree=3, campos=cam["campos"].cuda(), prefiltered=False, debug=False)
        with torch.no_grad():
            color, _, allmap = GaussianRasterizer(rs)(
                means3D=scene["means3D"], means2D=torch.zeros(P, 3).cuda(), shs=scene["shs"],
                opacities=scene["opacities"], scales=scene["scales"], rotations=scene["rotations"])
            view = types.SimpleNamespace(world_view_transform=cam["viewmatrix"].cuda(),
                                         full_proj_transform=cam["projmatrix"].cuda(), image_width=W, image_height=H)
            depth = surface_outputs(allmap, view, 0.0)["surf_depth"]
        views.append((types.SimpleNamespace(full_proj_transform=cam["projmatrix"]), depth.cpu(), color.cpu()))
    return views


def test_rendered_depth_maps_100_frames_800x800():
    views = _rendered_views(100, 800, 800)
    rng = np.random.default_rng(0)
    center, radius = np.array([0.0, 0.0, 7.0], F), 6.0
    pts = np.concatenate([rng.uniform(-1.9, 1.9, (40000, 3)), TS.special_points(1.9)]).astype(F)
    cpts = (rng.uniform(-1, 1, (20000, 3)) * [3, 3, 5] + [0, 0, 7]).astype(F)
    field = _check_both_modes(views, center, radius, radius * 2 / 1024, pts, cpts)
    t = field(torch.from_numpy(pts).cuda())
    assert (t != -1).sum() > 500


def test_one_256_cubed_call():
    views = TS.analytic_views([(64, 48), (80, 60), (50, 50), (72, 40)], 4)
    g = torch.linspace(-1.9, 1.9, 256)
    pts = torch.stack(torch.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).contiguous()
    field = _field(views, [0.0, 0.0, 0.0], 2.8, 2.8 * 2 / 1024)
    got = field(pts.cuda())
    _same(got, TR.emulate(pts.numpy(), TS.frames_of(views), [0.0, 0.0, 0.0], 2.8, 5 * 2.8 * 2 / 1024))
    assert (got != -1).sum() > 10000


def test_empty_and_degenerate_inputs():
    from diff_surfel_rasterization.tsdf import UnboundedTSDF
    rng = np.random.default_rng(5)
    pts = rng.uniform(-1.9, 1.9, (3000, 3)).astype(F)
    none = UnboundedTSDF([], [], [], torch.zeros(3).cuda(), 2.0, 0.01)
    assert torch.equal(none(torch.from_numpy(pts).cuda()), torch.full((3000,), -1.0).cuda())
    assert torch.equal(none.colors(torch.from_numpy(pts).cuda()), torch.zeros(3000, 3).cuda())
    views = TS.analytic_views([(1, 1), (1, 37), (41, 1), (2, 2), (30, 20)], 6, dist=2.0)
    field = _check_both_modes(views, [0, 0, 0], 2.5, 0.02, pts, (pts * 1.5).astype(F))
    assert field(torch.zeros(0, 3).cuda()).shape == (0,)
    assert field.colors(torch.zeros(0, 3).cuda()).shape == (0, 3)


@pytest.mark.parametrize("V", [31, 32, 33, 64, 65])
def test_frame_counts_around_the_batch(V):
    base = TS.analytic_views([(23 + k, 17 + 2 * k) for k in range(11)], 7, dist=2.2)
    views = [base[k % len(base)] for k in range(V)]
    rng = np.random.default_rng(V)
    pts = rng.uniform(-1.9, 1.9, (5000, 3)).astype(F)
    _check_both_modes(views, [0.02, -0.01, 0.0], 2.4, 0.015, pts, (rng.uniform(-1.5, 1.5, (3000, 3))).astype(F))


def test_nan_and_inf_in_maps_and_points():
    views = TS.analytic_views([(40, 30), (35, 28), (44, 33)], 8, dist=2.0)
    for k, (_, d, c) in enumerate(views):
        d[0, 5:9, 5:20] = [np.inf, -np.inf, np.nan, 0.0][k % 4]
        d[0, 10, 10:30] = np.inf
        c[:, 3:6, 3:30] = np.nan
        c[1, 20, :] = np.inf
    rng = np.random.default_rng(9)
    pts = rng.uniform(-1.9, 1.9, (20000, 3)).astype(F)
    pts[:6] = [[np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 0], [np.inf, np.inf, np.inf], [1e30, 0, 0], [0, 0, 1e-30]]
    cpts = rng.uniform(-1.5, 1.5, (20000, 3)).astype(F)
    cpts[:3] = [[np.nan, 0, 0], [np.inf, 0, 1], [0, 0, -np.inf]]
    _check_both_modes(views, [0, 0, 0], 2.2, 0.02, pts, cpts)


def test_maps_beyond_2_to_the_31_pixels():
    """1040 frames of 1080x1920: 2.16e9 pixels, so the last frames' offsets need 64 bits."""
    H, W, V = 1080, 1920, 1040
    cam = TS.ring_camera(W, H, 20.0, 0.1, 2.5)
    rng = np.random.default_rng(10)
    a, _ = TS.analytic_maps(cam, rng, n_nan=0)
    b = a + np.float32(0.05) * rng.standard_normal(a.shape).astype(F)
    view = types.SimpleNamespace(full_proj_transform=cam["projmatrix"])
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    maps = [da] * (V - 3) + [db] * 3
    from diff_surfel_rasterization.tsdf import UnboundedTSDF
    field = UnboundedTSDF(maps, None, [view] * V, torch.zeros(3).cuda(), 2.5, 0.01)
    assert field.map_pixels > 2 ** 31 and field.frames[V - 1].offset > 2 ** 31
    pts = TS.sphere_surface_points(3000, rng, [0, 0, 0], 2.5)[0]
    got = field(torch.from_numpy(pts).cuda())
    want = TR.emulate(pts, [(view.full_proj_transform.numpy(), m, None) for m in [a[0]] * (V - 3) + [b[0]] * 3],
                      [0, 0, 0], 2.5, 0.05)
    _same(got, want)
    assert (got != -1).sum() > 500
    del field, da, db, maps
    torch.cuda.empty_cache()


def test_side_stream_noncontiguous_points_and_second_device():
    views = TS.analytic_views([(40, 30), (35, 28)], 12, dist=2.0)
    rng = np.random.default_rng(12)
    pts = rng.uniform(-1.9, 1.9, (50000, 3)).astype(F)
    want = TR.emulate(pts, TS.frames_of(views), [0, 0, 0], 2.2, 0.1)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        field = _field(views, [0, 0, 0], 2.2, 0.02)
        wide = torch.zeros(50000, 6, device="cuda")
        wide[:, ::2] = torch.from_numpy(pts).cuda()
        got = field(wide[:, ::2])
    s.synchronize()
    _same(got, want)
    _same(field(torch.from_numpy(pts).cuda().t().contiguous().t()), want)
    if torch.cuda.device_count() > 1:
        f1 = _field(views, [0, 0, 0], 2.2, 0.02, dev="cuda:1")
        _same(f1(torch.from_numpy(pts).to("cuda:1")), want)
        with pytest.raises(RuntimeError, match="cuda:1"):
            f1(torch.from_numpy(pts).cuda())


def test_rejected_arguments():
    from diff_surfel_rasterization.tsdf import UnboundedTSDF
    views = TS.analytic_views([(10, 8)], 13)
    field = _field(views, [0, 0, 0], 2.0, 0.02)
    with pytest.raises(RuntimeError, match="CUDA"):
        field(torch.zeros(4, 3))
    with pytest.raises(RuntimeError, match="float32"):
        field(torch.zeros(4, 3, dtype=torch.float64).cuda())
    with pytest.raises(RuntimeError, match=r"\(N,3\)"):
        field.colors(torch.zeros(4, 4).cuda())
    no_rgb = UnboundedTSDF([views[0][1]], None, [views[0][0]], torch.zeros(3).cuda(), 2.0, 0.02)
    with pytest.raises(RuntimeError, match="without RGB"):
        no_rgb.colors(torch.zeros(4, 3).cuda())
    with pytest.raises(RuntimeError, match="RGB map"):
        UnboundedTSDF([views[0][1]], [torch.zeros(3, 8, 11)], [views[0][0]], torch.zeros(3).cuda(), 2.0, 0.02)
