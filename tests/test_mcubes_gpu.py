"""Device marching cubes of `UnboundedTSDF.extract_mesh` (csrc/mcubes.cu, DESIGN.md §7j) on the GPU: the grid-mode
field against `field(points)` on the reference's own points, bit-for-bit equality with the NumPy restatement of
tests/mcubes_ref.py (golden scene, rendered frames, analytic volumes through the C ABI), seams, determinism, the
colour pass, streams, poisoned memory, devices, rejected arguments and peak memory."""
import types

import numpy as np
import pytest
import torch

import mcubes_ref as MR
import tsdf_ref as TR
import tsdf_scenes as TS
from test_mcubes_cpu import check_closed_oriented, sphere, torus
from test_tsdf_gpu import _field, _rendered_views, _same

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _lib():
    from diff_surfel_rasterization import _cabi
    return _cabi.load()


def _grid_volume(field, bounds, side=512):
    """The grid-mode field of one crop (the values extract_mesh meshes)."""
    from diff_surfel_rasterization import _cabi
    out = torch.empty(side ** 3, dtype=torch.float32, device=field.device)
    b = (_cabi.ctypes.c_double * 6)(*bounds)
    stream = torch.cuda.current_stream(field.device)
    stream.wait_event(field._depth_ready)
    _cabi.check(_cabi.load().surfel_tsdf_eval_grid(side, b, field.n_frames, field.frames, field.map_pixels,
                                                   field.depth.data_ptr(), field.center, field.radius, field.trunc,
                                                   out.data_ptr(), stream.cuda_stream))
    return out


def _reference_points(x_min, x_max, y_min, y_max, z_min, z_max, cropN=512):
    """mcube_utils.py:50-55 with the axes built on the device."""
    x = torch.linspace(x_min, x_max, cropN, device="cuda")
    y = torch.linspace(y_min, y_max, cropN, device="cuda")
    z = torch.linspace(z_min, z_max, cropN, device="cuda")
    xx, yy, zz = torch.meshgrid(x, y, z, indexing="ij")
    return torch.vstack([xx.ravel(), yy.ravel(), zz.ravel()]).T.float().contiguous()


def _bits_equal(got, want):
    got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape)
    if got.dtype == np.float32:
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan)
        g, w = got[~nan].view(np.uint32), want[~nan].view(np.uint32)
        assert np.array_equal(g, w), f"{int((g != w).sum())} of {g.size} values differ"
    else:
        assert np.array_equal(got, want), f"{int((got != want).sum())} of {got.size} entries differ"


def test_linspace_axis_is_torch_cuda_linspace():
    for R in (0.3, 1.23, 1.9):
        for n in (1, 2, 4):
            xs = MR.crop_bounds(R, n)
            for i in range(n):
                got = torch.linspace(xs[i], xs[i + 1], 512, device="cuda").cpu().numpy()
                _bits_equal(got, MR.linspace32(xs[i], xs[i + 1], 512))
    for a, b, s in ((-1.0, 1.0, 7), (0.1, 0.7, 9), (-0.33, 1.9, 511)):
        _bits_equal(torch.linspace(a, b, s, device="cuda").cpu().numpy(), MR.linspace32(a, b, s))


_views = {}


def _analytic_field():
    if "a" not in _views:
        _views["a"] = TS.analytic_views([(64, 48), (80, 60), (50, 50), (72, 40)], 4)
    return _field(_views["a"], [0.0, 0.0, 0.0], 2.5, 2.5 * 2 / 1024)


@pytest.mark.parametrize("R", [0.3, 1.23, 1.9])
@pytest.mark.parametrize("N", [512, 1024, 2048])
def test_grid_mode_equals_the_field_of_the_reference_points(R, N):
    field = _analytic_field()
    n = N // 512
    xs = MR.crop_bounds(R, n)
    for (i, j, k) in {(0, 0, 0), (n - 1, n - 1, n - 1)}:
        b = (xs[i], xs[i + 1], xs[j], xs[j + 1], xs[k], xs[k + 1])
        want = field(_reference_points(*b))
        got = _grid_volume(field, b)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32))
        del want, got
    torch.cuda.empty_cache()


def _restate_field(field, resolution, R):
    n = resolution // 512
    xs = MR.crop_bounds(R, n)

    def values(ijk, axes):
        i, j, k = ijk
        return _grid_volume(field, (xs[i], xs[i + 1], xs[j], xs[j + 1], xs[k], xs[k + 1])).cpu().numpy()
    c = np.array(list(field.center), F)
    return MR.mesh(n, 512, xs, values, c, field.radius)


def _check_extract(field, resolution, R, min_faces=100):
    verts, faces = field.extract_mesh(resolution, R)
    assert verts.dtype == torch.float32 and faces.dtype == torch.int64
    assert verts.device == field.device and faces.device == field.device
    want_v, want_f, _, _ = _restate_field(field, resolution, R)
    _bits_equal(verts, want_v)
    _bits_equal(faces, want_f)
    assert len(want_f) >= min_faces
    return verts, faces


def test_golden_tsdf_scene():
    from test_tsdf_cpu import golden
    g, frames, (center, radius, trunc) = golden()
    views = [(types.SimpleNamespace(full_proj_transform=torch.from_numpy(M)), torch.from_numpy(d[None].copy()),
              torch.from_numpy(c)) for M, d, c in frames]
    field = _field(views, center, radius, float(g["voxel_size"]))
    verts, faces = _check_extract(field, 512, 1.2)
    # the colour pass on the mesh's vertices, as INTEGRATION §11 calls it
    _same(field.colors(verts), TR.emulate(verts.cpu().numpy(), frames, center, radius, trunc, colour=True))


@pytest.fixture(scope="module")
def rendered():
    return _rendered_views(100, 800, 800)


@pytest.mark.parametrize("resolution", [512, 1024])
def test_rendered_frames_100_800x800(rendered, resolution):
    center, radius = np.array([0.0, 0.0, 7.0], F), 6.0
    field = _field(rendered, center, radius, radius * 2 / resolution)
    verts, faces = _check_extract(field, resolution, 1.2, min_faces=10000)
    # deterministic run to run
    v2, f2 = field.extract_mesh(resolution, 1.2)
    assert torch.equal(verts.view(torch.int32), v2.view(torch.int32)) and torch.equal(faces, f2)
    if resolution == 512:
        frames = TS.frames_of(rendered)
        _same(field.colors(verts), TR.emulate(verts.cpu().numpy(), frames, center, radius, 5 * radius * 2 / 512,
                                              colour=True))


# ---- analytic volumes through the C ABI ------------------------------------------------------------------------------

def _device_mesh(fn, n, side, R=1.0, center=(0.1, -0.2, 0.3), radius=2.0, stream=None):
    from diff_surfel_rasterization import _cabi
    from diff_surfel_rasterization.tsdf import _mesh_crops
    xs = MR.crop_bounds(R, n)
    axes = MR.crop_axes(xs, side)
    crops = {}
    for i in range(n):
        for j in range(n):
            for k in range(n):
                crops[(i, j, k)] = MR.analytic(fn)((i, j, k), [axes[i], axes[j], axes[k]])
    lookup = {}
    for key, v in crops.items():
        b = (xs[key[0]], xs[key[0] + 1], xs[key[1]], xs[key[1] + 1], xs[key[2]], xs[key[2] + 1])
        lookup[b] = torch.from_numpy(v.reshape(-1).copy()).cuda()

    def field(lib, bounds, out, st):
        out.copy_(lookup[tuple(bounds)])
    cen = (_cabi.c_float * 3)(*center)
    stream = stream or torch.cuda.current_stream()
    v, f = _mesh_crops(_cabi.load(), stream, n, side, xs, cen, radius, field)
    want = MR.mesh(n, side, xs, lambda ijk, axes: crops[ijk], np.array(center, F), radius)
    return v, f, want


def _noise(seed, scale=1.0):
    def fn(X, Y, Z):
        rng = np.random.default_rng(seed)
        k = rng.normal(size=(6, 3)) * 9
        ph = rng.uniform(0, 6.3, 6)
        v = sum(np.sin(X * F(a) + Y * F(b) + Z * F(c) + F(p)) for (a, b, c), p in zip(k, ph))
        return (v * F(scale)).astype(F)
    return fn


def _planes_through_grid(side, n):
    g = np.concatenate([a[:-1] for a in MR.crop_axes(MR.crop_bounds(1.0, n), side)])
    return lambda X, Y, Z: np.minimum(X - g[side // 2], (Y - g[3]) * (Z - g[(side + 1) % len(g)]))


def _zeros(side, n):
    g = np.concatenate([a[:-1] for a in MR.crop_axes(MR.crop_bounds(1.0, n), side)])
    return lambda X, Y, Z: np.where((X >= g[4]) & (Y < g[len(g) // 2 + 1]), F(0), sphere(0.5)(X, Y, Z)).astype(F)


SCENES = {
    "sphere": lambda side, n: sphere(0.63, (0.02, -0.03, 0.01)),
    "torus": lambda side, n: torus(0.5, 0.2),
    "planes_through_grid_points": _planes_through_grid,
    "noise": lambda side, n: _noise(1),
    "noise_fine": lambda side, n: _noise(2, 0.5),
    "exact_zeros": _zeros,
    "all_inside": lambda side, n: lambda X, Y, Z: np.full(X.shape, F(-0.5)),
    "all_outside": lambda side, n: lambda X, Y, Z: np.full(X.shape, F(0.5)),
    "all_zero": lambda side, n: lambda X, Y, Z: np.zeros(X.shape, F),
    "nearly_far": lambda side, n: sphere(1.7),          # vertices beyond |y| = 1: uncontraction's outer branch
}


@pytest.mark.parametrize("n,side", [(1, 33), (2, 17), (3, 12), (1, 64)])
@pytest.mark.parametrize("scene", list(SCENES))
def test_analytic_volumes_through_the_c_abi(scene, n, side):
    R = 1.95 if scene == "nearly_far" else 1.0
    v, f, (want_v, want_f, _, _) = _device_mesh(SCENES[scene](side, n), n, side, R=R)
    _bits_equal(v, want_v)
    _bits_equal(f, want_f)
    if scene in ("all_inside", "all_outside", "all_zero"):
        assert v.shape == (0, 3) and f.shape == (0, 3)
    elif scene in ("sphere", "torus"):
        check_closed_oriented(f.cpu().numpy(), len(v), 2 if scene == "sphere" else 0)


def test_seam_vertices_are_shared_by_both_crops():
    side, n = 17, 2
    v, f, (want_v, want_f, pos, keys) = _device_mesh(sphere(0.6), n, side)
    _bits_equal(v, want_v)
    # crop (0,0,0)'s faces come first; faces of later crops reuse vertices on its planes
    G = (side - 1) * n + 1
    P = keys // 4
    on_seam = (P // (G * G) == side - 1) | (P // G % G == side - 1) | (P % G == side - 1)
    fn = f.cpu().numpy()
    per_crop = MR.Mesher(n, side, MR.crop_bounds(1.0, n))
    axes = per_crop.axes
    per_crop.add_crop((0, 0, 0), MR.analytic(sphere(0.6))((0, 0, 0), [axes[0]] * 3))
    first = len(np.concatenate(per_crop.tri_keys))
    shared = np.intersect1d(fn[:first].ravel(), fn[first:].ravel())
    assert len(shared) > 10 and on_seam[shared].all()
    check_closed_oriented(fn, len(v), 2)


def test_side_stream_poisoned_memory_and_second_device():
    field = _analytic_field()
    want_v, want_f = field.extract_mesh(512, 0.8)
    assert len(want_f) > 1000
    # every block the call allocates was 0xFF before it
    junk = torch.full((6 << 30,), 255, dtype=torch.uint8, device="cuda")
    del junk
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        v, f = field.extract_mesh(512, 0.8)
    s.synchronize()
    assert torch.equal(v.view(torch.int32), want_v.view(torch.int32)) and torch.equal(f, want_f)
    if torch.cuda.device_count() > 1:
        f1 = _field(_views["a"], [0.0, 0.0, 0.0], 2.5, 2.5 * 2 / 1024, dev="cuda:1")
        v1, ff1 = f1.extract_mesh(512, 0.8)
        assert v1.device == torch.device("cuda:1")
        assert torch.equal(v1.cpu().view(torch.int32), want_v.cpu().view(torch.int32))
        assert torch.equal(ff1.cpu(), want_f.cpu())


def test_rejected_arguments():
    field = _analytic_field()
    for res in (0, 1000, 256, -512, 512.5):
        with pytest.raises(RuntimeError, match="multiple of 512"):
            field.extract_mesh(res, 1.0)
    for R in (0.0, -0.5, float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match="finite and > 0"):
            field.extract_mesh(512, R)


def test_peak_memory_is_at_most_the_reference_points_and_field():
    field = _analytic_field()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    verts, faces = field.extract_mesh(1024, 1.0)
    torch.cuda.synchronize()
    ours = torch.cuda.max_memory_allocated() - base
    del verts, faces
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    xs = MR.crop_bounds(1.0, 2)
    pts = _reference_points(xs[0], xs[1], xs[0], xs[1], xs[0], xs[1])
    z = torch.cat([field(p) for p in torch.split(pts, 256 ** 3, dim=0)])
    torch.cuda.synchronize()
    ref = torch.cuda.max_memory_allocated() - base
    del pts, z
    print(f"peak device memory: extract_mesh {ours / 2**20:.0f} MiB, reference points + field per crop "
          f"{ref / 2**20:.0f} MiB")
    assert ours <= ref


def test_golden_inverse_contraction_and_clip_through_the_merge():
    """The reference's recorded inv_contraction + clip (tests/golden/ref_mcubes.npz) replayed by the merge kernel."""
    from diff_surfel_rasterization import _cabi
    from test_mcubes_cpu import _golden, golden_uncontract_check
    g = _golden()
    y = torch.from_numpy(g["contracted"].astype(F)).cuda().contiguous()
    n = y.shape[0]
    keys = torch.arange(n, dtype=torch.int64, device="cuda") * 4
    lib = _cabi.load()
    wb = lib.surfel_mcubes_merge_workspace_bytes(n)
    ws = torch.full((wb,), 255, dtype=torch.uint8, device="cuda")
    verts = torch.full((n, 3), float("nan"), device="cuda")
    count = torch.zeros(1, dtype=torch.int64, device="cuda")
    cen = (_cabi.c_float * 3)(*g["center"].tolist())
    _cabi.check(lib.surfel_mcubes_merge(n, keys.data_ptr(), y.data_ptr(), 0, None, 40, cen, float(g["radius"]),
                                        ws.data_ptr(), wb, verts.data_ptr(), None, count.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream))
    assert int(count.item()) == n
    golden_uncontract_check(verts.cpu().numpy(), g)
    _bits_equal(verts, MR.uncontract_clip(g["contracted"], g["center"], float(g["radius"])))
