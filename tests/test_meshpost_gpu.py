"""Device cluster filtering of `meshpost.post_process_mesh` (csrc/meshpost.cu, DESIGN.md §7k) on the GPU: cluster ids
and counts through the C ABI and the whole call against the reference's recorded outputs (tests/golden/
ref_meshpost.npz), meshes of `extract_mesh` and stress meshes against the vectorised restatement (b) of
tests/meshpost_ref.py, determinism, streams, poisoned memory, layouts, devices and rejected arguments."""
import types

import numpy as np
import pytest
import torch

import meshpost_ref as MP
from test_meshpost_cpu import golden, golden_cases

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _pp(*a, **k):
    from diff_surfel_rasterization.meshpost import post_process_mesh
    return post_process_mesh(*a, **k)


def _bits(got, want):
    got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    want = np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    if got.dtype == F32:
        got, want = got.view(np.uint32), want.view(np.uint32)
    assert np.array_equal(got, want), f"{int((got != want).sum())} of {got.size} entries differ"


def _check(out, want, colors=True):
    v, f, c = out
    _bits(v, want[1].astype(F32))
    _bits(f, np.asarray(want[2], np.int64).reshape(-1, 3))
    if want[3] is None:
        assert c is None
    else:
        _bits(c, want[3].astype(F32))
    assert f.dtype == torch.int64 and v.dtype == torch.float32 and v.shape[1] == 3 and f.shape[1] == 3


def _clusters_c_abi(M, faces):
    """(face ids, counts[:C], bad) of surfel_meshpost_clusters, workspace poisoned with 0xFF."""
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    F = faces.shape[0]
    wb = lib.surfel_meshpost_workspace_bytes(M, F)
    ws = torch.full((wb,), 255, dtype=torch.uint8, device="cuda")
    ids = torch.full((F,), -7, dtype=torch.int32, device="cuda")
    counts = torch.full((F,), -7, dtype=torch.int32, device="cuda")
    info = torch.full((2,), -7, dtype=torch.int64, device="cuda")
    _cabi.check(lib.surfel_meshpost_clusters(M, F, faces.data_ptr(), ws.data_ptr(), wb, ids.data_ptr(),
                                             counts.data_ptr(), info.data_ptr(), torch.cuda.current_stream().cuda_stream))
    C, bad = info.tolist()
    return ids.cpu().numpy(), counts[:C].cpu().numpy(), bad


# ---- the golden ----------------------------------------------------------------------------------------------------

def test_golden_cluster_ids_and_counts_through_the_c_abi():
    for name, v, f, _, _ in golden_cases(golden()):
        if len(f) == 0:
            continue
        ids, counts, bad = _clusters_c_abi(len(v), torch.from_numpy(f).cuda())
        want_ids, want_counts = MP.clusters_literal(f)
        assert bad == 0
        assert np.array_equal(ids, want_ids) and np.array_equal(counts, want_counts), name


def test_golden_post_process_mesh_bit_for_bit():
    g = golden()
    for name, v, f, c, ks in golden_cases(g):
        vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
        ct = None if c is None else torch.from_numpy(c).cuda()
        for k in ks:
            tag = f"{name}.k{k}"
            if f"{tag}.error" in g.files:
                with pytest.raises(IndexError):
                    _pp(vt, ft, ct, cluster_to_keep=k)
                continue
            out = _pp(vt, ft, ct, cluster_to_keep=k)
            want = (None, g[f"{tag}.verts"], g[f"{tag}.faces"], g[f"{tag}.colors"] if c is not None else None)
            _check(out, want)


# ---- extract_mesh ----------------------------------------------------------------------------------------------------

def _against_b(verts, faces, colors, ks):
    v, f = verts.cpu().numpy(), faces.cpu().numpy()
    c = None if colors is None else colors.cpu().numpy()
    cl = MP.clusters_vectorised(f, len(v))
    ids, counts, bad = _clusters_c_abi(len(v), faces.contiguous())
    assert bad == 0 and np.array_equal(ids, cl[0]) and np.array_equal(counts, cl[1])
    for k in ks:
        try:
            want = MP.post_process_vectorised(v, f, c, k, clusters=cl)
        except IndexError:
            with pytest.raises(IndexError):
                _pp(verts, faces, colors, cluster_to_keep=k)
            continue
        _check(_pp(verts, faces, colors, cluster_to_keep=k), want)
    return cl


def test_extract_mesh_of_the_tsdf_golden_scene():
    from test_mcubes_gpu import _field
    from test_tsdf_cpu import golden as tsdf_golden
    g, frames, (center, radius, trunc) = tsdf_golden()
    views = [(types.SimpleNamespace(full_proj_transform=torch.from_numpy(M)), torch.from_numpy(d[None].copy()),
              torch.from_numpy(c)) for M, d, c in frames]
    field = _field(views, center, radius, float(g["voxel_size"]))
    verts, faces = field.extract_mesh(512, 1.2)
    rgbs = field.colors(verts)
    cl = _against_b(verts, faces, rgbs, (1, 2, 3, 1000, 0, -1))
    assert len(cl[1]) >= 2


def test_extract_mesh_of_100_rendered_frames_at_1024():
    from test_mcubes_gpu import _field, _rendered_views
    views = _rendered_views(100, 800, 800)
    center, radius = np.array([0.0, 0.0, 7.0], F32), 6.0
    field = _field(views, center, radius, radius * 2 / 1024)
    verts, faces = field.extract_mesh(1024, 1.2)
    assert len(faces) > 10000
    rgbs = field.colors(verts)
    _against_b(verts, faces, rgbs, (1000, 1, 2, 10, 0, -1))


# ---- stress ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("order", ["forward", "reversed", "shuffled"])
def test_strip_of_10m_faces_is_one_cluster(order):
    n = 10_000_000
    f = MP.strip(n)
    if order == "reversed":
        f = f[::-1].copy()
    elif order == "shuffled":
        f = f[np.random.default_rng(1).permutation(n)]
    v = np.random.default_rng(2).normal(size=(n + 2, 3)).astype(F32)
    ids, counts, _ = _clusters_c_abi(n + 2, torch.from_numpy(f).cuda())
    assert np.array_equal(counts, [n]) and not ids.any()
    want = MP.post_process_vectorised(v, f, None, 1)
    _check(_pp(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), cluster_to_keep=1), want)


def test_4m_isolated_faces_are_all_removed():
    n = 4_000_000
    f = torch.arange(3 * n, device="cuda").view(n, 3)
    v = torch.randn(3 * n, 3, device="cuda")
    c = torch.rand(3 * n, 3, device="cuda")
    for k in (1, 1000, 0):
        vo, fo, co = _pp(v, f, c, cluster_to_keep=k)
        assert vo.shape == (0, 3) and fo.shape == (0, 3) and co.shape == (0, 3)
    with pytest.raises(IndexError):
        _pp(v, f, cluster_to_keep=n + 1)


def test_giant_grid_and_clusters_around_the_threshold():
    rng = np.random.default_rng(4)
    parts = [MP.grid(1200, 1500)]
    v0 = 1200 * 1500
    for n in rng.integers(40, 61, 3000):
        parts.append(MP.fan(int(n), v0))
        v0 += int(n) + 2
    f = np.concatenate(parts)
    f = f[rng.permutation(len(f))]
    v = rng.normal(size=(v0 + 10, 3)).astype(F32)
    c = rng.uniform(size=(v0 + 10, 3)).astype(F32)
    _against_b(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(c).cuda(),
               (1, 2, 500, 1000, 2900, 3001, 3002, 0, -1, -2000))


def test_vertex_indices_near_2_to_the_28():
    """Keys of more than 32 bits.  The rules only compare indices, so (b) on the used vertices, renumbered in order,
    gives the answer."""
    M = (1 << 28) - 3
    rng = np.random.default_rng(6)
    parts = [MP.grid(40, 30, M - 1200), MP.strip(60, M - 62), MP.fan(55, 1 << 27), MP.strip(80, 0)]
    parts += [MP.fan(int(n), (1 << 26) + 100 * i) for i, n in enumerate(rng.integers(45, 56, 40))]
    f = np.concatenate(parts)
    f = f[rng.permutation(len(f))]
    used = np.unique(f)
    small = np.searchsorted(used, f)
    vf = lambda idx: np.stack([idx % 1000, idx % 7, idx % 13], 1).astype(F32)
    verts = torch.arange(M, device="cuda")
    verts = torch.stack([verts % 1000, verts % 7, verts % 13], 1).float()
    ft = torch.from_numpy(f).cuda()
    for k in (1, 2, 20, 0, -1):
        _, vs, fs, _ = MP.post_process_vectorised(vf(used), small, None, k)
        vo, fo, _ = _pp(verts, ft, cluster_to_keep=k)
        _bits(fo, fs)
        _bits(vo, vs)


# ---- behaviour ------------------------------------------------------------------------------------------------------

def _mesh(seed=8):
    rng = np.random.default_rng(seed)
    parts, v0 = [MP.grid(300, 200)], 60000
    for n in rng.integers(1, 200, 400):
        parts.append(MP.bipyramid(int(n) + 3, v0))
        v0 += int(n) + 5
    parts.append(rng.integers(0, v0, (5000, 3)))                       # random faces, degenerate ones among them
    f = np.concatenate(parts)
    f = f[rng.permutation(len(f))]
    return (torch.from_numpy(rng.normal(size=(v0, 3)).astype(F32)).cuda(), torch.from_numpy(f).cuda(),
            torch.from_numpy(rng.uniform(size=(v0, 4)).astype(F32)).cuda())


def test_deterministic_streams_layouts_and_devices():
    v, f, c = _mesh()
    v0, f0, c0 = v.clone(), f.clone(), c.clone()
    want = MP.post_process_vectorised(v.cpu().numpy(), f.cpu().numpy(), c.cpu().numpy(), 100)
    a = _pp(v, f, c, cluster_to_keep=100)
    _check(a, want)
    b = _pp(v, f, c, cluster_to_keep=100)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32) if x.is_floating_point() else x,
                           y.view(torch.int32) if y.is_floating_point() else y)
    # inputs unmodified
    assert torch.equal(v.view(torch.int32), v0.view(torch.int32)) and torch.equal(f, f0)
    assert torch.equal(c.view(torch.int32), c0.view(torch.int32))
    # workspace and outputs in memory that held 0xFF, on a side stream
    junk = torch.full((4 << 30,), 255, dtype=torch.uint8, device="cuda")
    del junk
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out = _pp(v, f, c, cluster_to_keep=100)
    s.synchronize()
    _check(out, want)
    # int32 faces, non-contiguous inputs
    _check(_pp(v, f.to(torch.int32), c, cluster_to_keep=100), want)
    vn = torch.empty((v.shape[0], 5), device="cuda")[:, 1:4]
    vn.copy_(v)
    fn = f.t().contiguous().t()
    cn = c.t().contiguous().t()
    assert not (vn.is_contiguous() or fn.is_contiguous() or cn.is_contiguous())
    _check(_pp(vn, fn, cn, cluster_to_keep=100), want)
    _check(_pp(v, f, cluster_to_keep=np.int64(100)), want[:3] + (None,))
    if torch.cuda.device_count() > 1:
        out = _pp(v.to("cuda:1"), f.to("cuda:1"), c.to("cuda:1"), cluster_to_keep=100)
        assert all(t.device == torch.device("cuda:1") for t in out)
        _check(out, want)


def test_rejected_arguments():
    v, f = torch.zeros(10, 3, device="cuda"), torch.tensor([[0, 1, 2]] * 60, device="cuda")
    for bad in (dict(verts=v.cpu()), dict(faces=f.cpu()), dict(colors=torch.zeros(10, 3))):
        args = dict(verts=v, faces=f, colors=None) | bad
        with pytest.raises(RuntimeError, match="CUDA tensor"):
            _pp(**args)
    for bad in (dict(verts=v.double()), dict(verts=v[:, :2]), dict(verts=v.view(-1)), dict(faces=f.float()),
                dict(faces=f.to(torch.int16)), dict(faces=f[:, :2]), dict(colors=torch.zeros(9, 3, device="cuda")),
                dict(colors=torch.zeros(10, device="cuda"))):
        args = dict(verts=v, faces=f, colors=None) | bad
        with pytest.raises(RuntimeError):
            _pp(**args)
    for k in (1.0, True, None, "1"):
        with pytest.raises(RuntimeError, match="integer"):
            _pp(v, f, cluster_to_keep=k)
    big_v = torch.zeros(1, 3, device="cuda").expand(1 << 31, 3)
    with pytest.raises(RuntimeError, match="2\\^31"):
        _pp(big_v, f)
    big_f = torch.zeros(1, 3, dtype=torch.int64, device="cuda").expand(((1 << 30) - 1) // 3 + 1, 3)
    with pytest.raises(RuntimeError, match="2\\^30"):
        _pp(v, big_f)
    if torch.cuda.device_count() > 1:
        with pytest.raises(RuntimeError, match="are on"):
            _pp(v, f.to("cuda:1"))
    # a face index outside [0, M): rejected before any index addresses memory, with no output
    for bad in (10, -1, 1 << 40):
        fb = f.clone()
        fb[37, 1] = bad
        with pytest.raises(RuntimeError, match="outside"):
            _pp(v, fb)
        ids, counts, flag = _clusters_c_abi(10, fb)
        assert flag == 1
