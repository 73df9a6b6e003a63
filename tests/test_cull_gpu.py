"""DTU mask culling on the device (csrc/cull.cu, DESIGN.md §7n): `cull_scan` against the reference's recorded runs
(tests/golden/ref_cull.npz) with the bars of test_cull_cpu.py, the dilation against scipy at DTU size, a DTU-size
scene against the reference's torch lines on this GPU (cuBLAS and grid_sample), outputs bit-identical to the
restatement tests/cull_ref.py given the same projections, input dtypes, colours, repeat calls, a side stream,
unchanged inputs, rejected arguments, and one chained run into sample_mesh and dtu_chamfer."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cull_ref as CR
from test_cull_cpu import GOLDEN, IMAGE, NAMES, case, golden, ref_dilated, ref_keep, same, same64

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _ch():
    from diff_surfel_rasterization import chamfer
    return chamfer


def _t(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).to(DEV)
    return t if dtype is None else t.to(dtype)


def _np(t):
    return t.detach().cpu().numpy()


def unpack(bits, W):
    """(N, H, ceil(W/32)) int32 words -> (N, H, W) bool; pixel x in bit x % 32 of word x / 32."""
    b = _np(bits).view(np.uint32)
    x = np.arange(W)
    return ((b[..., x // 32] >> (x % 32).astype(np.uint32)) & 1).astype(bool)


def run_case(c, proj=None, **kw):
    ch = _ch()
    colors = _t(c["colors"]) if "colors" in c else None
    masks = _t(c["masks"])
    if proj is None:
        proj = ch.dtu_projections(c["world_mats"], c["scale_mats"])
    return ch._cull("test", _t(c["verts"]), _t(c["faces"]), masks, proj, c["scale_mats"], colors, IMAGE,
                    int(c["radius"]))


@pytest.mark.parametrize("name", NAMES)
def test_golden(name):
    c = case(golden(), name)
    r = run_case(c)
    W = c["masks"].shape[2]
    assert np.array_equal(unpack(r["dilated"], W), ref_dilated(c)), "dilated masks"
    keep = ref_keep(c)
    mine = _np(r["keep"])
    if str(c["kind"]) == "exact":
        assert np.array_equal(mine, keep), "decisions"
        assert same64(_np(r["verts"]), c["out_verts"]) and same(_np(r["faces"]), c["out_faces"])
        if "colors" in c:
            assert same(_np(r["colors"]), c["out_colors"])
        else:
            assert r["colors"] is None
        return
    differ = np.flatnonzero(mine != keep)
    # the device forms A itself (within 1e-6 of each row's scale of the reference's) and orders the dot products
    tie = CR.near_tie(c["verts"][differ], c["A"][:, :3], IMAGE, c["masks"].shape[1:], a_rel=1e-6)
    assert tie.any(0).all(), f"{int((~tie.any(0)).sum())} of {len(differ)} differing decisions are not near a tie"
    print(f"{name}: {len(differ)} of {len(keep)} decisions differ from the reference, all within rule 3's bound")
    # with the recorded A: bit for bit against the restatement
    r2 = run_case(c, proj=c["A"][:, :3])
    ref = CR.cull(c["verts"], c["faces"], c["masks"], c["A"][:, :3], c["scale_mats"], c.get("colors"), IMAGE,
                  int(c["radius"]))
    assert np.array_equal(_np(r2["keep"]), ref["keep"])
    assert same64(_np(r2["verts"]), ref["verts"]) and same(_np(r2["faces"]), ref["faces"])


def test_dilation_matches_scipy_at_dtu_size():
    import scipy.ndimage as ndi
    rng = np.random.default_rng(11)
    H, W = 1200, 1600
    masks = np.zeros((3, H, W), np.uint8)
    masks[0, 300:900, 400:1200] = (rng.random((600, 800)) < 0.002) * 255
    masks[0, [100, 1199, 0], [5, 1599, 800]] = 1
    yy, xx = np.mgrid[0:H, 0:W]
    masks[1] = (((yy - 500) / 300.0) ** 2 + ((xx - 900) / 500.0) ** 2 <= 1) * 255
    masks[1] |= (rng.random((H, W)) < 0.0003).astype(np.uint8)
    masks[2] = (rng.random((H, W)) < 0.00005).astype(np.uint8) * 7
    ch = _ch()
    proj = np.zeros((3, 3, 4), np.float32)
    r = ch._cull("test", torch.zeros((0, 3), device=DEV), torch.zeros((0, 3), dtype=torch.int64, device=DEV),
                 _t(masks), proj, np.eye(4)[None].repeat(3, 0), None, IMAGE, 24)
    got = unpack(r["dilated"], W)
    for k in range(3):
        ref = ndi.binary_dilation(masks[k] != 0, structure=CR.disk(24), border_value=0)
        assert np.array_equal(got[k], ref), k
    assert r["verts"].shape == (0, 3) and r["faces"].shape == (0, 3)


def _dtu_scene(rng, views=49, n_verts=2_000_000):
    """A DTU-size scene: 49 cameras around a blob surface, 1600 x 1200 masks, about 2 M vertices in mesh order
    (a triangulated sphere-like height field) and its faces."""
    from test_cull_cpu import case as _case
    g = golden()
    world0, scale0 = _case(g, "dtu_size")["world_mats"], _case(g, "dtu_size")["scale_mats"]
    K = np.array([[2892.33, 0.0, 823.205], [0.0, 2883.18, 619.07], [0.0, 0.0, 1.0]])
    S = scale0[0]
    world = []
    for k in range(views):
        th, ph = 2 * np.pi * k / views, 0.3 + 0.6 * ((k * 7) % views) / views
        c = 2.5 * np.array([np.cos(th) * np.sin(ph), np.sin(th) * np.sin(ph), -np.cos(ph)])
        f = -c / np.linalg.norm(c)
        r0 = np.cross([0.0, 1.0, 0.1], f)
        r0 /= np.linalg.norm(r0)
        R = np.stack([r0, np.cross(f, r0), f])
        Cw = S[:3, :3] @ c + S[:3, 3]
        Wm = np.eye(4)
        Wm[:3, :4] = (0.5 if k % 2 else -0.5) * K @ np.hstack([R, -R @ Cw[:, None]])
        world.append(Wm)
    world, scale = np.array(world), np.array([S] * views)
    side = int(np.sqrt(n_verts))
    u, v = np.meshgrid(np.linspace(0, np.pi, side), np.linspace(0, 2 * np.pi, side), indexing="ij")
    rad = 0.6 + 0.1 * np.sin(5 * u) * np.cos(3 * v)
    verts = np.stack([rad * np.sin(u) * np.cos(v), rad * np.sin(u) * np.sin(v), rad * np.cos(u)], -1).reshape(-1, 3)
    idx = np.arange(side * side).reshape(side, side)
    a, b, cc, d = idx[:-1, :-1].ravel(), idx[1:, :-1].ravel(), idx[:-1, 1:].ravel(), idx[1:, 1:].ravel()
    faces = np.concatenate([np.stack([a, b, cc], 1), np.stack([b, d, cc], 1)])
    # masks: each view's silhouette of a smaller blob, so that culling bites
    proj = CR.projections(world, scale).astype(np.float64)
    H, W = 1200, 1600
    masks = np.zeros((views, H, W), np.uint8)
    pts = verts[::37] * 0.85
    for k in range(views):
        c = proj[k] @ np.hstack([pts, np.ones((len(pts), 1))]).T
        px, py = np.rint(c[0] / c[2]).astype(int), np.rint(c[1] / c[2]).astype(int)
        ok = (px >= 0) & (px < W) & (py >= 0) & (py < H)
        masks[k, py[ok], px[ok]] = 255
    return verts, faces, masks, world, scale


def torch_lines(verts, A, D, image_size):
    """The reference's vertex test (evaluate_single_scene.py:61-88) on this GPU: cuBLAS for A @ V and grid_sample,
    view by view, with the dilated masks D (N, H, W) given."""
    W, H = image_size
    V = torch.cat((verts, torch.ones_like(verts[:, :1])), dim=-1).permute(1, 0).float()
    keep = torch.ones(verts.shape[0], dtype=torch.bool, device=verts.device)
    for i in range(A.shape[0]):
        cam_points = A[i] @ V
        pix_coords = cam_points[:2, :] / (cam_points[2, :].unsqueeze(0) + 1e-6)
        pix_coords = pix_coords.permute(1, 0)
        pix_coords[..., 0] /= W - 1
        pix_coords[..., 1] /= H - 1
        pix_coords = (pix_coords - 0.5) * 2
        valid = ((pix_coords > -1.) & (pix_coords < 1.)).all(dim=-1).float()
        sampled = F.grid_sample(D[i].float()[None, None], pix_coords[None, None], mode='nearest',
                                padding_mode='zeros', align_corners=True)[0, -1, 0]
        keep &= (sampled + (1. - valid)) > 0.
    return keep


def test_dtu_size_against_torch_lines():
    rng = np.random.default_rng(5)
    verts, faces, masks, world, scale = _dtu_scene(rng)
    ch = _ch()
    A = ch.dtu_projections(world, scale)
    v, f, m = _t(verts), _t(faces), _t(masks)
    r = ch._cull("test", v, f, m, A, scale, None, IMAGE, 24)
    D = torch.from_numpy(unpack(r["dilated"], 1600)).to(DEV)
    A4 = torch.zeros((len(A), 4, 4), dtype=torch.float32, device=DEV)
    A4[:, :3] = torch.from_numpy(A).to(DEV)
    A4[:, 3, 3] = 1
    ref = _np(torch_lines(v, A4, D, IMAGE))
    mine = _np(r["keep"])
    differ = np.flatnonzero(mine != ref)
    tie = CR.near_tie(verts[differ], A, IMAGE, masks.shape[1:])
    assert tie.any(0).all(), f"{int((~tie.any(0)).sum())} of {len(differ)} differing decisions are not near a tie"
    print(f"DTU size ({len(A)} views, {len(verts)} vertices, {int(mine.sum())} kept): {len(differ)} decisions differ "
          f"from the torch lines, all within rule 3's bound")
    assert 0 < mine.sum() < len(mine)
    fk = mine[faces].all(1)
    assert r["faces"].shape[0] == int(fk.sum()) and r["verts"].shape[0] == int(mine.sum())


def _random_case(rng, M=200_000, views=8, shape=(300, 400), radius=6):
    """Cameras of the golden's dtu_size case, random blob masks of another shape and random vertices."""
    g = golden()
    c = case(g, "dtu_size")
    world = np.concatenate([c["world_mats"]] * 3)[:views]
    scale = np.concatenate([c["scale_mats"]] * 3)[:views]
    H, W = shape
    yy, xx = np.mgrid[0:H, 0:W]
    masks = np.zeros((views, H, W), np.uint8)
    for k in range(views):
        for _ in range(3):
            cy, cx, ry, rx = rng.uniform(0, H), rng.uniform(0, W), rng.uniform(20, 120), rng.uniform(20, 160)
            masks[k][((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1] = 255
    verts = rng.normal(size=(M, 3)) * 0.4
    faces = rng.integers(0, M - 50, (M, 3))
    colors = rng.integers(0, 256, (M, 3)).astype(np.uint8)
    return verts, faces, masks, world, scale, colors, radius


def test_outputs_match_restatement_given_the_same_projections():
    rng = np.random.default_rng(8)
    verts, faces, masks, world, scale, colors, radius = _random_case(rng)
    ch = _ch()
    A = ch.dtu_projections(world, scale)
    ref = CR.cull(verts, faces, masks, A, scale, colors, IMAGE, radius)
    for vd, fd, cd in ((torch.float64, torch.int64, torch.uint8), (torch.float32, torch.int32, torch.float32),
                       (torch.float64, torch.int32, torch.int16)):
        v = _t(verts, vd)
        f = _t(faces, fd)
        col = _t(colors, cd)
        ref_v = CR.cull(_np(v), faces, masks, A, scale, None, IMAGE, radius) if vd == torch.float32 else ref
        r = ch._cull("test", v, f, _t(masks), A, scale, col, IMAGE, radius)
        assert np.array_equal(unpack(r["dilated"], masks.shape[2]), ref["dilated"])
        assert np.array_equal(_np(r["keep"]), ref_v["keep"])
        assert same64(_np(r["verts"]), ref_v["verts"]) and same(_np(r["faces"]), ref_v["faces"])
        assert r["colors"].dtype == cd and np.array_equal(_np(r["colors"]), colors[ref_v["keep"]].astype(
            _np(col).dtype))
    # the public call forms the same A
    out_v, out_f, out_c = ch.cull_scan(_t(verts), _t(faces), _t(masks), world, scale, colors=_t(colors),
                                       image_size=IMAGE, radius=radius)
    assert same64(_np(out_v), ref["verts"]) and same(_np(out_f), ref["faces"]) and same(_np(out_c), ref["colors"])
    # bool masks, tensor cameras
    out2 = ch.cull_scan(_t(verts), _t(faces), _t(masks != 0), torch.from_numpy(world), torch.from_numpy(scale),
                        image_size=IMAGE, radius=radius)
    assert same64(_np(out2[0]), ref["verts"]) and same(_np(out2[1]), ref["faces"]) and out2[2] is None


def test_repeat_side_stream_and_unchanged_inputs():
    rng = np.random.default_rng(9)
    verts, faces, masks, world, scale, colors, radius = _random_case(rng, M=300_000)
    ch = _ch()
    v, f, m, col = _t(verts), _t(faces), _t(masks), _t(colors)
    copies = [x.clone() for x in (v, f, m, col)]
    first = ch.cull_scan(v, f, m, world, scale, colors=col, radius=radius)
    again = ch.cull_scan(v, f, m, world, scale, colors=col, radius=radius)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        side = ch.cull_scan(v, f, m, world, scale, colors=col, radius=radius)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for out in (again, side):
        for a, b in zip(first, out):
            assert torch.equal(a, b)
    for a, b in zip(copies, (v, f, m, col)):
        assert torch.equal(a, b)
    assert first[0].shape[0] > 0 and first[1].dtype == torch.int64 and first[0].dtype == torch.float64


def test_rejects_bad_arguments():
    ch = _ch()
    c = case(golden(), "dyadic")
    v, f, m = _t(c["verts"]), _t(c["faces"]), _t(c["masks"])
    w, s = c["world_mats"], c["scale_mats"]
    bad = f.clone()
    bad[3, 1] = v.shape[0]
    with pytest.raises(ValueError, match="outside"):
        ch.cull_scan(v, bad, m, w, s)
    bad[3, 1] = -1
    with pytest.raises(ValueError, match="outside"):
        ch.cull_scan(v, bad, m, w, s)
    for x in (float("nan"), float("inf"), 1e39):
        vv = v.clone()
        vv[5, 2] = x
        with pytest.raises(ValueError, match="finite"):
            ch.cull_scan(vv, f, m, w, s)
    with pytest.raises(ValueError, match="masks and"):
        ch.cull_scan(v, f, m[:1], w, s)
    with pytest.raises(ValueError):
        ch.cull_scan(v, f, m.float(), w, s)
    with pytest.raises(ValueError):
        ch.cull_scan(v, f, m, w, s, radius=-1)
    with pytest.raises(ValueError):
        ch.cull_scan(v, f, m, w, s, radius=2.5)
    with pytest.raises(ValueError):
        ch.cull_scan(v, f, m, w, s, image_size=(0, 10))
    with pytest.raises(ValueError):
        ch.cull_scan(v, f, m, w, s, colors=_t(c["colors"])[:-1])
    with pytest.raises(ValueError):
        ch.cull_scan(v[:, :2], f, m, w, s)
    with pytest.raises(TypeError):
        ch.cull_scan(v.cpu(), f, m, w, s)
    with pytest.raises(ValueError):
        ch.cull_scan(v, f.float(), m, w, s)
    with pytest.raises(ValueError):
        ch.cull_scan(v, f, torch.zeros((2, 40000, 4), dtype=torch.uint8, device=DEV), w, s)
    # nothing was changed by the failed calls
    assert torch.equal(v, _t(c["verts"])) and torch.equal(f, _t(c["faces"]))


def test_chain_into_chamfer():
    """cull_scan -> sample_mesh -> dtu_chamfer: the stages compose on device tensors."""
    ch = _ch()
    c = case(golden(), "dtu_size")
    rng = np.random.default_rng(4)
    # a watertight-ish mesh: a height field over the blob, culled by the golden's masks
    n = 120
    X, Y = np.meshgrid(np.linspace(-0.6, 0.6, n), np.linspace(-0.6, 0.6, n), indexing="ij")
    Z = 0.1 * np.sin(4 * X) * np.cos(3 * Y)
    verts = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)
    idx = np.arange(n * n).reshape(n, n)
    a, b, cc, d = idx[:-1, :-1].ravel(), idx[1:, :-1].ravel(), idx[:-1, 1:].ravel(), idx[1:, 1:].ravel()
    faces = np.concatenate([np.stack([a, b, cc], 1), np.stack([b, d, cc], 1)])
    out_v, out_f, _ = ch.cull_scan(_t(verts), _t(faces), _t(c["masks"]), c["world_mats"], c["scale_mats"])
    assert 0 < out_f.shape[0] < faces.shape[0]
    pcd = ch.sample_mesh(out_v, out_f, density=2.0)
    pts = _np(pcd)
    stl = pts[rng.choice(len(pts), min(len(pts), 20000), replace=False)] + rng.normal(size=(min(len(pts), 20000), 3))
    lo, hi = pts.min(0) - 5, pts.max(0) + 5
    res = 4.0
    shape = tuple(int(x) for x in np.ceil((hi - lo) / res) + 1)
    r = ch.dtu_chamfer(pcd, _t(stl), torch.ones(shape, dtype=torch.bool, device=DEV), np.stack([lo, hi]), res,
                       np.array([0.0, 0.0, 0.0, 1.0]), downsample_density=2.0)
    assert np.isfinite(r.overall) and r.overall > 0
    print(f"chain: {out_v.shape[0]} vertices, {out_f.shape[0]} faces kept, {pcd.shape[0]} samples, "
          f"overall {r.overall:.4f}")
