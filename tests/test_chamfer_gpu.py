"""DTU Chamfer evaluation on the device (csrc/chamfer.cu, DESIGN.md §7m): `sample_mesh` and `dtu_chamfer` against the
reference's recorded eval.py runs (tests/golden/ref_chamfer.npz) bit for bit, stress scenes against the restatement
tests/chamfer_ref.py, the greedy set and the 1-NN distances checked directly at about a million points,
determinism, a side stream, unchanged inputs and rejected arguments."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import chamfer_ref as CR
from test_chamfer_cpu import case, case_names, close, golden, same

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _ch():
    from diff_surfel_rasterization import chamfer
    return chamfer


def _t(a, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


def _np(t):
    return t.detach().cpu().numpy()


def run_gpu(c):
    ch = _ch()
    thresh, patch, md, vis = (float(x) for x in c["args"])
    if str(c["mode"]) == "mesh":
        pcd = ch.sample_mesh(_t(c["verts"]), _t(c["faces"], torch.int64), density=thresh)
    else:
        pcd = _t(c["pcd_in"])
    r = ch.dtu_chamfer(pcd, _t(c["stl"]), _t(c["obs"], torch.bool), c["bb"], c["res"], c["plane"],
                       perm=_t(c["perm"], torch.int64), downsample_density=thresh, patch_size=patch, max_dist=md,
                       visualize_threshold=vis)
    return pcd, r


@pytest.mark.parametrize("name", case_names(np.load(__import__("test_chamfer_cpu").GOLDEN))
                         if __import__("os").path.exists(__import__("test_chamfer_cpu").GOLDEN) else [])
def test_golden(name):
    c = case(golden(), name)
    if str(c["error"]):
        with pytest.raises(ValueError):
            run_gpu(c)
        return
    pcd, r = run_gpu(c)
    md = float(c["args"][2])
    assert same(_np(pcd), c["pcd"]), "samples"
    assert same(_np(r.data_down), c["d2s_points"]), "data_down"
    assert same(_np(r.data_color), c["d2s_colors"]), "d2s colours"
    assert same(_np(r.stl_color), c["s2d_colors"]), "s2d colours"
    for got, k in ((r.dist_d2s, 0), (r.dist_s2d, 1)):
        ref = c[f"knn{k}_dist"]
        assert same(_np(got), np.where(ref < md, ref, np.inf)), f"pass {k}"
    res = c["results"]
    assert close(r.mean_d2s, res[0]) and close(r.mean_s2d, res[1]) and close(r.overall, res[2])
    assert r.rounds >= 1


def _scene(pcd, stl, perm, thresh=0.2, md=20.0, vis=10.0):
    lo = np.minimum(pcd.min(0), stl.min(0)) - 1
    hi = np.maximum(pcd.max(0), stl.max(0)) + 1
    bb = np.stack([lo, hi])
    shape = tuple(int(x) for x in np.ceil((hi - lo) / 1.0) + 1)
    obs = np.ones(shape, bool)
    plane = np.array([0.0, 0.0, 0.0, 1.0])                       # every STL point above
    return bb, 1.0, plane, obs


def _compare(pcd, stl, thresh=0.2, md=20.0, vis=10.0, seed=0):
    perm = np.random.default_rng(seed).permutation(len(pcd))
    bb, res, plane, obs = _scene(pcd, stl, perm)
    want = CR.evaluate(pcd, stl, obs, bb, res, plane, perm, thresh, 60.0, md, vis)
    r = _ch().dtu_chamfer(_t(pcd), _t(stl), _t(obs, torch.bool), bb, res, plane, perm=_t(perm, torch.int64),
                          downsample_density=thresh, max_dist=md, visualize_threshold=vis)
    assert same(_np(r.data_down), want["data_down"])
    assert same(_np(r.dist_d2s), want["dist_d2s"])
    assert same(_np(r.dist_s2d), want["dist_s2d"])
    assert same(_np(r.data_color), want["data_color"])
    assert same(_np(r.stl_color), want["stl_color"])
    assert close(r.mean_d2s, want["mean_d2s"]) and close(r.mean_s2d, want["mean_s2d"])
    return r


def test_thousands_of_copies():
    rng = np.random.default_rng(1)
    pcd = np.concatenate([np.tile([[1.0, 2.0, 3.0]], (5000, 1)), rng.uniform(0, 4, (3000, 3))])
    stl = rng.uniform(0, 4, (2000, 3))
    r = _compare(pcd, stl)
    assert r.rounds <= 64


def test_one_triangle():
    v = np.array([[0, 0, 0], [3, 0, 0], [0.5, 2, 0.3]], np.float64)
    pcd = _ch().sample_mesh(_t(v), _t([[0, 1, 2]], torch.int64))
    assert same(_np(pcd), CR.sample_mesh(v, [[0, 1, 2]], 0.2))
    rng = np.random.default_rng(2)
    _compare(_np(pcd), rng.uniform(0, 3, (500, 3)))


def test_large_triangle():
    # n1 * n2 of about 9e6: about 4.5 M samples from one triangle, written by one warp
    v = np.array([[0, 0, 0], [600, 0, 0], [0, 600, 1.0], [5, 5, 5], [6, 5, 5], [5, 6, 5]], np.float64)
    f = np.array([[3, 4, 5], [0, 1, 2], [3, 5, 4]])
    got = _np(_ch().sample_mesh(_t(v), _t(f, torch.int64)))
    want = CR.sample_mesh(v, f, 0.2)
    assert len(want) > 4_000_000
    assert same(got, want)


def test_greedy_and_nn_characterisation_at_a_million_points():
    rng = np.random.default_rng(3)
    n = 1_000_000
    pcd = rng.uniform(0, 40, (n, 3)) * [1, 1, 0.05]               # a slab: about 30 neighbours within r each
    stl = rng.uniform(0, 40, (400_000, 3)) * [1, 1, 0.05] + [0, 0, 0.3]
    perm = rng.permutation(n)
    r = 0.2
    bb, res, plane, obs = _scene(pcd, stl, perm)
    out = _ch().dtu_chamfer(_t(pcd), _t(stl), _t(obs, torch.bool), bb, res, plane, perm=_t(perm, torch.int64),
                            max_dist=0.5)
    x = pcd[perm]
    pairs = CR.neighbour_pairs(x, r)
    # recover the kept mask from data_down (rows keep the shuffled order)
    down = _np(out.data_down)
    kept = np.zeros(n, bool)
    pos = {tuple(p): i for i, p in enumerate(x)}
    idx = np.array([pos[tuple(p)] for p in down])
    assert np.all(np.diff(idx) > 0)
    kept[idx] = True
    i, j = pairs[:, 0], pairs[:, 1]
    assert not (kept[i] & kept[j]).any(), "two kept points are neighbours"
    has_kept_earlier = np.zeros(n, bool)
    has_kept_earlier[j[kept[i]]] = True
    assert np.array_equal(~kept, has_kept_earlier), "a removed point without an earlier kept neighbour"
    # 1-NN: each distance below max_dist is the exact rule at some point and no larger than the exact nearest
    q = down
    d = _np(out.dist_d2s)
    dk, ik = cKDTree(stl).query(q, k=1)
    exact = np.sqrt(CR.rdist(q, stl[ik]))
    fin = np.isfinite(d)
    assert np.all(d[fin] <= exact[fin])
    assert np.all(exact[~fin] >= 0.5 * (1 - 1e-12))
    assert np.all(d[fin] < 0.5)
    t = cKDTree(stl)
    cand = t.query_ball_point(q[fin][:2000], d[fin][:2000] * (1 + 1e-9))
    for row, c in zip(np.nonzero(fin)[0][:2000], cand):
        assert np.sqrt(CR.rdist(q[row][None], stl[c]).min()) == d[row]
    print("greedy rounds at 1 M points:", out.rounds)


def _small():
    c = case(golden(), "bumpy")
    return c


def test_two_calls_bit_identical_and_inputs_unchanged():
    c = _small()
    verts, faces, stl = _t(c["verts"]), _t(c["faces"], torch.int64), _t(c["stl"])
    keep = [verts.clone(), faces.clone(), stl.clone()]
    a = _ch().sample_mesh(verts, faces)
    b = _ch().sample_mesh(verts, faces)
    assert torch.equal(a, b)
    perm = _t(c["perm"], torch.int64)
    obs = _t(c["obs"], torch.bool)
    r1 = _ch().dtu_chamfer(a, stl, obs, c["bb"], c["res"], c["plane"], perm=perm)
    r2 = _ch().dtu_chamfer(a, stl, obs, c["bb"], c["res"], c["plane"], perm=perm)
    for f in ("data_down", "data_color", "stl_color", "dist_d2s", "dist_s2d"):
        assert same(_np(getattr(r1, f)), _np(getattr(r2, f)))
    assert r1.mean_d2s == r2.mean_d2s and r1.mean_s2d == r2.mean_s2d
    for x, y in zip(keep, (verts, faces, stl)):
        assert torch.equal(x, y)
    # float32 inputs widen exactly; uint8 mask and int32 faces are accepted
    v32 = verts.float()
    assert torch.equal(_ch().sample_mesh(v32, faces.int()), _ch().sample_mesh(v32.double(), faces))
    r3 = _ch().dtu_chamfer(a, stl, obs.to(torch.uint8), c["bb"], c["res"], c["plane"], perm=perm.int())
    assert r3.mean_d2s == r1.mean_d2s


def test_generator_draws_the_permutation():
    c = _small()
    pcd, stl, obs = _t(c["pcd"]), _t(c["stl"]), _t(c["obs"], torch.bool)
    g1 = torch.Generator(device=DEV).manual_seed(5)
    g2 = torch.Generator(device=DEV).manual_seed(5)
    r1 = _ch().dtu_chamfer(pcd, stl, obs, c["bb"], c["res"], c["plane"], generator=g1)
    r2 = _ch().dtu_chamfer(pcd, stl, obs, c["bb"], c["res"], c["plane"], generator=g2)
    assert same(_np(r1.data_down), _np(r2.data_down))


def test_side_stream():
    c = _small()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        pcd = _ch().sample_mesh(_t(c["verts"]), _t(c["faces"], torch.int64))
        r = _ch().dtu_chamfer(pcd, _t(c["stl"]), _t(c["obs"], torch.bool), c["bb"], c["res"], c["plane"],
                              perm=_t(c["perm"], torch.int64))
    s.synchronize()
    assert same(_np(r.data_down), c["d2s_points"])
    assert close(r.overall, c["results"][2])


def test_rejects_bad_arguments():
    ch = _ch()
    c = _small()
    v, f = _t(c["verts"]), _t(c["faces"], torch.int64)
    with pytest.raises(ValueError):
        ch.sample_mesh(v, f.clone().fill_(-1))
    with pytest.raises(ValueError):
        ch.sample_mesh(v, f + len(v))
    bad = v.clone()
    bad[3, 1] = math.nan
    with pytest.raises(ValueError):
        ch.sample_mesh(bad, f)
    with pytest.raises(TypeError):
        ch.sample_mesh(v.cpu(), f)
    with pytest.raises(ValueError):
        ch.sample_mesh(v[:, :2], f)
    pcd, stl, obs = _t(c["pcd"]), _t(c["stl"]), _t(c["obs"], torch.bool)
    args = (obs, c["bb"], c["res"], c["plane"])
    perm = _t(c["perm"], torch.int64)
    for p in (perm.clone().fill_(0), perm - 1, perm[:-1]):
        with pytest.raises(ValueError):
            ch.dtu_chamfer(pcd, stl, *args, perm=p)
    inf = stl.clone()
    inf[0, 0] = math.inf
    with pytest.raises(ValueError):
        ch.dtu_chamfer(pcd, inf, *args, perm=perm)
    with pytest.raises(ValueError):
        ch.dtu_chamfer(pcd, stl[:0], *args, perm=perm)
    with pytest.raises(ValueError):
        ch.dtu_chamfer(pcd, stl, obs, c["bb"][:1], c["res"], c["plane"], perm=perm)
    with pytest.raises(ValueError):
        ch.dtu_chamfer(pcd, stl, obs.float(), c["bb"], c["res"], c["plane"], perm=perm)
