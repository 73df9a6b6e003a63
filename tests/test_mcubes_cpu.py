"""Device marching cubes without a device (DESIGN.md §7j): the committed table against its generator, the table's
polygons, orientation and face agreement, the NumPy restatement on analytic volumes (closed oriented 2-manifolds,
vertices within the float64 bound, exact zeros, near-coincident vertices), the reference's recorded structure, and
the C ABI's argument checks."""
import ctypes
import itertools
import os
import types

import numpy as np
import pytest

import mcubes_ref as MR
from diff_surfel_rasterization import mcubes_table as T

F = np.float32
U = 2.0 ** -24
TABLE, COUNT = T.generate()
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_mcubes.npz")


def test_committed_table_is_the_generators_output():
    with open(T.INC) as f:
        assert f.read() == T.render()


def _crossing(case):
    return {e for e in range(12) if (case >> T.EDGE_CORNERS[e][0] & 1) != (case >> T.EDGE_CORNERS[e][1] & 1)}


def _boundary(tris):
    """Directed boundary segments of a set of triangles (interior diagonals cancel)."""
    seg = {}
    for t in tris:
        for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            if (b, a) in seg:
                del seg[(b, a)]
            else:
                assert (a, b) not in seg
                seg[(a, b)] = True
    return list(seg)


def _face_of(a, b):
    fs = [f for f in T.FACES if a in T.FACE_EDGES[f] and b in T.FACE_EDGES[f]]
    assert len(fs) == 1, (a, b)
    return fs[0]


@pytest.mark.parametrize("case", range(256))
def test_every_case_is_closed_polygons_on_crossing_edges_and_oriented(case):
    table, count = TABLE, COUNT
    tris = [tuple(int(e) for e in r) for r in table[case, :count[case]]]
    cross = _crossing(case)
    used = {e for t in tris for e in t}
    assert used == cross
    seg = _boundary(tris)
    # every crossing edge has one segment in and one out, and each segment lies on one cube face
    assert sorted(a for a, _ in seg) == sorted(cross) == sorted(b for _, b in seg)
    for a, b in seg:
        _face_of(a, b)
    # oriented: no triangle's normal points against the inside -> outside direction of its edges (the field
    # increases through the surface towards free space), and the case's triangles together point along it
    total = 0.0
    for t in tris:
        A, B, C = (T.edge_midpoint(e) for e in t)
        nrm = np.cross(B - A, C - A)
        flux = 0.0
        for e in t:
            lo, hi = T.EDGE_CORNERS[e]
            step = T.CORNERS[hi] - T.CORNERS[lo]
            flux += np.dot(nrm, step if case >> lo & 1 else -step)
        assert flux >= 0, (case, t)
        total += flux
    assert total > 0 or not tris


def _face_segments(case, face):
    """The boundary segments of `case` on `face`, as directed pairs of face-local edge slots."""
    table, count = TABLE, COUNT
    tris = [tuple(int(e) for e in r) for r in table[case, :count[case]]]
    d = face[0]
    local = lambda e: (T.EDGE_AXIS[e], tuple(int(x) for x in np.delete(T.edge_midpoint(e), d)))
    return {(local(a), local(b)) for a, b in _boundary(tris) if _face_of(a, b) == face}


def test_cases_that_share_a_face_pair_it_the_same_way():
    for d in range(3):
        lo_face, hi_face = (d, 0), (d, 1)
        for a, b in itertools.product(range(256), range(256)):
            # cube a below cube b along d: a's upper face is b's lower face
            sa = [a >> c & 1 for c in T.FACE_CORNERS[hi_face]]
            sb = [b >> c & 1 for c in T.FACE_CORNERS[lo_face]]
            if sa != sb or b % 17:          # every a, a sample of the b that match it
                continue
            ua, ub = _face_segments(a, hi_face), _face_segments(b, lo_face)
            # the same segments, walked in opposite directions: the mesh is closed and consistently oriented
            assert ua == {(y, x) for x, y in ub}, (d, a, b)


# ---- the restatement on analytic volumes ----------------------------------------------------------------------------

def sphere(r, c=(0.0, 0.0, 0.0)):
    return lambda X, Y, Z: np.sqrt((X - F(c[0])) ** 2 + (Y - F(c[1])) ** 2 + (Z - F(c[2])) ** 2) - F(r)


def torus(R0, r):
    return lambda X, Y, Z: np.sqrt((np.sqrt(X * X + Y * Y) - F(R0)) ** 2 + Z * Z) - F(r)


def _run(fn, n, side, R=1.0):
    xs = MR.crop_bounds(R, n)
    return MR.mesh(n, side, xs, MR.analytic(fn)), xs


def check_closed_oriented(faces, n_verts, euler):
    f = np.asarray(faces)
    assert len(f) > 0
    assert (f[:, 0] != f[:, 1]).all() and (f[:, 1] != f[:, 2]).all() and (f[:, 0] != f[:, 2]).all()
    directed = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    d = directed[:, 0] * n_verts + directed[:, 1]
    r = directed[:, 1] * n_verts + directed[:, 0]
    assert len(np.unique(d)) == len(d), "a directed edge is used twice: not oriented"
    assert np.array_equal(np.sort(d), np.sort(r)), "an edge has no opposite: not closed"
    E = len(d) // 2
    assert len(np.unique(f)) == n_verts
    assert n_verts - E + len(f) == euler


def _signed_volume(v, f):
    v = np.asarray(v, np.float64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6


def _global_axis(xs, side):
    axes = MR.crop_axes(xs, side)
    out = np.concatenate([a[:-1] for a in axes] + [axes[-1][-1:]])
    for i in range(1, len(axes)):         # neighbouring crops share their plane bit for bit
        assert axes[i - 1][-1].view(np.uint32) == axes[i][0].view(np.uint32)
    return out


def _check_positions_in_bound(fn, xs, side, pos, keys):
    g = _global_axis(xs, side)
    G = len(g)
    P, slot = keys // 4, keys % 4
    idx = np.stack([P // (G * G), P // G % G, P % G], 1)
    pa = g[idx].astype(np.float64)
    corner = slot == 3
    assert np.array_equal(pos[corner].astype(np.float64), pa[corner])
    e = ~corner
    d = slot[e]
    ib = idx[e].copy()
    ib[np.arange(len(d)), d] += 1
    pb = g[ib].astype(np.float64)
    va = np.asarray(fn(*g[idx[e]].T), F).astype(np.float64)
    vb = np.asarray(fn(*g[ib].T), F).astype(np.float64)
    assert ((va < 0) != (vb < 0)).all(), "a vertex off a sign-changing edge"
    t = va / (va - vb)
    exact = pa[e] + t[:, None] * (pb - pa[e])
    span = np.abs(pb - pa[e])
    bound = 4 * U * (span + np.abs(exact))
    assert (np.abs(pos[e] - exact) <= bound).all()


@pytest.mark.parametrize("n,side", [(1, 17), (2, 9), (3, 7)])
def test_sphere_is_a_closed_oriented_sphere(n, side):
    fn = sphere(0.61, (0.013, -0.021, 0.007))
    (verts, faces, pos, keys), xs = _run(fn, n, side)
    check_closed_oriented(faces, len(verts), 2)
    assert _signed_volume(pos, faces) > 0          # counter-clockwise seen from outside: normals point out
    _check_positions_in_bound(fn, xs, side, pos, keys)


@pytest.mark.parametrize("n,side", [(1, 25), (3, 9)])
def test_torus_is_a_closed_oriented_torus(n, side):
    fn = torus(0.55, 0.23)
    (verts, faces, pos, keys), xs = _run(fn, n, side)
    check_closed_oriented(faces, len(verts), 0)
    assert _signed_volume(pos, faces) > 0
    _check_positions_in_bound(fn, xs, side, pos, keys)


def test_crop_seams_do_not_change_the_mesh():
    """The same global grid cut into 1 or 3 crops per axis gives the same vertex keys and triangles; only the face
    order moves, and the positions by the last bits of the crops' own linspace axes."""
    fn = sphere(0.7)
    a, _ = _run(fn, 1, 19)
    b, _ = _run(fn, 3, 7)
    assert np.array_equal(a[3], b[3])
    assert np.abs(a[2].astype(np.float64) - b[2]).max() <= 1e-6
    ta = np.sort(np.sort(a[1], 1), 0)
    tb = np.sort(np.sort(b[1], 1), 0)
    assert np.array_equal(np.unique(ta, axis=0), np.unique(tb, axis=0))


def test_exact_zeros_vertex_count():
    """Planes through grid points and a sphere with a zero at grid corners: the vertex count is the crossing edges
    whose vertex is inside them plus the distinct corners where t is 0 or 1, counted over the global grid."""
    side, n = 9, 2
    xs = MR.crop_bounds(1.0, n)
    g = _global_axis(xs, side)
    fns = [lambda X, Y, Z: X - g[6], lambda X, Y, Z: np.where(Y >= g[9], F(0), F(-1)) + Z * F(0),
           lambda X, Y, Z: np.minimum(X - g[4], np.abs(Y - g[8]) - F(0.3)) + Z * F(0)]
    for fn in fns:
        verts, faces, pos, keys = MR.mesh(n, side, xs, MR.analytic(fn))
        X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
        V = np.asarray(fn(X, Y, Z), F)
        assert (V == 0).any()
        edges, corners = 0, set()
        G = len(g)
        for d in range(3):
            sa = [slice(None)] * 3
            sb = [slice(None)] * 3
            sa[d], sb[d] = slice(0, G - 1), slice(1, G)
            va, vb = V[tuple(sa)], V[tuple(sb)]
            cross = (va < 0) != (vb < 0)
            with np.errstate(all="ignore"):
                t = (va / (va - vb)).astype(F)
            edges += int((cross & (t != 0) & (t != 1)).sum())
            for which, m in ((0, cross & (t == 0)), (1, cross & (t == 1))):
                for p in zip(*np.nonzero(m)):
                    p = list(p)
                    p[d] += which
                    corners.add(tuple(p))
        assert len(verts) == edges + len(corners)
        assert len(corners) > 0


def test_near_coincident_vertices_are_reported():
    """Rule 5: distinct vertices within 1e-6 stay distinct.  On these scenes: counted, and reported."""
    reports = {}
    side, n = 9, 2
    xs = MR.crop_bounds(1.0, n)
    g = _global_axis(xs, side)
    scenes = {"sphere": sphere(0.61, (0.013, -0.021, 0.007)), "torus": torus(0.55, 0.23),
              "near_plane": lambda X, Y, Z: (X - g[6]) + (Y - g[4]) + F(3e-7) + Z * F(0)}
    for name, fn in scenes.items():
        verts, faces, pos, keys = MR.mesh(n, side, xs, MR.analytic(fn))
        reports[name] = MR.near_pairs(pos)
    print("near-coincident vertex pairs (within 1e-6, not merged):", reports)
    assert reports["sphere"] == 0 and reports["torus"] == 0
    assert reports["near_plane"] > 0


def test_linspace_halves_meet_at_the_ends():
    for R, n in ((0.3, 2), (1.23, 4), (1.9, 2)):
        xs = MR.crop_bounds(R, n)
        for a in MR.crop_axes(xs, 512):
            assert np.all(np.diff(a.astype(np.float64)) > 0)
        g = _global_axis(xs, 512)
        assert g[0] == F(-R) and g[-1] == F(R) and len(g) == 511 * n + 1


# ---- the reference's recorded structure (tests/golden/make_golden_mcubes.py) ------------------------------------------

def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("ref_mcubes.npz not generated")
    return np.load(GOLDEN)


def test_golden_crop_structure():
    g = _golden()
    R, N = float(g["R"]), int(g["resolution"])
    n = N // 512
    xs = MR.crop_bounds(R, n)
    assert np.array_equal(g["xs"], xs)
    ijk = [c for c in itertools.product(range(n), repeat=3)]
    assert np.array_equal(g["crops"], np.array(ijk))
    for c, (i, j, k) in enumerate(ijk):
        lo = np.array([xs[i], xs[j], xs[k]])
        hi = np.array([xs[i + 1], xs[j + 1], xs[k + 1]])
        if g["called"][c]:
            assert np.array_equal(g["offset"][c], lo)
            assert np.array_equal(g["spacing"][c], (hi - lo) / 511)
        # the reference builds each axis with torch.linspace on the host, then copies it to the device; this path
        # computes torch's CUDA linspace.  The two agree to one float32 ulp (the host kernel steps from its vector
        # base) - measured here, not assumed
        for d, v in enumerate((i, j, k)):
            want = MR.linspace32(xs[v], xs[v + 1], 512)
            got = g["axis"][c, d]
            assert got[0] == want[0] and got[-1] == want[-1]
            assert np.all(np.abs(got.view(np.int32) - want.view(np.int32)) <= 1)
    # the reference's skip rule: marching cubes runs on a crop iff its values straddle 0 (min <= 0 <= max)
    assert np.array_equal(g["called"], (g["zmin"] <= 0) & (g["zmax"] >= 0))


def golden_uncontract_check(got, g):
    """The reference's uncontraction and clip (run on the CPU) against `got`: bit for bit where |y| is exact in
    float32 whatever the order of the norm's sum (the chosen points), else within the first-order effect of the
    norm's rounding, which CPU torch computes in its own order."""
    import tsdf_ref as TR
    y = g["contracted"].astype(np.float64)
    want = g["clipped"].astype(F)
    got = np.asarray(got, F)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    exact = TR._norm_exact(y)
    assert exact.sum() >= 10
    rows = exact & ~nan.any(1)
    assert np.array_equal(got[rows].view(np.uint32), want[rows].view(np.uint32))
    m = np.linalg.norm(y, axis=1)
    c = g["center"].astype(np.float64)
    rel = 8 * U * (1 + m / np.maximum(np.abs(2 - m), 1e-30)) + 8 * U
    bound = rel[:, None] * np.abs(want.astype(np.float64) - c) + 4 * U * (np.abs(c) + np.abs(want))
    ok = nan | (np.abs(got.astype(np.float64) - want) <= bound)
    assert ok.all()


def test_golden_inverse_contraction_and_clip():
    g = _golden()
    golden_uncontract_check(MR.uncontract_clip(g["contracted"], g["center"], float(g["radius"])), g)


# ---- the C ABI's argument checks -----------------------------------------------------------------------------------

def test_c_abi_rejects_bad_arguments():
    from diff_surfel_rasterization import _cabi
    from diff_surfel_rasterization.tsdf import UnboundedTSDF
    lib = _cabi.load()
    err = lambda: lib.surfel_last_error().decode()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    crop = (ctypes.c_int * 3)(0, 0, 0)
    bounds = (ctypes.c_double * 6)(-1, 1, -1, 1, -1, 1)
    ws = lib.surfel_mcubes_crop_workspace_bytes(9)
    assert ws > 0 and lib.surfel_mcubes_crop_workspace_bytes(1) == 0 and lib.surfel_mcubes_crop_workspace_bytes(513) == 0
    count = lambda side=9, vol=p, cr=crop, n=1, w=p, wb=ws, tot=p: lib.surfel_mcubes_crop_count(
        side, vol, cr, n, w, wb, tot, None)
    assert count(side=1) != 0 and "side" in err()
    assert count(side=513) != 0 and "side" in err()
    assert count(n=0) != 0 and "crops per axis" in err()
    assert count(cr=(ctypes.c_int * 3)(0, 2, 0), n=2) != 0 and "crop index" in err()
    assert count(cr=(ctypes.c_int * 3)(-1, 0, 0)) != 0 and "crop index" in err()
    assert count(cr=None) != 0 and "NULL crop" in err()
    assert count(vol=None) != 0 and "NULL volume" in err()
    assert count(w=None) != 0 and "NULL workspace" in err()
    assert count(wb=ws - 1) != 0 and "workspace of" in err()
    emit = lambda nr=4, nt=2, b=bounds, o=p: lib.surfel_mcubes_crop_emit(9, p, b, crop, 1, p, ws, nr, nt, o, o, o, None)
    assert emit(b=None) != 0 and "NULL bounds" in err()
    assert emit(nr=-1) != 0 and "negative" in err()
    assert emit(o=None) != 0 and "NULL output" in err()
    assert lib.surfel_mcubes_merge_workspace_bytes(1 << 30) == 0 and lib.surfel_mcubes_merge_workspace_bytes(-1) == 0
    cen = (ctypes.c_float * 3)(0, 0, 0)
    mb = lib.surfel_mcubes_merge_workspace_bytes(10)
    merge = lambda nr=10, nt=4, kb=20, c=cen, w=p, wb=mb, o=p: lib.surfel_mcubes_merge(
        nr, o, o, nt, o, kb, c, 1.0, w, wb, o, o, p, None)
    assert merge(nr=1 << 30) != 0 and "2^30" in err()
    assert merge(nr=0) != 0 and "without vertices" in err()
    assert merge(nr=-1) != 0 and "negative" in err()
    assert merge(kb=0) != 0 and "key_bits" in err()
    assert merge(kb=65) != 0 and "key_bits" in err()
    assert merge(c=None) != 0 and "NULL center" in err()
    assert merge(wb=mb - 1) != 0 and "workspace of" in err()
    assert merge(o=None) != 0 and "NULL input or output" in err()
    frames = (_cabi.TsdfFrame * 1)()
    frames[0].height, frames[0].width = 4, 4
    grid = lambda side=9, b=bounds, mp=16, o=p: lib.surfel_tsdf_eval_grid(side, b, 1, frames, mp, p, cen, 1.0, 0.05,
                                                                          o, None)
    assert grid(side=1) != 0 and "side" in err()
    assert grid(side=513) != 0 and "side" in err()
    assert grid(b=None) != 0 and "NULL bounds" in err()
    assert grid(mp=15) != 0 and "outside" in err()
    assert grid(o=None) != 0 and "NULL points or output" in err()
    # the wrapper's checks come before any device work
    dummy = types.SimpleNamespace()
    for res in (0, -512, 1000, 511, 512.0, True):
        with pytest.raises(RuntimeError, match="multiple of 512"):
            UnboundedTSDF.extract_mesh(dummy, res, 1.0)
    for R in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match="finite and > 0"):
            UnboundedTSDF.extract_mesh(dummy, 512, R)
