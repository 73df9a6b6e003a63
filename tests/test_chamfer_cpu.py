"""DTU Chamfer evaluation without a device (DESIGN.md §7m): the restatement tests/chamfer_ref.py replays every array
the reference's own eval.py recorded (tests/golden/ref_chamfer.npz) bit for bit, raises where it raised, and agrees
with its means to 1e-12 relative; plus the C ABI's argument checks, which run before any device work."""
import ctypes
import math
import os

import numpy as np
import pytest

import chamfer_ref as CR

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_chamfer.npz")


def golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("ref_chamfer.npz not generated")
    return np.load(GOLDEN)


def case_names(g):
    return sorted({k.split(".")[0] for k in g.files})


def case(g, n):
    return {k.split(".", 1)[1]: g[k] for k in g.files if k.split(".")[0] == n}


def run_ref(c):
    """(pcd, result dict) of the restatement on a recorded case; raises as the rules say."""
    thresh, patch, md, vis = (float(x) for x in c["args"])
    if str(c["mode"]) == "mesh":
        pcd = CR.sample_mesh(c["verts"], c["faces"], thresh)
    else:
        pcd = c["pcd_in"]
    return pcd, CR.evaluate(pcd, c["stl"], c["obs"], c["bb"], c["res"], c["plane"], c["perm"], thresh, patch, md, vis)


def same(a, b):
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def close(a, b):
    return (math.isnan(a) and math.isnan(b)) or abs(a - b) <= 1e-12 * abs(b)


@pytest.mark.parametrize("name", case_names(np.load(GOLDEN)) if os.path.exists(GOLDEN) else [])
def test_restatement_matches_reference(name):
    g = golden()
    c = case(g, name)
    err = str(c["error"])
    if err:
        with pytest.raises(ValueError):
            run_ref(c)
        assert err == "ValueError"
        return
    pcd, r = run_ref(c)
    thresh = float(c["args"][0])
    assert same(pcd, c["pcd"]), "samples"
    assert same(r["shuffled"], c["pcd"][c["perm"]])
    # the kept mask against the reference's loop over its recorded radius neighbours
    ptr, idx = c["rnn_ptr"], c["rnn_idx"]
    mask = np.ones(len(pcd), bool)
    for k in range(len(pcd)):
        if mask[k]:
            mask[idx[ptr[k]:ptr[k + 1]]] = False
            mask[k] = True
    assert np.array_equal(r["kept"], mask), "kept mask"
    # every recorded radius neighbour pair is a pair of the exact rule, and the other way round
    x = r["shuffled"]
    pairs = CR.neighbour_pairs(x, thresh)
    mine = {(int(i), int(j)) for i, j in pairs} | {(int(j), int(i)) for i, j in pairs}
    rows = np.repeat(np.arange(len(x)), np.diff(ptr))
    theirs = {(int(i), int(j)) for i, j in zip(rows, idx) if i != j}
    assert mine == theirs, f"{len(mine ^ theirs)} pairs differ"
    assert same(r["data_down"], c["d2s_points"])
    assert same(r["data_color"], c["d2s_colors"]), "d2s colours"
    assert same(c["s2d_points"], c["stl"])
    assert same(r["stl_color"], c["s2d_colors"]), "s2d colours"
    md = float(c["args"][2])
    for k, mine_d in ((0, r["dist_d2s"]), (1, r["dist_s2d"])):
        ref = c[f"knn{k}_dist"]
        want = np.where(ref < md, ref, np.inf)
        assert same(mine_d, want), f"pass {k}: {int((mine_d != want).sum())} distances differ"
    res = c["results"]
    assert close(r["mean_d2s"], res[0]) and close(r["mean_s2d"], res[1]) and close(r["overall"], res[2])


def test_golden_covers_the_cases():
    g = golden()
    names = case_names(g)
    errors = {n: str(g[f"{n}.error"]) for n in names}
    assert sum(1 for e in errors.values() if e == "ValueError") == 4
    assert any(str(g[f"{n}.mode"]) == "pcd" for n in names)
    # exact pairs at r in the dyadic cloud, distances at exactly max_dist, a point on the plane
    c = case(g, "dyadic_pcd")
    x = c["pcd"][c["perm"]]
    d = CR.rdist(x[:, None], x[None])
    assert (d == 0.25 * 0.25).sum() > 100
    c = case(g, "maxdist_plane_pcd")
    assert (c["knn1_dist"] == 20.0).any() or (c["knn0_dist"] == 20.0).any()
    P = c["plane"]
    s = c["stl"]
    assert ((((P[0] * s[:, 0] + P[1] * s[:, 1]) + P[2] * s[:, 2]) + P[3]) == 0).any()


def test_sampling_rules():
    # n = 0 emits nothing; zero area is dropped; a vertex is always emitted
    v = np.array([[0, 0, 0], [0.1, 0, 0], [0, 0.1, 0], [9, 9, 9]], np.float64)
    out = CR.sample_mesh(v, [[0, 1, 2]], 0.2)
    assert same(out, v)
    with pytest.raises(ValueError):
        CR.sample_mesh(v, [[0, 0, 1]], 0.2)
    with pytest.raises(ValueError):
        CR.sample_mesh(v, [[0, 1, -1]], 0.2)


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
    info = ctypes.c_void_p(32)
    assert lib.surfel_chamfer_sample_workspace_bytes(-1) == 0
    assert lib.surfel_chamfer_workspace_bytes(-1, 5) == 0
    assert lib.surfel_chamfer_workspace_bytes(1 << 31, 5) == 0
    assert lib.surfel_chamfer_sample_count(-1, 1, p, p, 0.2, p, 1 << 20, info, None) != 0
    assert lib.surfel_chamfer_sample_count(3, 1, None, p, 0.2, p, 1 << 20, info, None) != 0
    assert b"NULL" in lib.surfel_last_error()
    assert lib.surfel_chamfer_sample_count(3, 1, p, p, 0.2, p, 1, info, None) != 0
    assert b"workspace" in lib.surfel_last_error()
    assert lib.surfel_chamfer_sample_emit(3, 1, p, p, 0.2, p, 1 << 20, 1 << 31, p, None) != 0
    rounds = ctypes.c_int(0)
    assert lib.surfel_chamfer_downsample(0, 5, p, 0.2, p, 1 << 20, ctypes.byref(rounds), None) != 0
    assert b"empty" in lib.surfel_last_error()
    assert lib.surfel_chamfer_downsample(5, 5, p, 0.2, p, 1, ctypes.byref(rounds), None) != 0
    d3 = (ctypes.c_double * 3)()
    sh = (ctypes.c_int * 3)(2, 0, 2)
    d4 = (ctypes.c_double * 4)()
    ws = lib.surfel_chamfer_workspace_bytes(5, 5)
    assert lib.surfel_chamfer_select(5, 5, p, p, d3, d3, d3, 1.0, p, sh, d4, p, ws, *([p] * 6), info, None) != 0
    assert b"zero side" in lib.surfel_last_error()
    assert lib.surfel_chamfer_distances(5, 5, p, 3, 2, p, 0, p, p, 1, p, p, 20.0, 10.0, p, ws,
                                        *([p] * 5), None) != 0
    assert b"non-empty" in lib.surfel_last_error()
