"""Cluster filtering without a device (DESIGN.md §7k): the reference's recorded post_process_mesh
(tests/golden/ref_meshpost.npz) replayed by restatement (a), restatement (a) against the vectorised (b) on the golden
and on random meshes, the reference's quirks one per case, and the argument checks of the C ABI and the wrapper."""
import ctypes
import os

import numpy as np
import pytest

import meshpost_ref as MP

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_meshpost.npz")
F32 = np.float32


def golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("ref_meshpost.npz not generated")
    return np.load(GOLDEN)


def golden_cases(g):
    """(name, verts, faces, colors or None, [k, ...]) of every recorded mesh."""
    names = sorted({k.split(".")[0] for k in g.files})
    return [(n, g[f"{n}.verts"], g[f"{n}.faces"], g[f"{n}.colors"] if f"{n}.colors" in g.files else None,
             [int(k) for k in g[f"{n}.ks"]]) for n in names]


def same_bits(got, want):
    got, want = np.ascontiguousarray(got, F32), np.ascontiguousarray(want, F32)
    return got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))


def check_result(got, g, tag, colors):
    mask, v, f, c = got
    assert np.array_equal(mask, g[f"{tag}.mask"])
    assert same_bits(v, g[f"{tag}.verts"])
    assert np.array_equal(np.asarray(f, np.int64).reshape(-1, 3), g[f"{tag}.faces"])
    if colors is None:
        assert c is None
    else:
        assert same_bits(c, g[f"{tag}.colors"])


def test_golden_replays_through_the_literal_restatement():
    g = golden()
    n_err = n_out = 0
    for name, v, f, c, ks in golden_cases(g):
        for k in ks:
            tag = f"{name}.k{k}"
            if f"{tag}.error" in g.files:
                assert str(g[f"{tag}.error"]) == "IndexError"
                with pytest.raises(IndexError):
                    MP.post_process_literal(v, f, c, k)
                n_err += 1
            else:
                check_result(MP.post_process_literal(v, f, c, k), g, tag, c)
                n_out += 1
    assert n_err >= 20 and n_out >= 25


def _same_ab(v, f, c, k):
    try:
        a = MP.post_process_literal(v, f, c, k)
    except IndexError:
        with pytest.raises(IndexError):
            MP.post_process_vectorised(v, f, c, k)
        return None
    b = MP.post_process_vectorised(v, f, c, k)
    assert np.array_equal(a[0], b[0])
    assert same_bits(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert (a[3] is None) == (b[3] is None) and (a[3] is None or same_bits(a[3], b[3]))
    return a


def test_literal_equals_vectorised_on_the_golden():
    for name, v, f, c, ks in golden_cases(golden()):
        ia, ca = MP.clusters_literal(f)
        ib, cb = MP.clusters_vectorised(f, len(v))
        assert np.array_equal(ia, ib) and np.array_equal(ca, cb), name
        for k in ks:
            _same_ab(v, f, c, k)


def _random_meshes(rng):
    out = []
    for M, F in ((4, 60), (6, 200), (10, 400), (30, 300)):           # few vertices: dense degeneracy and duplicates
        out.append((M, rng.integers(0, M, (F, 3))))
    g = MP.grid(12, 9)
    out.append((108, g[rng.permutation(len(g))]))                     # shuffled face order
    s = np.concatenate([MP.strip(70), MP.strip(55, 80), MP.strip(49, 150), MP.grid(6, 6, 210)])
    out.append((250, s[rng.permutation(len(s))]))
    parts, v0 = [], 0
    for n in rng.integers(1, 80, 30):                                  # many clusters around the floor of 50
        parts.append(MP.fan(int(n), v0))
        v0 += int(n) + 2
    f = np.concatenate(parts)
    out.append((v0 + 5, f[rng.permutation(len(f))]))
    return out


def test_literal_equals_vectorised_on_random_meshes():
    rng = np.random.default_rng(3)
    for M, f in _random_meshes(rng):
        v = rng.normal(size=(M, 3)).astype(F32)
        c = rng.uniform(size=(M, 2)).astype(F32)
        C = len(MP.clusters_literal(f)[1])
        for k in (1, 2, 3, 50, 0, -1, -2, C, C + 1):
            _same_ab(v, f, c, k)


# ---- the quirks, one per case ----------------------------------------------------------------------------------------

def _counts_mesh():
    """Clusters of 120, 60, 52, 52 and 10 faces (bipyramids), in that order of their first face."""
    parts, v0 = [], 0
    for n in (60, 30, 26, 26, 5):
        parts.append(MP.bipyramid(n, v0))
        v0 += n + 2
    return np.zeros((v0, 3), F32), np.concatenate(parts)


def test_k_zero_selects_the_smallest_count():
    v, f = _counts_mesh()
    mask = MP.post_process_literal(v, f, None, 0)[0]
    assert not mask[:-10].any() and mask[-10:].all()         # threshold max(10, 50): only the 10-face cluster goes
    mask = MP.post_process_literal(v, f, None, 1)[0]
    assert mask.sum() == len(f) - 120                        # k = 1: only the largest stays


def test_negative_k_counts_from_the_bottom():
    v, f = _counts_mesh()
    # sorted counts 10, 52, 52, 60, 120: k = -3 reads index 3 -> 60
    assert MP.post_process_literal(v, f, None, -3)[0].sum() == 10 + 52 + 52
    # ties at the threshold all stay: k = 3 reads 52, and both 52-face clusters are kept (four clusters, not three)
    assert MP.post_process_literal(v, f, None, 3)[0].sum() == 10
    with pytest.raises(IndexError):
        MP.post_process_literal(v, f, None, -5)


def test_index_error_on_empty_meshes_and_past_the_cluster_count():
    v, f = _counts_mesh()
    MP.post_process_literal(v, f, None, 5)
    for k in (6, 1000):
        with pytest.raises(IndexError):
            MP.post_process_literal(v, f, None, k)
    for k in (0, 1, -1, 1000):
        with pytest.raises(IndexError):
            MP.post_process_literal(v, np.zeros((0, 3), np.int64), None, k)


def test_vertex_of_degenerate_faces_only_survives_unreferenced():
    g = MP.grid(8, 8)
    f = np.concatenate([g, [[9, 9, 10], [9, 9, 70]]])         # (9,9,70) joins the grid through the pair (9,9)
    v = np.arange(71 * 3, dtype=F32).reshape(71, 3)
    _, vo, fo, _ = MP.post_process_literal(v, f, None, 1)
    assert len(fo) == len(g) and len(vo) == 65
    assert vo[-1, 0] == 70 * 3 and 64 not in fo               # vertex 70 is kept, now 64, and no face uses it


def test_bowtie_is_two_clusters():
    a, b = MP.fan(60, 0), MP.fan(60, 61)
    b[:, 0] = 0                                               # the fans share vertex 0 only
    ids, counts = MP.clusters_literal(np.concatenate([a, b]))
    assert np.array_equal(counts, [60, 60]) and np.array_equal(ids, [0] * 60 + [1] * 60)


# ---- argument checks ---------------------------------------------------------------------------------------------

def test_c_abi_rejects_bad_arguments():
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    err = lambda: lib.surfel_last_error().decode()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    maxf = ((1 << 30) - 1) // 3
    ws_bytes = lib.surfel_meshpost_workspace_bytes
    assert ws_bytes(10, 8) > 0 and ws_bytes(0, 0) > 0 and ws_bytes((1 << 31) - 1, maxf) > 0
    for m, f in ((-1, 8), (10, -1), (1 << 31, 8), (10, maxf + 1)):
        assert ws_bytes(m, f) == 0
    ws = ws_bytes(10, 8)
    clusters = lambda m=10, f=8, fa=p, w=p, wb=ws, o=p: lib.surfel_meshpost_clusters(m, f, fa, w, wb, o, o, o, None)
    assert clusters(m=-1) != 0 and "negative" in err()
    assert clusters(f=-1) != 0 and "negative" in err()
    assert clusters(m=1 << 31) != 0 and "2^31" in err()
    assert clusters(f=maxf + 1) != 0 and "2^30" in err()
    assert clusters(fa=None) != 0 and "NULL" in err()
    assert clusters(o=None) != 0 and "NULL" in err()
    assert clusters(w=None) != 0 and "NULL workspace" in err()
    assert clusters(wb=ws - 1) != 0 and "workspace of" in err()
    compact = lambda m=10, f=8, c=3, i=0, w=p, wb=ws, o=p: lib.surfel_meshpost_compact(
        m, f, p, p, p, c, i, w, wb, o, o, o, None)
    assert compact(m=-1) != 0 and "negative" in err()
    assert compact(m=1 << 31) != 0 and "2^31" in err()
    assert compact(f=maxf + 1) != 0 and "2^30" in err()
    assert compact(c=0) != 0 and "clusters" in err()
    assert compact(c=9) != 0 and "clusters" in err()
    assert compact(i=-1) != 0 and "index" in err()
    assert compact(i=3) != 0 and "index" in err()
    assert compact(o=None) != 0 and "NULL" in err()
    assert compact(w=None) != 0 and "NULL workspace" in err()
    assert compact(wb=ws - 1) != 0 and "workspace of" in err()


def test_wrapper_rejects_bad_arguments_before_any_device_work():
    import torch
    from diff_surfel_rasterization.meshpost import post_process_mesh, threshold_index
    v, f = torch.zeros(4, 3), torch.tensor([[0, 1, 2]])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        post_process_mesh(v, f)
    for k in (1.0, True, "3", None):
        with pytest.raises(RuntimeError, match="integer"):
            post_process_mesh(v, f, cluster_to_keep=k)
    # Python's indexing of np.sort(counts)[-k]
    assert [threshold_index(k, 5) for k in (1, 5, 0, -1, -4, np.int64(2))] == [4, 0, 0, 1, 4, 3]
    for k, C in ((6, 5), (-5, 5), (0, 0), (1, 0)):
        with pytest.raises(IndexError):
            threshold_index(k, C)
