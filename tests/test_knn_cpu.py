"""simple_knn.distCUDA2 without a GPU: the certified CPU restatement (tests/knn_oracle.py) against the definition,
the rules on hand-built inputs, the import path, and the reference's call site (tests/golden/ref_init_knn.npz)."""
import os

import numpy as np
import pytest

import knn_oracle as KO
import knn_scenes as KS

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def assert_same(got, want):
    """Bit for bit, NaN rows included (both produce the canonical quiet NaN)."""
    assert got.shape == want.shape
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    np.testing.assert_array_equal(bits(got[ok]), bits(want[ok]))


CLOUDS = {
    "uniform": lambda: KS.uniform(3000, 1),
    "colmap_like": lambda: KS.colmap_like(3000, 2),
    "plane": lambda: KS.plane(2000, 3),
    "line": lambda: KS.line(1500, 4),
    "lattice": lambda: KS.lattice(12),
    "dup_2_3_4": lambda: KS.duplicate_groups([2] * 200 + [3] * 150 + [4] * 100, 5),
    "dup_500": lambda: np.concatenate([KS.duplicate_groups([500, 500], 6), KS.uniform(1000, 6)]),
    "large_offset": lambda: KS.large_offset(2000, 7),
    "nonfinite": lambda: KS.with_nonfinite(2000, 8),
    "duplicated": lambda: KS.duplicated(3000, 9),
    "shell": lambda: KS.sphere_shell(40, 10),
}


@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_restatement_equals_brute_force(name):
    pts = CLOUDS[name]()
    assert pts.dtype == F32 and pts.shape[1] == 3 and len(pts) <= 3000
    assert_same(KO.mean_sq_dist(pts), KO.brute_force(pts))


@pytest.mark.parametrize("P", range(6))
def test_tiny_clouds(P):
    pts = KS.uniform(P, 11 + P)
    assert_same(KO.mean_sq_dist(pts), KO.brute_force(pts))


def test_certificate_escalation_happens_and_stays_exact():
    pts = KS.sphere_shell(40, 12)
    st = {}
    got = KO.mean_sq_dist(pts, stats=st)
    assert st["rounds"] >= 3 and st["escalated"] >= 1, st      # K = 16, 32 tie within rounding; K = 64 covers all
    assert_same(got, KO.brute_force(pts))
    # a cloud whose ties resolve at K = 16 needs no second round
    st = {}
    KO.mean_sq_dist(KS.uniform(2000, 13), stats=st)
    assert st["rounds"] == 1 and st["escalated"] == 0


def test_rule_2_operation_order_and_division():
    a = np.array([[0, 0, 0], [0.1, 0.2, 0.3], [-0.7, 0.05, 0.2], [1.3, -1.1, 0.4]], F32)
    q, o = a[0], a[1:]
    dx, dy, dz = [(q[c] - o[:, c]).astype(F32) for c in range(3)]
    d2 = np.sort(((dx * dx) + (dy * dy)) + (dz * dz))
    want = (((d2[0] + d2[1]) + d2[2]) / F32(3)).astype(F32)
    assert bits(KO.brute_force(a)[:1])[0] == bits(np.array([want]))[0]


def test_rule_3_fewer_than_three_neighbours():
    assert KO.mean_sq_dist(np.zeros((0, 3), F32)).shape == (0,)
    np.testing.assert_array_equal(KO.mean_sq_dist(np.array([[1, 2, 3]], F32)), [0.0])          # k = 0
    two = np.array([[0, 0, 0], [3, 4, 0]], F32)
    np.testing.assert_array_equal(KO.mean_sq_dist(two), [25.0, 25.0])                        # k = 1
    three = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0]], F32)
    np.testing.assert_array_equal(KO.mean_sq_dist(three), [(F32(1) + F32(4)) / F32(2), (F32(1) + F32(5)) / F32(2),
                                                           (F32(4) + F32(5)) / F32(2)])      # k = 2
    # only finite points count: two finite rows among NaN / inf rows behave like a two-point cloud
    mixed = np.array([[0, 0, 0], [np.nan, 0, 0], [3, 4, 0], [0, np.inf, 0], [0, 0, -np.inf]], F32)
    got = KO.mean_sq_dist(mixed)
    np.testing.assert_array_equal(got[[0, 2]], [25.0, 25.0])
    assert np.isnan(got[[1, 3, 4]]).all()


def test_rule_1_duplicates_are_neighbours_at_zero():
    pts = np.array([[1, 1, 1], [1, 1, 1], [1, 1, 1], [1, 1, 1], [5, 5, 5]], F32)
    got = KO.mean_sq_dist(pts)
    np.testing.assert_array_equal(got[:4], [0, 0, 0, 0])
    two = np.array([[1, 1, 1], [1, 1, 1], [2, 1, 1], [1, 3, 1]], F32)
    np.testing.assert_array_equal(KO.mean_sq_dist(two)[0], (F32(0) + F32(1) + F32(4)) / F32(3))


def test_rule_4_nonfinite_rows_are_nobodys_neighbour():
    base = KS.uniform(500, 14)
    poisoned = np.concatenate([base, np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan] * 3], F32)])
    got = KO.mean_sq_dist(poisoned)
    assert np.isnan(got[500:]).all()
    assert_same(got[:500], KO.mean_sq_dist(base))


def test_import_without_gpu_and_cpu_tensor_raises():
    import torch
    from simple_knn._C import distCUDA2
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        distCUDA2(torch.zeros(4, 3))
    with pytest.raises(RuntimeError):
        distCUDA2(np.zeros((4, 3), F32))


def test_cabi_rejects_bad_arguments_without_a_device():
    import ctypes
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    err = lambda: lib.surfel_last_error().decode()
    buf = (ctypes.c_float * 16)()
    p = ctypes.addressof(buf)
    n = lib.surfel_knn_workspace_bytes(1000)
    assert n >= 1000 * (16 + 24)
    assert lib.surfel_knn_workspace_bytes(-1) == 0 and lib.surfel_knn_workspace_bytes(1 << 30) == 0
    assert lib.surfel_knn_mean_sq_dist(0, None, None, None, 0, None) == 0              # P = 0: nothing to do
    assert lib.surfel_knn_mean_sq_dist(-1, p, p, p, n, None) != 0 and "P < 0" in err()
    assert lib.surfel_knn_mean_sq_dist((1 << 30), p, p, p, n, None) != 0 and "exceeds" in err()
    assert lib.surfel_knn_mean_sq_dist(5, None, p, p, n, None) != 0 and "NULL" in err()
    assert lib.surfel_knn_mean_sq_dist(5, p, None, p, n, None) != 0 and "NULL" in err()
    assert lib.surfel_knn_mean_sq_dist(5, p, p, None, n, None) != 0 and "NULL" in err()
    small = lib.surfel_knn_workspace_bytes(5) - 1
    assert lib.surfel_knn_mean_sq_dist(5, p, p, p, small, None) != 0 and "workspace" in err()


def test_golden_call_site():
    """The reference's own create_from_pcd (tests/golden/make_golden_knn.py) fed the restatement's values to
    its two lines; the stored input is what it passes to distCUDA2 and the stored distances what the
    restatement returns for it."""
    import torch
    g = np.load(os.path.join(HERE, "golden", "ref_init_knn.npz"))
    assert g["received"].dtype == F32 and g["received"].shape == (5000, 3)
    np.testing.assert_array_equal(g["received"], g["points"].astype(F32))
    assert_same(KO.mean_sq_dist(g["received"]), g["dist2"])
    d = torch.from_numpy(g["dist2"])
    scales = torch.log(torch.sqrt(torch.clamp_min(d, 0.0000001)))[..., None].repeat(1, 2)
    np.testing.assert_array_equal(scales.numpy(), g["scaling"])
