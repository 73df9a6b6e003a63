"""Seeded point clouds for simple_knn.distCUDA2 (tests and profiles/run_knn.py).  All return (P,3) float32."""
import numpy as np

F32 = np.float32


def uniform(P, seed=0):
    """The reference's random initialisation (/root/reference/scene/dataset_readers.py:236-242):
    uniform in [-1.3, 1.3]^3."""
    return (np.random.default_rng(seed).random((P, 3)) * 2.6 - 1.3).astype(F32)


def colmap_like(P, seed=0, outlier_frac=0.01):
    """A COLMAP sparse cloud's shape: anisotropic Gaussian clusters whose densities span four decades, plus
    `outlier_frac` of the points scattered uniformly over 100x the scene's extent."""
    rng = np.random.default_rng(seed)
    n_out = int(round(P * outlier_frac))
    n_in = P - n_out
    n_cl = 96
    w = np.exp(rng.uniform(0.0, np.log(1e3), n_cl))
    sizes = rng.multinomial(n_in, w / w.sum())
    parts = []
    for c in range(n_cl):
        if sizes[c] == 0:
            continue
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        sig = np.exp(rng.uniform(np.log(1e-3), np.log(2e-1), 3))
        parts.append(rng.uniform(-1, 1, 3) + (rng.normal(size=(sizes[c], 3)) * sig) @ q.T)
    parts.append(rng.uniform(-100, 100, (n_out, 3)))
    pts = np.concatenate(parts).astype(F32)
    return pts[rng.permutation(P)]


def duplicated(P, seed=0):
    """Heavy duplication: groups of 2..10 000 exact copies, about half the cloud in groups of 100 or more."""
    rng = np.random.default_rng(seed)
    base = uniform(P, seed)
    n_src = max(1, P // 20)
    counts = np.concatenate([np.full(max(1, n_src // 2), 2), rng.integers(3, 40, max(1, n_src // 2))])
    big = [10_000, 5_000, 2_000] + [500] * 40 + [100] * 200
    total, rows = 0, []
    for c in big + list(counts):
        if total + c > P // 2 + P // 4:
            break
        rows.append(np.repeat(base[rng.integers(P)][None], c, axis=0))
        total += c
    pts = np.concatenate([base[:P - total]] + rows).astype(F32)
    return pts[rng.permutation(P)]


def plane(P, seed=0):
    rng = np.random.default_rng(seed)
    p = rng.uniform(-1, 1, (P, 3))
    p[:, 2] = 0.25
    return p.astype(F32)


def line(P, seed=0):
    rng = np.random.default_rng(seed)
    t = rng.uniform(-1, 1, P)
    return np.stack([t, 0.5 * t + 0.1, -0.25 * t], 1).astype(F32)


def lattice(side):
    """Integer lattice side^3: every point has six neighbours at exactly 1 (massive ties)."""
    g = np.arange(side, dtype=F32)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(F32)


def duplicate_groups(group_sizes, seed=0, spread=1.0):
    """Groups of exact copies of distinct uniform points."""
    rng = np.random.default_rng(seed)
    src = rng.uniform(-spread, spread, (len(group_sizes), 3)).astype(F32)
    pts = np.concatenate([np.repeat(src[i][None], s, axis=0) for i, s in enumerate(group_sizes)])
    return pts[rng.permutation(len(pts))]


def large_offset(P, seed=0):
    """Coordinates about 1e4 with a spread of 1e-2: a float32 ulp there is ~1e-3 of the spacing."""
    rng = np.random.default_rng(seed)
    return (np.array([1.0e4, -2.0e4, 1.5e4]) + rng.uniform(-1e-2, 1e-2, (P, 3))).astype(F32)


def with_nonfinite(P, seed=0, frac=0.02):
    """Uniform cloud with NaN / +inf / -inf in one coordinate of a few rows."""
    rng = np.random.default_rng(seed)
    p = uniform(P, seed)
    rows = rng.choice(P, max(3, int(P * frac)), replace=False)
    vals = np.array([np.nan, np.inf, -np.inf], F32)
    p[rows, rng.integers(0, 3, len(rows))] = vals[np.arange(len(rows)) % 3]
    return p


def sphere_shell(n_shell, seed=0):
    """A centre point plus n_shell points at distance ~1 from it: the centre's K nearest candidates tie within
    float32 rounding, so a certificate with K < n_shell cannot separate them (forces escalation)."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n_shell, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([np.zeros((1, 3)), d, 3.0 * d[:8]]).astype(F32)
