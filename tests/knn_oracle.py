"""CPU restatement of simple_knn.distCUDA2 (csrc/knn.cu, DESIGN.md §7g) with a per-row certificate.

For each finite query: cKDTree (float64, on the float32 coordinates) proposes its K nearest other points; their
d2 is evaluated in float32 in rule 2's operation order (numpy float32 elementwise arithmetic rounds every
operation to nearest and never contracts to FMA); the result follows rules 2-5.  The row is CERTIFIED when the
K-th candidate's float64 squared distance, shrunk by 1e-6 relative, is still >= the third-smallest float32 d2:
a float32 d2 lies within ~3e-7 relative of its exact value, so no point outside the candidate set can be below
the third-best, and the value (which depends only on the multiset of the three smallest d2) is exact.  Rows
that fail are re-queried with K doubled until every row is certified (K >= number of others certifies trivially).
"""
import numpy as np
from scipy.spatial import cKDTree

F32 = np.float32


def sq_dist_f32(q, p):
    """Rule 2: d2 = (dx*dx + dy*dy) + dz*dz in float32, dx = q - p; broadcasts over leading axes."""
    q = np.asarray(q, F32)
    p = np.asarray(p, F32)
    dx = q[..., 0] - p[..., 0]
    dy = q[..., 1] - p[..., 1]
    dz = q[..., 2] - p[..., 2]
    return (dx * dx + dy * dy) + dz * dz


def mean_of_smallest(d2_sorted, k):
    """Rules 2 and 3 on rows of ascending float32 d2 (at least k columns)."""
    n = d2_sorted.shape[0]
    if k == 0:
        return np.zeros(n, F32)
    s = d2_sorted[:, 0].astype(F32)
    for c in range(1, k):
        s = s + d2_sorted[:, c]
    return (s / F32(k)).astype(F32)


def mean_sq_dist(points, k0=16, stats=None):
    """points: (P,3) float32 -> (P,) float32, what distCUDA2 returns.  `stats`, if a dict, receives the number
    of query rounds and of rows that needed a larger K."""
    pts = np.ascontiguousarray(points, dtype=F32).reshape(-1, 3)
    P = pts.shape[0]
    out = np.full(P, np.nan, F32)
    finite = np.isfinite(pts).all(axis=1)
    idx = np.nonzero(finite)[0]
    fp = pts[idx]
    n = fp.shape[0]
    if stats is not None:
        stats.update(rounds=0, escalated=0)
    if n == 0:
        return out
    k_mean = min(3, n - 1)
    res = np.zeros(n, F32)
    if n > 1:
        tree = cKDTree(fp.astype(np.float64))
        pending = np.arange(n)
        K = k0
        while pending.size:
            Kq = min(K + 1, n)                                       # +1: the query itself
            dist, nb = tree.query(fp[pending].astype(np.float64), k=Kq, workers=-1)
            dist = dist.reshape(len(pending), Kq)
            nb = nb.reshape(len(pending), Kq)
            # drop the query by index; when copies of it fill the list it may be absent: drop the last column
            is_self = nb == pending[:, None]
            drop = np.where(is_self.any(axis=1), is_self.argmax(axis=1), Kq - 1)
            keep = np.ones_like(is_self)
            keep[np.arange(len(pending)), drop] = False
            nb = nb[keep].reshape(len(pending), Kq - 1)
            dist = dist[keep].reshape(len(pending), Kq - 1)
            d2 = np.sort(sq_dist_f32(fp[pending][:, None, :], fp[nb]), axis=1)
            third = d2[:, k_mean - 1]
            if Kq == n:
                ok = np.ones(len(pending), bool)                      # every other point is a candidate
            else:
                ok = dist[:, -1] ** 2 * (1.0 - 1e-6) >= third.astype(np.float64)
            res[pending[ok]] = mean_of_smallest(d2[ok], k_mean)
            if stats is not None:
                stats["rounds"] += 1
                if stats["rounds"] > 1:
                    stats["escalated"] += int(len(pending))
            pending = pending[~ok]
            K *= 2
    out[idx] = res
    return out


def brute_force(points):
    """All pairs, rule 2 arithmetic, rules 3-5: the definition itself (small P only)."""
    pts = np.ascontiguousarray(points, dtype=F32).reshape(-1, 3)
    P = pts.shape[0]
    out = np.full(P, np.nan, F32)
    finite = np.isfinite(pts).all(axis=1)
    idx = np.nonzero(finite)[0]
    fp = pts[idx]
    n = fp.shape[0]
    if n == 0:
        return out
    k = min(3, n - 1)
    res = np.zeros(n, F32)
    for s in range(0, n, 512):
        d2 = sq_dist_f32(fp[s:s + 512, None, :], fp[None, :, :])
        d2[np.arange(d2.shape[0]), np.arange(s, s + d2.shape[0])] = np.inf   # exclude the query by index
        if k:
            res[s:s + 512] = mean_of_smallest(np.sort(d2, axis=1)[:, :k], k)
    out[idx] = res
    return out
