"""Restatement in numpy of the DTU Chamfer rules of DESIGN.md §7m (diff_surfel_rasterization.chamfer), written from
the rules: sampling (rule 1), the shuffle (2), the greedy radius downsampling (3), the float32 box (4), the
observation grid (5), the two bounded nearest-neighbour passes (6, 7) and the colours (8).  Candidate pairs and
nearest points come from scipy's cKDTree with a relative margin, and every decision is then taken with the exact
float64 rule, so the tree's own rounding never decides anything."""
import numpy as np
from scipy.spatial import cKDTree

MARGIN = 1e-9


def rdist(a, b):
    d = a - b
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _norm(v):
    return np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])


def tri_grid(verts, faces, thresh):
    """(kept mask, t0, v1, v2, n1, n2) of rule 1."""
    t0 = verts[faces[:, 0]]
    v1, v2 = verts[faces[:, 1]] - t0, verts[faces[:, 2]] - t0
    l1, l2 = _norm(v1), _norm(v2)
    cr = np.stack([v1[:, 1] * v2[:, 2] - v1[:, 2] * v2[:, 1], v1[:, 2] * v2[:, 0] - v1[:, 0] * v2[:, 2],
                   v1[:, 0] * v2[:, 1] - v1[:, 1] * v2[:, 0]], 1)
    area2 = _norm(cr)
    keep = area2 > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        thr = thresh * np.sqrt((l1 * l2) / area2)
        n1, n2 = np.floor(l1 / thr), np.floor(l2 / thr)
    return keep, t0, v1, v2, n1, n2


def sample_triangle(t0, v1, v2, n1, n2):
    a = (np.arange(n1 + 1) + 0.5) / max(n1, 1e-7)
    b = (np.arange(n2 + 1) + 0.5) / max(n2, 1e-7)
    A, B = np.meshgrid(a, b, indexing="ij")
    m = (A + B) < 1
    A, B = A[m][:, None], B[m][:, None]
    return (v1[None] * A + v2[None] * B) + t0[None]


def sample_mesh(verts, faces, thresh):
    """All vertices, then every positive-area triangle's samples in triangle and row-major order."""
    verts, faces = np.asarray(verts, np.float64), np.asarray(faces, np.int64).reshape(-1, 3)
    if faces.size and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError("face index outside [0, M)")
    if not np.isfinite(verts).all():
        raise ValueError("non-finite vertex")
    keep, t0, v1, v2, n1, n2 = tri_grid(verts, faces, thresh)
    if not keep.any():
        raise ValueError("no triangle of positive area")
    pts = [verts] + [sample_triangle(t0[f], v1[f], v2[f], n1[f], n2[f]) for f in np.nonzero(keep)[0]]
    return np.concatenate(pts, 0)


def neighbour_pairs(x, r):
    """(i, j) with i < j and rdist <= r*r (rule 3), from a superset of candidate pairs."""
    pairs = cKDTree(x).query_pairs(r * (1 + MARGIN), output_type="ndarray")
    if len(pairs) == 0:
        return np.zeros((0, 2), np.int64)
    pairs = np.sort(pairs, 1)
    return pairs[rdist(x[pairs[:, 0]], x[pairs[:, 1]]) <= r * r]


def greedy(n, pairs):
    """Kept mask of the sequential rule: a point is kept iff no earlier kept point is its neighbour."""
    order = np.argsort(pairs[:, 1], kind="stable")
    i, j = pairs[order, 0], pairs[order, 1]
    start = np.searchsorted(j, np.arange(n + 1))
    kept = np.zeros(n, bool)
    for k in range(n):
        kept[k] = not kept[i[start[k]:start[k + 1]]].any()
    return kept


def box(bb, patch):
    bb32 = np.asarray(bb).astype(np.float32)
    return (bb32[:1] - patch)[0].astype(np.float64), (bb32[1:] + patch * 2)[0].astype(np.float64), bb32


def nearest(q, x, max_dist):
    """Rule 6: sqrt of the exact rdist to the nearest point of x, +inf where it is >= max_dist."""
    if len(q) == 0:
        return np.zeros(0)
    tree = cKDTree(x)
    k = min(8, len(x))
    d, idx = tree.query(q, k=k)
    d, idx = d.reshape(len(q), k), idx.reshape(len(q), k)
    best = rdist(q[:, None, :], x[idx]).min(1)
    unsure = d[:, -1] <= d[:, 0] * (1 + MARGIN) + 1e-300
    if k < len(x):
        for r in np.nonzero(unsure)[0]:
            cand = tree.query_ball_point(q[r], d[r, 0] * (1 + MARGIN) + 1e-300)
            best[r] = rdist(q[r][None], x[cand]).min()
    dist = np.sqrt(best)
    return np.where(dist < max_dist, dist, np.inf)


def colours(n, rows, dist, max_dist, vis):
    c = np.tile(np.array([[0.0, 0.0, 1.0]]), (n, 1))
    alpha = np.minimum(dist, vis) / vis
    near = dist < max_dist
    R, W = np.array([1.0, 0.0, 0.0]), np.array([1.0, 1.0, 1.0])
    c[rows[near]] = R * alpha[near][:, None] + W * (1 - alpha[near][:, None])
    c[rows[~near]] = np.array([0.0, 1.0, 0.0])
    return c


def masked_mean(d, max_dist):
    sel = d[d < max_dist]
    return float(sel.sum() / len(sel)) if len(sel) else float("nan")


def evaluate(pcd, stl, obs_mask, bb, res, plane, perm, thresh=0.2, patch=60.0, max_dist=20.0, vis=10.0):
    """Every intermediate of rules 2-8 as a dict; ValueError where the reference raises."""
    pcd, stl = np.asarray(pcd, np.float64), np.asarray(stl, np.float64)
    if len(pcd) == 0 or len(stl) == 0 or not np.isfinite(pcd).all() or not np.isfinite(stl).all():
        raise ValueError("empty or non-finite cloud")
    x = pcd[np.asarray(perm)]
    kept = greedy(len(x), neighbour_pairs(x, thresh))
    down = x[kept]
    lo, hi, bb32 = box(bb, patch)
    inbound = ((down >= lo) & (down < hi)).all(1)
    data_in = down[inbound]
    g = np.rint((data_in - bb32[0].astype(np.float64)) / float(np.asarray(res).reshape(())))
    shape = np.asarray(obs_mask.shape)
    gin = ((g >= 0) & (g < shape)).all(1)
    gi = g[gin].astype(np.int64)
    obs = np.zeros(len(data_in), bool)
    obs[np.nonzero(gin)[0]] = np.asarray(obs_mask)[gi[:, 0], gi[:, 1], gi[:, 2]] != 0
    data_in_obs = data_in[obs]
    if len(data_in_obs) == 0:
        raise ValueError("empty data_in_obs")
    P = np.asarray(plane, np.float64).reshape(4)
    above = (((P[0] * stl[:, 0] + P[1] * stl[:, 1]) + P[2] * stl[:, 2]) + P[3]) > 0
    if len(data_in) == 0 or not above.any():
        raise ValueError("empty data_in or stl_above")
    d2s = nearest(data_in_obs, stl, max_dist)
    s2d = nearest(stl[above], data_in, max_dist)
    obs_rows = np.nonzero(inbound)[0][obs]
    out = dict(shuffled=x, kept=kept, data_down=down, inbound=inbound, obs=obs, data_in_obs=data_in_obs,
               dist_d2s=d2s, dist_s2d=s2d, above=above,
               data_color=colours(len(down), obs_rows, d2s, max_dist, vis),
               stl_color=colours(len(stl), np.nonzero(above)[0], s2d, max_dist, vis),
               mean_d2s=masked_mean(d2s, max_dist), mean_s2d=masked_mean(s2d, max_dist))
    out["overall"] = (out["mean_d2s"] + out["mean_s2d"]) / 2
    return out
