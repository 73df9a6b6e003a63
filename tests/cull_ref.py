"""A numpy restatement of the DTU mask culling rules (DESIGN.md §7n): cull_scan of the reference's
scripts/eval_dtu/evaluate_single_scene.py, as diff_surfel_rasterization.chamfer.cull_scan computes it.

 1. Cameras: P = (world_mat @ scale_mat)[:3, :4] in float32; A = sign(det P[:, :3]) * P / |P[2, :3]| in float64,
    rounded once to float32 (what cv2.decomposeProjectionMatrix, K / K[2, 2] and intrinsics @ inverse(pose) give).
 2. Dilation: D = binary_dilation(mask != 0, disk(r)) with a zero border, disk(r) = {dx^2 + dy^2 <= r^2}.
 3. Vertex test in float32, per view: c_k = ((A_k0 x + A_k1 y) + A_k2 z) + A_k3, d = c_2 + float32(1e-6),
    g = ((c / d) / float32(side - 1) - 0.5) * 2, valid iff -1 < gx < 1 and -1 < gy < 1 (NaN is not valid),
    i = nearbyint(((g + 1) / 2) * (mask side - 1)), half to even.  A view passes iff it is not valid or (ix, iy) lies
    in the mask and D[iy, ix] is set; a vertex is kept iff every view passes.
 4. Faces: kept iff their three vertices are; kept vertices (unreferenced ones too) and faces keep their order.
 5. World units: out = (v64 * f64(s00)) + f64(t), s00 = scale_mats[0][0, 0] and t = scale_mats[0][:3, 3] as float32.

`near_tie` gives rule 3's bound: where a decision may differ from one computed with another operation order.
"""
import numpy as np

U32 = 2.0 ** -24          # unit roundoff of float32
EPS = np.float32(1e-6)


def projections(world_mats, scale_mats):
    """(N,3,4) float32 from the (N,4,4) world and scale matrices of cameras.npz (rule 1)."""
    wm = np.asarray(world_mats).astype(np.float32)
    sm = np.asarray(scale_mats).astype(np.float32)
    P = np.stack([w @ s for w, s in zip(wm, sm)])[:, :3, :4].astype(np.float64)
    sign = np.sign(np.linalg.det(P[:, :, :3]))
    norm = np.sqrt((P[:, 2, :3] ** 2).sum(1))
    return (sign[:, None, None] * P / norm[:, None, None]).astype(np.float32)


def disk(r):
    d = np.arange(-r, r + 1)
    return (d[:, None] ** 2 + d[None, :] ** 2) <= r * r


def dilate(mask, r):
    """Rule 2 by row distances: a pixel is set iff some |dy| <= r has a set pixel in row y + dy within the disk's
    half-width isqrt(r^2 - dy^2)."""
    m = np.asarray(mask) != 0
    H, W = m.shape
    big = r + 1
    xs = np.arange(W)[None, :]
    left = np.maximum.accumulate(np.where(m, xs, -10 ** 9), axis=1)
    right = np.minimum.accumulate(np.where(m, xs, 10 ** 9)[:, ::-1], axis=1)[:, ::-1]
    hd = np.minimum(np.minimum(xs - left, right - xs), big)
    out = np.zeros((H, W), bool)
    for dy in range(-r, r + 1):
        hw = int(np.sqrt(r * r - dy * dy))
        while hw * hw > r * r - dy * dy:
            hw -= 1
        while (hw + 1) ** 2 <= r * r - dy * dy:
            hw += 1
        lo, hi = max(0, -dy), min(H, H - dy)
        if lo < hi:
            out[lo:hi] |= hd[lo + dy:hi + dy] <= hw
    return out


def project(verts, A, image_size):
    """Rule 3's float32 chain for every view: (gx, gy) of shape (N, M)."""
    v = np.asarray(verts).astype(np.float32)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    A = np.asarray(A, np.float32)
    W, H = image_size
    with np.errstate(all="ignore"):
        c = [((A[:, k, 0:1] * x + A[:, k, 1:2] * y) + A[:, k, 2:3] * z) + A[:, k, 3:4] for k in range(3)]
        d = c[2] + EPS
        gx = ((c[0] / d) / np.float32(W - 1) - np.float32(0.5)) * np.float32(2)
        gy = ((c[1] / d) / np.float32(H - 1) - np.float32(0.5)) * np.float32(2)
    return gx, gy


def keep_vertices(verts, A, dilated, image_size):
    """Rule 3: (M,) bool.  dilated: (N, Hm, Wm) bool."""
    gx, gy = project(verts, A, image_size)
    N, Hm, Wm = dilated.shape
    valid = (gx > -1) & (gx < 1) & (gy > -1) & (gy < 1)
    with np.errstate(all="ignore"):
        fx = ((gx + np.float32(1)) / np.float32(2)) * np.float32(Wm - 1)
        fy = ((gy + np.float32(1)) / np.float32(2)) * np.float32(Hm - 1)
    ix = np.where(valid, np.rint(fx), -1).astype(np.int64)
    iy = np.where(valid, np.rint(fy), -1).astype(np.int64)
    inside = valid & (ix >= 0) & (ix < Wm) & (iy >= 0) & (iy < Hm)
    hit = np.zeros_like(valid)
    for k in range(N):
        hit[k, inside[k]] = dilated[k][iy[k, inside[k]], ix[k, inside[k]]]
    return (~valid | hit).all(0)


def cull(verts, faces, masks, A, scale_mats, colors=None, image_size=(1600, 1200), radius=24):
    """Rules 2-5: dict with dilated (N,Hm,Wm) bool, keep (M,) bool, verts (M',3) float64, faces (F',3) int64,
    colors or None."""
    verts = np.asarray(verts)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    dilated = np.stack([dilate(m, radius) for m in masks])
    keep = keep_vertices(verts, A, dilated, image_size)
    fkeep = keep[faces].all(1) if len(faces) else np.zeros(0, bool)
    new = np.cumsum(keep) - 1
    sm = np.asarray(scale_mats[0]).astype(np.float32)
    s, t = np.float64(sm[0, 0]), sm[:3, 3].astype(np.float64)
    out = verts[keep].astype(np.float64) * s + t[None]
    return dict(dilated=dilated, keep=keep, verts=out, faces=new[faces[fkeep]].astype(np.int64),
                colors=None if colors is None else np.asarray(colors)[keep])


def near_tie(verts, A, image_size, mask_shape, a_rel=0.0):
    """(N, M) bool: where rule 3's decision rests on rounding.  Any evaluation of the chain whose dot products take
    another order or fused multiply-adds, whose A differs by at most a_rel relative per element, or which multiplies
    by a rounded reciprocal of W - 1 instead of dividing, stays within the first-order bounds below (u = 2^-24):
      e_c = (4u + a_rel) * S_c, S_c = |A0 x| + |A1 y| + |A2 z| + |A3| (in float64),
      e_d = e_c2 + u |d|,  e_q = (e_c + |q| e_d) / |d| + u |q| for q = c / d,
      e_g = 2 e_q / (W - 1) + 8u (|q| / (W - 1) + 1),  e_i = e_g (Wm - 1) / 2 + 4u (Wm - 1)(1 + |g|).
    A decision may then differ only where g lies within e_g of -1 or 1, or the unrounded pixel coordinate lies within
    e_i of k + 1/2; where |d| <= 2 e_d every decision of the view is treated as such."""
    v = np.asarray(verts).astype(np.float32).astype(np.float64)
    A64 = np.asarray(A, np.float32).astype(np.float64)
    W, H = image_size
    Hm, Wm = mask_shape
    e_tot = 4 * U32 + a_rel
    with np.errstate(all="ignore"):
        terms = A64[:, :, :3, None] * v.T[None, None]                     # (N, 3, 3, M)
        c = terms.sum(2) + A64[:, :, 3:4]
        S = np.abs(terms).sum(2) + np.abs(A64[:, :, 3:4])
        e_c = e_tot * S
        d = c[:, 2] + 1e-6
        e_d = e_c[:, 2] + U32 * np.abs(d)
        tie = ~(np.abs(d) > 2 * e_d)
        for k, side, mside in ((0, W, Wm), (1, H, Hm)):
            q = c[:, k] / d
            e_q = (e_c[:, k] + np.abs(q) * e_d) / np.abs(d) + U32 * np.abs(q)
            g = (q / (side - 1) - 0.5) * 2
            e_g = 2 * e_q / (side - 1) + 8 * U32 * (np.abs(q) / (side - 1) + 1)
            f = (g + 1) / 2 * (mside - 1)
            e_i = e_g * (mside - 1) / 2 + 4 * U32 * (mside - 1) * (1 + np.abs(g))
            half = np.floor(f) + 0.5
            tie |= (np.abs(g - 1) <= e_g) | (np.abs(g + 1) <= e_g) | (np.abs(f - half) <= e_i)
            tie |= ~np.isfinite(q)
    return tie
