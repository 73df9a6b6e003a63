"""Three statements of the reference's unbounded TSDF field (utils/mesh_utils.py:184-279; rules in DESIGN.md §7i):

* `emulate`: numpy float32, operation for operation what csrc/tsdf.cu computes (uncontracted, correctly rounded,
  the bilinear taps summed nw, ne, sw, se).  The kernel must match it bit for bit.
* `evaluate64`: the reference's expressions in float64 on the same float32 inputs, with a first-order bound per
  output on what float32 rounding can change, for ANY implementation of the reference's operations (a norm, matmul
  or grid_sample summed in another order, with or without FMA).  A (sample, frame) pair whose decision margin
  (|y| against 1 and 2, pix against +-1, w against 0, sdf against -trunc, a bilinear floor next to a
  non-finite tap) lies inside its bound is flagged, and a sample with a flagged pair is held only to range.
* `eager`: the reference's loop restated in eager torch (a mask and an indexed update per frame), for the profile.

A frame is (M, depth, rgb): M the (4,4) float32 full_proj_transform, depth (H,W) float32, rgb (3,H,W) float32
or None.  `center` is 3 float32 values, `radius` and `trunc` (= 5 * voxel_size) the doubles the reference forms.
"""
import numpy as np

F = np.float32
U = 2.0 ** -24          # unit roundoff of float32


# ---- float32 emulation of csrc/tsdf.cu ------------------------------------------------------------------------------

def _proj(M, X, Y, Z, j):
    return ((X * M[0, j] + Y * M[1, j]) + Z * M[2, j]) + M[3, j]


def _bilinear32(m, px, py):
    H, W = m.shape
    wm1, hm1 = F(W - 1), F(H - 1)
    sx = np.minimum(np.maximum(((px + F(1)) * F(0.5)) * wm1, F(0)), wm1)
    sy = np.minimum(np.maximum(((py + F(1)) * F(0.5)) * hm1, F(0)), hm1)
    x0, y0 = np.floor(sx), np.floor(sy)
    w = sx - x0
    e = F(1) - w
    n = sy - y0
    s = F(1) - n
    ix, iy = x0.astype(np.int64), y0.astype(np.int64)
    flat = m.reshape(-1)
    base = iy * W + ix
    east, south = ix + 1 < W, iy + 1 < H
    v = flat[base] * (s * e)
    v = np.where(east, v + flat[np.where(east, base + 1, base)] * (s * w), v)
    v = np.where(south, v + flat[np.where(south, base + W, base)] * (n * e), v)
    both = east & south
    v = np.where(both, v + flat[np.where(both, base + W + 1, base)] * (n * w), v)
    return v.astype(F)


def world_and_trunc32(points, center, radius, trunc, colour):
    P = np.asarray(points, F)
    X, Y, Z = P[:, 0].copy(), P[:, 1].copy(), P[:, 2].copy()
    t0 = F(trunc)
    tr = np.full(len(P), t0, F)
    if not colour:
        mag = np.sqrt((X * X + Y * Y) + Z * Z)
        big = mag > 1
        tr[big] = t0 * (F(1) / (F(2) - np.minimum(mag[big], F(1.9))))
        un = ~(mag < 1)
        r = F(1) / (F(2) - mag[un])
        for A in (X, Y, Z):
            A[un] = r * (A[un] / mag[un])
        rf, c = F(radius), np.asarray(center, F).reshape(3)
        X, Y, Z = X * rf + c[0], Y * rf + c[1], Z * rf + c[2]
    return X, Y, Z, tr


def emulate(points, frames, center, radius, trunc, colour=False):
    """(N,) TSDF (field mode) or (N,3) RGB (colour mode), bit for bit as csrc/tsdf.cu."""
    with np.errstate(all="ignore"):
        X, Y, Z, tr = world_and_trunc32(points, center, radius, trunc, colour)
        N = len(X)
        t = np.full(N, F(-1))
        rgb = np.zeros((N, 3), F)
        wt = np.ones(N, F)
        for M, depth, cmap in frames:
            M = np.asarray(M, F)
            hw = _proj(M, X, Y, Z, 3)
            px, py = _proj(M, X, Y, Z, 0) / hw, _proj(M, X, Y, Z, 1) / hw
            idx = np.nonzero((px > -1) & (px < 1) & (py > -1) & (py < 1) & (hw > 0))[0]
            if len(idx) == 0:
                continue
            depth = np.asarray(depth, F).reshape(np.shape(depth)[-2:])
            sdf = _bilinear32(depth, px[idx], py[idx]) - hw[idx]
            acc = sdf > -tr[idx]
            j = idx[acc]
            wp = wt[j] + F(1)
            if colour:
                cmap = np.asarray(cmap, F)
                for c in range(3):
                    v = _bilinear32(cmap[c], px[j], py[j])
                    rgb[j, c] = (rgb[j, c] * wt[j] + v) / wp
            else:
                s = np.clip(sdf[acc] / tr[j], F(-1), F(1))
                t[j] = (t[j] * wt[j] + s) / wp
            wt[j] = wp
    return rgb if colour else t


# ---- float64 evaluation with a first-order rounding bound ------------------------------------------------------------

def _tri(m, e):
    """The reference decides `m > 0` from a float32 m within e of this one: (sure true, sure false, undecided)."""
    sure_t = m > e
    sure_f = np.isnan(m) | np.where(e > 0, m < -e, m <= 0)
    return sure_t, sure_f, ~sure_t & ~sure_f


def _norm_exact(P):
    """|y| is exact in float32 whatever the order of the sum: every square, partial sum and the root are."""
    sq = P * P
    ok = np.all(sq.astype(F).astype(np.float64) == sq, axis=1)
    for a, b in ((0, 1), (1, 2), (0, 2)):
        s = sq[:, a] + sq[:, b]
        ok &= s.astype(F).astype(np.float64) == s
    S = sq.sum(1)
    r = np.sqrt(S)
    ok &= (S.astype(F).astype(np.float64) == S) & (r.astype(F).astype(np.float64) == r) & (r * r == S)
    return ok


def _bilinear64(m, px, py, e_px, e_py):
    """grid_sample's value in float64, its bound, and whether the floor may differ next to a non-finite tap."""
    H, W = m.shape
    m64 = m.astype(np.float64)
    sx = np.clip((px + 1) / 2 * (W - 1), 0, W - 1)
    sy = np.clip((py + 1) / 2 * (H - 1), 0, H - 1)
    e_sx = e_px * (W - 1) / 2 + 2 * U * sx
    e_sy = e_py * (H - 1) / 2 + 2 * U * sy
    ix, iy = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
    fx, fy = sx - ix, sy - iy
    tap = lambda r, c: m64[np.clip(r, 0, H - 1), np.clip(c, 0, W - 1)]
    east, south = ix + 1 < W, iy + 1 < H
    v = tap(iy, ix) * (1 - fx) * (1 - fy)
    v = v + np.where(east, tap(iy, ix + 1) * fx * (1 - fy), 0)
    v = v + np.where(south, tap(iy + 1, ix) * (1 - fx) * fy, 0)
    v = v + np.where(east & south, tap(iy + 1, ix + 1) * fx * fy, 0)
    near = ((np.abs(sx - np.round(sx)) <= e_sx) & (e_sx > 0)) | ((np.abs(sy - np.round(sy)) <= e_sy) & (e_sy > 0))
    k = np.arange(-1, 3)
    rows, cols = np.clip(iy[:, None] + k, 0, H - 1), np.clip(ix[:, None] + k, 0, W - 1)
    nb = m64[rows[:, :, None], cols[:, None, :]]                            # (n, 4, 4) neighbourhood
    cell = nb[:, 1:3, 1:3]
    use = np.where(near[:, None, None], nb, np.pad(cell, ((0, 0), (1, 1), (1, 1)), mode="edge"))
    with np.errstate(invalid="ignore"):
        lx = np.abs(np.diff(use, axis=2)).max(axis=(1, 2))
        ly = np.abs(np.diff(use, axis=1)).max(axis=(1, 2))
        big = np.abs(cell).max(axis=(1, 2))
    flag = near & ~np.isfinite(nb).all(axis=(1, 2))
    e = lx * e_sx + ly * e_sy + 8 * U * big
    e = np.where(np.isfinite(v), e, 0.0)
    return v, e, flag


def evaluate64(points, frames, center, radius, trunc, colour=False):
    """Returns (value, bound, flagged): value (N,) or (N,3) float64, bound of the same shape, flagged (N,) bool.
    Unflagged, every correct float32 implementation of the reference lies within `bound` of `value`."""
    with np.errstate(all="ignore"):
        P = np.asarray(points, F).astype(np.float64)
        N = len(P)
        t0 = float(F(trunc))
        flagged = np.zeros(N, bool)
        if colour:
            Xw, e_X = P, np.zeros_like(P)
            tr, e_tr = np.full(N, t0), np.zeros(N)
        else:
            mag = np.sqrt((P * P).sum(1))
            e_mag = np.where(_norm_exact(P), 0.0, 4 * U * mag)
            for edge in (1.0, 2.0):
                flagged |= (np.abs(mag - edge) <= e_mag) & (e_mag > 0)
            a = 2 - np.minimum(mag, float(F(1.9)))
            e_a = np.where(mag < float(F(1.9)) + e_mag, e_mag, 0.0)
            big = mag > 1
            tr = np.where(big, t0 / a, t0)
            e_tr = np.where(big, tr * (e_a / a + 2 * U), 0.0)
            un = ~(mag < 1)
            d = 2 - mag
            p = np.where(un[:, None], (1 / d)[:, None] * (P / mag[:, None]), P)
            rel = np.where(un, e_mag / np.abs(d) + e_mag / mag + 3 * U, 0.0)
            flagged |= un & (e_mag / np.abs(d) > 2.0 ** -5)       # first order no longer holds next to |y| = 2
            e_p = np.abs(p) * rel[:, None]
            rf, c = float(F(radius)), np.asarray(center, F).astype(np.float64).reshape(3)
            Xw = p * rf + c
            e_X = e_p * rf + U * np.abs(p * rf) + U * np.abs(Xw)
        t, e_t = np.full(N, -1.0), np.zeros(N)
        rgb, e_rgb = np.zeros((N, 3)), np.zeros((N, 3))
        wt = np.ones(N)
        for M, depth, cmap in frames:
            M = np.asarray(M, F).astype(np.float64)
            h = Xw @ M[:3] + M[3]
            e_h = e_X @ np.abs(M[:3]) + 4 * U * (np.abs(Xw) @ np.abs(M[:3]) + np.abs(M[3]))
            hw, e_hw = h[:, 3], e_h[:, 3]
            pix = h[:, :2] / hw[:, None]
            e_pix = (e_h[:, :2] + np.abs(pix) * e_hw[:, None]) / np.abs(hw)[:, None] + U * np.abs(pix)
            conds = [_tri(pix[:, 0] + 1, e_pix[:, 0]), _tri(1 - pix[:, 0], e_pix[:, 0]),
                     _tri(pix[:, 1] + 1, e_pix[:, 1]), _tri(1 - pix[:, 1], e_pix[:, 1]), _tri(hw, e_hw)]
            no = np.any([cf for _, cf, _ in conds], axis=0)
            und = ~no & np.any([cu for _, _, cu in conds], axis=0)
            flagged |= und
            idx = np.nonzero(~no & ~und & ~flagged)[0]
            if len(idx) == 0:
                continue
            depth = np.asarray(depth, F).reshape(np.shape(depth)[-2:])
            dv, e_d, fl = _bilinear64(depth, pix[idx, 0], pix[idx, 1], e_pix[idx, 0], e_pix[idx, 1])
            sdf = dv - hw[idx]
            e_sdf = np.where(np.isfinite(sdf), e_d + e_hw[idx] + U * np.abs(sdf), 0.0)
            yes, no2, und2 = _tri(sdf + tr[idx], e_sdf + e_tr[idx])
            flagged[idx[fl | und2]] = True
            keep = yes & ~fl
            j, sdf, e_sdf = idx[keep], sdf[keep], e_sdf[keep]
            w = wt[j]
            if colour:
                cmap = np.asarray(cmap, F)
                for ch in range(3):
                    cv, e_c, flc = _bilinear64(cmap[ch], pix[j, 0], pix[j, 1], e_pix[j, 0], e_pix[j, 1])
                    flagged[j[flc]] = True
                    old = rgb[j, ch]
                    rgb[j, ch] = (old * w + cv) / (w + 1)
                    e_rgb[j, ch] = ((w * e_rgb[j, ch] + e_c + 2 * U * (np.abs(old) * w + np.abs(cv))) / (w + 1)
                                    + U * np.abs(rgb[j, ch]))
            else:
                q = sdf / tr[j]
                e_q = np.where(np.isfinite(q), (e_sdf + np.abs(q) * e_tr[j]) / tr[j] + U * np.abs(q), 0.0)
                s = np.clip(q, -1, 1)
                e_s = np.where((q > 1 + e_q) | (q < -1 - e_q), 0.0, e_q)
                old = t[j]
                t[j] = (old * w + s) / (w + 1)
                e_t[j] = (w * e_t[j] + e_s + 2 * U * (np.abs(old) * w + np.abs(s))) / (w + 1) + U * np.abs(t[j])
            wt[j] = w + 1
    return (rgb, e_rgb, flagged) if colour else (t, e_t, flagged)


def check_within(got, value, bound, flagged, factor=2.0):
    """Indices of unflagged samples where `got` is outside factor * bound of `value` (NaN must match NaN), and
    of flagged samples outside [-1, 1] (field) / non-finite mismatches.  Returns (bad unflagged, bad flagged)."""
    got = np.asarray(got, np.float64)
    if got.ndim == 1:
        got, value, bound = got[:, None], value[:, None], bound[:, None]
    nan_ok = np.isnan(got) == np.isnan(value)
    with np.errstate(invalid="ignore"):
        close = (np.abs(got - value) <= factor * bound) | (np.isnan(got) & np.isnan(value)) | (got == value)
    bad = np.nonzero(~flagged & ~np.all(close & nan_ok, axis=1))[0]
    return bad


# ---- eager torch restatement of the reference loop -------------------------------------------------------------------

def eager(points, depthmaps, rgbmaps, cameras, center, radius, voxel_size, colour=False):
    """The reference's compute_unbounded_tsdf restated in eager torch: per frame a projection, two grid_samples,
    masks and indexed updates.  Maps may live on the host (copied to the device every frame, as the reference
    does) or on the device.  Returns (N,) TSDF or (N,3) RGB."""
    import torch
    import torch.nn.functional as Fn
    dev = points.device
    x = points
    trunc = 5 * voxel_size
    if not colour:
        mag = torch.linalg.norm(x, dim=-1)
        tr = trunc * torch.ones_like(x[:, 0])
        far = mag > 1
        tr[far] *= 1 / (2 - mag[far].clamp(max=1.9))
        m = mag[..., None]
        x = torch.where(m < 1, x, 1 / (2 - m) * (x / m))
        x = x * radius + center
    else:
        tr = trunc
    t = -torch.ones_like(x[:, 0])
    rgb = torch.zeros((x.shape[0], 3), device=dev)
    w = torch.ones_like(x[:, 0])
    hom = torch.cat([x, torch.ones_like(x[:, :1])], -1)
    for i, cam in enumerate(cameras):
        h = hom @ cam.full_proj_transform
        z = h[:, 3:]
        pix = h[:, :2] / z
        mask = ((pix > -1) & (pix < 1) & (z > 0)).all(-1)
        grid = pix[None, None]
        d = Fn.grid_sample(depthmaps[i].to(dev)[None], grid, mode="bilinear", padding_mode="border",
                           align_corners=True).reshape(-1, 1)
        c = Fn.grid_sample(rgbmaps[i].to(dev)[None], grid, mode="bilinear", padding_mode="border",
                           align_corners=True).reshape(3, -1).T
        sdf = (d - z).flatten()
        mask = mask & (sdf > -tr)
        s = torch.clamp(sdf / tr, -1.0, 1.0)[mask]
        wm = w[mask]
        wp = wm + 1
        t[mask] = (t[mask] * wm + s) / wp
        rgb[mask] = (rgb[mask] * wm[:, None] + c[mask]) / wp[:, None]
        w[mask] = wp
    return rgb if colour else t
