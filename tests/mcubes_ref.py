"""NumPy restatement of the device marching cubes of `UnboundedTSDF.extract_mesh` (csrc/mcubes.cu, DESIGN.md §7j).
The kernels must match it bit for bit: positions as uint32, faces exactly, in the same order.  Its rules:

1. Crops.  xs = np.linspace(-R, R, n + 1) in float64; crops run in (i, j, k) order; each crop's axis is
   torch.linspace(x_min, x_max, side) on CUDA in float32 (`linspace32`); points are laid out by
   meshgrid(indexing="ij"), x slowest.  Neighbouring crops sample their shared plane at bit-identical coordinates, so
   the crops form one global grid of (side - 1) * n + 1 points per axis and every cube belongs to one crop.
2. Field.  The values are UnboundedTSDF's own (§7i); here any callable that returns a crop's side^3 values.
3. Inside and outside.  A corner is inside iff its value is < 0; exactly 0 is outside (not verified against skimage).
4. Vertex positions.  On every edge whose ends differ in side: t = va / (va - vb) and p = pa + t * (pb - pa) per
   component in float32, from the lower end a; where t is exactly 0 or 1 the vertex is that grid corner.
5. Identity.  A vertex's key is its global grid edge, point * 4 + axis, or its grid corner, point * 4 + 3; equal keys
   are one vertex.  Distinct vertices within 1e-6 of each other are not merged (`near_pairs` counts them).
   Triangles whose corners merged are kept.
6. Triangulation.  The table of diff_surfel_rasterization/mcubes_table.py (its docstring states its rule).
7. Order.  Vertices in ascending key order; faces in crop order, then cube order (x slowest), then table order.
8. Inverse contraction and clip.  §7i rule 3's uncontraction, x * radius + center, then clip to [-32, 32] (NaN stays
   NaN), after merging.
"""
from fractions import Fraction

import numpy as np

import tsdf_ref as TR
from diff_surfel_rasterization.mcubes_table import EDGE_CORNERS, generate

F = np.float32
TABLE, COUNT = generate()
MAX_RANGE = 32.0
# kLinspaceFma of csrc/contraction.cuh: torch's CUDA linspace contracts start + step * i into one FMA
LINSPACE_FMA = True


def _round32(x):
    """The float32 nearest to the Fraction x, ties to even."""
    f = np.float32(float(x))
    best = None
    for c in (np.nextafter(f, F(-np.inf)), f, np.nextafter(f, F(np.inf))):
        d = abs(Fraction(float(c)) - x)
        key = (d, int(np.array(c).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return F(best[1])


def linspace32(start, end, steps, fma=LINSPACE_FMA):
    """torch.linspace(start, end, steps) in float32 as torch's CUDA kernel computes it: start and end rounded once,
    step = (end - start) / (steps - 1) in float32, start + step * i for i < steps // 2, else
    end - step * (steps - 1 - i), each an FMA when `fma`."""
    a, b = F(start), F(end)
    if steps == 1:
        return np.array([a], F)
    step = F(F(b - a) / F(steps - 1))
    out = np.empty(steps, F)
    half = steps // 2
    for i in range(steps):
        base, s, k = (a, step, i) if i < half else (b, -step, steps - 1 - i)
        if fma:
            out[i] = _round32(Fraction(float(s)) * k + Fraction(float(base)))
        else:
            out[i] = F(base + F(s * F(k)))
    return out


def crop_bounds(R, n):
    return np.linspace(-R, R, n + 1)


def crop_axes(xs, side):
    """The float32 axis of each crop: [n] arrays of `side` values."""
    return [linspace32(xs[i], xs[i + 1], side) for i in range(len(xs) - 1)]


def _edge_t(va, vb):
    with np.errstate(all="ignore"):
        return (va / (va - vb)).astype(F)


def _keys(P, stride, d, t):
    return np.where(t == 0, P * 4 + 3, np.where(t == 1, (P + stride) * 4 + 3, P * 4 + d)).astype(np.int64)


class Mesher:
    """Marching cubes over n^3 crops of side^3 points; `add_crop` in (i, j, k) order, then `finish`."""

    def __init__(self, n, side, xs):
        self.n, self.s, self.xs = n, side, xs
        self.axes = crop_axes(xs, side)
        self.G = (side - 1) * n + 1
        self.rec_keys, self.rec_pos, self.tri_keys = [], [], []

    def add_crop(self, ijk, vol):
        s, n, G = self.s, self.n, self.G
        vol = np.asarray(vol, F).reshape(s, s, s)
        g0 = [c * (s - 1) for c in ijk]
        ax = [self.axes[c] for c in ijk]
        last = [c == n - 1 for c in ijk]
        inside = vol < 0
        strides = (G * G, G, 1)
        gp = lambda a, b, c: ((np.int64(g0[0]) + a) * G + (g0[1] + b)) * G + (g0[2] + c)
        # records: every crossing edge the crop owns
        for d in range(3):
            hi = [s if last[e] else s - 1 for e in range(3)]
            hi[d] = s - 1
            sl_a = tuple(slice(0, h) for h in hi)
            sl_b = tuple(slice(1, h + 1) if e == d else slice(0, h) for e, h in enumerate(hi))
            cross = inside[sl_a] != inside[sl_b]
            a, b, c = np.nonzero(cross)
            if len(a) == 0:
                continue
            loc = [a, b, c]
            va, vb = vol[sl_a][cross], vol[sl_b][cross]
            t = _edge_t(va, vb)
            P = gp(a, b, c)
            self.rec_keys.append(_keys(P, strides[d], d, t))
            pos = np.empty((len(a), 3), F)
            with np.errstate(all="ignore"):
                for k in range(3):
                    pa = ax[k][loc[k]]
                    pb = ax[k][loc[k] + 1] if k == d else pa
                    x = (pa + t * (pb - pa)).astype(F)
                    x = np.where(t == 0, pa, np.where(t == 1, pb, x))
                    pos[:, k] = x
            self.rec_pos.append(pos)
        # triangles: cubes in x-slowest order, then table order
        m = s - 1
        case = np.zeros((m, m, m), np.uint8)
        for k in range(8):
            dx, dy, dz = k & 1, k >> 1 & 1, k >> 2 & 1
            case |= (inside[dx:dx + m, dy:dy + m, dz:dz + m].astype(np.uint8) << k)
        ntri = COUNT[case]
        a, b, c = np.nonzero(ntri > 0)
        if len(a) == 0:
            return
        cs = case[a, b, c]
        cv = np.stack([vol[a + (k & 1), b + (k >> 1 & 1), c + (k >> 2 & 1)] for k in range(8)], 1)
        P0 = gp(a, b, c)
        rows = TABLE[cs]                                         # (cubes, MAX_TRIS, 3)
        keys = np.zeros(rows.shape, np.int64)
        for e in range(12):
            lo, hi_ = EDGE_CORNERS[e]
            d = e // 4
            off = (lo & 1) * strides[0] + (lo >> 1 & 1) * strides[1] + (lo >> 2 & 1) * strides[2]
            ke = _keys(P0 + off, strides[d], d, _edge_t(cv[:, lo], cv[:, hi_]))
            keys = np.where(rows == e, ke[:, None, None], keys)
        valid = np.arange(TABLE.shape[1])[None, :] < COUNT[cs][:, None]
        self.tri_keys.append(keys[valid])

    def finish(self, center, radius):
        """(verts (M,3) float32 world, faces (F,3) int64, contracted (M,3) float32, keys (M,) int64)."""
        keys = np.concatenate(self.rec_keys) if self.rec_keys else np.zeros(0, np.int64)
        pos = np.concatenate(self.rec_pos) if self.rec_pos else np.zeros((0, 3), F)
        tk = np.concatenate(self.tri_keys) if self.tri_keys else np.zeros((0, 3), np.int64)
        order = np.argsort(keys, kind="stable")
        ks, ps = keys[order], pos[order]
        first = np.ones(len(ks), bool)
        first[1:] = ks[1:] != ks[:-1]
        ukeys, upos = ks[first], ps[first]
        # equal keys carry equal positions (bits; NaN only from NaN values)
        rank = np.cumsum(first) - 1
        assert np.array_equal(ps.view(np.uint32), upos[rank].view(np.uint32)) or np.isnan(ps).any()
        faces = np.searchsorted(ukeys, tk).astype(np.int64)
        assert len(tk) == 0 or np.array_equal(ukeys[faces], tk)
        verts = uncontract_clip(upos, center, radius)
        return verts, faces, upos, ukeys


def uncontract_clip(pos, center, radius):
    X, Y, Z, _ = TR.world_and_trunc32(pos, center, radius, 0.0, False)
    with np.errstate(invalid="ignore"):
        return np.clip(np.stack([X, Y, Z], 1).astype(F), F(-MAX_RANGE), F(MAX_RANGE))


def mesh(n, side, xs, crop_values, center=(0, 0, 0), radius=1.0):
    """crop_values(ijk, axes) -> side^3 values, axes being the crop's three float32 axes."""
    m = Mesher(n, side, xs)
    for i in range(n):
        for j in range(n):
            for k in range(n):
                ijk = (i, j, k)
                m.add_crop(ijk, crop_values(ijk, [m.axes[c] for c in ijk]))
    return m.finish(center, radius)


def analytic(fn):
    """crop_values of an analytic field fn(X, Y, Z) -> float32 over the crop's meshgrid."""
    def values(ijk, axes):
        X, Y, Z = np.meshgrid(*axes, indexing="ij")
        return np.asarray(fn(X, Y, Z), F)
    return values


def near_pairs(pos, tol=1e-6):
    """Pairs of distinct vertices within tol of each other in every coordinate (what merge_vertices(digits=6)
    could join; this path does not)."""
    if len(pos) < 2:
        return 0
    q = np.floor(np.asarray(pos, np.float64) / tol).astype(np.int64)
    count = 0
    from collections import defaultdict
    cells = defaultdict(list)
    for idx, c in enumerate(map(tuple, q)):
        cells[c].append(idx)
    for c, members in cells.items():
        cand = list(members)
        for dx in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dz in (-1, 0, 1):
                    nb = (c[0] + dx, c[1] + dy, c[2] + dz)
                    if nb > c and nb in cells:
                        cand_nb = cells[nb]
                        for a in members:
                            for b in cand_nb:
                                count += bool(np.all(np.abs(pos[a] - pos[b]) <= tol))
        for x in range(len(cand)):
            for y in range(x + 1, len(cand)):
                count += bool(np.all(np.abs(pos[cand[x]] - pos[cand[y]]) <= tol))
    return count
