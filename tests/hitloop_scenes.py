"""Certified scenes aimed at the structure of the render kernels' hit loops (tests only).

Every scene here is built from fronto-parallel or tilted surfels placed in PIXEL units in front of the identity
camera, so a generator controls exactly which tiles a splat reaches, how many list slots a tile has, where the
transmittance of a pixel crosses 0.5 and where it saturates.  Each generator then

  * certifies the scene: every (pixel, splat) pair the A.3 walk evaluates stays at least DELTA (relative) away from
    every discontinuity of the forward (alpha >= 1/255, the 0.99 clamp, rho3d <= rho2d, depth < near,
    T (1 - alpha) < 1e-4, T > 0.5, p.z == 0), measured in float64 on the float32 preprocess output
    (oracle.decision_margins).  Offending splats are jittered until the certificate holds.  The CUDA path sits a
    few 1e-7 from the exact evaluation, so on a certified scene it cannot take a different decision from the
    float64 oracle: the GPU tests compare every entry, with no budget for flipped pixels;
  * asserts the structure it claims (list lengths, saturation, median positions, near-plane and low-pass pairs),
    from the oracle's tile ranges and n_contrib.

Frames are at most 96x96 so the float64 oracle stays fast.
"""
import functools

import numpy as np

import surfel_scenes as S

DELTA = 1e-4                       # certified: every decision margin above this (relative)
BG = np.array([0.1, 0.2, 0.3], np.float32)
NEAR = 0.2
COUNTS = (1, 31, 32, 33, 255, 256, 257, 383, 384, 385, 511, 512, 513, 1100)


class Layer:
    """Accumulates splats given in pixel units (centre cx, cy; std dev sx, sy in pixels at depth z)."""

    def __init__(self, W, H, seed):
        self.W, self.H = W, H
        self.cam = S.to_numpy(S.make_camera(W, H))
        self.f = W / (2.0 * self.cam["tanfovx"])
        self.rng = np.random.default_rng(seed)
        self.cols = {k: [] for k in ("cx", "cy", "z", "sx", "sy", "opa", "quat")}

    def add(self, cx, cy, z, sx, sy, opa, quat=(1.0, 0.0, 0.0, 0.0)):
        n = max(np.size(cx), np.size(cy), np.size(z), np.size(opa))
        b = lambda v: np.broadcast_to(np.asarray(v, np.float64), (n,))
        for k, v in (("cx", cx), ("cy", cy), ("z", z), ("sx", sx), ("sy", sy), ("opa", opa)):
            self.cols[k].append(b(v).copy())
        self.cols["quat"].append(np.broadcast_to(np.asarray(quat, np.float64), (n, 4)).copy())
        return self

    def scene(self):
        c = {k: np.concatenate(v) for k, v in self.cols.items()}
        P = c["z"].shape[0]
        W, H, f = self.W, self.H, self.f
        means = np.stack([(c["cx"] - (W - 1) / 2) * c["z"] / f, (c["cy"] - (H - 1) / 2) * c["z"] / f, c["z"]], 1)
        scales = np.stack([c["sx"] * c["z"] / f, c["sy"] * c["z"] / f], 1)
        q = c["quat"] / np.linalg.norm(c["quat"], axis=1, keepdims=True)
        shs = self.rng.normal(0.0, 0.25, (P, 16, 3))
        shs[:, 0] = self.rng.uniform(-0.5, 1.2, (P, 3))
        return dict(means3D=means.astype(np.float32), scales=scales.astype(np.float32),
                    rotations=q.astype(np.float32), opacities=c["opa"][:, None].astype(np.float32),
                    shs=shs.astype(np.float32)), c


def uniform(layer, n, z0, z1, alpha=(0.0045, 0.0065)):
    """n splats that cover the whole frame with G ~ 1 (std dev 400 px): every pixel of every tile gets them, with
    alpha far from both thresholds."""
    r = layer.rng
    return layer.add(layer.W / 2 + r.uniform(-3, 3, n) + 0.37, layer.H / 2 + r.uniform(-3, 3, n) + 0.29,
                     np.sort(r.uniform(z0, z1, n)), 400.0, 400.0, r.uniform(*alpha, n))


def fillers(layer, n, tx, ty, z0, z1):
    """n small splats inside tile (tx, ty) with opacity 0.003 < 1/255: they occupy list slots of that tile only and
    never contribute (alpha stays 23 % below the threshold everywhere)."""
    r = layer.rng
    return layer.add(tx * 16 + 7.5 + r.uniform(-0.5, 0.5, n), ty * 16 + 7.5 + r.uniform(-0.5, 0.5, n),
                     np.sort(r.uniform(z0, z1, n)), 2.0, 2.0, 0.003)


def hot(layer, n, cx, cy, sigma, z0, z1, opa):
    """n splats centred at (cx, cy) (usually outside the frame) with a strong alpha gradient across it; the caller
    keeps alpha above 1/255 on every evaluated pixel, so no alpha contour lies inside the frame."""
    r = layer.rng
    return layer.add(cx + r.uniform(-1, 1, n), cy + r.uniform(-1, 1, n), np.sort(r.uniform(z0, z1, n)),
                     sigma, sigma, opa * r.uniform(0.9, 1.0, n))


# ---------------------------------------------------------------------------------------------- certification
def run_oracle(O, scene, cam, rows=None):
    W, H = cam["W"], cam["H"]
    gy = (H + 15) // 16
    r0, r1 = (0, gy) if rows is None else rows
    pre = O.preprocess_fwd(scene["means3D"], scene["scales"], scene["rotations"], scene["opacities"], scene["shs"],
                           cam["viewmatrix"], cam["projmatrix"], cam["campos"], W, H, 3, 1.0, None, None, r0, r1)
    binned = O.bin_sort(pre, W, H, r0, r1)
    return pre, binned


def certify(O, layer, rows=None, max_iter=40):
    """Jitter the splats that take part in a pair closer than DELTA to a discontinuity, or that set the transmittance
    such a pair is tested against (opacity by up to 3 %, centre by up to 0.05 px), until none is left.  Returns a dict
    with the scene, camera, preprocess, binning, float64 forward and the margins."""
    scene, _ = layer.scene()
    cam = layer.cam
    W, H = cam["W"], cam["H"]
    for it in range(max_iter):
        pre, binned = run_oracle(O, scene, cam, rows)
        margins, per_splat = O.decision_margins(pre, binned, W, H)
        bad = np.nonzero(per_splat < DELTA)[0]
        if bad.size == 0:
            img = O.render_fwd(pre, binned, BG, W, H, f64=True)
            worst = min(float(m.min()) for m in margins.values())
            return dict(scene=scene, cam=cam, pre=pre, binned=binned, img=img, margins=margins, worst=worst,
                        rows=rows, jitter_rounds=it)
        r = layer.rng
        scene = {k: v.copy() for k, v in scene.items()}
        scene["opacities"][bad, 0] = (scene["opacities"][bad, 0] * r.uniform(0.97, 1.03, bad.size)).astype(np.float32)
        z = scene["means3D"][bad, 2].astype(np.float64)
        shift = r.uniform(-0.05, 0.05, (bad.size, 2)) * z[:, None] / layer.f
        scene["means3D"][bad, :2] = (scene["means3D"][bad, :2] + shift).astype(np.float32)
    raise AssertionError(f"scene not certified after {max_iter} rounds of jitter: {bad.size} splats within {DELTA}")


def tile_lengths(s):
    r = s["binned"]["ranges"].astype(np.int64)
    return r[:, 1] - r[:, 0]


def assert_certified(s):
    for name, m in s["margins"].items():
        assert m.min() >= DELTA, f"margin {name} = {m.min():.3e} < {DELTA}"


# ---------------------------------------------------------------------------------------------- generators
# Each returns the certified scene dict; they are cached per process (the GPU test and the CPU structure test
# share them).  `O` is the oracle module.

@functools.lru_cache(maxsize=None)
def count_sweep(O, k):
    """Every tile of a 32x32 frame holds exactly k contributors, and every pixel blends all k (T stays > 1e-4)."""
    layer = Layer(32, 32, seed=1000 + k)
    uniform(layer, k, 2.0, 12.0)
    s = certify(O, layer)
    assert (tile_lengths(s) == k).all(), tile_lengths(s)
    assert (s["img"]["n_contrib"][0] == k).all()
    return s


@functools.lru_cache(maxsize=None)
def warps_apart(O):
    """Lists of 540 slots (two forward rounds, three backward rounds).  Splats with a strong alpha gradient from the
    top-left corner saturate the pixels near it within the first 40 slots, while the far pixels never saturate and
    run to the end of the list: warps (and pixels inside one warp) finish in different rounds."""
    layer = Layer(32, 32, seed=7)
    hot(layer, 40, -5.0, -5.0, 20.0, 2.0, 2.5, 0.9)
    uniform(layer, 500, 3.0, 12.0)
    s = certify(O, layer)
    n0 = s["img"]["n_contrib"][0].astype(np.int64)
    assert (tile_lengths(s) == 540).all()
    assert n0.min() <= 40 and n0.max() == 540, (n0.min(), n0.max())
    # at least one warp footprint (8x4) mixes saturated and unsaturated pixels, and one is all saturated early
    fp = n0.reshape(8, 4, 4, 8).transpose(0, 2, 1, 3).reshape(32, 32)
    assert ((fp.min(1) < 540) & (fp.max(1) == 540)).any()
    assert (fp.max(1) <= 40).any()
    return s


@functools.lru_cache(maxsize=None)
def all_saturate(O):
    """Lists of 1000 slots; every pixel saturates between slots ~410 and ~430 (second forward round, second backward
    round): the forward leaves through the CTA-wide early exit and the backward starts at cta_max < list length."""
    layer = Layer(32, 32, seed=8)
    uniform(layer, 400, 2.0, 4.0)
    hot(layer, 60, -8.0, -8.0, 40.0, 4.5, 5.0, 0.5)
    uniform(layer, 540, 6.0, 12.0)
    s = certify(O, layer)
    n0 = s["img"]["n_contrib"][0].astype(np.int64)
    assert (tile_lengths(s) == 1000).all()
    assert (s["img"]["accum"][0] < 1e-3).all(), "every pixel must saturate"
    assert n0.max() < 768 and n0.max() > 384 and n0.min() > 384 and n0.min() < n0.max(), (n0.min(), n0.max())
    return s


MEDIAN_TARGETS = (32, 64, 96, 256, 288, 512)      # each tile puts medians on target - 1, target, target + 1


@functools.lru_cache(maxsize=None)
def median_boundaries(O):
    """A 64x48 frame (12 tiles).  Big splats with an alpha gradient across the frame make T cross 0.5 after 5 to 15
    of them, depending on the pixel; per-tile fillers in front of them (never blended) shift the crossing so that
    it lands on list positions 32n +- 1 and 256n +- 1 in different tiles."""
    W, H = 64, 48
    probe = Layer(W, H, seed=9)
    hot(probe, 24, -10.0, -5.0, 30.0, 6.0, 8.0, 0.3)
    ps = certify(O, probe)
    med = ps["img"]["n_contrib"][1].astype(np.int64)
    # tiles whose pixels put the crossing on at least three consecutive positions c-1, c, c+1
    good = []
    for t in range(12):
        tm = med[(t // 4) * 16:(t // 4 + 1) * 16, (t % 4) * 16:(t % 4 + 1) * 16]
        c = int(np.median(tm))
        if all((tm == c + d).any() for d in (-1, 0, 1)):
            good.append((t, c))
    assert len(good) >= len(MEDIAN_TARGETS), good
    layer = Layer(W, H, seed=9)
    hot(layer, 24, -10.0, -5.0, 30.0, 6.0, 8.0, 0.3)
    for (t, c), target in zip(good, MEDIAN_TARGETS):
        fillers(layer, target - c, t % 4, t // 4, 2.0, 5.0)
    s = certify(O, layer)
    med = s["img"]["n_contrib"][1].astype(np.int64)
    for target in MEDIAN_TARGETS:
        for d in (-1, 0, 1):
            assert (med == target + d).any(), f"no pixel has its median at list position {target + d}"
    return s


@functools.lru_cache(maxsize=None)
def near_plane(O):
    """Tilted splats close to the camera whose ray-splat depth crosses the near plane (0.2) inside a tile: the
    forward skips their pairs in front of it and the backward writes zero rows for them.  Big splats behind keep
    the pixels covered."""
    W = H = 48
    layer = Layer(W, H, seed=10)
    r = layer.rng
    for i in range(4):
        a = np.deg2rad(r.uniform(37, 43)) * (1 if i < 2 else -1) / 2
        axis = (0.0, 1.0, 0.0) if i % 2 == 0 else (1.0, 0.0, 0.0)
        quat = (np.cos(a), np.sin(a) * axis[0], np.sin(a) * axis[1], np.sin(a) * axis[2])
        layer.add(r.uniform(18, 30), r.uniform(18, 30), r.uniform(0.24, 0.26), 20.0, 20.0, r.uniform(0.3, 0.5), quat)
    uniform(layer, 40, 2.0, 6.0, alpha=(0.03, 0.05))
    s = certify(O, layer)
    flagged = near_pairs(s)
    assert flagged["skipped"] > 50 and flagged["blended"] > 50, flagged
    return s


@functools.lru_cache(maxsize=None)
def low_pass(O):
    """Sub-pixel splats (std dev 0.15-0.45 px, below the low-pass filter's 0.707): most of their blended pairs take the low-pass branch
    (rho2d < rho3d), over a background of big splats."""
    W = H = 48
    layer = Layer(W, H, seed=13)
    r = layer.rng
    n = 400
    layer.add(r.uniform(0, W - 1, n), r.uniform(0, H - 1, n), r.uniform(2.0, 3.0, n), r.uniform(0.15, 0.45, n),
              r.uniform(0.15, 0.45, n), r.uniform(0.3, 0.9, n))
    uniform(layer, 40, 3.5, 12.0, alpha=(0.03, 0.05))
    s = certify(O, layer)
    lp = low_pass_pairs(s)
    assert lp > 1000, lp
    return s


RAGGED = ((49, 33), (40, 36), (41, 37), (13, 37), (41, 1))


@functools.lru_cache(maxsize=None)
def ragged(O, W, H):
    """W mod 16 in {1, 8, 9}, H mod 16 in {1, 4, 5}, W < 16 and H = 1: whole warps of the edge tiles lie outside the
    image.  Lists of 300 slots (two backward rounds), saturation near the bottom-right corner."""
    layer = Layer(W, H, seed=100 * W + H)
    uniform(layer, 260, 3.0, 12.0)
    hot(layer, 40, W + 6.0, H + 6.0, 20.0, 2.0, 2.5, 0.9)
    s = certify(O, layer)
    assert (tile_lengths(s) == 300).all()
    return s


@functools.lru_cache(maxsize=None)
def tile_band(O):
    """The warps-apart construction on a 32x64 frame rendered as the tile band of rows [1, 4): row0 > 0."""
    layer = Layer(32, 64, seed=12)
    hot(layer, 40, 10.0, 20.0, 20.0, 2.0, 2.5, 0.9)
    uniform(layer, 500, 3.0, 12.0)
    s = certify(O, layer, rows=(1, 4))
    L = tile_lengths(s).reshape(4, 2)
    assert (L[0] == 0).all() and (L[1:] == 540).all(), L
    return s


def all_scenes(O):
    """(name, certified scene) of every generator."""
    out = [(f"count{k}", count_sweep(O, k)) for k in COUNTS]
    out += [("warps_apart", warps_apart(O)), ("all_saturate", all_saturate(O)),
            ("median_boundaries", median_boundaries(O)), ("near_plane", near_plane(O)), ("low_pass", low_pass(O)),
            ("tile_band", tile_band(O))]
    out += [(f"ragged{W}x{H}", ragged(O, W, H)) for W, H in RAGGED]
    return out


# ---------------------------------------------------------------------------------------------- structure probes
def _pairs(s):
    """float64 evaluation of every (pixel, splat) pair of every tile list, in list order (small scenes only)."""
    pre, binned, cam = s["pre"], s["binned"], s["cam"]
    W, H = cam["W"], cam["H"]
    gx = (W + 15) // 16
    for tile, (a, b) in enumerate(binned["ranges"].astype(np.int64)):
        if b <= a:
            continue
        tx, ty = tile % gx, tile // gx
        ys, xs = np.mgrid[ty * 16:min(H, ty * 16 + 16), tx * 16:min(W, tx * 16 + 16)]
        px, py = xs.ravel().astype(np.float64), ys.ravel().astype(np.float64)
        ids = binned["vals_sorted"][a:b]
        T = pre["transMat"][ids].astype(np.float64)
        Tu, Tv, Tw = T[:, None, 0:3], T[:, None, 3:6], T[:, None, 6:9]
        k = px[None, :, None] * Tw - Tu
        l = py[None, :, None] * Tw - Tv
        p = np.cross(k, l)
        sx, sy = p[..., 0] / p[..., 2], p[..., 1] / p[..., 2]
        rho3d = sx * sx + sy * sy
        c = pre["xy"][ids].astype(np.float64)
        rho2d = 2.0 * ((c[:, None, 0] - px) ** 2 + (c[:, None, 1] - py) ** 2)
        depth = np.where(rho3d <= rho2d, sx * Tw[..., 0] + sy * Tw[..., 1] + Tw[..., 2], Tw[..., 2])
        alpha = np.minimum(0.99, pre["normal_opacity"][ids, 3].astype(np.float64)[:, None]
                           * np.exp(-0.5 * np.minimum(rho3d, rho2d)))
        yield ids, px.astype(np.int64), py.astype(np.int64), rho3d, rho2d, depth, alpha


def near_pairs(s):
    """Pairs that pass the alpha test with the ray-splat depth below / above the near plane, among pixels that get
    as far as the pair (n_contrib): the forward skips the first, blends the second."""
    n0 = s["img"]["n_contrib"][0].astype(np.int64)
    skipped = blended = 0
    for ids, px, py, rho3d, rho2d, depth, alpha in _pairs(s):
        pos = np.arange(1, len(ids) + 1)[:, None]
        reached = pos <= n0[py, px][None, :]
        ok = (alpha >= 1 / 255) & reached
        skipped += int((ok & (depth < NEAR)).sum())
        blended += int((ok & (depth >= NEAR) & (depth < 0.3)).sum())
    return dict(skipped=skipped, blended=blended)


def low_pass_pairs(s):
    """Number of blended pairs in the low-pass branch."""
    n0 = s["img"]["n_contrib"][0].astype(np.int64)
    count = 0
    for ids, px, py, rho3d, rho2d, depth, alpha in _pairs(s):
        pos = np.arange(1, len(ids) + 1)[:, None]
        count += int(((alpha >= 1 / 255) & (rho2d < rho3d) & (pos <= n0[py, px][None, :])).sum())
    return count


# ---------------------------------------------------------------------------------------------- cotangents
CHANNEL_GROUPS = ("all", "color", "depth", "alpha", "normal", "median", "distortion")


def cotangent(W, H, group, seed=0):
    """(dL_dcolor (3,H,W), dL_dothers (7,H,W)): random normal in every channel ("all") or in one group only."""
    rng = np.random.default_rng(seed)
    gc = rng.normal(size=(3, H, W)).astype(np.float32)
    go = rng.normal(size=(7, H, W)).astype(np.float32)
    if group == "all":
        return gc, go
    keep = dict(depth=[0], alpha=[1], normal=[2, 3, 4], median=[5], distortion=[6]).get(group, [])
    mask = np.zeros((7, 1, 1), np.float32)
    mask[keep] = 1.0
    return (gc if group == "color" else np.zeros_like(gc)), go * mask
