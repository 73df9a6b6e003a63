"""Certified scenes for preprocess backward (tests only).

Every scene is seen through a rotated, offset camera (look_at_rotation, t != 0) on a non-square frame, with splats
placed in view space (pixel position, depth, pixel-sized extents) and carried to world space.  Each builder asserts
the feature it is named for and certifies, in float64, the one decision preprocess backward takes on its own: the
dual-visible normal sign, |c| / |p_view| >= SIGN_MARGIN with c = -p_view . n_view (offending splats are re-drawn).
The clamp scene also certifies |raw rgb| >= RGB_MARGIN for every active degree, so the clamp bits cannot depend
on rounding.  SH rows carry 25 coefficients; a case slices the M it needs.
"""
import functools

import numpy as np

import surfel_scenes as S

SIGN_MARGIN = 1e-3
RGB_MARGIN = 1e-3
CAMS = {"A": (200, 120, 20.0, -10.0, (0.3, -0.2, 0.5)), "B": (333, 171, -35.0, 15.0, (-0.4, 0.1, 0.2))}
LAYOUT_P = (1, 31, 32, 33, 127, 128, 129, 1000, 4097)
SCENES = ("orient", "grazing", "unnormalised", "clamp", "low_pass", "near", "distance") + tuple(f"layout{P}" for P in LAYOUT_P)
C0 = 0.28209479177387814


def camera(which):
    W, H, yaw, pitch, t = CAMS[which]
    return S.make_camera(W, H, R=S.look_at_rotation(yaw, pitch), t=list(t))


def _vm(cam):
    return np.asarray(cam["viewmatrix"], np.float64)


def rotmat_to_quat(R):
    """(P,3,3) proper rotations -> (P,4) unit quaternions (w, x, y, z) in the convention of dense_torch.quat_to_R."""
    q = np.zeros((R.shape[0], 4))
    for i, m in enumerate(R):
        tr = np.trace(m)
        if tr > 0:
            s = 2.0 * np.sqrt(tr + 1.0)
            q[i] = (0.25 * s, (m[2, 1] - m[1, 2]) / s, (m[0, 2] - m[2, 0]) / s, (m[1, 0] - m[0, 1]) / s)
        else:
            k = int(np.argmax(np.diag(m)))
            a, b = (k + 1) % 3, (k + 2) % 3
            s = 2.0 * np.sqrt(1.0 + m[k, k] - m[a, a] - m[b, b])
            v = np.zeros(3)
            v[k] = 0.25 * s
            v[a] = (m[a, k] + m[k, a]) / s
            v[b] = (m[b, k] + m[k, b]) / s
            q[i] = ((m[b, a] - m[a, b]) / s, *v)
    return q


def quat_to_R(q):
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)


def frame_from_normal(n, rng):
    """Rotations (columns a, b, n with a x b = n) for unit view-space normals n, random in-plane angle."""
    t = rng.normal(size=n.shape)
    a = t - (t * n).sum(1, keepdims=True) * n
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    b = np.cross(n, a)
    return np.stack([a, b, n], 2)


class Builder:
    """Splats in view space: pixel (u, v), view depth z, extents in pixels, view-space rotation."""

    def __init__(self, which, seed):
        self.cam = camera(which)
        self.W, self.H = self.cam["W"], self.cam["H"]
        self.f = self.W / (2.0 * self.cam["tanfovx"])
        self.rng = np.random.default_rng(seed)
        self.p, self.s, self.Rv, self.opa = [], [], [], []

    def view_point(self, u, v, z):
        return np.stack([(u - (self.W - 1) / 2) * z / self.f, (v - (self.H - 1) / 2) * z / self.f, z], 1)

    def add(self, pv, su_px, sv_px, Rv, opa):
        n = pv.shape[0]
        depth = np.abs(pv[:, 2]).clip(0.2)
        self.p.append(pv)
        self.s.append(np.stack([np.broadcast_to(su_px, (n,)) * depth / self.f, np.broadcast_to(sv_px, (n,)) * depth / self.f], 1))
        self.Rv.append(Rv)
        self.opa.append(np.broadcast_to(opa, (n,)).astype(np.float64))
        return self

    def random_rot(self, n):
        q = self.rng.normal(size=(n, 4))
        return quat_to_R(q)

    def build(self, qscale=None, shs=None):
        V = _vm(self.cam)
        V3, t = V[:3, :3], V[3, :3]
        pv, Rv = np.concatenate(self.p), np.concatenate(self.Rv)
        P = pv.shape[0]
        means = (pv - t) @ V3.T                 # p_view = p_world V3 + t, V3 orthonormal
        Rw = np.einsum("ij,pjk->pik", V3, Rv)   # directions: d_world = V3 d_view
        q = rotmat_to_quat(Rw)
        if qscale is not None:
            q = q * qscale[:, None]
        if shs is None:
            shs = self.rng.normal(0.0, 0.25, (P, 25, 3))
            shs[:, 0] = self.rng.uniform(-0.5, 1.2, (P, 3))
        scene = dict(means3D=means.astype(np.float32), scales=np.concatenate(self.s).astype(np.float32),
                     rotations=q.astype(np.float32), opacities=np.concatenate(self.opa)[:, None].astype(np.float32),
                     shs=np.asarray(shs, np.float32))
        return scene


# ---------------------------------------------------------------------------------------------- float64 geometry
def view_geometry(scene, cam):
    """(p_view (P,3), view-space normal (P,3), c = -p_view . n) in float64 from the float32 inputs."""
    V = _vm(cam)
    m = scene["means3D"].astype(np.float64)
    pv = m @ V[:3, :3] + V[3, :3]
    R = quat_to_R(scene["rotations"].astype(np.float64))
    nv = R[:, :, 2] @ V[:3, :3]
    return pv, nv, -(pv * nv).sum(1)


def sign_margin(scene, cam):
    """|c| / |p_view| per splat in front of the near plane (inf elsewhere)."""
    pv, nv, c = view_geometry(scene, cam)
    m = np.abs(c) / np.linalg.norm(pv, axis=1)
    return np.where(pv[:, 2] > 0.2, m, np.inf)


def raw_rgb(scene, cam, D):
    from oracle import dense_torch as DT
    import torch
    m = torch.tensor(scene["means3D"], dtype=torch.float64)
    d = m - torch.as_tensor(np.asarray(cam["campos"], np.float64))[None]
    sh = torch.tensor(scene["shs"], dtype=torch.float64)
    return (DT.eval_sh(D, sh, d / d.norm(dim=1, keepdim=True)) + 0.5).numpy()


def _certify_sign(b, scene, redraw, tries=20):
    """Re-draw (redraw(idx) -> new view-space rotations) the splats under SIGN_MARGIN until none is left."""
    for _ in range(tries):
        bad = np.nonzero(sign_margin(scene, b.cam) < SIGN_MARGIN)[0]
        if bad.size == 0:
            return scene
        Rv = np.concatenate(b.Rv)
        Rv[bad] = redraw(bad)
        b.Rv = [Rv]
        q = scene["rotations"].astype(np.float64)
        qn = np.linalg.norm(q, axis=1)
        V3 = _vm(b.cam)[:3, :3]
        Rw = np.einsum("ij,pjk->pik", V3, Rv[bad])
        q[bad] = rotmat_to_quat(Rw) * qn[bad, None]
        scene["rotations"] = q.astype(np.float32)
    raise AssertionError("dual-visible sign margin not certified")


def _done(name, b, scene, **features):
    scene = _certify_sign(b, scene, lambda idx: b.random_rot(idx.size))
    assert sign_margin(scene, b.cam).min() >= SIGN_MARGIN
    return dict(name=name, scene=scene, cam=b.cam, features=features)


# ---------------------------------------------------------------------------------------------- scenes
def _uv(b, n, margin=10.0):
    r = b.rng
    return r.uniform(margin, b.W - 1 - margin, n), r.uniform(margin, b.H - 1 - margin, n)


@functools.lru_cache(maxsize=None)
def orient():
    """Uniformly random orientations, anisotropy 1..300, half front-facing and half back-facing."""
    b = Builder("A", seed=1)
    r, n = b.rng, 240
    u, v = _uv(b, n)
    pv = b.view_point(u, v, r.uniform(2.0, 8.0, n))
    s0 = r.uniform(3.0, 12.0, n)
    aniso = np.exp(r.uniform(0.0, np.log(300.0), n))
    swap = r.random(n) < 0.5
    su, sv = np.where(swap, s0 / aniso, s0), np.where(swap, s0, s0 / aniso)
    Rv = b.random_rot(n)
    # split by the sign of c: even splats face the camera, odd ones face away (flip the normal: R diag(1, -1, -1))
    c = -(pv * Rv[:, :, 2]).sum(1)
    want = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    flip = np.sign(c) != want
    Rv[flip] = Rv[flip] * np.array([1.0, -1.0, -1.0])[None, None, :]
    b.add(pv, su, sv, Rv, r.uniform(0.2, 0.6, n))
    s = _done("orient", b, b.build(), max_aniso=float(aniso.max()))
    _, _, c = view_geometry(s["scene"], b.cam)
    s["features"].update(front=int((c > 0).sum()), back=int((c < 0).sum()))
    return s


def _grazing_rot(b, pv, lo=2.0, hi=10.0):
    n_ = pv.shape[0]
    r = b.rng
    ray = pv / np.linalg.norm(pv, axis=1, keepdims=True)
    t = r.normal(size=(n_, 3))
    e = t - (t * ray).sum(1, keepdims=True) * ray
    e /= np.linalg.norm(e, axis=1, keepdims=True)
    phi = np.deg2rad(r.uniform(lo, hi, n_)) * np.where(r.random(n_) < 0.5, 1.0, -1.0)
    nrm = np.sin(phi)[:, None] * ray + np.cos(phi)[:, None] * e
    return frame_from_normal(nrm, r)


@functools.lru_cache(maxsize=None)
def grazing():
    """Normals 2-10 degrees from perpendicular to the view ray, both signs."""
    b = Builder("B", seed=2)
    r, n = b.rng, 200
    u, v = _uv(b, n)
    pv = b.view_point(u, v, r.uniform(2.0, 8.0, n))
    Rv = _grazing_rot(b, pv)
    b.add(pv, r.uniform(4.0, 12.0, n), r.uniform(4.0, 12.0, n), Rv, r.uniform(0.2, 0.6, n))
    scene = b.build()
    pvw, nv, c = view_geometry(scene, b.cam)
    ang = np.rad2deg(np.arcsin(np.abs(c) / np.linalg.norm(pvw, axis=1)))
    assert ang.min() > 1.9 and ang.max() < 10.1, (ang.min(), ang.max())
    s = _done("grazing", b, scene, min_angle_deg=float(ang.min()), max_angle_deg=float(ang.max()),
              front=int((c > 0).sum()), back=int((c < 0).sum()))
    return s


@functools.lru_cache(maxsize=None)
def unnormalised():
    """|q| log-uniform in [1e-2, 1e2]."""
    b = Builder("A", seed=3)
    r, n = b.rng, 200
    u, v = _uv(b, n)
    pv = b.view_point(u, v, r.uniform(2.0, 8.0, n))
    b.add(pv, r.uniform(3.0, 10.0, n), r.uniform(1.0, 10.0, n), b.random_rot(n), r.uniform(0.2, 0.6, n))
    qs = np.exp(r.uniform(np.log(1e-2), np.log(1e2), n))
    scene = b.build(qscale=qs)
    qn = np.linalg.norm(scene["rotations"].astype(np.float64), axis=1)
    return _done("unnormalised", b, scene, min_qnorm=float(qn.min()), max_qnorm=float(qn.max()))


def clamp_patterns(scene, cam, D):
    raw = raw_rgb(scene, cam, D)
    return (raw < 0).astype(np.int64) @ np.array([1, 2, 4]), raw


@functools.lru_cache(maxsize=None)
def clamp():
    """Every one of the 8 clamp patterns on 16 splats: DC chosen so that raw rgb = +-(0.2..0.5) at degree 3, with
    higher coefficients small enough (0.01) that every degree keeps the pattern and |raw| >= RGB_MARGIN."""
    b = Builder("B", seed=4)
    r, n = b.rng, 128
    u, v = _uv(b, n)
    pv = b.view_point(u, v, r.uniform(2.0, 8.0, n))
    b.add(pv, r.uniform(3.0, 10.0, n), r.uniform(3.0, 10.0, n), b.random_rot(n), r.uniform(0.2, 0.6, n))
    shs = r.normal(0.0, 0.01, (n, 25, 3))
    shs[:, 0] = 0.0
    scene = b.build(shs=shs)
    pat = np.arange(n) % 8
    bits = (pat[:, None] >> np.arange(3)[None]) & 1
    target = np.where(bits == 1, -1.0, 1.0) * r.uniform(0.2, 0.5, (n, 3))
    rest = raw_rgb(scene, b.cam, 3) - 0.5
    shs = scene["shs"].astype(np.float64)
    shs[:, 0] = (target - 0.5 - rest) / C0
    scene["shs"] = shs.astype(np.float32)
    s = _done("clamp", b, scene)
    for D in range(4):
        got, raw = clamp_patterns(s["scene"], s["cam"], D)
        assert np.abs(raw).min() >= RGB_MARGIN and (got == pat).all(), D
    s["features"]["splats_per_pattern"] = int(np.bincount(pat, minlength=8).min())
    return s


@functools.lru_cache(maxsize=None)
def low_pass():
    """Sub-pixel splats (std dev 0.15-0.45 px) over big background splats: the low-pass branch writes dL_dmean2D and
    Zl into their records."""
    b = Builder("A", seed=5)
    r, n = b.rng, 260
    u, v = _uv(b, n, 2.0)
    pv = b.view_point(u, v, r.uniform(2.0, 3.0, n))
    b.add(pv, r.uniform(0.15, 0.45, n), r.uniform(0.15, 0.45, n), b.random_rot(n), r.uniform(0.3, 0.9, n))
    m = 40
    u, v = _uv(b, m)
    b.add(b.view_point(u, v, r.uniform(4.0, 10.0, m)), r.uniform(20, 40, m), r.uniform(20, 40, m), b.random_rot(m),
          r.uniform(0.05, 0.1, m))
    return _done("low_pass", b, b.build(), sub_pixel=n)


def near_crossing(scene, cam):
    """Splats in front of the near plane whose cutoff disk (3 sigma) reaches behind it in view depth."""
    V = _vm(cam)
    pv, _, _ = view_geometry(scene, cam)
    R = quat_to_R(scene["rotations"].astype(np.float64))
    s = scene["scales"].astype(np.float64)
    dz = np.hypot((R[:, :, 0] @ V[:3, 2]) * s[:, 0], (R[:, :, 1] @ V[:3, 2]) * s[:, 1])
    return (pv[:, 2] > 0.2) & (pv[:, 2] - 3.0 * dz < 0.2)


@functools.lru_cache(maxsize=None)
def near():
    """Tilted splats just beyond the near plane whose extent reaches in front of it (the render record's near flag),
    over background splats."""
    b = Builder("B", seed=6)
    r, n = b.rng, 24
    u, v = _uv(b, n, 30.0)
    pv = b.view_point(u, v, r.uniform(0.24, 0.3, n))
    tilt = np.deg2rad(r.uniform(30, 50, n))
    axis = r.normal(size=(n, 3)) * np.array([1.0, 1.0, 0.0])
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    nrm = np.cos(tilt)[:, None] * np.array([0.0, 0.0, -1.0]) + np.sin(tilt)[:, None] * axis
    b.add(pv, r.uniform(25.0, 40.0, n), r.uniform(25.0, 40.0, n), frame_from_normal(nrm, r), r.uniform(0.2, 0.4, n))
    m = 60
    u, v = _uv(b, m)
    b.add(b.view_point(u, v, r.uniform(2.0, 6.0, m)), r.uniform(5, 15, m), r.uniform(5, 15, m), b.random_rot(m),
          r.uniform(0.2, 0.5, m))
    s = _done("near", b, b.build())
    s["features"]["near_crossing"] = int(near_crossing(s["scene"], s["cam"]).sum())
    return s


@functools.lru_cache(maxsize=None)
def distance():
    """|p - campos| log-uniform from 0.25 to 90, on rays through the central part of the frame."""
    b = Builder("A", seed=7)
    r, n = b.rng, 200
    u, v = r.uniform(0.35 * b.W, 0.65 * b.W, n), r.uniform(0.35 * b.H, 0.65 * b.H, n)
    ray = b.view_point(u, v, np.ones(n))
    ray /= np.linalg.norm(ray, axis=1, keepdims=True)
    dist = np.exp(np.linspace(np.log(0.25), np.log(90.0), n))
    r.shuffle(dist)
    pv = ray * dist[:, None]
    b.add(pv, r.uniform(2.0, 8.0, n), r.uniform(2.0, 8.0, n), b.random_rot(n), r.uniform(0.1, 0.4, n))
    scene = b.build()
    d = np.linalg.norm(scene["means3D"].astype(np.float64) - np.asarray(b.cam["campos"], np.float64), axis=1)
    return _done("distance", b, scene, min_dist=float(d.min()), max_dist=float(d.max()))


@functools.lru_cache(maxsize=None)
def layout(P):
    """P generic splats; every third one behind the camera, so warps mix culled and visible rows."""
    b = Builder("A" if P % 2 else "B", seed=100 + P)
    r = b.rng
    u, v = _uv(b, P, 4.0)
    z = np.where(np.arange(P) % 3 == 2, r.uniform(-2.0, 0.1, P), r.uniform(2.0, 10.0, P))
    pv = b.view_point(u, v, z)
    b.add(pv, r.uniform(2.0, 8.0, P), r.uniform(1.0, 8.0, P), b.random_rot(P), r.uniform(0.1, 0.5, P))
    scene = b.build()
    pvw, _, _ = view_geometry(scene, b.cam)
    return _done(f"layout{P}", b, scene, behind=int((pvw[:, 2] <= 0.2).sum()))


def get(name):
    if name.startswith("layout"):
        return layout(int(name[6:]))
    return globals()[name]()


def with_sh(scene, M):
    """The scene with its SH rows cut to M coefficients."""
    s = dict(scene)
    s["shs"] = np.ascontiguousarray(scene["shs"][:, :M])
    return s


def colors_precomp(scene, seed=0):
    s = {k: v for k, v in scene.items() if k != "shs"}
    s["colors_precomp"] = np.random.default_rng(seed).uniform(0.0, 1.0, (scene["means3D"].shape[0], 3)).astype(np.float32)
    return s


def transmat_precomp(scene, transMat, radii, seed=0):
    """transMat_precomp + colors_precomp from a forward's T (culled rows get a harmless T)."""
    s = colors_precomp(scene, seed)
    T = np.asarray(transMat, np.float32).copy()
    T[np.asarray(radii) == 0] = np.array([1, 0, 0, 0, 1, 0, 0, 0, 5], np.float32)
    s["transMat_precomp"] = T
    del s["scales"], s["rotations"]
    return s
