"""Float64 reference of preprocess backward (csrc/preprocess_bwd.cu, SURVEY A.5), evaluated on the GPU's own
records (tests only).

Preprocess backward is a deterministic per-splat function of the inputs, the forward's transform record (T, screen
centre c, clamp bits) and the render backward's 22-float gradient record (common.cuh: A, Bx, By, Zd, Zl,
dL_dmean2D, dL_dopacity, dL_dnormal, dL_dcolor).  This module restates it with torch autograd in float64,
independently of the kernel and of the C oracle:

  1. record -> dL_dT: the vjp of (Pc, P1, P2) = (Tu' x Tv', Tv' x Tw, Tw x Tu'), Tu' = Tu - c.x Tw, Tv' = Tv - c.y Tw,
     weighted by A, Bx, By, plus Zd * d det(T) / dT and Zl on Tw.  It is linearised at the forward's STORED float32
     T and c (evaluated in float64): Tu.z and c.x Tw.z cancel to a few units in 1e5, so T recomputed from the inputs
     would sit further from the record's point than the tolerance;
  2. the AABB-centre fold: dL_dmean2D through the vjp of xy(T) (oracle/dense_torch.preprocess), at the same T;
  3. T, the normal and the colour to the leaves: autograd through oracle/dense_torch.preprocess at the float32
     inputs, with the gradient taken w.r.t. the unit quaternion (q / |q| formed outside the graph), the
     dual-visible normal sign as in the forward and the colour gradient masked by the forward's clamp bits;
  4. the densification proxy (dense_torch.densification_proxy): the raw dL_dT[2|5] of step 1 on the
     scales+rotations path, the folded one on the transMat_precomp path, times the stored Tw.z * 0.5 * W|H;
  5. the scale_modifier convention (`scale_modifier_quirk`).  Upstream's backward rebuilds L = R diag(s) with the
     modifier fixed to 1 (SURVEY A.5), so both dL_dscale and the scale-weighted columns 0 and 1 of dL_dR are those
     of modifier 1: the exact autograd values divided by scale_modifier.  The normal column is unaffected.

Everything above is linear in the record, so each leaf entry's Jacobian J w.r.t. the 22 record floats follows from
22 evaluations with unit records, and |J| . |rec| bounds the float32 rounding a per-splat evaluation can pick up.
The low-pass depth setting (lowpass_quirk) only changes what render backward writes into Zl and dL_dmean2D; the
preprocess step is the same for both.
"""
import numpy as np
import torch

from oracle import dense_torch as DT

F64 = torch.float64
REC_FLOATS = 22
# output keys of surfel_backward; the first group is computed, the second copied from the record
BOUNDED_KEYS = ("dL_dtransMat", "dL_dmeans2D", "dL_dmeans3D", "dL_dscales", "dL_drotations", "dL_dshs")


def _t(x):
    return None if x is None else torch.as_tensor(np.asarray(x, np.float64), dtype=F64)


def _cross(a, b):
    return torch.cross(a, b, dim=-1)


def _grad(out, leaf):
    g = torch.autograd.grad(out, leaf, retain_graph=True, allow_unused=True)[0]
    return torch.zeros_like(leaf) if g is None else g


def record_to_dT(T, c, rec):
    """Step 1 as a scalar: sum_splats A.Pc + Bx.P1 + By.P2 + Zd det T + Zl.Tw, with c held fixed."""
    Tu, Tv, Tw = T[:, 0:3], T[:, 3:6], T[:, 6:9]
    Tu_, Tv_ = Tu - c[:, 0:1] * Tw, Tv - c[:, 1:2] * Tw
    Pc, P1, P2 = _cross(Tu_, Tv_), _cross(Tv_, Tw), _cross(Tw, Tu_)
    det = (Tu * _cross(Tv, Tw)).sum(1)
    return ((rec[:, 0:3] * Pc).sum(1) + (rec[:, 3:6] * P1).sum(1) + (rec[:, 6:9] * P2).sum(1)
            + rec[:, 9] * det + (rec[:, 10:13] * Tw).sum(1))


def aabb_centre(T, means, cam):
    """xy(T): the screen centre formula of dense_torch.preprocess (A.1 step 5)."""
    P = T.shape[0]
    pre = DT.preprocess(means, None, None, torch.zeros(P, 1, dtype=F64), None, cam["vm"], cam["pm"], cam["campos"],
                        cam["W"], cam["H"], transMat_precomp=T, colors_precomp=torch.zeros(P, 3, dtype=F64))
    return pre["xy"]


def scale_modifier_quirk(g, scale_modifier):
    """Upstream's convention at scale_modifier != 1 on top of the exact gradients g (dict with the parts below):
    the backward treats L = R diag(s) as if the modifier were 1, so dL_dscale and the rotation gradient that flows
    through the scaled tangent columns L0, L1 are the exact ones divided by the modifier; the rotation gradient
    through the normal column is kept."""
    return dict(dL_dscales=g["scales_T"] / scale_modifier,
                dL_drotations=g["rot_T"] / scale_modifier + g["rot_N"])


class Reference:
    """The linear map record -> outputs of one (scene, camera, forward record, SH setting)."""

    def __init__(self, scene, cam, fwd, sh_degree=3, scale_modifier=1.0, quirk=True):
        self.D, self.mod, self.quirk = int(sh_degree), float(scale_modifier), quirk
        self.W, self.H = int(cam["W"]), int(cam["H"])
        self.cam = dict(vm=_t(cam["viewmatrix"]), pm=_t(cam["projmatrix"]), campos=_t(cam["campos"]), W=self.W, H=self.H)
        self.means = _t(scene["means3D"])
        self.P = self.means.shape[0]
        self.geom = scene.get("transMat_precomp") is None
        self.scales, self.rots = _t(scene.get("scales")), _t(scene.get("rotations"))
        self.shs = _t(scene.get("shs")) if scene.get("colors_precomp") is None else None
        self.M = 0 if scene.get("shs") is None else np.asarray(scene["shs"]).shape[1]
        self.vis = torch.as_tensor(np.asarray(fwd["radii"]) > 0)
        self.T0 = _t(fwd["transMat"]).reshape(self.P, 9)
        self.c0 = _t(fwd["xy"]).reshape(self.P, 2)
        cl = np.asarray(fwd["clamped"])
        self.clamped = torch.as_tensor(cl.reshape(self.P, 3) != 0)
        self._jac = None

    def _leaf(self, x):
        return x.detach().clone().requires_grad_(True)

    def evaluate(self, rec):
        """Exact outputs for a (P, >=22) float64 record; rows of culled splats are zero."""
        rec = _t(rec)[:, :REC_FLOATS].clone()
        rec[~self.vis] = 0.0
        P, cam = self.P, self.cam
        # steps 1-2 at the stored T and c
        T = self._leaf(self.T0)
        s_rec = record_to_dT(T, self.c0, rec).sum()
        g_raw = _grad(s_rec, T)
        s_fold = (rec[:, 13:15] * aabb_centre(T, self.means, cam)).sum()
        gT = g_raw + _grad(s_fold, T)
        out = dict(dL_dtransMat_raw=g_raw, dL_dtransMat=gT)
        src = g_raw if self.geom else gT
        prox = DT.densification_proxy(self.T0, src, self.W, self.H)
        out["dL_dmeans2D"] = torch.cat([prox, torch.zeros(P, 1, dtype=F64)], 1)
        out["dL_dopacity"] = rec[:, 15:16].clone()
        gn, gc = rec[:, 16:19], rec[:, 19:22]
        out["dL_dcolors_raw"] = gc.clone()
        dR = torch.where(self.clamped, torch.zeros_like(gc), gc)
        out["dL_dcolors_masked"] = dR
        means = self._leaf(self.means)
        g3 = torch.zeros(P, 3, dtype=F64)
        # step 3: T and the normal to the leaves
        if self.geom:
            qn = self.rots / self.rots.norm(dim=1, keepdim=True)       # unit quaternion, outside the graph
            scales, q = self._leaf(self.scales), self._leaf(qn)
            pre = DT.preprocess(means, scales, q, torch.zeros(P, 1, dtype=F64), None, cam["vm"], cam["pm"],
                                cam["campos"], self.W, self.H, self.D, self.mod, None,
                                torch.zeros(P, 3, dtype=F64), normalize_quat=False)
            s_T = (gT * pre["T"]).sum()
            s_N = (gn * pre["normal"]).sum()
            parts = dict(scales_T=_grad(s_T, scales), rot_T=_grad(s_T, q), rot_N=_grad(s_N, q))
            g3 = g3 + _grad(s_T, means)
            out["exact_dL_dscales"] = parts["scales_T"]
            out["exact_dL_drotations"] = parts["rot_T"] + parts["rot_N"]
            q_ = scale_modifier_quirk(parts, self.mod)
            out["quirk_dL_dscales"], out["quirk_dL_drotations"] = q_["dL_dscales"], q_["dL_drotations"]
            pick = "quirk_" if self.quirk else "exact_"
            out["dL_dscales"], out["dL_drotations"] = out[pick + "dL_dscales"], out[pick + "dL_drotations"]
        # SH: the clamp-masked colour gradient through raw rgb = SH(dir) + 0.5
        if self.shs is not None:
            shs = self._leaf(self.shs)
            d = means - cam["campos"][None]
            raw = DT.eval_sh(self.D, shs, d / d.norm(dim=1, keepdim=True)) + 0.5
            s_C = (dR * raw).sum()
            g3 = g3 + _grad(s_C, means)
            out["dL_dshs"] = _grad(s_C, shs)
        out["dL_dmeans3D"] = g3
        for k, v in out.items():
            out[k] = torch.where(self.vis.reshape((-1,) + (1,) * (v.dim() - 1)), v, torch.zeros_like(v)).detach()
        return out

    def jacobian(self):
        """{key: (22, P, ...)} signed Jacobian of every output w.r.t. the record (cached)."""
        if self._jac is None:
            cols = []
            for j in range(REC_FLOATS):
                e = np.zeros((self.P, REC_FLOATS))
                e[:, j] = 1.0
                cols.append(self.evaluate(e))
            self._jac = {k: torch.stack([c[k] for c in cols]) for k in cols[0]}
        return self._jac

    def bound(self, rec):
        """Per entry sum_j |J_j| |rec_j|."""
        a = _t(np.abs(np.asarray(rec, np.float64)[:, :REC_FLOATS]))
        a[~self.vis] = 0.0
        return {k: torch.einsum("jp...,pj->p...", J.abs(), a).numpy() for k, J in self.jacobian().items()}


def preprocess_bwd_exact(scene, cam, fwd, rec, sh_degree=3, scale_modifier=1.0, lowpass_quirk=True, defer_sh=False,
                         quirk=True, ref=None):
    """Every output of surfel_backward's preprocess step, and a per-entry bound, for the record `rec` (P, 24).

    fwd: radii, transMat, xy, clamped of the forward (CudaPipeline.preprocess()).  quirk: apply the scale_modifier
    convention (scale_modifier_quirk); False gives the exact derivative.  lowpass_quirk is accepted for symmetry
    with surfel_backward: it shapes the record, not this step.  ref: a Reference to reuse (its Jacobian is cached).
    Returns (outputs, bounds), both dicts of numpy float64 arrays keyed like surfel_backward's outputs."""
    del lowpass_quirk
    ref = Reference(scene, cam, fwd, sh_degree, scale_modifier, quirk) if ref is None else ref
    ev = {k: v.numpy() for k, v in ref.evaluate(rec).items()}
    ev["dL_dcolors"] = ev["dL_dcolors_masked"] if defer_sh else ev["dL_dcolors_raw"]
    bd = ref.bound(rec)
    return ev, bd
