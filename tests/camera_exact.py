"""Float64 restatement of the rasterizer's camera gradients (csrc/camera_bwd.cu, DESIGN.md §7p), evaluated on a
gradient record (tests only).

The camera gradient is a sum over the visible splats of per-splat terms that are linear in what surfel_backward
leaves per splat: the full dL_dT after the AABB-centre fold (gT), the gradient of the stored normal (gn, record
16..18) and the clamp-masked colour gradient (dR, record 19..21).  gT is itself linear in the 22-float record
(preprocess_exact.Reference, steps 1-2), so everything here is linear in the record.  With row-vector matrices,
pr = projmatrix, vm = viewmatrix (16 contiguous floats each), L0 = mod s_u R[:,0], L1 = mod s_v R[:,1], L2 = R[:,2]
and p the splat's position:

  1. projmatrix, through T:  G_j[r] = gT[3j] L0[r] + gT[3j+1] L1[r] + gT[3j+2] p[r] (r < 3), G_j[3] = gT[3j+2];
     dpr[4r] = W/2 G_0[r], dpr[4r+1] = H/2 G_1[r], dpr[4r+2] = 0, dpr[4r+3] = (W-1)/2 G_0[r] + (H-1)/2 G_1[r] + G_2[r];
  2. viewmatrix, through the normal:  dvm[4r+c] = mult L2[r] gn[c] (r, c < 3), every other entry 0;
  3. campos, through the SH view direction:  -(the SH term of dL_dmeans3D);
  4. with transMat_precomp only 3 remains.
Rules 1 and 2 are written out; rule 3 is the negated SH part of preprocess_exact's dL_dmeans3D, taken separately.
"""
import numpy as np
import torch

import preprocess_exact as PE
from oracle import dense_torch as DT

F64 = torch.float64
KEYS = ("viewmatrix", "projmatrix", "campos")
GT_ROW_FLOOR = 1e-3       # x the largest |J|.|rec| of the splat's dL_dT row, as preprocess backward's own bound


class CameraReference(PE.Reference):
    """The linear map record -> (dL_dviewmatrix, dL_dprojmatrix, dL_dcampos) of one forward."""

    def _frame(self):
        q = self.rots / self.rots.norm(dim=1, keepdim=True)
        R = DT.quat_to_R(q)
        L0 = R[:, :, 0] * (self.mod * self.scales[:, 0:1])
        L1 = R[:, :, 1] * (self.mod * self.scales[:, 1:2])
        L2 = R[:, :, 2]
        vm = self.cam["vm"]
        p_view = torch.cat([self.means, torch.ones(self.P, 1, dtype=F64)], 1) @ vm[:, :3]
        nv = L2 @ vm[:3, :3]
        mult = torch.where(-(p_view * nv).sum(1) > 0, 1.0, -1.0).to(F64)
        return L0, L1, L2, mult

    def sh_direction_term(self, dR, shs=None):
        """(P,3) SH part of dL_dmeans3D for the masked colour gradient dR (zero without SH); shs: other coefficients."""
        if self.shs is None or self.D == 0:
            return torch.zeros(self.P, 3, dtype=F64)
        means = self._leaf(self.means)
        d = means - self.cam["campos"][None]
        raw = DT.eval_sh(self.D, self.shs if shs is None else shs, d / d.norm(dim=1, keepdim=True)) + 0.5
        g = PE._grad((dR * raw).sum(), means)
        return torch.where(self.vis[:, None], g, torch.zeros_like(g)).detach()

    def terms(self, rec, gT=None):
        """Per-splat terms (G (P,3,4), V (P,3,3), C (P,3)) and the pieces they were formed from."""
        rec = PE._t(rec)[:, :PE.REC_FLOATS].clone()
        rec[~self.vis] = 0.0
        if gT is None:
            gT = self.evaluate(rec)["dL_dtransMat"]
        gn = rec[:, 16:19]
        dR = torch.where(self.clamped, torch.zeros_like(rec[:, 19:22]), rec[:, 19:22])
        G = torch.zeros(self.P, 3, 4, dtype=F64)
        V = torch.zeros(self.P, 3, 3, dtype=F64)
        if self.geom:
            L0, L1, L2, mult = self._frame()
            for j in range(3):
                G[:, j, :3] = gT[:, 3 * j:3 * j + 1] * L0 + gT[:, 3 * j + 1:3 * j + 2] * L1 + gT[:, 3 * j + 2:3 * j + 3] * self.means
                G[:, j, 3] = gT[:, 3 * j + 2]
            V = (mult[:, None] * L2)[:, :, None] * gn[:, None, :]
        C = -self.sh_direction_term(dR)
        return G, V, C

    def _assemble(self, G, V, C):
        W, H = self.W, self.H
        G = G.sum(0)
        dpr = torch.zeros(4, 4, dtype=F64)
        dpr[:, 0] = W / 2 * G[0]
        dpr[:, 1] = H / 2 * G[1]
        dpr[:, 3] = (W - 1) / 2 * G[0] + (H - 1) / 2 * G[1] + G[2]
        dvm = torch.zeros(4, 4, dtype=F64)
        dvm[:3, :3] = V.sum(0)
        return dict(viewmatrix=dvm.reshape(16).numpy(), projmatrix=dpr.reshape(16).numpy(), campos=C.sum(0).numpy())

    def camera(self, rec):
        """{viewmatrix (16,), projmatrix (16,), campos (3,)} float64: the exact camera gradient for the record."""
        return self._assemble(*self.terms(rec))

    def camera_bound(self, rec):
        """Per entry, sum over splats of |J| |rec| along the chain the kernel evaluates in float32: dL_dT's own bound
        (preprocess_exact, with its row floor) through |L0|, |L1|, |p|; |L2| |gn|; and, for the SH term, |J| |dR| taken
        per coefficient."""
        a = np.abs(np.asarray(rec, np.float64)[:, :PE.REC_FLOATS]).copy()
        a[~self.vis.numpy()] = 0.0
        bT = torch.as_tensor(self.bound(rec)["dL_dtransMat"])
        bT = bT + GT_ROW_FLOOR * bT.max(1, keepdim=True).values
        gn, gc = torch.as_tensor(a[:, 16:19]), torch.as_tensor(a[:, 19:22])
        dRabs = torch.where(self.clamped, torch.zeros_like(gc), gc)
        G = torch.zeros(self.P, 3, 4, dtype=F64)
        V = torch.zeros(self.P, 3, 3, dtype=F64)
        if self.geom:
            L0, L1, L2, _ = self._frame()
            for j in range(3):
                G[:, j, :3] = bT[:, 3 * j:3 * j + 1] * L0.abs() + bT[:, 3 * j + 1:3 * j + 2] * L1.abs() + \
                    bT[:, 3 * j + 2:3 * j + 3] * self.means.abs()
                G[:, j, 3] = bT[:, 3 * j + 2]
            V = L2.abs()[:, :, None] * gn[:, None, :]
        C = torch.zeros(self.P, 3, dtype=F64)
        if self.shs is not None:
            # one coefficient and one channel at a time: the float32 sum runs over these products
            for k in range(1, (self.D + 1) ** 2):
                for c in range(3):
                    e = torch.zeros(self.P, 3, dtype=F64)
                    e[:, c] = 1.0
                    shs = torch.zeros_like(self.shs)
                    shs[:, k, c] = self.shs[:, k, c].abs()
                    C = C + self.sh_direction_term(e, shs).abs() * dRabs[:, c:c + 1]
        return self._assemble(G, V, C)


def autograd_camera(ref, rec, gT):
    """The same gradient by float64 autograd of oracle/dense_torch.preprocess in viewmatrix, projmatrix and campos:
    sum over visible splats of gT . T + gn . normal + dR . rgb, with gT, gn and dR those the restatement uses."""
    rec = PE._t(rec)[:, :PE.REC_FLOATS].clone()
    rec[~ref.vis] = 0.0
    gn = rec[:, 16:19]
    dR = torch.where(ref.clamped, torch.zeros_like(rec[:, 19:22]), rec[:, 19:22])
    vm, pm, cp = (ref.cam[k].detach().clone().requires_grad_(True) for k in ("vm", "pm", "campos"))
    P = ref.P
    shs = ref.shs
    q = None if ref.rots is None else ref.rots / ref.rots.norm(dim=1, keepdim=True)
    T0 = None if ref.geom else ref.T0
    pre = DT.preprocess(ref.means, ref.scales, q, torch.zeros(P, 1, dtype=F64), shs, vm, pm, cp, ref.W, ref.H, ref.D,
                        ref.mod, T0, None if shs is not None else torch.zeros(P, 3, dtype=F64), normalize_quat=False)
    s = (gT * pre["T"]).sum() + (gn * pre["normal"]).sum() + (dR * pre["rgb"]).sum()
    out = {}
    for key, leaf in (("viewmatrix", vm), ("projmatrix", pm), ("campos", cp)):
        g = torch.autograd.grad(s, leaf, retain_graph=True, allow_unused=True)[0] if s.requires_grad else None
        out[key] = (torch.zeros_like(leaf) if g is None else g).reshape(-1).detach().numpy()
    return out


def dense_camera_grad(scene, cam, bg, gc, go, dtype, sh_degree=3, upstream_lowpass_depth=True, band_rows=32):
    """dL/d(viewmatrix, projmatrix, campos) of sum(color * gc) + sum(allmap * go) by autograd through
    oracle/dense_torch.render in `dtype`, on the device of the cotangents.  The frame is rendered in bands of
    band_rows rows (a multiple of the 16-pixel tile) to bound memory: a band starting at row y0 is the full-frame
    rasterization with the pixel rows shifted, i.e. Tv - y0 Tw, xy - (0, y0) and the tile rectangles moved by y0 / 16.
    Returns numpy float64 arrays (16,), (16,), (3,)."""
    dev = gc.device
    W, H = int(cam["W"]), int(cam["H"])
    t = lambda x: torch.as_tensor(np.asarray(x)).to(dev, dtype)
    s = {k: t(v) for k, v in scene.items()}
    leaves = [t(cam[k]).clone().requires_grad_(True) for k in ("viewmatrix", "projmatrix", "campos")]
    acc = [torch.zeros_like(x) for x in leaves]
    gc, go = gc.to(dtype), go.to(dtype)
    with torch.device(dev):
        for y0 in range(0, H, band_rows):
            hb = min(band_rows, H - y0)
            pre = DT.preprocess(s["means3D"], s["scales"], s["rotations"], s["opacities"], s["shs"], *leaves, W, H,
                                sh_degree)
            T = pre["T"]
            band = dict(pre)
            band["T"] = torch.cat([T[:, 0:3], T[:, 3:6] - y0 * T[:, 6:9], T[:, 6:9]], 1)
            band["xy"] = pre["xy"] - torch.tensor([0.0, float(y0)], dtype=dtype)
            band["rect"] = pre["rect"] - torch.tensor([0, y0 // 16, 0, y0 // 16])
            color, others, _, _ = DT.rasterize(band, t(bg), W, hb, upstream_lowpass_depth=upstream_lowpass_depth)
            loss = (color * gc[:, y0:y0 + hb]).sum() + (others * go[:, y0:y0 + hb]).sum()
            for a, g in zip(acc, torch.autograd.grad(loss, leaves, allow_unused=True)):
                if g is not None:
                    a += g
    return tuple(a.detach().double().reshape(-1).cpu().numpy() for a in acc)
