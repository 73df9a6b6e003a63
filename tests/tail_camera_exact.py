"""Float64 restatement of the camera gradients of the fused render() tail and of the 2DGS regularisers
(DESIGN §7q), in the layouts of csrc/postprocess.cu:

    rot[3r+c]:  n_world_c = sum_r n_view_r rot[3r+c]
    rays[3k+j]: dir_j = x rays[j] + y rays[3+j] + rays[6+j];   rays[9+j]: the camera centre o_j

Over the pixels p, with q = (x, y, 1), d = surf_depth and dP the gradient of the point P = d dir + o:

    G_rot[3r+c]  = sum_p allmap[2+r](p) gw_c(p)          gw: the cotangent of rend_normal
    G_rays[3k+j] = sum_p d(p) q_k(p) dP_j(p)
    G_rays[9+j]  = sum_p dP_j(p)

dP is the four-neighbour gather of the six-plane point gradient tmp6 (the vjp of normalize(dx x dy) for the
cotangent of surf_normal times the detached alpha).  For surface_outputs gw = g_rend_normal and the surf_normal
cotangent is g_surf_normal; for the regularisers, with s = dL/dnormal_loss * lambda_normal / N, gw = -s sn and the
surf_normal cotangent is -s rend_normal (sn the alpha-weighted surf_normal, zero on the border).  `chain` carries the
21 sums through the algebra of postprocess._view_matrices to world_view_transform and full_proj_transform.

`sums_from` also returns a first-order bound (units of u = 2^-24) on what a float32 evaluation of the per-pixel terms,
summed in double, may add, given bounds on its factors' own errors.
"""
import numpy as np
import torch
import torch.nn.functional as F

import tail_loss_exact as X

U = X.U


def view_matrices(view, proj, W, H):
    """rot (3,3) and rays (12,) in float64 from the two camera matrices (autograd flows through)."""
    rot, M, o = X.camera_f64(view, proj, W, H)
    return rot, torch.cat([M.reshape(-1), o])


def surf_depth(a, ratio):
    """surf_depth (H,W) of the reference's tail from a float64 allmap."""
    ex = torch.nan_to_num(a[0] / a[1], 0.0, 0.0, X.F32_LOWEST)
    return ex * (1 - ratio) + ratio * torch.nan_to_num(a[5], 0.0, 0.0, X.F32_LOWEST)


def _grid(H, W, dev):
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=dev),
                            torch.arange(W, dtype=torch.float64, device=dev), indexing="ij")
    return torch.stack([xs, ys, torch.ones_like(xs)], -1)                     # q (H, W, 3)


def _stencil(d, rays):
    H, W = d.shape
    P = d[..., None] * (_grid(H, W, d.device) @ rays[:9].reshape(3, 3)) + rays[9:]
    dx, dy = P[2:, 1:-1] - P[:-2, 1:-1], P[1:-1, 2:] - P[1:-1, :-2]
    return dx, dy, torch.cross(dx, dy, dim=-1)


def surf_normal(a, d, rays):
    """(3,H,W): normalize(dx x dy) * alpha, zero on the border."""
    H, W = d.shape
    out = torch.zeros(H, W, 3, dtype=torch.float64, device=d.device)
    if H > 2 and W > 2:
        out[1:-1, 1:-1] = F.normalize(_stencil(d, rays)[2], dim=-1)
    return out.permute(2, 0, 1) * a[1]


def point_grads(d, rays, g):
    """tmp6 (6,H,W): d(dx) and d(dy) at each interior pixel for the surf_normal cotangent g (3,H,W, alpha folded in),
    with F.normalize's eps rule (|v| <= 1e-12: dv = g / 1e-12)."""
    H, W = d.shape
    tmp = torch.zeros(6, H, W, dtype=torch.float64, device=d.device)
    if H > 2 and W > 2:
        dx, dy, v = _stencil(d, rays)
        gi = g.permute(1, 2, 0)[1:-1, 1:-1]
        ln = v.norm(dim=-1, keepdim=True)
        live = ln > 1e-12
        lns = torch.where(live, ln, torch.ones_like(ln))
        n = v / lns
        dv = torch.where(live, (gi - n * (n * gi).sum(-1, keepdim=True)) / lns, gi * 1e12)
        tmp[0:3, 1:-1, 1:-1] = torch.cross(dy, dv, dim=-1).permute(2, 0, 1)
        tmp[3:6, 1:-1, 1:-1] = torch.cross(dv, dx, dim=-1).permute(2, 0, 1)
    return tmp


def gather(tmp, absolute=False):
    """dP (H,W,3): the point gradient gathered from the four neighbours' tmp6 (absolute=True: of |tmp6|, the
    magnitude behind the gather's rounding)."""
    t = tmp.abs() if absolute else tmp
    sg = 1.0 if absolute else -1.0
    dP = torch.zeros_like(t[0:3])
    dP[:, 1:] += t[0:3, :-1]
    dP[:, :-1] += sg * t[0:3, 1:]
    dP[:, :, 1:] += t[3:6, :, :-1]
    dP[:, :, :-1] += sg * t[3:6, :, 1:]
    return dP.permute(1, 2, 0)


def sums_from(nv, gw, d, dP, e_gw=None, e_d=None, e_dP=None):
    """(G (21,), B (21,)): the sums of the module docstring from the per-pixel factors nv, gw (3,H,W), d (H,W) and
    dP (H,W,3), and the bound on a float32 evaluation given the factors' error bounds (units of u; None: exact):
    each term t = nv_r gw_c, (d q_k) dP_j or dP_j rounds once per product, and the double sum adds N 2^-29 |t|."""
    H, W = d.shape
    q = _grid(H, W, d.device)
    z3, z1 = torch.zeros_like(gw), torch.zeros_like(d)
    e_gw = z3 if e_gw is None else e_gw
    e_d = z1 if e_d is None else e_d
    e_dP = torch.zeros_like(dP) if e_dP is None else e_dP
    N = H * W
    red = N * 2.0 ** -29
    G_rot = torch.einsum("rhw,chw->rc", nv, gw)
    G_dir = torch.einsum("hw,hwk,hwj->kj", d, q, dP)
    G_o = dP.sum((0, 1))
    G = torch.cat([G_rot.reshape(-1), G_dir.reshape(-1), G_o])
    an, ag, ad, aq, aP = nv.abs(), gw.abs(), d.abs(), q.abs(), dP.abs()
    B_rot = torch.einsum("rhw,chw->rc", an, e_gw + (1 + red) * ag)
    B_dir = torch.einsum("hw,hwk,hwj->kj", e_d, aq, aP) + torch.einsum("hw,hwk,hwj->kj", ad, aq, e_dP) \
        + (2 + red) * torch.einsum("hw,hwk,hwj->kj", ad, aq, aP)
    B_o = (e_dP + red * aP).sum((0, 1))
    return G, torch.cat([B_rot.reshape(-1), B_dir.reshape(-1), B_o])


def magnitudes(nv, gw, d, tmp):
    """(21,): each sum of sums_from evaluated on the factors' absolute values, with dP gathered from |tmp6|: the scale
    a sum's rounding is measured against."""
    return sums_from(nv.abs(), gw.abs(), d.abs(), gather(tmp, absolute=True))[0]


def outputs_sums(allmap, rot, rays, ratio, cot):
    """(G, B): the 21 sums for surface_outputs with cotangents cot (keys rend_normal, surf_normal; a missing or None one
    is zero); float64 throughout.  The pass reads neither rot nor surf_depth's cotangent."""
    a = X._t(allmap)
    rays = X._t(rays, a.device)
    d = surf_depth(a, ratio)
    z = torch.zeros(3, *d.shape, dtype=torch.float64, device=a.device)
    g_rn = z if cot.get("rend_normal") is None else X._t(cot["rend_normal"], a.device)
    g_sn = z if cot.get("surf_normal") is None else X._t(cot["surf_normal"], a.device)
    tmp = point_grads(d, rays, g_sn * a[1])
    return sums_from(a[2:5], g_rn, d, gather(tmp))[0], magnitudes(a[2:5], g_rn, d, tmp)


def reg_sums(allmap, rot, rays, ratio, lambda_normal, g_normal=1.0):
    """(G, B): the 21 sums for surface_regularizers with dL/dnormal_loss = g_normal (the distortion term does not depend on
    the camera)."""
    a = X._t(allmap)
    rot, rays = X._t(rot, a.device).reshape(3, 3), X._t(rays, a.device)
    s = g_normal * lambda_normal / (a.shape[1] * a.shape[2])
    d = surf_depth(a, ratio)
    rn = torch.einsum("rhw,rc->chw", a[2:5], rot)
    tmp = point_grads(d, rays, -s * rn * a[1])
    gw = -s * surf_normal(a, d, rays)
    return sums_from(a[2:5], gw, d, gather(tmp))[0], magnitudes(a[2:5], gw, d, tmp)


def chain(G, view, proj, W, H):
    """(dL/dworld_view_transform, dL/dfull_proj_transform) (4,4 float64) for the 21 sums G, by float64 autograd
    through view_matrices."""
    v = X._t(view).clone().requires_grad_(True)
    p = X._t(proj).clone().requires_grad_(True)
    rot, rays = view_matrices(v, p, W, H)
    G = X._t(G, v.device)
    gv, gp = torch.autograd.grad((rot.reshape(-1) * G[:9]).sum() + (rays * G[9:]).sum(), [v, p])
    return gv, gp


def chain_bound(B, view, proj, W, H):
    """|J|^T B for the Jacobian J of (rot, rays) with respect to (view, proj): what a bound B (21,) on the sums
    becomes on the two matrices."""
    v, p = X._t(view), X._t(proj)
    Jv, Jp = torch.autograd.functional.jacobian(lambda a, b: torch.cat([t.reshape(-1) for t in view_matrices(a, b, W, H)]),
                                                (v, p))
    B = X._t(B, v.device)
    return torch.einsum("kij,k->ij", Jv.abs(), B), torch.einsum("kij,k->ij", Jp.abs(), B)


def reference_camera_grads(allmap, view, proj, ratio, loss_fn, dtype=torch.float64, dev="cpu"):
    """Autograd of the reference's tail (test_postprocess_gpu.reference_tail) in `dtype` with both camera matrices as
    leaves: (dL/dview, dL/dproj) for the scalar loss_fn(outputs)."""
    import types
    from test_postprocess_gpu import reference_tail
    a = torch.as_tensor(np.asarray(allmap)).to(dev, dtype)
    v = torch.as_tensor(np.asarray(view)).to(dev, dtype).requires_grad_(True)
    p = torch.as_tensor(np.asarray(proj)).to(dev, dtype).requires_grad_(True)
    cam = types.SimpleNamespace(world_view_transform=v, full_proj_transform=p, image_width=a.shape[2],
                                image_height=a.shape[1])
    out = reference_tail(a, cam, ratio)
    return torch.autograd.grad(loss_fn(out), [v, p], allow_unused=True, materialize_grads=True)


def outputs_loss(cot):
    """sum_k cot_k * out_k over the tail's outputs."""
    return lambda out: sum((out[k] * torch.as_tensor(np.asarray(c)).to(out[k])).sum() for k, c in cot.items())


def reg_loss(lambda_normal, lambda_dist):
    """train.py's normal_loss + dist_loss on the tail's outputs."""
    def f(out):
        normal_error = (1 - (out["rend_normal"] * out["surf_normal"]).sum(dim=0))[None]
        return lambda_normal * normal_error.mean() + lambda_dist * out["rend_dist"].mean()
    return f
