"""Float64 evaluations of the render() tail (SURVEY §8f row f1) and of the L1+SSIM loss (row f2), each with
a per-entry bound on the rounding a float32 implementation of the same operation may add.

The exact value is the reference's algebra evaluated in float64 on the same float32 inputs (allmap, the
camera matrices, image and gt): c2w, intrins and their inverses are formed in float64 from the float32
matrices, and the loss uses the reference's float32 1-D window with an exact (float64) outer product.

Every bound is returned in units of u = 2^-24 (float32's unit roundoff) times a magnitude, so
`|got - exact| <= K * bound` with a constant K of order one is the check.  The bounds are first order:
  * tail forward: a point P = d * (x M0 + y M1 + M2) + o is held to its magnitude
    |d|(|x||M0| + |y||M1| + |M2|) + |o|, which covers a float32 M and the cancellation of P[y+1] - P[y-1];
    normalize() turns the error of dx and dy into ((|a|+|b|)|dy| + |dx|(|c|+|d|)) / |v| (a..d the four
    neighbouring points' magnitudes, v = dx x dy);
  * tail backward: the same terms evaluated on absolute values and carried through the vjp of normalize,
    the cross product, the four-neighbour gather, the ray dot product and D/alpha (as oracle
    render_bwd_f64 does for the render backward);
  * loss: n u sum_m |df/dm| conv(|m|) over the five raw window moments (mu1, mu2, E[x^2], E[y^2], E[xy])
    plus a few u|f|, for the SSIM map and for the backward's three derivative maps (whose moment
    derivatives are the second derivatives of f, taken by float64 autograd), carried through the
    backward's convolution; the loss value's bound is the mean of the per-pixel bounds plus the share of
    its reduction.
"""
from math import exp

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24
KEYS = ("rend_alpha", "rend_normal", "rend_dist", "surf_depth", "surf_normal")
F32_LOWEST = float(np.finfo(np.float32).min)      # torch.nan_to_num's default for -inf on a float32 tensor
N_PT = 16          # roundings behind one float32 point (the float32 ray matrix, its dot product, x depth, + o)
N_MOM = 24         # roundings of one float32 window moment (11 + 11 taps of the separable convolution)
N_CONV = 24        # roundings of the backward's separable convolution of one derivative map


def _t(a, dev=None):
    t = a if torch.is_tensor(a) else torch.from_numpy(np.asarray(a))
    return t.to(device=dev or t.device, dtype=torch.float64)


def camera_f64(view, proj, W, H, dev=None):
    """rot (n_world = n_view @ rot), ray matrix M (dir = (x, y, 1) @ M) and camera centre o, in float64
    from the float32 world_view_transform and full_proj_transform (reference utils/point_utils.py:9-24)."""
    wvt, full = _t(view, dev), _t(proj, dev)
    c2w = wvt.T.inverse()
    ndc2pix = torch.tensor([[W / 2, 0, 0, W / 2], [0, H / 2, 0, H / 2], [0, 0, 0, 1]],
                           dtype=torch.float64, device=wvt.device).T
    intrins = ((c2w.T @ full) @ ndc2pix)[:3, :3].T
    M = intrins.inverse().T @ c2w[:3, :3].T
    return wvt[:3, :3].T, M, c2w[:3, 3]


def _abs_cross(a, b):
    """The cross product evaluated on absolute values (last dimension 3)."""
    a, b = a.abs(), b.abs()
    return torch.stack([a[..., 1] * b[..., 2] + a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] + a[..., 0] * b[..., 2],
                        a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]], -1)


def _interior(t):
    """Embed an (H-2, W-2, ...) interior array into a zero (H, W, ...) one."""
    out = t.new_zeros((t.shape[0] + 2, t.shape[1] + 2) + tuple(t.shape[2:]))
    out[1:-1, 1:-1] = t
    return out


def tail_f64(allmap, view, proj, ratio, cot=None, dev=None):
    """The reference render() tail in float64.

    Returns (out, grad, out_bound, grad_bound, hole_grad):
      out         dict of the five outputs (float64);
      grad        d(sum_k out[k] * cot[k]) / d allmap by float64 autograd, NaN where the reference's is
                  (D / alpha not finite: 0 * inf behind nan_to_num), or None without `cot`;
      out_bound   per-entry rounding bounds of `out` (units of u; 0 means the entry is exact);
      grad_bound  per-entry bounds of `grad` (units of u) where it is finite;
      hole_grad   what a NaN-free backward gives where `grad` is NaN: the D/alpha term contributes 0, so
                  channel 0 is 0 and channel 1 is the cotangent of rend_alpha.
    """
    a = _t(allmap, dev).clone()
    dev = a.device
    _, H, W = a.shape
    rot, M, o = camera_f64(view, proj, W, H, dev)
    a.requires_grad_(cot is not None)
    alpha = a[1:2]
    rend_normal = torch.einsum("khw,kc->chw", a[2:5], rot)
    med = torch.nan_to_num(a[5:6], 0.0, 0.0, F32_LOWEST)
    ex = torch.nan_to_num(a[0:1] / alpha, 0.0, 0.0, F32_LOWEST)
    surf_depth = ex * (1 - ratio) + ratio * med
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=dev),
                            torch.arange(W, dtype=torch.float64, device=dev), indexing="ij")
    pix = torch.stack([xs, ys, torch.ones_like(xs)], -1)
    rays = pix @ M                                                          # (H, W, 3)
    points = surf_depth[0][..., None] * rays + o
    normal = torch.zeros_like(points)
    if H > 2 and W > 2:
        dx = points[2:, 1:-1] - points[:-2, 1:-1]
        dy = points[1:-1, 2:] - points[1:-1, :-2]
        normal[1:-1, 1:-1] = F.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    surf_normal = normal.permute(2, 0, 1) * alpha.detach()
    out = {"rend_alpha": alpha, "rend_normal": rend_normal, "rend_dist": a[6:7], "surf_depth": surf_depth,
           "surf_normal": surf_normal}
    grad = None
    if cot is not None:
        c = {k: _t(v, dev) for k, v in cot.items()}
        grad, = torch.autograd.grad(sum((out[k] * c[k]).sum() for k in KEYS), a)
    out = {k: v.detach() for k, v in out.items()}

    with torch.no_grad():
        A, D = a[1].detach(), a[0].detach()
        medr = a[5].detach()
        ex_fin = torch.isfinite(D / A)
        med_fin = torch.isfinite(medr)
        exd = torch.nan_to_num(D / A, 0.0, 0.0, F32_LOWEST)
        medd = torch.nan_to_num(medr, 0.0, 0.0, F32_LOWEST)
        sd_mag = exd.abs() * (1 - ratio) + ratio * medd.abs()                # (H, W)
        rmag = xs[..., None] * M[0].abs() + ys[..., None] * M[1].abs() + M[2].abs()   # (H, W, 3)
        pmag = sd_mag[..., None] * rmag + o.abs()                             # |P| with everything that rounds into it
        ob = {"rend_alpha": torch.zeros_like(alpha), "rend_dist": torch.zeros_like(alpha),
              "rend_normal": 4 * torch.einsum("khw,kc->chw", a[2:5].detach().abs(), rot.abs()),
              "surf_depth": 6 * sd_mag[None]}
        sn_b = torch.zeros(H, W, device=dev, dtype=torch.float64)
        if H > 2 and W > 2:
            P = points.detach()
            dx, dy = P[2:, 1:-1] - P[:-2, 1:-1], P[1:-1, 2:] - P[1:-1, :-2]
            edx, edy = pmag[2:, 1:-1] + pmag[:-2, 1:-1], pmag[1:-1, 2:] + pmag[1:-1, :-2]
            v = torch.cross(dx, dy, dim=-1)
            ln = v.norm(dim=-1)
            live = ln > 0                     # v == 0 exactly (a flat 3x3 hole): both paths give exactly 0
            lns = torch.where(live, ln, torch.ones_like(ln))
            kappa = N_PT * (edx.norm(dim=-1) * dy.norm(dim=-1) + dx.norm(dim=-1) * edy.norm(dim=-1)) / lns
            kappa = torch.where(live, kappa, torch.zeros_like(kappa))
            sn_b = _interior(torch.where(live, kappa + 4, torch.zeros_like(kappa)))
        ob["surf_normal"] = sn_b[None] * A.abs()[None] * torch.ones(3, 1, 1, dtype=torch.float64, device=dev)

        gb = None
        if cot is not None:
            gb = torch.zeros(7, H, W, dtype=torch.float64, device=dev)
            gsd = c["surf_depth"][0].abs()
            dPb = torch.zeros(H, W, 3, dtype=torch.float64, device=dev)
            dPa = torch.zeros_like(dPb)
            if H > 2 and W > 2:
                g = (c["surf_normal"].permute(1, 2, 0) * A[..., None])[1:-1, 1:-1].abs()
                n = v / lns[..., None]
                dv_abs = (g + n.abs() * (n.abs() * g).sum(-1, keepdim=True)) / lns[..., None]
                dv_abs = torch.where(live[..., None], dv_abs, g * 1e12)    # normalize's v / eps branch
                amp = (2 * kappa + N_PT + 4)[..., None]
                t_dx, t_dy = _interior(amp * _abs_cross(edy, dv_abs)), _interior(amp * _abs_cross(dv_abs, edx))
                a_dx, a_dy = _interior(_abs_cross(dy, dv_abs)), _interior(_abs_cross(dv_abs, dx))
                for src_b, src_a, sh, dim in ((t_dx, a_dx, 1, 0), (t_dx, a_dx, -1, 0), (t_dy, a_dy, 1, 1), (t_dy, a_dy, -1, 1)):
                    # pixel p gathers the neighbour at p - sh along `dim` (zero beyond the frame)
                    dPb += _shift(src_b, sh, dim)
                    dPa += _shift(src_a, sh, dim)
            gd_u = (dPb * rmag).sum(-1) + (N_PT + 4) * (dPa * rmag).sum(-1) + 4 * gsd      # error of gd, units of u
            gd_abs = (dPa * rmag).sum(-1) + gsd
            Asafe = torch.where(ex_fin, A.abs(), torch.ones_like(A))
            gb[0] = torch.where(ex_fin, (gd_u + 3 * gd_abs) * (1 - ratio) / Asafe, torch.zeros_like(A))
            gb[1] = torch.where(ex_fin, (gd_u + 4 * gd_abs) * (1 - ratio) * D.abs() / Asafe ** 2, torch.zeros_like(A)) \
                + 2 * c["rend_alpha"][0].abs()
            gb[2:5] = 4 * torch.einsum("chw,kc->khw", c["rend_normal"].abs(), rot.abs())
            gb[5] = torch.where(med_fin, (gd_u + 3 * gd_abs) * ratio, torch.zeros_like(A))
        hole = None
        if cot is not None:
            hole = torch.zeros(7, H, W, dtype=torch.float64, device=dev)
            hole[1] = c["rend_alpha"][0]
    return out, (None if grad is None else grad.detach()), ob, gb, hole


def _shift(t, sh, dim):
    """out[p] = t[p - sh] along `dim` (0: rows, 1: columns), zero where p - sh leaves the frame."""
    out = torch.zeros_like(t)
    n = t.shape[dim]
    if abs(sh) >= n:
        return out
    if sh > 0:
        out.narrow(dim, sh, n - sh).copy_(t.narrow(dim, 0, n - sh))
    else:
        out.narrow(dim, 0, n + sh).copy_(t.narrow(dim, -sh, n + sh))
    return out


# ---------------------------------------------------------------------------------------------- loss (f2)

def window_1d():
    """The reference's window: exp(-(x-5)^2 / (2 * 1.5^2)) as float32, normalised in float32."""
    g = torch.tensor([exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)], dtype=torch.float32)
    return g / g.sum()


def _conv(t, g):
    """Zero-padded 11x11 window (the exact outer product of g with itself) over each (H, W) plane of t."""
    C, H, W = t.shape
    k = g.to(t)
    t = F.conv2d(t[:, None], k.view(1, 1, 1, 11), padding=(0, 5))
    return F.conv2d(t, k.view(1, 1, 11, 1), padding=(5, 0))[:, 0]


def _ssim_parts(m):
    mu1, mu2, e11, e22, e12 = m
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    A = 2 * mu1 * mu2 + C1
    B = 2 * (e12 - mu1 * mu2) + C2
    Cc = mu1 * mu1 + mu2 * mu2 + C1
    Dd = (e11 - mu1 * mu1) + (e22 - mu2 * mu2) + C2
    return A, B, Cc, Dd


def loss_f64(img, gt, lam, gout=1.0, dev=None):
    """(1 - lam) * mean|img - gt| + lam * (1 - mean SSIM) in float64, for (..., C, H, W) input (leading
    dimensions fold into channels, as the reference's 4-D call does).

    Returns (value, grad, value_bound, grad_bound, ssim_map, ssim_bound): grad is gout * d value / d img;
    the bounds are in units of u (value_bound a scalar, the others per entry).
    """
    x, y = _t(img, dev), _t(gt, dev)
    shape = x.shape
    H, W = shape[-2:]
    x, y = x.reshape(-1, H, W), y.reshape(-1, H, W)
    N = x.numel()
    g = window_1d().double().to(x.device)
    conv = lambda t: _conv(t, g)
    m = [t.requires_grad_(True) for t in (conv(x), conv(y), conv(x * x), conv(y * y), conv(x * y))]
    A, B, Cc, Dd = _ssim_parts(m)
    f = A * B / (Cc * Dd)
    df = torch.autograd.grad(f.sum(), m, create_graph=True)                 # per pixel: f depends on its own moments
    maps = (df[0], df[2], df[4])                                             # d f / d (mu1, E[x^2], E[xy])
    mabs = [conv(x.abs()), conv(y.abs()), conv(x * x), conv(y * y), conv((x * y).abs())]
    with torch.no_grad():
        mom_err = lambda d: N_MOM * sum(di.abs() * mi for di, mi in zip(d, mabs))
        f_b = mom_err(df) + 8 * f.abs()
        A_, B_, Cc_, Dd_ = (t.detach() for t in (A, B, Cc, Dd))
        mu1, mu2 = m[0].detach(), m[1].detach()
        P = Cc_ * Dd_
        q_abs = (((2 * mu2.abs() * (B_.abs() + A_.abs())) * Cc_.abs() * Dd_.abs()
                  + A_.abs() * B_.abs() * (2 * mu1.abs() * (Dd_.abs() + Cc_.abs()))) / P ** 2,
                 maps[1].detach().abs(), maps[2].detach().abs())
    q_b = []
    for q, qa in zip(maps, q_abs):
        d2 = torch.autograd.grad(q.sum(), m, retain_graph=True, allow_unused=True, materialize_grads=True)
        with torch.no_grad():
            q_b.append(mom_err(d2) + 8 * qa)
    with torch.no_grad():
        f = f.detach()
        qs = [q.detach() for q in maps]
        l1 = (x - y).abs()
        value = (1.0 - lam) * l1.mean() + lam * (1.0 - f.mean())
        s0, s1 = gout * (1.0 - lam) / N, -gout * lam / N
        sgn = torch.sign(x - y)
        inner = conv(qs[0]) + 2 * x * conv(qs[1]) + y * conv(qs[2])
        grad = s0 * sgn + s1 * inner
        inner_b = conv(q_b[0]) + 2 * x.abs() * conv(q_b[1]) + y.abs() * conv(q_b[2]) \
            + N_CONV * (conv(qs[0].abs()) + 2 * x.abs() * conv(qs[1].abs()) + y.abs() * conv(qs[2].abs()))
        grad_b = abs(s1) * inner_b + 2 * abs(s0) * sgn.abs() + 4 * grad.abs()
        red = N * 2.0 ** -29                                                 # a float64 sum of N terms, in units of u
        value_b = (1.0 - lam) * (2 * l1.mean() + red * l1.mean()) + lam * (f_b.mean() + red * f.abs().mean()) \
            + 2 * abs(float(value))
    return float(value), grad.reshape(shape), float(value_b), grad_b.reshape(shape), f.reshape(shape), f_b.reshape(shape)


def loss_f32_emulation(img, gt, lam, gout=1.0):
    """An honest float32 implementation of the fused loss's algorithm (separable window moments, the SSIM
    map and its three derivative maps, their convolution), in torch on whatever device `img` is on: the
    rehearsal that the bounds above are met by float32 arithmetic and are not vacuous."""
    H, W = img.shape[-2:]
    x, y = img.float().reshape(-1, H, W), gt.float().reshape(-1, H, W)
    N = x.numel()
    g = window_1d().to(x.device)
    conv = lambda t: _conv(t, g)
    mu1, mu2, e11, e22, e12 = conv(x), conv(y), conv(x * x), conv(y * y), conv(x * y)
    C1, C2 = np.float32(0.01) * np.float32(0.01), np.float32(0.03) * np.float32(0.03)
    mu1s, mu2s, m12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    A, B = 2 * m12 + C1, 2 * (e12 - m12) + C2
    Cc, Dd = mu1s + mu2s + C1, (e11 - mu1s) + (e22 - mu2s) + C2
    inv = 1.0 / (Cc * Dd)
    f = A * B * inv
    dmu1 = ((2 * mu2 * (B - A)) * Cc * Dd - A * B * (2 * mu1 * (Dd - Cc))) * inv * inv
    ds11 = -A * B * inv / Dd
    ds12 = 2 * A * inv
    value = (1.0 - lam) * (x - y).abs().double().sum() / N + lam * (1.0 - f.double().sum() / N)
    s = torch.tensor([gout * (1.0 - lam) / N, -gout * lam / N], dtype=torch.float32)
    grad = s[0] * torch.sign(x - y) + s[1] * (conv(dmu1) + 2 * x * conv(ds11) + y * conv(ds12))
    return float(value.float()), grad.reshape(img.shape), f.reshape(img.shape)
