"""Float64 evaluation of the 2DGS regularisers of the reference's train.py (lines 80-85) on the render() tail's
outputs, with bounds on the rounding a float32 implementation may add (SURVEY §8f row f2, DESIGN §7l):

    normal_loss = lambda_normal * mean(1 - sum_c rend_normal_c * surf_normal_c)
    dist_loss   = lambda_dist * mean(rend_dist)

Built on tail_loss_exact.tail_f64, whose outputs, per-entry output bounds and gradient bounds it reuses:
  * the values are the reference's lines evaluated in float64 on tail_f64's float64 outputs;
  * a value's bound (units of u = 2^-24) is lambda times the mean over pixels of
    sum_c |r_c| ob_s_c + |s_c| ob_r_c + 3 |r_c s_c| + |1 - r.s| (the output errors, the dot product's and the
    subtraction's own rounding), plus the share of a double reduction of N terms and 2 |value| for the final
    cast to float32 (r = rend_normal, s = surf_normal, ob their tail_f64 bounds);
  * the gradient is tail_f64's float64 autograd with train.py's cotangents c_rn = -lambda_normal/N s,
    c_sn = -lambda_normal/N r and c_dist = lambda_dist/N; its bound is tail_f64's bound for those cotangents
    plus tail_f64's bound for the cotangents' own float32 error (|lambda_normal|/N (ob + 2|.|) for the two normal
    cotangents, known from out_bound): the tail bound carries a cotangent through the vjp on absolute values
    with weight >= 3, so it covers that error's first-order effect.  rend_dist is a copy, so channel 6's bound is
    the rounding of its constant cotangent alone, 2 |lambda_dist| / N.
"""
import types

import numpy as np
import torch
import torch.nn.functional as F

import tail_loss_exact as X

U = X.U
MISTAKES = ("alpha_not_detached", "mean_over_3hw", "view_space_rend_normal", "surf_normal_dropped",
            "depth_ratio_ignored", "dist_grad_missing")


def reg_f64(allmap, view, proj, ratio, lambda_normal, lambda_dist, dev=None):
    """Returns (values, grad, value_bounds, grad_bound, hole):
      values        (normal_loss, dist_loss) in float64;
      grad          d(normal_loss + dist_loss) / d allmap by float64 autograd, NaN where the reference's is
                    (D / alpha not finite);
      value_bounds  the two values' bounds, units of u;
      grad_bound    (7,H,W) per-entry bound of grad where it is finite, units of u;
      hole          what the NaN-free D/alpha rule of DESIGN §7b gives where grad is NaN (0: train.py's graph
                    leaves rend_alpha unused).
    """
    a = X._t(allmap, dev)
    dev = a.device
    _, H, W = a.shape
    N = H * W
    out, _, ob, _, _ = X.tail_f64(a, view, proj, ratio, dev=dev)
    r, s, dist = out["rend_normal"], out["surf_normal"], out["rend_dist"]
    dot = (r * s).sum(0)
    ne = 1 - dot
    values = (lambda_normal * float(ne.mean()), lambda_dist * float(dist.mean()))
    red = N * 2.0 ** -29                                        # a double sum of N terms, units of u
    e = (r.abs() * ob["surf_normal"] + s.abs() * ob["rend_normal"]).sum(0) + 3 * (r * s).abs().sum(0) + ne.abs()
    vb = (abs(lambda_normal) * float(e.mean() + red * ne.abs().mean()) + 2 * abs(values[0]),
          abs(lambda_dist) * red * float(dist.abs().mean()) + 2 * abs(values[1]))

    zero1 = torch.zeros(1, H, W, dtype=torch.float64, device=dev)
    cot = {"rend_alpha": zero1, "surf_depth": zero1, "rend_normal": -lambda_normal / N * s,
           "surf_normal": -lambda_normal / N * r, "rend_dist": zero1 + lambda_dist / N}
    _, grad, _, gb, hole = X.tail_f64(a, view, proj, ratio, cot, dev=dev)
    dcot = {"rend_alpha": zero1, "surf_depth": zero1, "rend_dist": zero1,
            "rend_normal": abs(lambda_normal) / N * (ob["surf_normal"] + 2 * s.abs()),
            "surf_normal": abs(lambda_normal) / N * (ob["rend_normal"] + 2 * r.abs())}
    gb = gb + X.tail_f64(a, view, proj, ratio, dcot, dev=dev)[3]
    gb[6] = 2 * abs(lambda_dist) / N
    return values, grad, vb, gb, hole


def _tail32(a, view, proj, ratio, mistake):
    """The render() tail in float32 (the fused kernels' per-pixel arithmetic), with an optional planted mistake."""
    _, H, W = a.shape
    rot, M, o = (t.float() for t in X.camera_f64(view, proj, W, H))
    alpha = a[1:2]
    rn = a[2:5] if mistake == "view_space_rend_normal" else torch.einsum("khw,kc->chw", a[2:5], rot)
    med = torch.nan_to_num(a[5:6], 0.0, 0.0, X.F32_LOWEST)
    ex = torch.nan_to_num(a[0:1] / alpha, 0.0, 0.0, X.F32_LOWEST)
    r = 0.0 if mistake == "depth_ratio_ignored" else ratio
    sd = ex * (1 - r) + r * med
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    points = sd[0][..., None] * (torch.stack([xs, ys, torch.ones_like(xs)], -1) @ M) + o
    normal = torch.zeros_like(points)
    if H > 2 and W > 2:
        dx = points[2:, 1:-1] - points[:-2, 1:-1]
        dy = points[1:-1, 2:] - points[1:-1, :-2]
        normal[1:-1, 1:-1] = F.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    sn = normal.permute(2, 0, 1) * (alpha if mistake == "alpha_not_detached" else alpha.detach())
    if mistake == "surf_normal_dropped":
        sn = sn.detach()
    dist = a[6:7].detach() if mistake == "dist_grad_missing" else a[6:7]
    return rn, sn, dist


def reg_f32_emulation(allmap, view, proj, ratio, lambda_normal, lambda_dist, mistake=None):
    """The fused op's algorithm in float32 on the CPU: per-pixel float32 terms summed in double, lambda * (sum / N)
    rounded once to float32; backward with float32 cotangents lambda / N and the per-pixel float32 vjp (float32
    autograd), with the kernels' rule where D / alpha is not finite: its term gives 0 to channels 0 and 1.
    `mistake` (one of MISTAKES) plants an error, for checking that the bounds reject it.
    Returns ((normal_loss, dist_loss), grad)."""
    a = torch.as_tensor(np.asarray(allmap, np.float32)).clone().requires_grad_(True)
    _, H, W = a.shape
    rn, sn, dist = _tail32(a, view, proj, ratio, mistake)
    ne = 1 - (rn * sn) if mistake == "mean_over_3hw" else 1 - (rn * sn).sum(0)
    n_ne, n = ne.numel(), H * W
    values = (float(np.float32(lambda_normal * (float(ne.detach().double().sum()) / n_ne))),
              float(np.float32(lambda_dist * (float(dist.detach().double().sum()) / n))))
    s_n = torch.tensor(lambda_normal / n_ne, dtype=torch.float32)
    s_d = torch.tensor(lambda_dist / n, dtype=torch.float32)
    loss = (ne * s_n).sum() + (dist * s_d).sum()
    if loss.requires_grad:
        loss.backward()
    grad = (a.grad if a.grad is not None else torch.zeros_like(a)).detach().clone()
    hole = ~torch.isfinite(a[0].detach() / a[1].detach())
    grad[0][hole] = 0.0
    grad[1][hole] = 0.0
    return values, grad


def worst_ratios(values, grad, exact, nan_rule):
    """Worst |got - exact| / bound for the two values and the gradient (where the exact one is finite).
    nan_rule: 'nan' -- got is NaN exactly where the exact gradient is; 'hole' -- got is finite and equals the hole
    value there.  A mismatch gives inf."""
    ev, eg, vb, gb, hole = exact
    out = {}
    for k, (g, e, b) in enumerate(zip(values, ev, vb)):
        err = abs(float(g) - e)
        out[("normal", "dist")[k]] = err / (U * b) if b > 0 else (np.inf if err > 0 else 0.0)
    grad = grad.to(eg).double()
    nan = torch.isnan(eg)
    if nan_rule == "nan":
        same = torch.equal(torch.isnan(grad), nan)
    else:
        same = bool(torch.isfinite(grad).all()) and torch.equal(grad[nan], hole[nan])
    err = (grad - eg).abs()[~nan]
    b = U * gb[~nan]
    r = torch.where(b > 0, err / b.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    out["grad"] = (float(r.max()) if r.numel() else 0.0) if same else np.inf
    return out, r


def view_of(scene, dev="cpu", dtype=torch.float32):
    H, W = scene["allmap"].shape[1:]
    return types.SimpleNamespace(world_view_transform=torch.from_numpy(scene["view"]).to(dev, dtype),
                                 full_proj_transform=torch.from_numpy(scene["proj"]).to(dev, dtype),
                                 image_width=W, image_height=H)
