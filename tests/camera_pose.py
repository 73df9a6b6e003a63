"""Pose refinement through the rasterizer (tests only): the loop a localisation or COLMAP-pose-refinement caller runs.

A seeded scene of textured surfels fills the view of a true camera.  The starting pose is the true one perturbed by
ROT_DEG about a random axis and by TRANS_FRAC of the scene depth along a random direction.  A 6-dof increment
xi = (omega, tau) acts on the starting world-to-camera transform, W2C(xi) = [Exp(omega) R0 | Exp(omega) t0 + tau],
and each step rebuilds world_view_transform, full_proj_transform and camera_center from it exactly as the reference's
Camera does (scene/cameras.py), renders, and takes an Adam step on the L1 loss against the true view.  The splats are
frozen.  `refine` runs the loop on any renderer with the signature of `dense_renderer()` / the public op.
"""
import math

import numpy as np
import torch

import surfel_scenes as S

SEED = 21
P_GPU, W_GPU, H_GPU = 2000, 256, 256
SMALL_P, SMALL_W, SMALL_H = 250, 64, 64
STEPS = 200
ROT_DEG, TRANS_FRAC, DEPTH = 1.0, 0.01, 5.0
LR_ROT, LR_TRANS = 1e-3, 3e-3
FOVY = 50.0


def make_scene(P, W, H, seed=SEED):
    """Surfels spread over depths 3-7 in front of the identity camera, mostly facing it, large enough to cover the
    frame several times, with SH degree 1 colours (view-dependent, so campos carries gradient too)."""
    rng = np.random.default_rng(seed)
    tanfovy = math.tan(math.radians(FOVY) / 2)
    tanfovx = tanfovy * W / H
    z = rng.uniform(3.0, 7.0, P)
    x = rng.uniform(-1.1, 1.1, P) * tanfovx * z
    y = rng.uniform(-1.1, 1.1, P) * tanfovy * z
    px = W / (2 * tanfovx)
    sigma = np.exp(rng.normal(0.0, 0.3, (P, 2))) * math.sqrt(6.0 * W * H / (math.pi * P)) / 3.0
    scales = z[:, None] * sigma / px
    q = np.concatenate([np.ones((P, 1)), rng.normal(0.0, 0.3, (P, 3))], 1)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    shs = np.zeros((P, 16, 3))
    shs[:, 0] = rng.uniform(-1.5, 1.5, (P, 3))
    shs[:, 1:4] = rng.normal(0.0, 0.3, (P, 3, 3))
    f = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32)
    return dict(means3D=f(np.stack([x, y, z], 1)), scales=f(scales), rotations=f(q),
                opacities=f(rng.uniform(0.6, 0.95, (P, 1))), shs=f(shs))


def hat(w):
    z = torch.zeros((), dtype=w.dtype)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def so3_exp(w):
    th2 = (w * w).sum()
    th = torch.sqrt(th2 + 1e-30)
    K = hat(w)
    a = torch.where(th2 > 1e-12, torch.sin(th) / th, 1.0 - th2 / 6.0)
    b = torch.where(th2 > 1e-12, (1.0 - torch.cos(th)) / (th2 + 1e-30), 0.5 - th2 / 24.0)
    return torch.eye(3, dtype=w.dtype) + a * K + b * (K @ K)


def camera_tensors(R, t, proj_T):
    """(world_view_transform, full_proj_transform, camera_center) from W2C = [R | t] (column-vector convention), as
    the reference's Camera builds them: the row-vector transpose, times the transposed projection, and the centre."""
    top = torch.cat([R, t[:, None]], 1)
    w2c = torch.cat([top, torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=R.dtype)], 0)
    wvt = w2c.transpose(0, 1)
    full = wvt @ proj_T
    center = -(R.transpose(0, 1) @ t)
    return wvt, full, center


def perturbation(seed=SEED):
    rng = np.random.default_rng(seed + 1)
    a = rng.normal(size=3)
    d = rng.normal(size=3)
    return (a / np.linalg.norm(a) * math.radians(ROT_DEG), d / np.linalg.norm(d) * TRANS_FRAC * DEPTH)


def pose_errors(R, t, R_true, t_true):
    """Rotation error (rad) and camera-centre error of [R | t] against the true pose."""
    dR = R @ R_true.T
    ang = math.acos(max(-1.0, min(1.0, (np.trace(dR) - 1.0) / 2.0)))
    c, c_true = -R.T @ t, -R_true.T @ t_true
    return ang, float(np.linalg.norm(c - c_true))


def dense_renderer(dtype=torch.float64):
    """Renderer on oracle/dense_torch (CPU, any dtype): render(scene, vm, pm, campos, W, H) -> color (3,H,W)."""
    from oracle import dense_torch as DT

    def render(scene, vm, pm, cp, W, H):
        s = {k: v.to(dtype) for k, v in scene.items()}
        color, _, _, _, _ = DT.render(s["means3D"], s["scales"], s["rotations"], s["opacities"], s["shs"], vm.to(dtype),
                                      pm.to(dtype), cp.to(dtype), torch.zeros(3, dtype=dtype), W, H, 1)
        return color
    return render


def refine(render, P, W, H, steps=STEPS, device="cpu", dtype=torch.float64):
    """Runs the loop; returns the per-step rotation / centre errors and losses."""
    scene = {k: v.to(device) for k, v in make_scene(P, W, H).items()}
    cam = S.make_camera(W, H, fovy_deg=FOVY)
    proj_T = torch.linalg.solve(cam["viewmatrix"].double(), cam["projmatrix"].double())   # full = viewmatrix proj^T
    R_true, t_true = np.eye(3), np.zeros(3)
    w0, d0 = perturbation()
    R0 = so3_exp(torch.tensor(w0)).numpy() @ R_true
    t0 = t_true + d0
    with torch.no_grad():
        vm, pm, cp = camera_tensors(torch.tensor(R_true), torch.tensor(t_true), proj_T)
        target = render(scene, vm.to(device, dtype), pm.to(device, dtype), cp.to(device, dtype), W, H).detach()
    omega = torch.zeros(3, dtype=torch.float64, requires_grad=True)
    tau = torch.zeros(3, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([dict(params=[omega], lr=LR_ROT), dict(params=[tau], lr=LR_TRANS)])
    R0t, t0t = torch.tensor(R0), torch.tensor(t0)
    rot_err, trans_err, losses = [], [], []
    for it in range(steps + 1):
        E = so3_exp(omega)
        R, t = E @ R0t, E @ t0t + tau
        e = pose_errors(R.detach().numpy(), t.detach().numpy(), R_true, t_true)
        rot_err.append(e[0]); trans_err.append(e[1])
        if it == steps:
            break
        vm, pm, cp = camera_tensors(R, t, proj_T)
        color = render(scene, vm.to(device, dtype), pm.to(device, dtype), cp.to(device, dtype), W, H)
        loss = (color - target).abs().mean()
        losses.append(loss.item())
        opt.zero_grad()
        loss.backward()
        opt.step()
    return dict(rot_err=rot_err, trans_err=trans_err, losses=losses)
