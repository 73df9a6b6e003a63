"""Inputs for the render() tail (f1) and L1+SSIM loss (f2) checks: allmaps with the holes, NaN medians,
frame sizes and cameras where the tail's kernels go wrong, cotangents, and image pairs at the sizes,
contents and layouts where the loss kernel goes wrong.  Everything is generated on the CPU from a seed;
the rasterized allmaps come from the CPU oracle, so the same scenes feed the CPU rehearsal and the GPU
tests."""
import numpy as np
import torch

import surfel_scenes as S

RATIOS = (0.0, 0.3, 1.0)


def _cam(W, H, yaw=12.0, pitch=-7.0, t=(0.15, -0.05, 0.4)):
    cam = S.make_camera(W, H, R=S.look_at_rotation(yaw, pitch), t=list(t))
    return cam["viewmatrix"].numpy(), cam["projmatrix"].numpy()


def synthetic_allmap(W, H, seed, hole_frac=0.12):
    """A plausible rasterizer output: alpha in (0, 1] with holes (alpha == 0, D == 0), alpha-weighted depth
    and normals, a median depth that is 0 where alpha <= 0.5 and a small distortion channel."""
    g = torch.Generator("cpu").manual_seed(seed)
    alpha = torch.rand(1, H, W, generator=g) * 0.99 + 0.01
    alpha[torch.rand(1, H, W, generator=g) < hole_frac] = 0.0
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    z = (3.0 + 1.5 * torch.sin(5 * xx) * torch.cos(4 * yy) + 0.3 * torch.rand(H, W, generator=g))[None]
    n = torch.nn.functional.normalize(torch.randn(3, H, W, generator=g), dim=0)
    median = torch.where(alpha > 0.5, z + 0.05 * torch.randn(1, H, W, generator=g), torch.zeros(1, H, W))
    dist = 0.01 * torch.rand(1, H, W, generator=g)
    return torch.cat([alpha * z, alpha, n * alpha, median, dist], 0).contiguous().numpy()


def rasterized_allmap(W, H, P, seed, depth_complexity, yaw=15.0, pitch=-8.0, t=(0.2, -0.1, 0.3)):
    """The allmap the CPU oracle rasterizes for a generated scene seen by a turned camera."""
    from oracle import surfel_oracle as O
    O.build()
    cam = S.make_camera(W, H, R=S.look_at_rotation(yaw, pitch), t=list(t))
    scene = S.make_scene(P, W, H, seed, depth_complexity=depth_complexity)
    m = torch.cat([scene["means3D"], torch.ones(P, 1)], 1) @ cam["viewmatrix"].inverse()
    scene["means3D"] = m[:, :3].contiguous()
    sc = {k: (v.numpy() if torch.is_tensor(v) else v) for k, v in scene.items()}
    cm = {k: (v.numpy() if torch.is_tensor(v) else v) for k, v in cam.items()}
    cm["W"], cm["H"] = W, H
    _, _, img = O.forward(sc, cm, np.zeros(3, np.float32))
    return np.ascontiguousarray(img["others"], np.float32), cam["viewmatrix"].numpy(), cam["projmatrix"].numpy()


def _scene(allmap, view, proj):
    return dict(allmap=np.ascontiguousarray(allmap, np.float32), view=np.float32(view), proj=np.float32(proj))


def golden():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_tail_loss.npz"))
    return _scene(g["allmap"], g["viewmatrix"], g["projmatrix"])


def dense_raster():
    """The 320x200 rasterized scene of the original parity test: no empty pixel."""
    return _scene(*rasterized_allmap(320, 200, 6000, 5, 20))


def sparse_raster():
    """Few splats over the same frame: at least 10 % of the pixels are empty."""
    am, v, p = rasterized_allmap(320, 200, 60, 7, 6)
    assert float((am[1] == 0).mean()) >= 0.10, float((am[1] == 0).mean())
    return _scene(am, v, p)


def holes():
    """An isolated hole, 5x5 empty blocks (their inner 3x3 points all sit at the camera centre, so v == 0
    exactly: normalize's eps branch), and holes along all four borders."""
    W, H = 64, 48
    am = synthetic_allmap(W, H, 31, hole_frac=0.0)
    empty = np.zeros((H, W), bool)
    empty[20, 30] = True
    empty[5:10, 5:10] = True
    empty[30:36, 40:47] = True
    empty[0, :] = empty[:, 0] = True
    empty[H - 1, 10:30] = True
    empty[15:40, W - 1] = True
    am[0][empty] = am[1][empty] = 0.0
    am[2:5, empty] = 0.0
    am[5][empty] = 0.0
    return _scene(am, *_cam(W, H))


def nan_medians():
    W, H = 40, 30
    am = synthetic_allmap(W, H, 37)
    g = np.random.default_rng(5)
    am[5][g.random((H, W)) < 0.15] = np.nan
    return _scene(am, *_cam(W, H))


def zero_alpha_depth():
    """alpha == 0 with D != 0: D / alpha = +-inf, which nan_to_num maps to 0 (+inf) or the lowest float (-inf).
    -inf only survives into surf_depth at depth_ratio 1, so the negative D sit where the caller uses ratio 1."""
    W, H = 40, 30
    am = synthetic_allmap(W, H, 41, hole_frac=0.0)
    g = np.random.default_rng(6)
    z = g.random((H, W)) < 0.1
    am[1][z] = 0.0
    am[0][z] = 2.5
    return _scene(am, *_cam(W, H))


def zero_alpha_negative_depth():
    s = zero_alpha_depth()
    s["allmap"][0][s["allmap"][1] == 0] = -2.5
    return s


def frame(W, H, seed=43):
    return _scene(synthetic_allmap(W, H, seed + W * 7 + H), *_cam(W, H))


def far_camera():
    """A camera about 100 units from the origin: the point cancellation P[y+1] - P[y-1] loses 2^-24 * 100."""
    W, H = 96, 64
    return _scene(synthetic_allmap(W, H, 47), *_cam(W, H, t=(60.0, -50.0, 60.0)))


# name -> (builder, depth ratios)
ALLMAPS = {
    "golden": (golden, RATIOS),
    "dense_raster": (dense_raster, RATIOS),
    "sparse_raster": (sparse_raster, RATIOS),
    "holes": (holes, RATIOS),
    "nan_medians": (nan_medians, RATIOS),
    "zero_alpha_depth": (zero_alpha_depth, RATIOS),
    "zero_alpha_negative_depth": (zero_alpha_negative_depth, (1.0,)),
    "far_camera": (far_camera, RATIOS),
    "f1x1": (lambda: frame(1, 1), RATIOS),
    "f2x2": (lambda: frame(2, 2), RATIOS),
    "f3x3": (lambda: frame(3, 3), RATIOS),
    "f1x64": (lambda: frame(1, 64), RATIOS),
    "f64x1": (lambda: frame(64, 1), RATIOS),
    **{f"f{W}x{H}": ((lambda W=W, H=H: frame(W, H)), (0.3,)) for W in (31, 32, 33) for H in (7, 8, 9)},
    "f1920x1080": (lambda: frame(1920, 1080), (0.3,)),
}
ALLMAP_CASES = [(name, r) for name, (_, rs) in ALLMAPS.items() for r in rs]


def cotangents(H, W, kind, out=None, seed=3):
    """'random': every output gets a random cotangent.  'train': train.py's graph, the float32 gradient of
    train_graph_loss with respect to the outputs `out` (surf_depth is unused, so autograd hands the backward
    zeros for it; rend_alpha is unused too)."""
    g = torch.Generator("cpu").manual_seed(seed + H * 131 + W)
    shapes = dict(rend_alpha=(1, H, W), rend_normal=(3, H, W), rend_dist=(1, H, W), surf_depth=(1, H, W),
                  surf_normal=(3, H, W))
    if kind == "random":
        return {k: torch.randn(*s, generator=g).numpy() for k, s in shapes.items()}
    o = {k: torch.as_tensor(v).detach().cpu().float().requires_grad_(True) for k, v in out.items()}
    train_graph_loss(o).backward()
    return {k: (o[k].grad if o[k].grad is not None else torch.zeros(*shapes[k])).numpy() for k in shapes}


def train_graph_loss(out, lambda_normal=0.05, lambda_dist=100.0):
    """train.py's regularisers on the tail's outputs (reference train.py:76-86, with both switched on)."""
    normal_error = (1 - (out["rend_normal"] * out["surf_normal"]).sum(dim=0))[None]
    return lambda_normal * normal_error.mean() + lambda_dist * out["rend_dist"].mean()


# ----------------------------------------------------------------------------------------- image pairs (f2)

def image_pair(shape, content, seed=0):
    g = torch.Generator("cpu").manual_seed(seed + sum(shape))
    if content == "noisy":
        base = torch.rand(*shape, generator=g)
        gt = (base + 0.1 * torch.randn(*shape, generator=g)).clamp(0, 1)
        img = (base + 0.15 * torch.randn(*shape, generator=g)).clamp(0, 1)
    elif content == "flat_bright":
        gt = 0.97 + 1e-3 * torch.rand(*shape, generator=g)
        img = 0.98 + 1e-3 * torch.rand(*shape, generator=g)
    elif content == "clamped":
        gt = (2 * torch.rand(*shape, generator=g) - 0.5).clamp(0, 1)
        img = (2 * torch.rand(*shape, generator=g) - 0.5).clamp(0, 1)
    elif content == "equal":
        img = torch.rand(*shape, generator=g)
        gt = img.clone()
    else:
        raise ValueError(content)
    return img.contiguous(), gt.contiguous()


# (shape, content, lambda)
LOSS_CASES = [
    ((3, 1, 1), "noisy", 0.2), ((3, 5, 7), "noisy", 0.2), ((3, 10, 10), "noisy", 1.0),
    ((3, 16, 16), "noisy", 0.2), ((3, 17, 33), "noisy", 0.2), ((3, 1, 57), "noisy", 0.2), ((3, 45, 1), "noisy", 1.0),
    ((3, 97, 131), "noisy", 0.2), ((3, 256, 320), "noisy", 0.2), ((3, 64, 48), "noisy", 1.0), ((3, 33, 17), "noisy", 0.0),
    ((3, 1080, 1920), "noisy", 0.2), ((3, 2160, 3840), "noisy", 0.2),
    ((3, 64, 80), "flat_bright", 0.2), ((3, 64, 80), "flat_bright", 1.0),
    ((3, 64, 80), "clamped", 0.2), ((3, 64, 80), "equal", 0.2), ((3, 64, 80), "equal", 1.0),
    ((1, 40, 56), "noisy", 0.2), ((4, 40, 56), "noisy", 0.2),
    ((1, 3, 40, 56), "noisy", 0.2), ((2, 3, 40, 56), "noisy", 0.2), ((2, 3, 1080, 1920), "noisy", 0.2),
]


def loss_case_id(case):
    shape, content, lam = case
    return "x".join(map(str, shape)) + f"-{content}-{lam}"
