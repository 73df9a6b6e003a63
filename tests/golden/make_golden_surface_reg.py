"""Pins the regularisers of the reference's train.py (normal consistency and depth distortion) to THE
REFERENCE'S OWN PYTHON; writes tests/golden/ref_surface_reg.npz.

The reference's unmodified gaussian_renderer.render() runs on the CPU against a stub rasterizer that returns
the 48x36 allmap of ref_tail_loss.npz (same construction as make_golden_tail_loss.py).  Then train.py's own
lines 80-85 (from reading render_pkg's three maps through normal_loss and dist_loss) are read as text from the
reference's file and executed on render()'s output, so the pinned arithmetic is the reference's.  Stored for
depth_ratio 0 and 1 and each (lambda_normal, lambda_dist) of PAIRS: normal_loss, dist_loss (the float32 values,
as float64) and the gradient of normal_loss + dist_loss with respect to allmap, NaNs included.

Usage:  python tests/golden/make_golden_surface_reg.py [reference checkout]
"""
import os
import sys
import textwrap
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "2d-gaussian-splatting_b200"))

RATIOS = (0.0, 1.0)
PAIRS = ((0.05, 0.0), (0.05, 100.0), (0.05, 1000.0), (0.0, 100.0), (0.0, 0.0))
TRAIN_LINES = (80, 85)          # train.py: rend_dist = ... through dist_loss = ...


def tag(ratio, ln, ld):
    return f"r{ratio:g}_n{ln:g}_d{ld:g}".replace(".", "p")


def train_lines(ref):
    with open(os.path.join(ref, "train.py")) as f:
        lines = f.read().splitlines()[TRAIN_LINES[0] - 1:TRAIN_LINES[1]]
    src = textwrap.dedent("\n".join(lines))
    assert src.startswith("rend_dist = ") and "normal_loss = " in src and src.rstrip().split("\n")[-1].startswith("dist_loss = "), src
    return src


def main(ref="/root/reference"):
    import make_golden as MG
    import make_golden_tail_loss as MT
    import surfel_scenes as S
    MG.cpu_patches()
    holder = {}
    MG.stub_modules({})                                                         # plyfile / simple_knn / cv2 stubs
    dsr = types.ModuleType("diff_surfel_rasterization")

    class Settings:
        def __init__(self, **kw):
            self.__dict__.update(kw)

    class Rasterizer:
        def __init__(self, raster_settings):
            self.rs = raster_settings

        def __call__(self, **kw):
            P = kw["means3D"].shape[0]
            H, W = self.rs.image_height, self.rs.image_width
            return torch.zeros(3, H, W), torch.ones(P, dtype=torch.int32), holder["allmap"]
    dsr.GaussianRasterizationSettings, dsr.GaussianRasterizer = Settings, Rasterizer
    sys.modules["diff_surfel_rasterization"] = dsr
    sys.path.insert(0, ref)
    from gaussian_renderer import render
    from scene.cameras import Camera
    from scene.gaussian_model import GaussianModel
    code = compile(train_lines(ref), os.path.join(ref, "train.py"), "exec")

    W, H, P = 48, 36, 8
    Rm = S.look_at_rotation(12, -7)
    tv = np.array([0.15, -0.05, 0.4])
    mycam = S.make_camera(W, H, R=Rm, t=tv)
    cam = Camera(colmap_id=0, R=Rm, T=tv, FoVx=mycam["FoVx"], FoVy=mycam["FoVy"], image=torch.zeros(3, H, W),
                 gt_alpha_mask=None, image_name="g", uid=0, data_device="cpu")
    scene = S.make_scene(P, W, H, 3, depth_complexity=2)
    pc = GaussianModel(3)
    pc.active_sh_degree = 3
    pc._xyz, pc._scaling, pc._rotation = scene["means3D"], torch.log(scene["scales"]), scene["rotations"]
    pc._opacity = torch.log(scene["opacities"] / (1 - scene["opacities"]))
    pc._features_dc, pc._features_rest = scene["shs"][:, :1].contiguous(), scene["shs"][:, 1:].contiguous()

    allmap0 = MT.make_allmap(W, H, 17)
    out = {"W": W, "H": H, "viewmatrix": cam.world_view_transform.numpy(), "projmatrix": cam.full_proj_transform.numpy(),
           "allmap": allmap0.numpy()}
    for ratio in RATIOS:
        for ln, ld in PAIRS:
            holder["allmap"] = allmap0.clone().requires_grad_(True)
            pipe = types.SimpleNamespace(compute_cov3D_python=False, convert_SHs_python=False, depth_ratio=ratio, debug=False)
            env = {"render_pkg": render(cam, pc, pipe, torch.zeros(3)), "lambda_normal": ln, "lambda_dist": ld}
            exec(code, env)
            (env["normal_loss"] + env["dist_loss"]).backward()
            t = tag(ratio, ln, ld)
            out[f"{t}_normal_loss"] = np.float64(env["normal_loss"].item())
            out[f"{t}_dist_loss"] = np.float64(env["dist_loss"].item())
            out[f"{t}_grad_allmap"] = holder["allmap"].grad.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_surface_reg.npz"), **out)
    print("wrote ref_surface_reg.npz with", len(out), "arrays")


if __name__ == "__main__":
    main(*sys.argv[1:])
