"""Pins the camera gradients of the render() tail and of train.py's regularisers to THE REFERENCE'S OWN PYTHON;
writes tests/golden/ref_tail_camera.npz.

The reference's unmodified gaussian_renderer.render() runs on the CPU against a stub rasterizer that returns the
48x36 allmap of ref_tail_loss.npz (as make_golden_surface_reg.py does), on a Camera whose world_view_transform and
full_proj_transform are replaced by leaves that require grad.  Stored for depth_ratio 0 and 1:
  * the gradients with respect to both matrices of sum_k cot_k * out_k over render()'s five tail outputs, for seeded
    float32 cotangents (stored too);
  * for each (lambda_normal, lambda_dist) of PAIRS, the gradients of normal_loss + dist_loss, with train.py's own
    lines 80-85 read as text from the reference's file and executed on render()'s output.

Usage:  python tests/golden/make_golden_tail_camera.py [reference checkout]
"""
import os
import sys
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
KEYS = ("rend_alpha", "rend_normal", "rend_dist", "surf_depth", "surf_normal")
CHANNELS = dict(rend_alpha=1, rend_normal=3, rend_dist=1, surf_depth=1, surf_normal=3)


def tag(ratio, ln, ld):
    return f"r{ratio:g}_n{ln:g}_d{ld:g}".replace(".", "p")


def cotangents(W, H, seed=29):
    g = torch.Generator("cpu").manual_seed(seed)
    return {k: torch.randn(CHANNELS[k], H, W, generator=g) for k in KEYS}


def main(ref="/root/reference"):
    import make_golden as MG
    import make_golden_surface_reg as MR
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
    code = compile(MR.train_lines(ref), os.path.join(ref, "train.py"), "exec")

    W, H, P = 48, 36, 8
    Rm = S.look_at_rotation(12, -7)
    tv = np.array([0.15, -0.05, 0.4])
    mycam = S.make_camera(W, H, R=Rm, t=tv)
    cam = Camera(colmap_id=0, R=Rm, T=tv, FoVx=mycam["FoVx"], FoVy=mycam["FoVy"], image=torch.zeros(3, H, W),
                 gt_alpha_mask=None, image_name="g", uid=0, data_device="cpu")
    view0, proj0 = cam.world_view_transform.detach().clone(), cam.full_proj_transform.detach().clone()
    scene = S.make_scene(P, W, H, 3, depth_complexity=2)
    pc = GaussianModel(3)
    pc.active_sh_degree = 3
    pc._xyz, pc._scaling, pc._rotation = scene["means3D"], torch.log(scene["scales"]), scene["rotations"]
    pc._opacity = torch.log(scene["opacities"] / (1 - scene["opacities"]))
    pc._features_dc, pc._features_rest = scene["shs"][:, :1].contiguous(), scene["shs"][:, 1:].contiguous()

    allmap0 = MT.make_allmap(W, H, 17)
    cot = cotangents(W, H)
    out = {"W": W, "H": H, "viewmatrix": view0.numpy(), "projmatrix": proj0.numpy(), "allmap": allmap0.numpy(),
           **{f"cot_{k}": v.numpy() for k, v in cot.items()}}

    def run(ratio):
        cam.world_view_transform = view0.clone().requires_grad_(True)
        cam.full_proj_transform = proj0.clone().requires_grad_(True)
        holder["allmap"] = allmap0.clone()
        pipe = types.SimpleNamespace(compute_cov3D_python=False, convert_SHs_python=False, depth_ratio=ratio, debug=False)
        return render(cam, pc, pipe, torch.zeros(3))

    def grads(loss):
        gv, gp = torch.autograd.grad(loss, [cam.world_view_transform, cam.full_proj_transform], allow_unused=True,
                                     materialize_grads=True)
        return gv.numpy(), gp.numpy()

    for ratio in RATIOS:
        pkg = run(ratio)
        t = f"r{ratio:g}_outputs"
        out[f"{t}_grad_view"], out[f"{t}_grad_proj"] = grads(sum((pkg[k] * cot[k]).sum() for k in KEYS))
        for ln, ld in PAIRS:
            env = {"render_pkg": run(ratio), "lambda_normal": ln, "lambda_dist": ld}
            exec(code, env)
            t = tag(ratio, ln, ld)
            out[f"{t}_grad_view"], out[f"{t}_grad_proj"] = grads(env["normal_loss"] + env["dist_loss"])
    np.savez_compressed(os.path.join(HERE, "ref_tail_camera.npz"), **out)
    print("wrote ref_tail_camera.npz with", len(out), "arrays")


if __name__ == "__main__":
    main(*sys.argv[1:])
