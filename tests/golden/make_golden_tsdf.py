"""Pins diff_surfel_rasterization.tsdf to THE REFERENCE'S OWN GaussianExtractor.extract_mesh_unbounded
(utils/mesh_utils.py:184-279 of the reference, `render.py --unbounded`).

The reference runs unmodified on the CPU (make_golden.py's cpu_patches / stub_modules, plus stubs for open3d,
trimesh, skimage and mediapy).  Its extractor is given eight analytic views of a sphere on a plane at small,
unequal sizes, with empty (0) and NaN pixels (tests/tsdf_scenes.py), as MiniCams of its own scene/cameras.py, and
its own estimate_bounding_sphere computes the center and radius from them.  `utils.mcube_utils` is replaced by a
capturing stub: its marching_cubes_with_contraction calls the `sdf` callable the reference hands it on chosen
contracted points (random in the grid's box, |y| = 0, 1 and 2 exactly, cube corners, points on the sphere) and
returns a fake mesh whose vertices are chosen world points (on the sphere and random), which drives the reference's
colour pass (:277).

Writes tests/golden/ref_tsdf.npz: the maps, the cameras' full_proj_transform, center, radius, voxel_size, the
box half-size R, the points of both passes and the reference's TSDF and RGB.

Usage:  python tests/golden/make_golden_tsdf.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "2d-gaussian-splatting_b200"))
REF = "/root/reference"

SIZES = [(40, 30), (33, 25), (48, 36), (24, 40), (37, 29), (45, 31), (29, 22), (52, 38)]
SEED, RESOLUTION = 11, 512
N_RANDOM, N_SURFACE, N_COLOUR = 5000, 600, 1200


def stub_mesh_modules(capture, rng):
    for name in ("open3d", "trimesh", "skimage", "skimage.measure", "mediapy"):
        sys.modules[name] = types.ModuleType(name)
    o3d = sys.modules["open3d"]
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a))
    mpl = sys.modules.get("matplotlib")
    if mpl is not None and not hasattr(mpl, "cm"):
        mpl.cm = types.ModuleType("matplotlib.cm")
    mc = types.ModuleType("utils.mcube_utils")

    def marching_cubes_with_contraction(sdf, bounding_box_min, bounding_box_max, level, resolution, inv_contraction):
        R = float(bounding_box_max[0])
        assert tuple(bounding_box_min) == (-R, -R, -R) and level == 0 and resolution == RESOLUTION
        import tsdf_scenes as TS
        y_surf, w_surf = TS.sphere_surface_points(N_SURFACE, rng, capture["center"], capture["radius"])
        pts = np.concatenate([rng.uniform(-R, R, (N_RANDOM, 3)).astype(np.float32), TS.special_points(R), y_surf])
        capture["R"] = R
        capture["points"] = pts
        capture["tsdf"] = sdf(torch.from_numpy(pts)).numpy().copy()
        cpts = np.concatenate([w_surf[:N_COLOUR // 2],
                               rng.uniform(-2.0, 2.0, (N_COLOUR - N_COLOUR // 2, 3)).astype(np.float32)])
        capture["colour_points"] = cpts
        mesh = types.SimpleNamespace(vertices=cpts.astype(np.float64))   # what `.as_open3d.vertices` holds
        return types.SimpleNamespace(as_open3d=mesh)
    mc.marching_cubes_with_contraction = marching_cubes_with_contraction
    sys.modules["utils.mcube_utils"] = mc


def main():
    import make_golden as MG
    import tsdf_scenes as TS
    MG.cpu_patches()
    MG.stub_modules({})
    capture = {}
    rng = np.random.default_rng(SEED)
    stub_mesh_modules(capture, rng)
    sys.path.insert(0, REF)
    import utils                                                           # noqa: F401 (the package, before the stub)
    sys.modules["utils"].mcube_utils = sys.modules["utils.mcube_utils"]
    from scene.cameras import MiniCam
    from utils.mesh_utils import GaussianExtractor

    views = TS.analytic_views(SIZES, SEED)
    cams = [MiniCam(v.image_width, v.image_height, v.camera["FoVy"], v.camera["FoVx"], v.camera["znear"],
                    v.camera["zfar"], v.world_view_transform, v.full_proj_transform) for v, _, _ in views]
    ex = GaussianExtractor(types.SimpleNamespace(), lambda *a, **k: None, types.SimpleNamespace())
    ex.viewpoint_stack = cams
    ex.depthmaps = [d for _, d, _ in views]
    ex.rgbmaps = [c for _, _, c in views]
    ex.estimate_bounding_sphere()
    capture["center"], capture["radius"] = ex.center.numpy().copy(), float(ex.radius)
    # gaussians spread widely, so R = min(q95 + 0.01, 1.9) = 1.9 (the largest box the reference uses)
    ex.gaussians = types.SimpleNamespace(
        get_xyz=torch.from_numpy(rng.normal(size=(2000, 3)).astype(np.float32) * 50 * ex.radius) + ex.center)
    mesh = ex.extract_mesh_unbounded(resolution=RESOLUTION)
    ref_rgb = np.asarray(mesh.vertex_colors, np.float32)
    out = dict(center=capture["center"].astype(np.float32), radius=np.float64(capture["radius"]),
               voxel_size=np.float64(capture["radius"] * 2 / RESOLUTION), R=np.float64(capture["R"]),
               points=capture["points"], ref_tsdf=capture["tsdf"].astype(np.float32),
               colour_points=capture["colour_points"], ref_rgb=ref_rgb,
               n_frames=np.int64(len(views)))
    for f, (v, d, c) in enumerate(views):
        out[f"proj{f}"] = v.full_proj_transform.numpy()
        out[f"depth{f}"] = d.numpy()
        out[f"rgb{f}"] = c.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_tsdf.npz"), **out)
    t = capture["tsdf"]
    print(f"wrote ref_tsdf.npz: radius {capture['radius']:.4f}, R {capture['R']}, {len(t)} samples "
          f"({int((t != -1).sum())} observed), {len(ref_rgb)} colour points "
          f"({int((ref_rgb != 0).any(1).sum())} observed)")


if __name__ == "__main__":
    main()
