"""Records what THE REFERENCE'S OWN marching_cubes_with_contraction (utils/mcube_utils.py:17-95 of the reference)
does around its marching cubes, for diff_surfel_rasterization.tsdf.UnboundedTSDF.extract_mesh (DESIGN.md §7j).

The reference's GaussianExtractor.extract_mesh_unbounded runs unmodified on the CPU (make_golden.cpu_patches /
stub_modules, the analytic views of make_golden_tsdf.py) at resolution 1024, and calls the reference's real
marching_cubes_with_contraction with its own inv_contraction; only the `sdf` it passes is replaced by a cheap analytic
one (a sphere in contracted space that meets two of the eight crops), so each 512^3 crop costs seconds, not hours.
skimage.measure and trimesh are stubs that record:
  * per crop: the three torch.linspace axes, the min and max of the crop's values, whether skimage was called, and
    the spacing and offset it was given;
  * the float32 contracted vertices passed to inv_contraction and the clipped result.  The first called crop's fake
    mesh holds chosen contracted points: |y| = 1 and 2 exactly, points beyond 2, points whose norm is exact in
    float32, and random points in the box.

Writes tests/golden/ref_mcubes.npz.  Needs about 6 GB of host memory while a crop is built.

Usage:  python tests/golden/make_golden_mcubes.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_tsdf as MGT  # noqa: E402  (sets the paths)

REF = MGT.REF
RESOLUTION = 1024
SPHERE_C, SPHERE_R = (0.1, 0.5, 0.45), 0.3


def chosen_points(R, rng):
    pts = [[1, 0, 0], [0, -1, 0], [0, 0, 1], [2, 0, 0], [0, 2, 0], [0, 0, -2], [2.5, 0, 0], [0, -3, 0],
           [0.75, 1, 0], [1.5, 2, 0], [0.375, 0.5, 0], [0, 0.75, -1], [-1.5, 0, 2], [0.5, 0.5, 0.5],
           [1.9, 0, 0], [1.25, 1.25, 1.25], [0, 0, 0], [1.999, 0, 0], [0, 2.001, 0], [1e-3, -2e-3, 3e-3]]
    rnd = rng.uniform(-R, R, (200, 3))
    return np.concatenate([np.asarray(pts, np.float64), rnd])


def main():
    import make_golden as MG
    MG.cpu_patches()
    MG.stub_modules({})
    rng = np.random.default_rng(7)
    rec = {"axes": [], "zmin": [], "zmax": [], "called": [], "spacing": [], "offset": [], "chunks": 0}
    for name in ("open3d", "trimesh", "trimesh.util", "skimage", "skimage.measure", "mediapy"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["open3d"].utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a))
    mpl = sys.modules.get("matplotlib")
    if mpl is not None and not hasattr(mpl, "cm"):
        mpl.cm = types.ModuleType("matplotlib.cm")

    lin = torch.linspace

    def linspace(*a, **k):
        out = lin(*a, **k)
        rec["axes"].append(out.numpy().copy())
        return out
    torch.linspace = linspace

    def marching_cubes(volume, level, spacing):
        assert level == 0 and volume.dtype == np.float32 and volume.shape == (512, 512, 512)
        rec["called"][-1] = True
        rec["spacing"][-1] = np.asarray(spacing, np.float64)
        verts = np.zeros((1, 3))                       # row 0 + offset: the offset itself
        if "first" not in rec:
            rec["first"] = len(rec["called"]) - 1
            rec["R"] = float(rec["bounds"])
            n = RESOLUTION // 512
            xs = np.linspace(-rec["bounds"], rec["bounds"], n + 1)
            c = len(rec["called"]) - 1
            offset = np.array([xs[c // (n * n)], xs[c // n % n], xs[c % n]])
            verts = np.concatenate([verts, rec["chosen"] - offset])      # the chosen points once offset
        rec["returned"] = verts
        return verts, np.zeros((0, 3), np.int64), np.zeros_like(verts), None

    class Trimesh:
        def __init__(self, verts, faces, normals):
            rec["offset"][-1] = np.asarray(verts[0], np.float64)
            self.vertices = np.asarray(verts, np.float64)

    class Combined:
        def __init__(self, vertices):
            self.vertices = vertices
            self.merged = None

        def merge_vertices(self, digits_vertex):
            self.merged = digits_vertex

        @property
        def as_open3d(self):
            return types.SimpleNamespace(vertices=self.vertices, vertex_colors=None)

    sys.modules["skimage"].measure = sys.modules["skimage.measure"]
    sys.modules["skimage.measure"].marching_cubes = marching_cubes
    sys.modules["trimesh"].Trimesh = Trimesh
    sys.modules["trimesh"].util = sys.modules["trimesh.util"]
    sys.modules["trimesh.util"].concatenate = lambda ms: Combined(np.concatenate([m.vertices for m in ms]))

    sys.path.insert(0, REF)
    import utils                                                           # noqa: F401
    import importlib.util
    spec = importlib.util.spec_from_file_location("utils.mcube_utils", os.path.join(REF, "utils", "mcube_utils.py"))
    real = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(real)
    wrapper = types.ModuleType("utils.mcube_utils")

    def sdf_analytic(p):
        v = torch.linalg.norm(p - torch.tensor(SPHERE_C, dtype=torch.float32), dim=-1) - SPHERE_R
        if rec["chunks"] % 8 == 0:                     # a 512^3 crop is evaluated in eight 256^3 calls
            rec["zmin"].append(np.inf), rec["zmax"].append(-np.inf)
            rec["called"].append(False), rec["spacing"].append(np.full(3, np.nan)), rec["offset"].append(
                np.full(3, np.nan))
        rec["chunks"] += 1
        rec["zmin"][-1] = min(rec["zmin"][-1], float(v.min()))
        rec["zmax"][-1] = max(rec["zmax"][-1], float(v.max()))
        return v

    def mcwc(sdf, bounding_box_min, bounding_box_max, level, resolution, inv_contraction):
        rec["bounds"] = bounding_box_max[0]
        rec["chosen"] = chosen_points(bounding_box_max[0], rng)

        def inv(x):
            rec["contracted"] = x.numpy().copy()
            out = inv_contraction(x)
            return out
        mesh = real.marching_cubes_with_contraction(sdf=sdf_analytic, bounding_box_min=bounding_box_min,
                                                    bounding_box_max=bounding_box_max, level=level,
                                                    resolution=resolution, inv_contraction=inv)
        rec["clipped"] = np.asarray(mesh.vertices).copy()
        rec["merged"] = mesh.merged
        return mesh
    wrapper.marching_cubes_with_contraction = mcwc
    sys.modules["utils.mcube_utils"] = wrapper
    sys.modules["utils"].mcube_utils = wrapper
    from scene.cameras import MiniCam
    from utils.mesh_utils import GaussianExtractor
    import tsdf_scenes as TS

    views = TS.analytic_views(MGT.SIZES[:3], MGT.SEED)
    cams = [MiniCam(v.image_width, v.image_height, v.camera["FoVy"], v.camera["FoVx"], v.camera["znear"],
                    v.camera["zfar"], v.world_view_transform, v.full_proj_transform) for v, _, _ in views]
    ex = GaussianExtractor(types.SimpleNamespace(), lambda *a, **k: None, types.SimpleNamespace())
    ex.viewpoint_stack = cams
    ex.depthmaps = [d for _, d, _ in views]
    ex.rgbmaps = [c for _, _, c in views]
    ex.estimate_bounding_sphere()
    ex.gaussians = types.SimpleNamespace(
        get_xyz=torch.from_numpy(rng.normal(size=(2000, 3)).astype(np.float32) * 0.4 * ex.radius) + ex.center)
    ex.extract_mesh_unbounded(resolution=RESOLUTION)

    n = RESOLUTION // 512
    crops = np.array([(i, j, k) for i in range(n) for j in range(n) for k in range(n)])
    axes = np.stack(rec["axes"]).reshape(len(crops), 3, 512)
    out = dict(resolution=np.int64(RESOLUTION), R=np.float64(rec["bounds"]),
               xs=np.linspace(-rec["bounds"], rec["bounds"], n + 1), crops=crops, axis=axes,
               zmin=np.array(rec["zmin"]), zmax=np.array(rec["zmax"]), called=np.array(rec["called"]),
               spacing=np.stack(rec["spacing"]), offset=np.stack(rec["offset"]),
               first_called=np.int64(rec["first"]), contracted=rec["contracted"].astype(np.float32),
               clipped=rec["clipped"].astype(np.float32), merge_digits=np.int64(rec["merged"]),
               center=ex.center.numpy().astype(np.float32), radius=np.float64(ex.radius))
    np.savez_compressed(os.path.join(HERE, "ref_mcubes.npz"), **out)
    print(f"wrote ref_mcubes.npz: R {rec['bounds']:.4f}, crops called {np.nonzero(out['called'])[0].tolist()}, "
          f"{len(out['contracted'])} vertices through inv_contraction")


if __name__ == "__main__":
    main()
