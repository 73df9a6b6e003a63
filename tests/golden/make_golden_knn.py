"""Pins simple_knn.distCUDA2's call site to THE REFERENCE'S OWN GaussianModel.create_from_pcd
(/root/reference/scene/gaussian_model.py:124-146, the call at :134-135).

The reference runs unmodified on the CPU (make_golden.py's cpu_patches / stub_modules, plus torch.rand, whose
device="cuda" cpu_patches does not cover).  Its point cloud is the reference's own random initialisation
(/root/reference/scene/dataset_readers.py:236-242: uniform in [-1.3, 1.3]^3), 5 000 points from a fixed seed.
The distCUDA2 stub records the tensor create_from_pcd passes and returns the certified CPU restatement
(tests/knn_oracle.py) of it.  Writes tests/golden/ref_init_knn.npz: points (what the cloud holds), received
(the distCUDA2 input), dist2 (what it returned) and scaling (the resulting _scaling).

Usage:  python tests/golden/make_golden_knn.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "2d-gaussian-splatting_b200"))
REF = "/root/reference"


def main():
    import knn_oracle as KO
    import make_golden as MG
    MG.cpu_patches()
    orig_rand = torch.rand

    def rand(*a, **k):
        if "device" in k:
            k["device"] = "cpu"
        return orig_rand(*a, **k)
    torch.rand = rand
    MG.stub_modules({})
    store = {}

    def distCUDA2(points):
        store["received"] = points.detach().clone().numpy()
        store["dist2"] = KO.mean_sq_dist(store["received"])
        return torch.from_numpy(store["dist2"].copy())
    sys.modules["simple_knn._C"].distCUDA2 = distCUDA2
    sys.path.insert(0, REF)
    from scene.gaussian_model import GaussianModel
    from utils.graphics_utils import BasicPointCloud
    from utils.sh_utils import SH2RGB

    num_pts = 5000
    rng = np.random.default_rng(20240)
    xyz = rng.random((num_pts, 3)) * 2.6 - 1.3
    shs = rng.random((num_pts, 3)) / 255.0
    pcd = BasicPointCloud(points=xyz, colors=SH2RGB(shs), normals=np.zeros((num_pts, 3)))
    torch.manual_seed(0)
    pc = GaussianModel(3)
    pc.create_from_pcd(pcd, 1.0)
    np.savez(os.path.join(HERE, "ref_init_knn.npz"), points=xyz, received=store["received"], dist2=store["dist2"],
             scaling=pc._scaling.detach().numpy())
    print("wrote ref_init_knn.npz:", num_pts, "points")


if __name__ == "__main__":
    main()
