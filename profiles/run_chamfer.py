"""chamfer.sample_mesh and chamfer.dtu_chamfer (csrc/chamfer.cu) on a synthetic scan-sized scene: a bumpy height
field of about --tris triangles (default 2 M) and a noisy STL cloud of --stl points (default 3 M) near it, with an
observation mask over the box and a plane that cuts the STL.  These are assumed sizes, not measured DTU sizes.

Per call: the wall time ended by torch.cuda.synchronize() (after a warm-up call), its split by the library's
per-stage CUDA events (chamfer_sample, chamfer_downsample, chamfer_select, chamfer_nn and the radix sort's stages),
the greedy round count and the set sizes.  Beside them, on this machine's host, sklearn's radius_neighbors and
kneighbors (kd_tree, n_jobs=-1, as eval.py calls them) on the same points.  Prints the card, its power limit and one
JSON line.

Usage:  python profiles/run_chamfer.py [--tris 2000000] [--stl 3000000] [--leg 0.6] [--no-sklearn]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import numpy as np
import torch

from diff_surfel_rasterization import _cabi
from diff_surfel_rasterization.chamfer import dtu_chamfer, sample_mesh

ap = argparse.ArgumentParser()
ap.add_argument("--tris", type=int, default=2_000_000)
ap.add_argument("--stl", type=int, default=3_000_000)
ap.add_argument("--leg", type=float, default=0.6, help="grid spacing: 0.6 gives three samples per triangle")
ap.add_argument("--no-sklearn", action="store_true")
args = ap.parse_args()

assert torch.cuda.is_available(), "run_chamfer.py needs a GPU"
dev = torch.device("cuda")
out = {"gpu": torch.cuda.get_device_name(dev)}
try:
    out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:   # noqa: BLE001
    out["power_limit"] = f"unknown ({type(e).__name__})"

lib = _cabi.load()
STAGES = [lib.surfel_profile_stage_name(i).decode() for i in range(lib.surfel_profile_num_stages())]


def stage_ms():
    ms = (ctypes.c_double * len(STAGES))()
    cnt = (ctypes.c_int * len(STAGES))()
    lib.surfel_profile_read(ms, cnt)
    return {s: round(m, 3) for s, m, c in zip(STAGES, ms, cnt) if c}


def timed(fn):
    fn()                                          # warm-up
    torch.cuda.synchronize()
    lib.surfel_profile_enable(0)
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t) * 1e3
    lib.surfel_profile_enable(1)
    fn()
    torch.cuda.synchronize()
    split = stage_ms()
    lib.surfel_profile_enable(0)
    return r, round(wall, 2), split


# scene: an n x n height field over [0, side]^2 whose triangles have legs of about --leg
rng = np.random.default_rng(0)
n = int(np.sqrt(args.tris / 2)) + 1
side = args.leg * (n - 1)
xs = np.linspace(0, side, n)
X, Y = np.meshgrid(xs, xs, indexing="ij")
Z = 3 * np.sin(X / 7) * np.cos(Y / 9)
verts = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)
idx = np.arange(n * n).reshape(n, n)
a, b, c, d = idx[:-1, :-1].ravel(), idx[1:, :-1].ravel(), idx[:-1, 1:].ravel(), idx[1:, 1:].ravel()
faces = np.concatenate([np.stack([a, b, c], 1), np.stack([b, d, c], 1)])
stl = verts[rng.integers(0, len(verts), args.stl)] + 0.2 * rng.standard_normal((args.stl, 3))
bb = np.array([[-1.0, -1.0, -5.0], [side + 1, side + 1, 5.0]])
res = 1.0
obs = torch.rand(tuple(int(x) for x in np.ceil((bb[1] - bb[0]) / res) + 1), device=dev) < 0.9
plane = np.array([0.01, 0.0, 1.0, 2.0])
v_d, f_d, s_d = (torch.as_tensor(x).to(dev) for x in (verts, faces, stl))
out.update(tris=len(faces), verts=len(verts), stl=len(stl))

pcd, out["sample_ms"], out["sample_stages"] = timed(lambda: sample_mesh(v_d, f_d))
out["points"] = pcd.shape[0]
perm = torch.randperm(pcd.shape[0], device=dev, generator=torch.Generator(device=dev).manual_seed(1))
r, out["chamfer_ms"], out["chamfer_stages"] = timed(lambda: dtu_chamfer(pcd, s_d, obs, bb, res, plane, perm=perm))
out.update(rounds=r.rounds, data_down=r.data_down.shape[0], data_in_obs=r.dist_d2s.shape[0],
           stl_above=r.dist_s2d.shape[0], mean_d2s=r.mean_d2s, mean_s2d=r.mean_s2d)
print(f"{out['gpu']} at {out['power_limit']}: {out['points']} points from {out['tris']} triangles, "
      f"sample_mesh {out['sample_ms']} ms, dtu_chamfer {out['chamfer_ms']} ms, {out['rounds']} greedy rounds")

if not args.no_sklearn:
    import sklearn.neighbors as skln
    x = pcd[perm].cpu().numpy()
    nn = skln.NearestNeighbors(n_neighbors=1, radius=0.2, algorithm="kd_tree", n_jobs=-1)
    t = time.perf_counter()
    nn.fit(x)
    nn.radius_neighbors(x, radius=0.2, return_distance=False)
    out["sklearn_radius_ms"] = round((time.perf_counter() - t) * 1e3, 1)
    t = time.perf_counter()
    nn.fit(stl)
    nn.kneighbors(r.data_down.cpu().numpy(), n_neighbors=1, return_distance=True)
    out["sklearn_knn_d2s_ms"] = round((time.perf_counter() - t) * 1e3, 1)
    out["host_cpus"] = os.cpu_count()
print(json.dumps(out))
