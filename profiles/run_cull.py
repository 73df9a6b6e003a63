"""chamfer.cull_scan (csrc/cull.cu) on a DTU-size scene: 49 views with 1600 x 1200 masks at disk(24) and about 2 M
vertices in mesh order (the scene of tests/test_cull_gpu.py).

Per call: the wall time ended by torch.cuda.synchronize() (after a warm-up call) and its split by the library's
per-stage CUDA events (cull_dilate, cull_vertices, cull_faces, cull_emit).  Beside it, the reference's way on the same
card: its torch lines (cuBLAS A @ V and grid_sample per view, with the device's dilated masks given), timed with CUDA
events, and the host dilation, for which scipy.ndimage.binary_dilation (what skimage calls) stands in for skimage,
timed on --scipy-views views of this machine's host and scaled to 49.  Prints the card, its power limit and one JSON
line.

Usage:  python profiles/run_cull.py [--scipy-views 3] [--repeat 10]"""
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

import cull_ref as CR
from diff_surfel_rasterization import _cabi
from diff_surfel_rasterization.chamfer import _cull, cull_scan, dtu_projections
from test_cull_gpu import _dtu_scene, torch_lines, unpack

ap = argparse.ArgumentParser()
ap.add_argument("--scipy-views", type=int, default=3)
ap.add_argument("--repeat", type=int, default=10)
args = ap.parse_args()

assert torch.cuda.is_available(), "run_cull.py needs a GPU"
dev = torch.device("cuda")
out = {"gpu": torch.cuda.get_device_name(dev)}
try:
    out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:   # noqa: BLE001
    out["power_limit"] = f"unknown ({type(e).__name__})"

lib = _cabi.load()
STAGES = [lib.surfel_profile_stage_name(i).decode() for i in range(lib.surfel_profile_num_stages())]

verts, faces, masks, world, scale = _dtu_scene(np.random.default_rng(5))
v, f, m = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (verts, faces, masks))
out.update(views=int(len(masks)), mask_shape=list(masks.shape[1:]), verts=int(len(verts)), faces=int(len(faces)))


def call():
    return cull_scan(v, f, m, world, scale, radius=24)


res = call()
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(args.repeat):
    res = call()
torch.cuda.synchronize()
out["cull_scan_ms"] = round((time.perf_counter() - t0) * 1e3 / args.repeat, 3)
out["kept_verts"], out["kept_faces"] = int(res[0].shape[0]), int(res[1].shape[0])

lib.surfel_profile_enable(1)
ms = (ctypes.c_double * len(STAGES))()
cnt = (ctypes.c_int * len(STAGES))()
lib.surfel_profile_read(ms, cnt)
for _ in range(args.repeat):
    call()
torch.cuda.synchronize()
lib.surfel_profile_read(ms, cnt)
lib.surfel_profile_enable(0)
out["stage_ms"] = {s: round(x / args.repeat, 3) for s, x, c in zip(STAGES, ms, cnt) if c and s.startswith("cull")}

# the reference's way: torch lines on this card, with the device's dilated masks
A = dtu_projections(world, scale)
r = _cull("profile", v, f, m, A, scale, None, (1600, 1200), 24)
D = torch.from_numpy(unpack(r["dilated"], masks.shape[2])).to(dev)
A4 = torch.zeros((len(A), 4, 4), dtype=torch.float32, device=dev)
A4[:, :3] = torch.from_numpy(A).to(dev)
A4[:, 3, 3] = 1
torch_lines(v, A4, D, (1600, 1200))
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(3):
    keep_ref = torch_lines(v, A4, D, (1600, 1200))
e1.record()
torch.cuda.synchronize()
out["torch_lines_ms"] = round(e0.elapsed_time(e1) / 3, 3)
out["torch_lines_decisions_differ"] = int((keep_ref != r["keep"]).sum())

import scipy.ndimage as ndi   # noqa: E402
disk = CR.disk(24)
t0 = time.perf_counter()
for k in range(args.scipy_views):
    ndi.binary_dilation(masks[k] != 0, structure=disk, border_value=0)
per_view = (time.perf_counter() - t0) / args.scipy_views
out["scipy_dilation_s_per_view"] = round(per_view, 3)
out["scipy_dilation_s_49_views_scaled"] = round(per_view * len(masks), 2)
out["host_cpus"] = os.cpu_count()

print(f"{out['gpu']} at {out['power_limit']}: cull_scan {out['cull_scan_ms']} ms on {out['views']} views of "
      f"{masks.shape[2]} x {masks.shape[1]} and {out['verts']} vertices; stages {out['stage_ms']}; torch lines "
      f"{out['torch_lines_ms']} ms; scipy dilation {out['scipy_dilation_s_per_view']} s per view on the host")
print(json.dumps(out))
