"""UnboundedTSDF.extract_mesh (csrc/tsdf.cu grid mode + csrc/mcubes.cu) at `--mesh_res` 1024 and 2048, V = 100 and
300 frames of 1920x1080 (eight analytic views of a sphere on a plane, tests/tsdf_scenes.py, cycled), box half-size
R = 1.9.  Per configuration: the wall time of one call ended by torch.cuda.synchronize() (after a warm-up call at
1024), its split into field passes and marching-cubes passes (the library's per-stage CUDA events: tsdf, mcubes_crop,
mcubes_merge and the radix sort's stages), the mesh size and the peak device memory of the call.

Against it, the part of the reference's marching_cubes_with_contraction that runs on the GPU, per crop as
mcube_utils.py:50-69 does it: the points (linspace x3, meshgrid, vstack(...).T, torch.tensor), the field in 256^3
calls (this project's fused field, so only the points and the copy differ from the reference's own loop) and the
device-to-host copy of the crop's values, summed over all crops, with its peak device memory.  skimage's marching
cubes, trimesh's concatenate and merge_vertices and the host side of the vertices' round trip are not measured: they
cannot run where this project runs.  Prints the card, its power limit and one JSON line."""
import json
import os
import subprocess
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ctypes

import numpy as np
import torch

import tsdf_scenes as TS
from diff_surfel_rasterization import _cabi
from diff_surfel_rasterization.tsdf import UnboundedTSDF

assert torch.cuda.is_available(), "run_mcubes.py needs a GPU"
dev = torch.device("cuda")
out = {"gpu": torch.cuda.get_device_name(dev)}
try:
    out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:   # noqa: BLE001
    out["power_limit"] = f"unknown ({type(e).__name__})"

lib = _cabi.load()
STAGES = [lib.surfel_profile_stage_name(i).decode() for i in range(lib.surfel_profile_num_stages())]
FIELD, MC = {"tsdf"}, {"mcubes_crop", "mcubes_merge", "sort_histogram", "sort_onesweep_pass"}


def stage_ms():
    ms = (ctypes.c_double * len(STAGES))()
    cnt = (ctypes.c_int * len(STAGES))()
    lib.surfel_profile_read(ms, cnt)
    return dict(zip(STAGES, ms))


def run_extract(field, res, R):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    lib.surfel_profile_enable(1)
    stage_ms()
    t = time.perf_counter()
    v, f = field.extract_mesh(res, R)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t
    ms = stage_ms()
    lib.surfel_profile_enable(0)
    peak = torch.cuda.max_memory_allocated() - base
    return v, f, {"extract_mesh_s": wall, "field_kernels_s": sum(ms[s] for s in FIELD) / 1e3,
                  "mcubes_kernels_s": sum(ms[s] for s in MC) / 1e3, "peak_MiB": peak / 2 ** 20,
                  "verts": int(v.shape[0]), "faces": int(f.shape[0])}


def reference_gpu_part(field, res, R):
    """mcube_utils.py:37-69 up to the host copy, every crop; the field is this project's."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    n, cropN = res // 512, 512
    xs = np.linspace(-R, R, n + 1)
    t = time.perf_counter()
    for i in range(n):
        for j in range(n):
            for k in range(n):
                x = torch.linspace(xs[i], xs[i + 1], cropN).cuda()
                y = torch.linspace(xs[j], xs[j + 1], cropN).cuda()
                z = torch.linspace(xs[k], xs[k + 1], cropN).cuda()
                xx, yy, zz = torch.meshgrid(x, y, z, indexing="ij")
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    points = torch.tensor(torch.vstack([xx.ravel(), yy.ravel(), zz.ravel()]).T,
                                          dtype=torch.float).cuda()
                points = points.reshape(cropN, cropN, cropN, 3).reshape(-1, 3)
                zs = torch.cat([field(p) for p in torch.split(points.contiguous(), 256 ** 3, dim=0)])
                zh = zs.detach().cpu().numpy()
                del points, zs, xx, yy, zz, zh
    torch.cuda.synchronize()
    return {"reference_gpu_part_s": time.perf_counter() - t,
            "reference_peak_MiB": (torch.cuda.max_memory_allocated() - base) / 2 ** 20}


views = TS.analytic_views([(1920, 1080)] * 8, 21, dist=3.0)
center, radius, R = torch.zeros(3, device=dev), 3.0, 1.9
rows = []
for V in (100, 300):
    vs = [views[k % len(views)] for k in range(V)]
    cams = [v for v, _, _ in vs]
    for cam in cams:
        cam.full_proj_transform = cam.full_proj_transform.to(dev)
    for res in (1024, 2048):
        field = UnboundedTSDF([d for _, d, _ in vs], [c for _, _, c in vs], cams, center, radius, radius * 2 / res)
        if not rows:
            run_extract(field, 1024, R)               # warm-up
        v, f, row = run_extract(field, res, R)
        del v, f
        row.update({"V": V, "mesh_res": res, "crops": (res // 512) ** 3})
        row.update(reference_gpu_part(field, res, R))
        row["speedup_vs_reference_gpu_part"] = row["reference_gpu_part_s"] / row["extract_mesh_s"]
        rows.append(row)
        print(json.dumps(row), flush=True)
        del field
        torch.cuda.empty_cache()
out["rows"] = rows
out["not_measured"] = ("skimage.measure.marching_cubes, trimesh concatenate + merge_vertices and the host side of "
                       "the reference's vertex round trip: they cannot run where this project runs")
print(f"{out['gpu']}, power limit {out['power_limit']}")
print(json.dumps(out))
