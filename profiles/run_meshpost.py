"""meshpost.post_process_mesh (csrc/meshpost.cu) on the meshes `render.py --unbounded` exports: the output of
UnboundedTSDF.extract_mesh at `--mesh_res` 1024 and 2048 of the analytic views profiles/run_mcubes.py uses (V = 100
frames of 1920x1080, box half-size R = 1.9), with their colours, and one synthetic strip of 10 M faces in reversed
order, the union-find's worst case (each face's union meets the chain built so far at its far end).

Per mesh, with cluster_to_keep = 1000 as render.py defaults to: the wall time of one call ended by
torch.cuda.synchronize() (after a warm-up call on the same mesh), its split by the library's per-stage CUDA events
(meshpost_edges, the radix sort's stages for both sorts, meshpost_union, meshpost_label, meshpost_compact), the peak
device memory of the call above its inputs, and F, C (clusters), F' and M'.  For scale it also times the vectorised
NumPy/SciPy restatement (tests/meshpost_ref.py, (b)) on this machine's host; that is not Open3D, whose
cluster_connected_triangles is not measured.  Prints the card, its power limit and one JSON line."""
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

import meshpost_ref as MP
import tsdf_scenes as TS
from diff_surfel_rasterization import _cabi
from diff_surfel_rasterization.meshpost import post_process_mesh
from diff_surfel_rasterization.tsdf import UnboundedTSDF

assert torch.cuda.is_available(), "run_meshpost.py needs a GPU"
dev = torch.device("cuda")
out = {"gpu": torch.cuda.get_device_name(dev)}
try:
    out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:   # noqa: BLE001
    out["power_limit"] = f"unknown ({type(e).__name__})"

lib = _cabi.load()
STAGES = [lib.surfel_profile_stage_name(i).decode() for i in range(lib.surfel_profile_num_stages())]
SPLIT = ["meshpost_edges", "sort_histogram", "sort_onesweep_pass", "meshpost_union", "meshpost_label",
         "meshpost_compact"]
K = 1000


def stage_ms():
    ms = (ctypes.c_double * len(STAGES))()
    cnt = (ctypes.c_int * len(STAGES))()
    lib.surfel_profile_read(ms, cnt)
    return dict(zip(STAGES, ms))


def n_clusters(verts, faces):
    F, M = faces.shape[0], verts.shape[0]
    wb = lib.surfel_meshpost_workspace_bytes(M, F)
    ws = torch.empty(wb, dtype=torch.uint8, device=dev)
    ids = torch.empty(F, dtype=torch.int32, device=dev)
    counts = torch.empty(F, dtype=torch.int32, device=dev)
    info = torch.empty(2, dtype=torch.int64, device=dev)
    _cabi.check(lib.surfel_meshpost_clusters(M, F, faces.data_ptr(), ws.data_ptr(), wb, ids.data_ptr(),
                                             counts.data_ptr(), info.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return int(info[0].item())


def measure(name, verts, faces, colors):
    k = min(K, n_clusters(verts, faces))
    post_process_mesh(verts, faces, colors, cluster_to_keep=k)          # warm-up
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    lib.surfel_profile_enable(1)
    stage_ms()
    t = time.perf_counter()
    v, f, c = post_process_mesh(verts, faces, colors, cluster_to_keep=k)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t
    ms = stage_ms()
    lib.surfel_profile_enable(0)
    peak = torch.cuda.max_memory_allocated() - base
    row = {"mesh": name, "F": int(faces.shape[0]), "M": int(verts.shape[0]), "C": n_clusters(verts, faces),
           "cluster_to_keep": k, "F_out": int(f.shape[0]), "M_out": int(v.shape[0]), "call_ms": wall * 1e3,
           "stages_ms": {s: round(ms[s], 3) for s in SPLIT}, "peak_MiB": peak / 2 ** 20}
    vh, fh = verts.cpu().numpy(), faces.cpu().numpy()
    ch = None if colors is None else colors.cpu().numpy()
    t = time.perf_counter()
    want = MP.post_process_vectorised(vh, fh, ch, k)
    row["numpy_scipy_restatement_host_s"] = time.perf_counter() - t
    row["equals_restatement"] = bool(np.array_equal(want[2], f.cpu().numpy())
                                     and np.array_equal(want[1].view(np.uint32), v.cpu().numpy().view(np.uint32)))
    print(json.dumps(row), flush=True)
    return row


rows = []
views = TS.analytic_views([(1920, 1080)] * 8, 21, dist=3.0)
vs = [views[k % len(views)] for k in range(100)]
cams = [v for v, _, _ in vs]
for cam in cams:
    cam.full_proj_transform = cam.full_proj_transform.to(dev)
center, radius, R = torch.zeros(3, device=dev), 3.0, 1.9
for res in (1024, 2048):
    field = UnboundedTSDF([d for _, d, _ in vs], [c for _, _, c in vs], cams, center, radius, radius * 2 / res)
    verts, faces = field.extract_mesh(res, R)
    rgbs = field.colors(verts)
    del field
    rows.append(measure(f"extract_mesh {res}", verts, faces, rgbs))
    del verts, faces, rgbs
    torch.cuda.empty_cache()
n = 10_000_000
faces = torch.from_numpy(MP.strip(n)[::-1].copy()).to(dev)
verts = torch.randn(n + 2, 3, device=dev)
rows.append(measure("strip 10M reversed", verts, faces, None))
out["rows"] = rows
out["not_measured"] = "Open3D's cluster_connected_triangles and mesh filtering on the host: Open3D is not available"
print(f"{out['gpu']}, power limit {out['power_limit']}")
print(json.dumps(out))
