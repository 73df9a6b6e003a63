"""diff_surfel_rasterization.tsdf.UnboundedTSDF (csrc/tsdf.cu) against the reference's loop restated in eager torch
(tests/tsdf_ref.py:eager, on the same GPU), for the field of `render.py --unbounded`: V = 100 and 300 frames at
1920x1080, eager with the maps on the host (copied to the device every frame, as the reference keeps them) and
resident on the device, on one call of 256^3 points (the reference's chunk, mcube_utils.py:60); the fused field also
on one 512^3 block (eight such calls).  Each time is the median of repeated calls ended by torch.cuda.synchronize()
(host clock) after a warm-up call.  The depth maps are eight analytic 1080p views of a sphere on a plane
(tests/tsdf_scenes.py) cycled over the frames; the points are the 256^3 grid of [-1.9, 1.9]^3 in contracted space.
Reports (sample, frame) pairs/s and the projected `--mesh_res 1024` field time (64 calls), checks that fused and
eager agree on the unobserved samples, and prints the card, its power limit and one JSON line."""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch

import tsdf_ref as TR
import tsdf_scenes as TS
from diff_surfel_rasterization.tsdf import UnboundedTSDF

assert torch.cuda.is_available(), "run_tsdf.py needs a GPU"
dev = torch.device("cuda")
out = {"gpu": torch.cuda.get_device_name(dev)}
try:
    out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:   # noqa: BLE001
    out["power_limit"] = f"unknown ({type(e).__name__})"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts)


views = TS.analytic_views([(1920, 1080)] * 8, 21, dist=3.0)
center, radius, voxel = torch.zeros(3, device=dev), 3.0, 3.0 * 2 / 1024
g = torch.linspace(-1.9, 1.9, 256, device=dev)
pts = torch.stack(torch.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).contiguous()
N = pts.shape[0]
rows = []
for V in (100, 300):
    vs = [views[k % len(views)] for k in range(V)]
    cams = [v for v, _, _ in vs]
    host_d, host_c = [d for _, d, _ in vs], [c for _, _, c in vs]
    for cam in cams:
        cam.full_proj_transform = cam.full_proj_transform.to(dev)
    t0 = time.perf_counter()
    field = UnboundedTSDF(host_d, host_c, cams, center, radius, voxel)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    fused = timed(lambda: field(pts), 5)
    ref = field(pts)
    row = {"V": V, "N": N, "fused_256^3_s": fused, "fused_pairs_per_s": N * V / fused, "construct_s": build_s,
           "fused_mesh_res_1024_projected_s": 64 * fused}
    if V == 300:
        blk = torch.stack(torch.meshgrid(*(torch.linspace(-1.9, 0.0, 512, device=dev),) * 3, indexing="ij"),
                          -1).reshape(-1, 3)
        row["fused_512^3_block_s"] = timed(lambda: [field(c) for c in torch.split(blk, 256 ** 3)], 3)
        del blk
    dev_d = [d.to(dev) for d in host_d[:len(views)]] * (V // len(views) + 1)
    dev_c = [c.to(dev) for c in host_c[:len(views)]] * (V // len(views) + 1)
    for where, (dm, cm) in (("host", (host_d, host_c)), ("device", (dev_d[:V], dev_c[:V]))):
        e = timed(lambda: TR.eager(pts, dm, cm, cams, center, radius, voxel), 2)
        row[f"eager_{where}_256^3_s"] = e
        row[f"eager_{where}_pairs_per_s"] = N * V / e
        row[f"eager_{where}_mesh_res_1024_projected_s"] = 64 * e
        row[f"speedup_vs_eager_{where}"] = e / fused
    te = TR.eager(pts, dev_d[:V], dev_c[:V], cams, center, radius, voxel)
    row["unobserved_agree"] = bool(torch.equal(te == -1, ref == -1))
    row["max_abs_diff_vs_eager"] = float((te - ref).abs().max())
    rows.append(row)
    print(json.dumps(row), flush=True)
    del field, dev_d, dev_c
    torch.cuda.empty_cache()
out["rows"] = rows
out["not_measured"] = "eager on the 512^3 block (eight 256^3 calls); the whole --mesh_res 1024 run (projected as 64 calls)"
print(f"{out['gpu']}, power limit {out['power_limit']}")
print(json.dumps(out))
