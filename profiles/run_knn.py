"""simple_knn.distCUDA2 (csrc/knn.cu) at model-initialisation sizes: the reference's random init (100 k uniform),
COLMAP-like clouds (clusters of widely varying density + 1 % far outliers) at 300 k and 1 M, 1 M points with heavy
duplication, 1 M and 10 M uniform.  Each GPU time is the median over 20 calls (CUDA events around each call, after
5 warm-ups); next to it the host's scipy cKDTree(...).query(k=4, workers=-1) (build + query, one run).  The first
100 k result is also compared bit for bit with the certified restatement.  Prints one JSON line."""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np
import torch
from scipy.spatial import cKDTree

import knn_oracle as KO
import knn_scenes as KS
from simple_knn._C import distCUDA2

assert torch.cuda.is_available(), "run_knn.py needs a GPU"
dev = torch.device("cuda")
out = {"gpu": torch.cuda.get_device_name(dev), "host_cores": os.cpu_count()}
try:
    out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:   # noqa: BLE001
    out["power_limit"] = f"unknown ({type(e).__name__})"


def gpu_ms(x, reps=20, warmup=5):
    for _ in range(warmup):
        distCUDA2(x)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        distCUDA2(x)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def host_ms(pts):
    t0 = time.perf_counter()
    cKDTree(pts).query(pts, k=4, workers=-1)
    return (time.perf_counter() - t0) * 1e3


clouds = [("uniform_100k", lambda: KS.uniform(100_000, 1)),
          ("colmap_like_300k", lambda: KS.colmap_like(300_000, 2)),
          ("uniform_1M", lambda: KS.uniform(1_000_000, 3)),
          ("colmap_like_1M", lambda: KS.colmap_like(1_000_000, 4)),
          ("duplicated_1M", lambda: KS.duplicated(1_000_000, 5)),
          ("uniform_10M", lambda: KS.uniform(10_000_000, 6))]
for name, make in clouds:
    pts = make()
    x = torch.from_numpy(pts).to(dev)
    out[f"{name}_gpu_ms"] = round(gpu_ms(x), 3)
    out[f"{name}_ckdtree_ms"] = round(host_ms(pts), 1)
    if name == "uniform_100k":
        want = KO.mean_sq_dist(pts)
        out["uniform_100k_bit_exact"] = bool(np.array_equal(distCUDA2(x).cpu().numpy().view(np.uint32), want.view(np.uint32)))
    del x
    torch.cuda.empty_cache()
print(json.dumps(out))
