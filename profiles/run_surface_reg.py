"""Times train.py's two regularisers (normal consistency and depth distortion), forward + backward from allmap, on
one GPU three ways: the eager reference tail + train.py's lines, surface_outputs + the lines, and the fused
surface_regularizers.  At 1920x1080 and at BASELINE config 3's 1600x1200, for (lambda_normal, lambda_dist) =
(0.05, 1000) and (0, 1000).  Prints one JSON line with the times, the bytes each path must move and the card's name
and power limit.  Usage: python profiles/run_surface_reg.py [--iters 50]"""
import argparse
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch

import tail_loss_scenes as TS
from diff_surfel_rasterization.postprocess import surface_outputs, surface_regularizers
from test_postprocess_gpu import reference_tail

SIZES = ((1920, 1080), (1600, 1200))
LAMBDAS = ((0.05, 1000.0), (0.0, 1000.0))


def lines(out, ln, ld):
    """train.py's regularisers on the render() tail's outputs."""
    normal_error = (1 - (out["rend_normal"] * out["surf_normal"]).sum(dim=0))[None]
    return ln * normal_error.mean(), ld * out["rend_dist"].mean()


def fused_planes(ln):
    """float32 planes of H x W the fused kernels read or write (neighbours of the stencil come from cache):
    forward 7 reads (1: rend_dist alone without the normal term); backward with the normal term: kernel 1 reads
    D, alpha, the median and the normal (6) and writes the 6 point-gradient planes and channels 2-4 (9), kernel 2
    reads those 6 planes and D, alpha, the median (9) and writes channels 0, 1, 5, 6 (4); without it, 7 writes."""
    return 7 + 6 + 9 + 9 + 4 if ln else 1 + 7


def outputs_planes():
    """surface_outputs + train.py's lines, each materialised plane counted once per read and write:
    forward: depth/normal kernel 6 reads + 4 writes, surf_normal kernel 2 + 3, rn * sn 6 + 3, sum 3 + 1, 1 - x 1 + 1,
    the two means 1 + 1 (32); backward: the neg of 1 - x 1 + 1, mul's two products 8 reads + 6 writes, the zero
    surf_depth cotangent 1, the allmap[6:7] slice gradient 1 read + 7 writes, the normal vjp 5 + 6, the allmap
    kernel 12 + 7, the two allmap gradients accumulated 14 + 7 (76).  The lambda_normal == 0 graph is the same."""
    return 32 + 76


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "run_surface_reg.py measures on a GPU"
    dev = "cuda"
    res = {"what": "train.py regularisers from allmap, forward + backward, CUDA events over --iters calls after a "
                   "warm-up; bytes are the float32 planes each path must move, computed from shapes (not measured; the "
                   "eager reference's ~20 kernels each way are not modelled: null)",
           "gpu": torch.cuda.get_device_name(0)}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        res["power_limit"] = f"unread: {ex}"
    runs = []
    for W, H in SIZES:
        scene = TS.frame(W, H)
        view = types.SimpleNamespace(world_view_transform=torch.from_numpy(scene["view"]).to(dev),
                                     full_proj_transform=torch.from_numpy(scene["proj"]).to(dev), image_width=W, image_height=H)
        allmap = torch.from_numpy(scene["allmap"]).to(dev).requires_grad_(True)
        plane = 4 * W * H
        for ln, ld in LAMBDAS:
            paths = {"eager_reference": lambda a: lines(reference_tail(a, view, 0.0), ln, ld),
                     "surface_outputs": lambda a: lines(surface_outputs(a, view, 0.0), ln, ld),
                     "fused": lambda a: surface_regularizers(a, view, 0.0, ln, ld)}
            row = {"W": W, "H": H, "lambda_normal": ln, "lambda_dist": ld,
                   "bytes": {"eager_reference": None, "surface_outputs": outputs_planes() * plane, "fused": fused_planes(ln) * plane}}
            for name, fn in paths.items():
                def step():
                    allmap.grad = None
                    n, d = fn(allmap)
                    (n + d).backward()
                for _ in range(5):
                    step()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    step()
                e1.record()
                torch.cuda.synchronize()
                row[name + "_ms"] = e0.elapsed_time(e1) / args.iters
            row["speedup_vs_eager"] = row["eager_reference_ms"] / row["fused_ms"]
            row["speedup_vs_surface_outputs"] = row["surface_outputs_ms"] / row["fused_ms"]
            row["fused_GBps"] = row["bytes"]["fused"] / (row["fused_ms"] * 1e-3) / 1e9
            runs.append(row)
    res["runs"] = runs
    print(json.dumps(res))


if __name__ == "__main__":
    main()
