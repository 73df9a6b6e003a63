"""diff_surfel_rasterization.densify.densify_and_prune (csrc/densify.cu) against the torch restatement of the same
rules (tests/densify_ref.py, eager torch on the same GPU) at 1 M and 3 M rows, with 5 % of the rows cloned, 5 % split
and 3 % below min_opacity (max_screen_size = 20).  Each time is the median over 20 calls, each on a fresh copy of the
model and ended by torch.cuda.synchronize() (host clock), after 3 warm-up calls.  Also: the peak of
torch.cuda.max_memory_allocated over what was allocated before the call, both outputs compared (bit for bit except
split rows' xyz), the plan + apply kernels alone (the library's per-launch CUDA events), and the HBM floor: the
state read once and written once, 58 floats x 3 (param, exp_avg, exp_avg_sq) x 4 B x (P + P') over 3.35 TB/s.
Prints the card, its power limit and one JSON line."""
import json
import os
import statistics
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch
from torch import nn

import densify_ref as DR
from diff_surfel_rasterization.densify import densify_and_prune

assert torch.cuda.is_available(), "run_densify.py needs a GPU"
dev = torch.device("cuda")
out = {"gpu": torch.cuda.get_device_name(dev)}
try:
    out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:   # noqa: BLE001
    out["power_limit"] = f"unknown ({type(e).__name__})"
ARGS = (0.0002, 0.005, 4.0, 20)


def copy_model(src):
    m = types.SimpleNamespace(percent_dense=src.percent_dense)
    groups = []
    for g in src.optimizer.param_groups:
        p = nn.Parameter(g["params"][0].detach().clone().requires_grad_(True))
        setattr(m, DR.ATTR[g["name"]], p)
        groups.append({"params": [p], "lr": g["lr"], "name": g["name"]})
    m.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    for g, gs in zip(m.optimizer.param_groups, src.optimizer.param_groups):
        st = src.optimizer.state[gs["params"][0]]
        m.optimizer.state[g["params"][0]] = {k: v.clone() for k, v in st.items()}
    m.xyz_gradient_accum, m.denom, m.max_radii2D = (src.xyz_gradient_accum.clone(), src.denom.clone(),
                                                    src.max_radii2D.clone())
    return m


def timed(fn, src, reps=20, warmup=3):
    ts = []
    for i in range(warmup + reps):
        m = copy_model(src)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(m, *ARGS)
        torch.cuda.synchronize()
        if i >= warmup:
            ts.append((time.perf_counter() - t0) * 1e3)
        del m
    return statistics.median(ts)


def peak(fn, src):
    m = copy_model(src)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    fn(m, *ARGS)
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20, m


def kernel_ms(src, reps=20):
    """Median over `reps` calls of the plan and apply kernels alone (the library's CUDA events around each launch)."""
    import ctypes
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    n = lib.surfel_profile_num_stages()
    stage = [lib.surfel_profile_stage_name(i).decode() for i in range(n)].index("densify")
    ms, cnt = (ctypes.c_double * n)(), (ctypes.c_int * n)()
    ts = []
    for _ in range(reps):
        m = copy_model(src)
        torch.cuda.synchronize()
        lib.surfel_profile_read(ms, cnt)
        lib.surfel_profile_enable(1)
        densify_and_prune(m, *ARGS)
        lib.surfel_profile_enable(0)
        _cabi.check(lib.surfel_profile_read(ms, cnt))
        assert cnt[stage] == 3                    # plan, apply f_rest, apply the rest
        ts.append(ms[stage])
        del m
    return statistics.median(ts)


for P in (1_000_000, 3_000_000):
    src = DR.build(DR.scene_arrays(P, 21, split_frac=0.05, clone_frac=0.05), dev)
    row = {}
    row["fused_ms"] = round(timed(densify_and_prune, src), 3)
    row["restatement_ms"] = round(timed(DR.densify_and_prune, src), 3)
    torch.manual_seed(1)
    row["fused_peak_mib"], a = peak(densify_and_prune, src)
    torch.manual_seed(1)
    row["restatement_peak_mib"], b = peak(DR.densify_and_prune, src)
    P_new = a._xyz.shape[0]
    row["P_new"] = P_new
    row["floor_ms"] = round(58 * 3 * 4 * (P + P_new) / 3.35e12 * 1e3, 3)
    same = all(torch.equal(x.view(torch.int32), y.view(torch.int32))
               for n in DR.GROUPS if n != "xyz"
               for x, y in [(getattr(a, DR.ATTR[n]).detach(), getattr(b, DR.ATTR[n]).detach())])
    row["outputs_equal_except_split_xyz"] = bool(same)
    row["kernels_ms"] = round(kernel_ms(src), 3)
    row["kernels_hbm_tbs"] = round(58 * 3 * 4 * (P + P_new) / (row["kernels_ms"] * 1e-3) / 1e12, 2)
    out[f"{P // 1_000_000}M"] = row
    del src, a, b
    torch.cuda.empty_cache()
print(json.dumps(out))
