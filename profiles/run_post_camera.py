"""Cost of the fused tail's camera gradients (surfel_post_camera_backward / surfel_post_reg_camera_backward,
DESIGN.md §7q) at 1920x1080, on one GPU.  For surface_outputs (random cotangents on all five outputs) and for
surface_regularizers (lambda_normal 0.05, lambda_dist 1000), CUDA events time:
  * the backward with and without camera gradients (the forward runs outside the timed window);
  * the camera pass alone (kernel and finish), repeated on the state one backward left, with its achieved bytes/s
    from the planes it must read (computed from shapes);
  * the reference's float32 torch tail backward with camera gradients, which is what a pose-refining caller ran
    before the fused tail had them.
Variants alternate round by round; each time is the median over rounds of the mean over --iters calls.  Prints one
JSON line with the card's name and power limit.  Usage: python profiles/run_post_camera.py [--iters 50 --rounds 5]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch

import tail_loss_scenes as TS
from diff_surfel_rasterization import _cabi
from diff_surfel_rasterization.postprocess import _view_matrices, surface_outputs, surface_regularizers
from test_postprocess_gpu import reference_tail

W, H = 1920, 1080
LN, LD = 0.05, 1000.0
# float32 planes of H x W the camera pass reads (stencil neighbours come from cache): surface_outputs: the normal
# (allmap 2-4), g_rend_normal, tmp6 and surf_depth; the regularisers: allmap 0-5 (depth, alpha, normal, median) and tmp6
PASS_PLANES = {"outputs": 3 + 3 + 6 + 1, "regularizers": 6 + 6}


def timed(fn, iters):
    """Mean ms per call of fn() over iters calls, CUDA events around the whole window."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def backward_ms(make_loss, iters):
    """Mean ms of loss.backward() over iters fresh graphs; the forwards run outside the events."""
    total = 0.0
    for _ in range(iters):
        loss = make_loss()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss.backward()
        b.record()
        b.synchronize()
        total += a.elapsed_time(b)
    return total / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "run_post_camera.py measures on a GPU"
    res = {"gpu": torch.cuda.get_device_name(0), "size": [W, H]}
    try:
        res["power_limit, clocks.max.sm"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        res["power_limit, clocks.max.sm"] = f"unavailable: {ex}"
    lib = _cabi.load()
    s = TS.frame(W, H)
    allmap = torch.from_numpy(s["allmap"]).cuda()
    cot = {k: torch.from_numpy(v).cuda() for k, v in TS.cotangents(H, W, "random").items()}
    view0, proj0 = torch.from_numpy(s["view"]).cuda(), torch.from_numpy(s["proj"]).cuda()

    def cam(camera_grad):
        return types.SimpleNamespace(world_view_transform=view0.clone().requires_grad_(camera_grad),
                                     full_proj_transform=proj0.clone().requires_grad_(camera_grad),
                                     image_width=W, image_height=H)

    def outputs_loss(out):
        return sum((out[k] * cot[k]).sum() for k in cot)

    def reg_loss(out):
        return LN * (1 - (out["rend_normal"] * out["surf_normal"]).sum(dim=0)).mean() + LD * out["rend_dist"].mean()

    a_leaf = lambda: allmap.clone().requires_grad_(True)
    variants = {
        "outputs backward, no camera": lambda: outputs_loss(surface_outputs(a_leaf(), cam(False), 0.3)),
        "outputs backward, camera": lambda: outputs_loss(surface_outputs(a_leaf(), cam(True), 0.3)),
        "torch tail backward, camera (outputs)": lambda: outputs_loss(reference_tail(a_leaf(), cam(True), 0.3)),
        "regularizers backward, no camera": lambda: sum(surface_regularizers(a_leaf(), cam(False), 0.3, LN, LD)),
        "regularizers backward, camera": lambda: sum(surface_regularizers(a_leaf(), cam(True), 0.3, LN, LD)),
        "torch tail backward, camera (regularizers)": lambda: reg_loss(reference_tail(a_leaf(), cam(True), 0.3)),
    }

    # the state one backward leaves, for the pass alone
    rot, rays = _view_matrices(view0, proj0, W, H)
    st = torch.cuda.current_stream().cuda_stream
    sd, rn, sn = (torch.empty(c, H, W, device="cuda") for c in (1, 3, 3))
    tmp, g_allmap = torch.empty(6, H, W, device="cuda"), torch.empty(7, H, W, device="cuda")
    partials = torch.empty(lib.surfel_post_camera_partials_bytes(W, H) // 8, dtype=torch.float64, device="cuda")
    out = torch.empty(21, device="cuda")
    _cabi.check(lib.surfel_post_forward(W, H, 0.3, allmap.data_ptr(), rot.data_ptr(), rays.data_ptr(), rn.data_ptr(),
                                        sd.data_ptr(), sn.data_ptr(), st))
    gp = [cot[k].data_ptr() for k in ("rend_normal", "surf_depth", "surf_normal")]
    _cabi.check(lib.surfel_post_backward(W, H, 0.3, allmap.data_ptr(), rot.data_ptr(), rays.data_ptr(), sd.data_ptr(),
                                         *gp, tmp.data_ptr(), g_allmap.data_ptr(), st))
    gscale = torch.tensor([LN / (W * H), LD / (W * H)], device="cuda")
    tmp_r = torch.empty(6, H, W, device="cuda")
    _cabi.check(lib.surfel_post_reg_backward(W, H, 0.3, LN, LD, allmap.data_ptr(), rot.data_ptr(), rays.data_ptr(),
                                             gscale.data_ptr(), tmp_r.data_ptr(), g_allmap.data_ptr(), st))
    passes = {
        "outputs camera pass": lambda: _cabi.check(lib.surfel_post_camera_backward(
            W, H, 0.3, allmap.data_ptr(), rot.data_ptr(), rays.data_ptr(), sd.data_ptr(), *gp, tmp.data_ptr(),
            partials.data_ptr(), out[:9].data_ptr(), out[9:].data_ptr(), st)),
        "regularizers camera pass": lambda: _cabi.check(lib.surfel_post_reg_camera_backward(
            W, H, 0.3, LN, LD, allmap.data_ptr(), rot.data_ptr(), rays.data_ptr(), gscale.data_ptr(),
            tmp_r.data_ptr(), partials.data_ptr(), out[:9].data_ptr(), out[9:].data_ptr(), st)),
    }

    for fn in variants.values():                          # warm-up: module loads, allocator, cuBLAS handles
        backward_ms(fn, 3)
    for fn in passes.values():
        timed(fn, 10)
    times = {k: [] for k in list(variants) + list(passes)}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            times[k].append(backward_ms(fn, args.iters))
        for k, fn in passes.items():
            times[k].append(timed(fn, args.iters * 4))
    res["ms"] = {k: round(statistics.median(v), 4) for k, v in times.items()}
    res["ms_spread"] = {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()}
    for kind in ("outputs", "regularizers"):
        gb = PASS_PLANES[kind] * 4 * W * H / 1e9
        res[f"{kind} camera pass GB (computed)"] = round(gb, 4)
        res[f"{kind} camera pass TB/s"] = round(gb / res["ms"][f"{kind} camera pass"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
