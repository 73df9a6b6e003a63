"""Cost of the rasterizer's camera gradients (surfel_camera_backward, DESIGN.md §7p) on the headline workload:
1 M splats at 1920x1080, SH degree 3.

Reports, in one run on one GPU:
  * the backward of the public op (autograd backward of sum(color * gc) + sum(allmap * go), after one forward) with
    and without camera gradients, as medians of alternating rounds of --reps calls each;
  * the camera kernel and its finish alone: CUDA events around repeated surfel_camera_backward calls on the state
    the last backward left, and the two stages' event times from the library's profiler;
  * the bytes the camera kernel reads per splat (from the layouts: visible splats only), over its time;
  * the card's name and power limit, read in this run.

Usage:  python profiles/run_camera_grad.py [--reps 10] [--rounds 5]
"""
import argparse
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200")]

import torch  # noqa: E402

import surfel_scenes as S  # noqa: E402
import diff_surfel_rasterization as dsr  # noqa: E402
from diff_surfel_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _cabi  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        pl = "unknown"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workload", default="headline")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_camera_grad.py needs a GPU")
    name, pl = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {pl}")
    dev = torch.device("cuda")
    P, W, H = S.CONFIGS[args.workload]
    scene, cam = S.named(args.workload)
    gc, go = (x.to(dev) for x in S.make_cotangents(W, H, 0))
    leaf = {k: v.to(dev).requires_grad_(True) for k, v in scene.items()}
    m2d = torch.zeros(P, 3, device=dev, requires_grad=True)
    lib = _cabi.load()

    def settings(camera_grad):
        t = lambda k: cam[k].to(dev).requires_grad_(camera_grad)
        return GaussianRasterizationSettings(H, W, cam["tanfovx"], cam["tanfovy"], torch.zeros(3, device=dev), 1.0,
                                             t("viewmatrix"), t("projmatrix"), 3, t("campos"), False, False)

    def backward_ms(camera_grad, reps):
        """Mean of reps backward calls, each after its own untimed forward."""
        rs = settings(camera_grad)
        total = 0.0
        for _ in range(reps):
            color, radii, allmap = GaussianRasterizer(rs)(means3D=leaf["means3D"], means2D=m2d, shs=leaf["shs"],
                                                          opacities=leaf["opacities"], scales=leaf["scales"],
                                                          rotations=leaf["rotations"])
            loss = (color * gc).sum() + (allmap * go).sum()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            loss.backward()
            e.record()
            e.synchronize()
            total += s.elapsed_time(e)
            for v in list(leaf.values()) + [m2d, rs.viewmatrix, rs.projmatrix, rs.campos]:
                v.grad = None
        return total / reps, int((radii > 0).sum())

    for cg in (False, True):
        backward_ms(cg, 2)
    plain, withcam = [], []
    for _ in range(args.rounds):
        plain.append(backward_ms(False, args.reps)[0])
        ms, visible = backward_ms(True, args.reps)
        withcam.append(ms)
    med = lambda v: sorted(v)[len(v) // 2]
    print(f"{args.workload}: P={P} {W}x{H}, visible {visible}")
    print(f"backward (median of {args.rounds} alternating rounds x {args.reps}): without camera gradients "
          f"{med(plain):.3f} ms, with {med(withcam):.3f} ms, difference {med(withcam) - med(plain):.3f} ms")
    print(f"  rounds without: {[round(x, 3) for x in plain]}")
    print(f"  rounds with:    {[round(x, 3) for x in withcam]}")

    # the camera step alone, on the state of one backward through the C ABI
    rs = settings(True)
    keep = []
    cs = dsr._settings_struct(rs, keep)
    sh = leaf["shs"].detach().contiguous()
    means, scales, rots = (leaf[k].detach().contiguous() for k in ("means3D", "scales", "rotations"))
    radii = torch.empty(P, dtype=torch.int32, device=dev)
    geom = torch.empty(lib.surfel_geom_bytes(P), dtype=torch.uint8, device=dev)
    img = torch.empty(lib.surfel_image_bytes(W, H), dtype=torch.uint8, device=dev)
    host_R = torch.zeros(1, dtype=torch.int32).pin_memory()
    st = torch.cuda.current_stream().cuda_stream
    opa = leaf["opacities"].detach().contiguous()
    _cabi.check(lib.surfel_forward_preprocess(ctypes.byref(cs), P, 16, means.data_ptr(), opa.data_ptr(), scales.data_ptr(),
                                              rots.data_ptr(), None, sh.data_ptr(), None, radii.data_ptr(), geom.data_ptr(),
                                              img.data_ptr(), host_R.data_ptr(), st))
    torch.cuda.synchronize()
    R = int(host_R.item())
    binning = torch.empty(lib.surfel_binning_bytes(R, W, H), dtype=torch.uint8, device=dev)
    color = torch.empty(3, H, W, device=dev)
    allmap = torch.empty(7, H, W, device=dev)
    _cabi.check(lib.surfel_forward_render(ctypes.byref(cs), P, R, radii.data_ptr(), geom.data_ptr(), binning.data_ptr(),
                                          img.data_ptr(), 1, color.data_ptr(), allmap.data_ptr(), st))
    e = lambda *s: torch.empty(*s, device=dev)
    scratch, dtm = e(P, lib.surfel_grad_scratch_floats()), e(P, 9)
    outs = [e(P, 3), e(P, 3), e(P, 1), e(P, 3), e(P, 16, 3), e(P, 2), e(P, 4)]
    _cabi.check(lib.surfel_backward(ctypes.byref(cs), P, 16, R, means.data_ptr(), scales.data_ptr(), rots.data_ptr(), None,
                                    sh.data_ptr(), 0, radii.data_ptr(), geom.data_ptr(), binning.data_ptr(), img.data_ptr(),
                                    gc.data_ptr(), go.data_ptr(), scratch.data_ptr(), outs[0].data_ptr(), None,
                                    outs[2].data_ptr(), outs[3].data_ptr(), dtm.data_ptr(), outs[4].data_ptr(),
                                    outs[5].data_ptr(), outs[6].data_ptr(), 1, st))
    partials = torch.empty(lib.surfel_camera_partials_bytes(P) // 8, dtype=torch.float64, device=dev)
    cam_out = e(35)

    def call():
        _cabi.check(lib.surfel_camera_backward(ctypes.byref(cs), P, 16, means.data_ptr(), scales.data_ptr(), rots.data_ptr(),
                                               None, sh.data_ptr(), 0, radii.data_ptr(), geom.data_ptr(), scratch.data_ptr(),
                                               dtm.data_ptr(), partials.data_ptr(), cam_out[0:16].data_ptr(),
                                               cam_out[16:32].data_ptr(), cam_out[32:35].data_ptr(), st))
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    n = args.reps * 20
    times = []
    for _ in range(args.rounds):
        s, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n):
            call()
        en.record()
        en.synchronize()
        times.append(s.elapsed_time(en) / n)
    lib.surfel_profile_enable(1)
    nst = lib.surfel_profile_num_stages()
    ms_arr, cnt_arr = (ctypes.c_double * nst)(), (ctypes.c_int * nst)()
    lib.surfel_profile_read(ms_arr, cnt_arr)
    for _ in range(n):
        call()
    torch.cuda.synchronize()
    lib.surfel_profile_read(ms_arr, cnt_arr)
    lib.surfel_profile_enable(0)
    stages = {lib.surfel_profile_stage_name(i).decode(): ms_arr[i] / cnt_arr[i] for i in range(nst) if cnt_arr[i]}
    vis = int((radii > 0).sum())
    # bytes per visible splat: radii 4, means 12, rotation 16, scale 8, dL_dT 36, record (gn, gc) 24, normal 16,
    # clamp bits 1, SH row 192; culled splats read their radius only
    nbytes = vis * (4 + 12 + 16 + 8 + 36 + 24 + 16 + 1 + 192) + (P - vis) * 4
    t = med(times)
    print(f"camera step alone (median of {args.rounds} x {n} calls): {t:.4f} ms; per stage with events around each "
          f"launch: " + ", ".join(f"{k} {v:.4f} ms" for k, v in stages.items() if k.startswith("camera")))
    print(f"  reads {nbytes / 1e6:.1f} MB ({nbytes / max(vis, 1):.0f} B per visible splat): {nbytes / (t * 1e-3) / 1e12:.2f} TB/s "
          f"against the 3.35 TB/s HBM3 data-sheet figure")
    print("  dL_dviewmatrix", [round(x, 4) for x in cam_out[0:16].tolist()])


if __name__ == "__main__":
    main()
