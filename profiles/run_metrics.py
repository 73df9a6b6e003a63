"""Per-view cost of the novel-view metrics (diff_surfel_rasterization.metrics, DESIGN.md §7o) at the two Mip-NeRF 360
sizes (1237x822 outdoor images_4, 1558x1039 indoor images_2), with seeded weights standing in for the real ones.

Reports, in one run on one GPU:
  * the per-view time of psnr + ssim + LPIPS on the device, and of LPIPS alone;
  * each conv layer's kernel time (CUDA events around repeated launches on the same input) and its achieved
    TFLOP/s from the algorithmic FLOPs 2 H_l W_l 9 Cin Cout per image (two images per view), against the H100 SXM
    data-sheet figure of 495 dense TF32 TFLOP/s;
  * the per-view time of a cached torchvision-layout module (the same convolutions through cuDNN at torch's
    default TF32, built once), alternated with the device path;
  * the card's name and power limit, read in this run.
The reference's own loop rebuilds the network and reloads its weights for every image; that cost needs the real
weight files and is not measured here.

Usage:  python profiles/run_metrics.py [--reps 10]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), os.path.join(ROOT, "tests")]

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import metrics_ref as R  # noqa: E402
from diff_surfel_rasterization import metrics as M  # noqa: E402

SIZES = ((822, 1237), (1039, 1558))
TF32_PEAK = 495.0


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        pl = "unknown"
    return name, pl


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps


class CudnnLPIPS:
    """The restatement as a cached module: float32 weights on the device once, cuDNN at torch's defaults."""

    def __init__(self, vgg, lin):
        self.layers = R.conv_layers(vgg, torch.float32, "cuda")
        self.lin = {k: v.cuda() for k, v in lin.items()}

    def __call__(self, x, y):
        with torch.no_grad():
            f = R.trunk(R.zscore(torch.cat([x, y], 0)), self.layers)
            return R.tap_values([t[:1] for t in f], [t[1:] for t in f], self.lin).sum()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_metrics.py needs a GPU")
    name, pl = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {pl}; cudnn.allow_tf32={torch.backends.cudnn.allow_tf32}")
    vgg, lin = R.vgg_weights(), R.lin_weights()
    dev = M.LPIPS(vgg, lin)
    ref = CudnnLPIPS(vgg, lin)
    lib = M._cabi.load()
    for H, W in SIZES:
        g = torch.Generator().manual_seed(H)
        x = (torch.rand((1, 3, H, W), generator=g) * 255).round().div(255).cuda()
        y = (torch.rand((1, 3, H, W), generator=g) * 255).round().div(255).cuda()
        full = lambda: (M.psnr(x, y), M.ssim(x, y), dev(x, y))
        for f in (full, lambda: ref(x, y)):
            f()
        torch.cuda.synchronize()
        t_full, t_dev, t_ref = [], [], []
        for _ in range(5):                               # alternate the two paths
            t_full.append(timed(full, args.reps))
            t_dev.append(timed(lambda: dev(x, y), args.reps))
            t_ref.append(timed(lambda: ref(x, y), args.reps))
        med = lambda v: sorted(v)[len(v) // 2]
        print(f"\n{W}x{H}: per view (median of 5 x {args.reps}): psnr+ssim+LPIPS {med(t_full):.2f} ms, "
              f"LPIPS {med(t_dev):.2f} ms, cached cuDNN TF32 module {med(t_ref):.2f} ms, "
              f"ratio device/cuDNN {med(t_dev) / med(t_ref):.3f}")
        print(f"  {'layer':8s} {'H_l x W_l':>11s} {'cin':>4s} {'cout':>4s} {'ms':>8s} {'TFLOP/s':>8s} {'of 495':>7s}")
        h, w, li = H, W, 0
        for k, n in enumerate(R.BLOCKS):
            for j in range(n):
                cin, cout, packed, bias = dev.layers[li]
                inp = torch.rand((2, h, w, cin), device="cuda")
                out = torch.empty((2, h, w, cout), device="cuda")
                call = lambda: lib.surfel_metrics_conv3x3(2, h, w, cin, cout, inp.data_ptr(), packed.data_ptr(),
                                                          bias.data_ptr(), out.data_ptr(), None)
                call()
                ms = timed(call, args.reps * 2)
                tf = 2 * 2 * h * w * 9 * cin * cout / (ms * 1e-3) / 1e12
                print(f"  conv{k + 1}_{j + 1}  {h:5d}x{w:<5d} {cin:4d} {cout:4d} {ms:8.3f} {tf:8.1f} {tf / TF32_PEAK:7.1%}")
                li += 1
            if k + 1 < len(R.BLOCKS):
                h, w = h // 2, w // 2


if __name__ == "__main__":
    main()
