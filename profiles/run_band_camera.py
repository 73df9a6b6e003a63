"""Cost of the tile-band camera gradients (surfel_camera_backward_sums, DESIGN.md §7r).

On one GPU (default):
  * the new entry point on one band of config 5 (2 M splats, 7680x4320, SH degree 3; the first band of an N-band
    equal partition), against surfel_camera_backward on the whole 1080p headline frame (1 M splats): CUDA events
    around repeated calls on the state the band's / frame's last backward left;
  * the band backward through rasterize_tile_band (rank 0 of N, no process group) with and without camera
    gradients, as medians of alternating rounds.
Under torchrun with N > 1 processes (one per GPU), additionally the band backward with and without camera gradients
inside the NCCL group, and the extra 35 x float64 (280-byte) all-reduce alone.  The card's name and power limit are
read in the same run.

Usage:  python profiles/run_band_camera.py [--bands 2] [--reps 20] [--rounds 5]
        torchrun --nproc_per_node N profiles/run_band_camera.py
"""
import argparse
import ctypes
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), os.path.join(ROOT, "profiles")]

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import surfel_parallel as SP  # noqa: E402
import surfel_scenes as S  # noqa: E402
from diff_surfel_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _cabi  # noqa: E402
from run_camera_grad import card  # noqa: E402


def event_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def state(workload, dev, rank, world, band):
    """Settings, leaves and cotangents of a workload; camera tensors are separate leaves per call."""
    P, W, H = S.CONFIGS[workload]
    scene, cam = S.named(workload)
    gc, go = (x.to(dev) for x in S.make_cotangents(W, H, 0))
    leaf = {k: v.to(dev).requires_grad_(True) for k, v in scene.items()}

    def settings(camera_grad):
        t = lambda k: cam[k].to(dev).requires_grad_(camera_grad)
        return GaussianRasterizationSettings(H, W, cam["tanfovx"], cam["tanfovy"], torch.zeros(3, device=dev), 1.0,
                                             t("viewmatrix"), t("projmatrix"), 3, t("campos"), False, False)

    def forward(camera_grad):
        m2d = torch.zeros(P, 3, device=dev, requires_grad=True)
        args = dict(means3D=leaf["means3D"], means2D=m2d, shs=leaf["shs"], opacities=leaf["opacities"],
                    scales=leaf["scales"], rotations=leaf["rotations"])
        rs = settings(camera_grad)
        if band:
            res = SP.rasterize_tile_band(GaussianRasterizer, rs, rank, world, **args)
            res["wait"]()
            s, e = SP.band_pixel_rows(H, res["band"])
            return ((res["render"][:, s:e] * gc[:, s:e]).sum() + (res["allmap"][:, s:e] * go[:, s:e]).sum())
        color, _, allmap = GaussianRasterizer(rs)(**args)
        return (color * gc).sum() + (allmap * go).sum()
    return forward


def backward_ms(forward, camera_grad, reps):
    """Median backward time of `reps` forward + backward steps (events around the backward only)."""
    out = []
    for _ in range(reps):
        loss = forward(camera_grad)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss.backward()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def camera_entry_ms(workload, dev, tile_rows, sums, reps):
    """CUDA-event time of one camera entry-point call on the state of a whole-frame / band backward (stage driver)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from cuda_stages import CudaPipeline
    scene, cam = S.named(workload)
    scene, cam = S.to_numpy(scene), S.to_numpy(cam)
    pipe = CudaPipeline(scene, cam, [0.0, 0.0, 0.0], 3, 1.0, tile_rows=tile_rows)
    pipe.preprocess(); pipe.bucket(); pipe.render()
    gc, go = S.make_cotangents(cam["W"], cam["H"], 0)
    got = pipe.backward(gc.numpy(), go.numpy())
    scratch = torch.tensor(got["grad_rec"], device=dev)
    dtm = torch.tensor(got["dL_dtransMat"], device=dev)
    lib = pipe.lib
    partials = torch.empty((lib.surfel_camera_partials_bytes(pipe.P) // 8,), dtype=torch.float64, device=dev)
    out = torch.empty((35,), dtype=torch.float64 if sums else torch.float32, device=dev)
    entry = lib.surfel_camera_backward_sums if sums else lib.surfel_camera_backward
    _p = lambda t: None if t is None else t.data_ptr()
    stream = torch.cuda.current_stream().cuda_stream

    def call():
        _cabi.check(entry(ctypes.byref(pipe.cs), pipe.P, pipe.M, _p(pipe.means3D), _p(pipe.scales), _p(pipe.rotations),
                          None, _p(pipe.shs), 0, pipe.radii.data_ptr(), pipe.geom.data_ptr(), scratch.data_ptr(),
                          dtm.data_ptr(), partials.data_ptr(), out[0:16].data_ptr(), out[16:32].data_ptr(),
                          out[32:35].data_ptr(), stream), lib)
    visible = int((pipe.radii > 0).sum())
    return event_ms(call, reps), visible


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bands", type=int, default=2, help="N of the equal-band partition on one GPU")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("run_band_camera.py needs a GPU")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        local = int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", torch.cuda.current_device())
    name, pl = card()
    if rank == 0:
        print(f"card: {name}; power.limit, clocks.max.sm: {pl}")

    if world == 1:
        H5 = S.CONFIGS["config5"][2]
        band = SP.equal_band(H5, 0, args.bands)
        t_band, v_band = camera_entry_ms("config5", dev, band, True, args.reps)
        t_head, v_head = camera_entry_ms("headline", dev, (0, 0), False, args.reps)
        print(f"surfel_camera_backward_sums, config5 band {band} of {args.bands} ({v_band} visible splats of 2 M): "
              f"{t_band:.3f} ms")
        print(f"surfel_camera_backward, headline 1080p whole frame ({v_head} visible of 1 M): {t_head:.3f} ms")
        n = args.bands
    else:
        n = world
    fwd = state("config5", dev, rank, n, band=True)
    with_cam, without = [], []
    for _ in range(args.rounds):
        without.append(backward_ms(fwd, False, args.reps // 4 or 1))
        with_cam.append(backward_ms(fwd, True, args.reps // 4 or 1))
    if rank == 0:
        print(f"config5 band backward, rank 0 of {n}{' (NCCL group)' if world > 1 else ' (no process group)'}: "
              f"{statistics.median(without):.3f} ms without camera gradients, "
              f"{statistics.median(with_cam):.3f} ms with them (medians of {args.rounds} rounds)")
    if world > 1:
        sums = torch.zeros(35, dtype=torch.float64, device=dev)
        t = event_ms(lambda: dist.all_reduce(sums), args.reps * 5)
        if rank == 0:
            print(f"35 x float64 all-reduce over {world} GPUs: {t * 1000:.1f} us")
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
