"""Camera gradients of the tile-band frame over 2 GPUs with NCCL (DESIGN.md §7r); skipped below 2 devices.

For every gather mode (sync, async, fused, and fused_multicast where the group has a multicast address) and every
grad_reduce ("all_reduce", "defer", "none"): the camera gradients are bit-identical on both ranks, they match the
single-GPU rasterizer's within test_band_camera_gpu's bar, and under "none" the two ranks' partials add up to it.
rasterize_tile_band -> postprocess.surface_regularizers on the gathered frame gives the single-GPU camera gradient
of rasterizer -> fused regularisers (the tail's part is whole-frame on every rank and is not reduced).  The pose loop
of tests/camera_pose.py on a tile-band frame ends in the same error band as on one GPU.
"""
import os
import socket
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
KEYS = ("viewmatrix", "projmatrix", "campos")
CAST = 2.0 ** -24
W, H, P = 640, 360, 20000


def _paths():
    for p in (ROOT, os.path.join(ROOT, "2d-gaussian-splatting_b200"), HERE):
        if p not in sys.path:
            sys.path.insert(0, p)


def _settings(cam, dev):
    from diff_surfel_rasterization import GaussianRasterizationSettings
    t = lambda k: cam[k].to(dev).clone().requires_grad_(True)
    return GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=dev),
        scale_modifier=1.0, viewmatrix=t("viewmatrix"), projmatrix=t("projmatrix"), sh_degree=3, campos=t("campos"),
        prefiltered=False, debug=False)


def _step(rs, leaf, rank, world, gc, go, band=True, tail=False, **kw):
    """One forward + backward; returns the camera gradients (numpy float32)."""
    import surfel_parallel as SP
    from diff_surfel_rasterization import GaussianRasterizer
    m2d = torch.zeros(P, 3, device=leaf["means3D"].device, requires_grad=True)
    args = dict(means3D=leaf["means3D"], means2D=m2d, shs=leaf["shs"], opacities=leaf["opacities"], scales=leaf["scales"],
                rotations=leaf["rotations"])
    if band:
        res = SP.rasterize_tile_band(GaussianRasterizer, rs, rank, world, **kw, **args)
        res["wait"]()
        color, allmap = res["render"], res["allmap"]
    else:
        color, _, allmap = GaussianRasterizer(rs)(**args)
    if tail:
        from diff_surfel_rasterization import postprocess as PP
        normal_loss, dist_loss = PP.surface_regularizers(allmap, _viewpoint(rs), 1.0, 0.05, 100.0)
        loss = (color * gc).sum() + normal_loss + dist_loss
    else:
        loss = (color * gc).sum() + (allmap * go).sum()
    for k in KEYS:
        getattr(rs, k).grad = None
    loss.backward()
    if kw.get("grad_reduce") == "defer":
        SP.last_sh_expand()()
    torch.cuda.synchronize()
    return {k: getattr(rs, k).grad.detach().cpu().numpy().reshape(-1).copy() for k in KEYS}


def _viewpoint(rs):
    from types import SimpleNamespace
    return SimpleNamespace(image_width=W, image_height=H, world_view_transform=rs.viewmatrix,
                           full_proj_transform=rs.projmatrix)


def _worker(rank, world, port, out):
    import torch.distributed as dist
    _paths()
    import surfel_scenes as S
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        cam = S.make_camera(W, H, R=S.look_at_rotation(12, -7), t=[0.15, -0.1, 0.4])
        scene = S.make_scene(P, W, H, 41)
        m = torch.cat([scene["means3D"], torch.ones(P, 1)], 1) @ cam["viewmatrix"].inverse()
        scene["means3D"] = m[:, :3].contiguous()
        gc, go = (x.to(dev) for x in S.make_cotangents(W, H, 41))
        leaf = {k: v.to(dev).requires_grad_(True) for k, v in scene.items()}
        rs = _settings(cam, dev)
        res = {"single": [_step(rs, leaf, rank, world, gc, go, band=False) for _ in range(2)],
               "single_tail": [_step(rs, leaf, rank, world, gc, go, band=False, tail=True) for _ in range(2)]}
        from surfel_parallel import symmetric_frame
        modes = ["sync", "async", "fused"]
        _, reps, _ = symmetric_frame(H, W, world, dev, multicast=True)
        if len(reps) == 1:
            modes.append("fused_multicast")
        for g in modes:
            for red in ("all_reduce", "defer", "none"):
                res[(g, red)] = _step(rs, leaf, rank, world, gc, go, gather=g, grad_reduce=red)
        res["band_tail"] = _step(rs, leaf, rank, world, gc, go, tail=True)
        import camera_pose as CP
        res["pose"] = CP.refine(_band_renderer(rank, world), P=CP.P_GPU, W=CP.W_GPU, H=CP.H_GPU, steps=CP.STEPS,
                                device=str(dev), dtype=torch.float32)
        torch.save(res, f"{out}.r{rank}")
    finally:
        import surfel_parallel as SP
        SP.release_symmetric_frames()
        dist.destroy_process_group()


def _band_renderer(rank, world):
    import math
    import camera_pose as CP
    import surfel_parallel as SP
    from diff_surfel_rasterization import GaussianRasterizationSettings, GaussianRasterizer

    def render(scene, vm, pm, cp, Wp, Hp):
        tanfovy = math.tan(math.radians(CP.FOVY) / 2)
        rs = GaussianRasterizationSettings(Hp, Wp, tanfovy * Wp / Hp, tanfovy, torch.zeros(3, device=vm.device), 1.0, vm,
                                           pm, 1, cp, False, False)
        m2d = torch.zeros(scene["means3D"].shape[0], 3, device=vm.device)
        res = SP.rasterize_tile_band(GaussianRasterizer, rs, rank, world, means3D=scene["means3D"], means2D=m2d,
                                     opacities=scene["opacities"], shs=scene["shs"], scales=scene["scales"],
                                     rotations=scene["rotations"])
        return res["render"]
    return render


def test_band_camera_two_gpus(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    _paths()
    import camera_pose as CP
    from test_camera_grad_gpu import device_renderer
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = str(tmp_path / "cam")
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    r = [torch.load(f"{out}.r{k}", weights_only=False) for k in range(2)]
    single, single2 = r[0]["single"]
    for key in ("sync", "async", "fused", "fused_multicast"):
        for red in ("all_reduce", "defer", "none"):
            if (key, red) not in r[0]:
                continue
            a, b = r[0][(key, red)], r[1][(key, red)]
            for k in KEYS:
                ref = single[k].astype(np.float64)
                scale = np.abs(ref).max()
                bar = max(2.0 * np.abs(single2[k] - ref).max(), 4e-6 * scale) + 2 * CAST * scale
                if red == "none":
                    got = a[k].astype(np.float64) + b[k]
                else:
                    assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), (key, red, k)
                    got = a[k].astype(np.float64)
                assert np.abs(got - ref).max() <= bar, (key, red, k, np.abs(got - ref).max(), bar)
    # the fused regularisers on the gathered frame: their camera term is whole-frame on each rank, not reduced
    t1, t2 = r[0]["single_tail"]
    for k in KEYS:
        ref = t1[k].astype(np.float64)
        scale = np.abs(ref).max()
        bar = max(2.0 * np.abs(t2[k] - ref).max(), 1.3e-5 * scale) + 2 * CAST * scale
        for rank in range(2):
            assert np.abs(r[rank]["band_tail"][k] - ref).max() <= bar, (rank, k)
    one = CP.refine(device_renderer(), P=CP.P_GPU, W=CP.W_GPU, H=CP.H_GPU, steps=CP.STEPS, device="cuda",
                    dtype=torch.float32)
    for rank in range(2):
        pose = r[rank]["pose"]
        assert pose["rot_err"][-1] < 0.25 * pose["rot_err"][0] and pose["trans_err"][-1] < 0.25 * pose["trans_err"][0]
        assert pose["rot_err"][-1] <= 2.0 * one["rot_err"][-1] + 1e-4 * one["rot_err"][0]
