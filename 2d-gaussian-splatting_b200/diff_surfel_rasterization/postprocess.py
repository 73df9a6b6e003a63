"""Opt-in fused post-process of the rasterizer's `allmap` (SURVEY §8(f) row f1).

`surface_outputs(allmap, camera, depth_ratio)` returns what the reference's render() derives with
about ten PyTorch kernels per direction (/root/reference/gaussian_renderer/__init__.py:118-147,
/root/reference/utils/point_utils.py:9-37): rend_alpha, rend_normal (world space), rend_dist,
surf_depth and surf_normal — computed by two CUDA kernels forward and two backward
(csrc/postprocess.cu).  The reference's render() keeps working unchanged on the plain op; a caller
that wants the fused path replaces lines :118-147 of its render() by

    out = surface_outputs(allmap, viewpoint_camera, pipe.depth_ratio)
    rets.update(out)
"""
import torch

from . import _cabi


def _view_matrices(world_view_transform, full_proj_transform, W, H):
    """rot (3,3): n_world = n_view @ rot;  rays (12,): pixel -> world ray matrix and camera centre.
    Same algebra as depths_to_points (reference utils/point_utils.py:9-24), done once per view."""
    wvt = world_view_transform.float()
    c2w = wvt.T.inverse()
    ndc2pix = torch.tensor([[W / 2, 0, 0, W / 2], [0, H / 2, 0, H / 2], [0, 0, 0, 1]],
                           dtype=torch.float32, device=wvt.device).T
    projection_matrix = c2w.T @ full_proj_transform.float()
    intrins = (projection_matrix @ ndc2pix)[:3, :3].T
    M = intrins.inverse().T @ c2w[:3, :3].T
    rays = torch.cat([M.reshape(-1), c2w[:3, 3]]).contiguous()
    rot = wvt[:3, :3].T.contiguous()
    return rot, rays


class _SurfaceOutputs(torch.autograd.Function):
    @staticmethod
    def forward(ctx, allmap, rot, rays, depth_ratio):
        lib = _cabi.load()
        if not allmap.is_cuda:
            raise RuntimeError("surface_outputs: allmap must be a CUDA tensor (no CPU path)")
        allmap = allmap.contiguous().float()
        _, H, W = allmap.shape
        dev = allmap.device
        rend_normal = torch.empty((3, H, W), device=dev)
        surf_depth = torch.empty((1, H, W), device=dev)
        surf_normal = torch.empty((3, H, W), device=dev)
        with torch.cuda.device(dev):
            _cabi.check(lib.surfel_post_forward(W, H, float(depth_ratio), allmap.data_ptr(), rot.data_ptr(),
                                                rays.data_ptr(), rend_normal.data_ptr(), surf_depth.data_ptr(),
                                                surf_normal.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        ctx.save_for_backward(allmap, rot, rays, surf_depth)
        ctx.depth_ratio = float(depth_ratio)
        return rend_normal, surf_depth, surf_normal

    @staticmethod
    def backward(ctx, g_rend_normal, g_surf_depth, g_surf_normal):
        lib = _cabi.load()
        allmap, rot, rays, surf_depth = ctx.saved_tensors
        _, H, W = allmap.shape
        dev = allmap.device
        c = lambda g: None if g is None else g.contiguous().float()
        g_rend_normal, g_surf_depth, g_surf_normal = c(g_rend_normal), c(g_surf_depth), c(g_surf_normal)
        p = lambda g: None if g is None else g.data_ptr()
        tmp = torch.empty((6, H, W), device=dev)
        g_allmap = torch.empty((7, H, W), device=dev)
        with torch.cuda.device(dev):
            _cabi.check(lib.surfel_post_backward(W, H, ctx.depth_ratio, allmap.data_ptr(), rot.data_ptr(), rays.data_ptr(),
                                                 surf_depth.data_ptr(), p(g_rend_normal), p(g_surf_depth), p(g_surf_normal),
                                                 tmp.data_ptr(), g_allmap.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        return g_allmap, None, None, None


def surface_outputs(allmap, viewpoint_camera, depth_ratio):
    """allmap (7,H,W) from GaussianRasterizer -> dict with the reference's keys."""
    W, H = int(viewpoint_camera.image_width), int(viewpoint_camera.image_height)
    if not torch.is_tensor(allmap) or not allmap.is_cuda:
        raise RuntimeError("surface_outputs: allmap must be a CUDA tensor (no CPU path)")
    if tuple(allmap.shape) != (7, H, W):
        raise RuntimeError(f"surface_outputs: allmap must be (7, {H}, {W}) for this camera, got {tuple(allmap.shape)}")
    for name in ("world_view_transform", "full_proj_transform"):
        m = getattr(viewpoint_camera, name)
        if not torch.is_tensor(m) or m.device != allmap.device or tuple(m.shape) != (4, 4):
            raise RuntimeError(f"surface_outputs: camera {name} must be a (4, 4) tensor on {allmap.device}")
    rot, rays = _view_matrices(viewpoint_camera.world_view_transform, viewpoint_camera.full_proj_transform, W, H)
    rend_normal, surf_depth, surf_normal = _SurfaceOutputs.apply(allmap, rot, rays, depth_ratio)
    return {"rend_alpha": allmap[1:2], "rend_normal": rend_normal, "rend_dist": allmap[6:7],
            "surf_depth": surf_depth, "surf_normal": surf_normal}
