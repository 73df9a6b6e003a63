"""Opt-in fused post-process of the rasterizer's `allmap` (SURVEY §8(f) row f1).

`surface_outputs(allmap, camera, depth_ratio)` returns what the reference's render() derives with
about ten PyTorch kernels per direction (/root/reference/gaussian_renderer/__init__.py:118-147,
/root/reference/utils/point_utils.py:9-37): rend_alpha, rend_normal (world space), rend_dist,
surf_depth and surf_normal — computed by two CUDA kernels forward and two backward
(csrc/postprocess.cu).  The reference's render() keeps working unchanged on the plain op; a caller
that wants the fused path replaces lines :118-147 of its render() by

    out = surface_outputs(allmap, viewpoint_camera, pipe.depth_ratio)
    rets.update(out)

`surface_regularizers(allmap, camera, depth_ratio, lambda_normal, lambda_dist)` goes from `allmap`
straight to the two regularisers of the reference's train.py (normal consistency and depth distortion),
two kernels each way with no intermediate plane (see its docstring).

Both are differentiable in the camera, as the reference's tail is: when world_view_transform or
full_proj_transform requires grad, the backward adds one more pass (csrc/postprocess.cu, DESIGN.md §7q) that sums
dL/drot and dL/drays over the frame, and torch autograd carries them through _view_matrices to the two matrices.
A caller that refines the pose through the rasterizer (DESIGN.md §7p) can keep the fused tail.  Without camera
gradients the backward runs the same launches as before.
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


def _camera_buffers(lib, W, H, dev):
    """Scratch and outputs of the camera pass: partials, dL/drot (3,3) and dL/drays (12,)."""
    partials = torch.empty(lib.surfel_post_camera_partials_bytes(W, H) // 8, dtype=torch.float64, device=dev)
    return partials, torch.empty((3, 3), device=dev), torch.empty((12,), device=dev)


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
            g_rot, g_rays = None, None
            if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
                partials, g_rot, g_rays = _camera_buffers(lib, W, H, dev)
                _cabi.check(lib.surfel_post_camera_backward(
                    W, H, ctx.depth_ratio, allmap.data_ptr(), rot.data_ptr(), rays.data_ptr(), surf_depth.data_ptr(),
                    p(g_rend_normal), p(g_surf_depth), p(g_surf_normal), tmp.data_ptr(), partials.data_ptr(),
                    g_rot.data_ptr(), g_rays.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        return g_allmap, g_rot, g_rays, None


class _SurfaceRegularizers(torch.autograd.Function):
    @staticmethod
    def forward(ctx, allmap, rot, rays, depth_ratio, lambda_normal, lambda_dist):
        lib = _cabi.load()
        allmap = allmap.contiguous().float()
        _, H, W = allmap.shape
        dev = allmap.device
        partials = torch.empty(lib.surfel_post_reg_partials_bytes(W, H) // 8, dtype=torch.float64, device=dev)
        normal_loss = torch.empty((), device=dev)
        dist_loss = torch.empty((), device=dev)
        with torch.cuda.device(dev):
            _cabi.check(lib.surfel_post_reg_forward(W, H, float(depth_ratio), lambda_normal, lambda_dist,
                                                    allmap.data_ptr(), rot.data_ptr(), rays.data_ptr(),
                                                    partials.data_ptr(), normal_loss.data_ptr(), dist_loss.data_ptr(),
                                                    torch.cuda.current_stream(dev).cuda_stream))
        ctx.save_for_backward(allmap, rot, rays)
        ctx.consts = (float(depth_ratio), lambda_normal, lambda_dist)
        return normal_loss, dist_loss

    @staticmethod
    def backward(ctx, g_normal, g_dist):
        lib = _cabi.load()
        allmap, rot, rays = ctx.saved_tensors
        depth_ratio, lambda_normal, lambda_dist = ctx.consts
        _, H, W = allmap.shape
        dev = allmap.device
        n = float(W * H)
        # the cotangents stay on the device (no sync): dL/d(sum over pixels) of each term
        gscale = torch.stack([g_normal * (lambda_normal / n), g_dist * (lambda_dist / n)]).float().contiguous()
        tmp = torch.empty((6, H, W), device=dev) if lambda_normal != 0.0 else None
        g_allmap = torch.empty((7, H, W), device=dev)
        with torch.cuda.device(dev):
            _cabi.check(lib.surfel_post_reg_backward(W, H, depth_ratio, lambda_normal, lambda_dist, allmap.data_ptr(),
                                                     rot.data_ptr(), rays.data_ptr(), gscale.data_ptr(),
                                                     None if tmp is None else tmp.data_ptr(), g_allmap.data_ptr(),
                                                     torch.cuda.current_stream(dev).cuda_stream))
            g_rot, g_rays = None, None
            if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
                partials, g_rot, g_rays = _camera_buffers(lib, W, H, dev)
                _cabi.check(lib.surfel_post_reg_camera_backward(
                    W, H, depth_ratio, lambda_normal, lambda_dist, allmap.data_ptr(), rot.data_ptr(), rays.data_ptr(),
                    gscale.data_ptr(), None if tmp is None else tmp.data_ptr(), partials.data_ptr(), g_rot.data_ptr(),
                    g_rays.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        return g_allmap, g_rot, g_rays, None, None, None


def _check_inputs(fn, allmap, viewpoint_camera):
    """Raise RuntimeError unless allmap is a (7,H,W) CUDA tensor for the camera's size and both camera matrices
    are (4,4) tensors on its device; returns (W, H)."""
    W, H = int(viewpoint_camera.image_width), int(viewpoint_camera.image_height)
    if not torch.is_tensor(allmap) or not allmap.is_cuda:
        raise RuntimeError(f"{fn}: allmap must be a CUDA tensor (no CPU path)")
    if tuple(allmap.shape) != (7, H, W):
        raise RuntimeError(f"{fn}: allmap must be (7, {H}, {W}) for this camera, got {tuple(allmap.shape)}")
    for name in ("world_view_transform", "full_proj_transform"):
        m = getattr(viewpoint_camera, name)
        if not torch.is_tensor(m) or m.device != allmap.device or tuple(m.shape) != (4, 4):
            raise RuntimeError(f"{fn}: camera {name} must be a (4, 4) tensor on {allmap.device}")
    return W, H


def surface_outputs(allmap, viewpoint_camera, depth_ratio):
    """allmap (7,H,W) from GaussianRasterizer -> dict with the reference's keys."""
    W, H = _check_inputs("surface_outputs", allmap, viewpoint_camera)
    rot, rays = _view_matrices(viewpoint_camera.world_view_transform, viewpoint_camera.full_proj_transform, W, H)
    rend_normal, surf_depth, surf_normal = _SurfaceOutputs.apply(allmap, rot, rays, depth_ratio)
    return {"rend_alpha": allmap[1:2], "rend_normal": rend_normal, "rend_dist": allmap[6:7],
            "surf_depth": surf_depth, "surf_normal": surf_normal}


def surface_regularizers(allmap, viewpoint_camera, depth_ratio, lambda_normal, lambda_dist):
    """allmap (7,H,W) from GaussianRasterizer -> (normal_loss, dist_loss), two 0-d float32 CUDA tensors equal to
    surface_outputs() followed by the reference's train.py regularisers:

        normal_error = (1 - (rend_normal * surf_normal).sum(dim=0))[None]
        normal_loss = lambda_normal * normal_error.mean()
        dist_loss = lambda_dist * rend_dist.mean()

    Gradients flow to allmap and, when they require grad, to the camera's world_view_transform and
    full_proj_transform (only the normal term depends on the camera); surf_normal's alpha is detached, as in the
    reference, and where D/alpha is not finite (a hole) its term contributes 0 to allmap's gradient, where the
    reference's is NaN.  lambda_normal and
    lambda_dist are Python numbers: lambda_normal == 0 skips the normal term (its loss and gradient are exactly
    0), and with both 0 nothing reads allmap.  Inputs are checked as surface_outputs checks them."""
    W, H = _check_inputs("surface_regularizers", allmap, viewpoint_camera)
    rot, rays = _view_matrices(viewpoint_camera.world_view_transform, viewpoint_camera.full_proj_transform, W, H)
    return _SurfaceRegularizers.apply(allmap, rot, rays, float(depth_ratio), float(lambda_normal), float(lambda_dist))
