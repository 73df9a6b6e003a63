"""diff_surfel_rasterization — H100-native drop-in for the reference's rasterizer module.

Same import name and public surface as the (un-vendored) upstream Python package
hbb1/diff-surfel-rasterization that the reference imports at
/root/reference/gaussian_renderer/__init__.py:14 and drives at :37-53 and :97-106:

    GaussianRasterizationSettings   NamedTuple, 12 fields in the reference's order
    GaussianRasterizer(nn.Module)   .forward(means3D, means2D, opacities, shs=None,
                                             colors_precomp=None, scales=None, rotations=None,
                                             cov3D_precomp=None) -> (color, radii, allmap)
                                    .markVisible(positions) -> bool (P,)
    rasterize_gaussians(...)        functional form

Return order and `allmap` channel layout follow SURVEY.md §8(b) / the consumer at
/root/reference/gaussian_renderer/__init__.py:110-135: color (3,H,W), radii (P,) int32,
allmap (7,H,W) = [sum w*depth, alpha, normal xyz (view space), median depth, distortion].
`means2D.grad` receives the densification proxy (SURVEY A.5), as train.py:127-128 expects.

All compute happens in libsurfel_b200.so (hand-written sm_90a CUDA behind the C ABI in
include/surfel_rasterizer.h) on the current PyTorch CUDA stream.  PyTorch is only used for
device memory, streams and autograd plumbing.  There is NO fallback path: a missing library or a
CPU tensor raises.
"""
import ctypes
import os
import threading
import time
from typing import NamedTuple, Optional, Tuple

import torch
import torch.nn as nn

from . import _cabi

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians"]

# Low-pass branch of the render backward.  The published upstream kernel propagates the depth gradient
# there as dL_dTw += (s.x, s.y, 1) * dL_dz ("Propagate the gradients of depth") although its forward
# uses depth = Tw.z in that branch; the reference's training consumes exactly these gradients
# (/root/reference/train.py:90), so that is the DEFAULT.  SURFEL_LOWPASS_EXACT_DERIVATIVE=1 selects
# the exact derivative of the forward, (0, 0, 1) * dL_dz, instead (opt-in; see DESIGN.md).
LOWPASS_DEPTH_QUIRK = not bool(int(os.environ.get("SURFEL_LOWPASS_EXACT_DERIVATIVE", "0")))

# Optional host-side trace (profiles/host_trace.py): when switched on, the autograd node appends
# (tag, perf_counter_ns, thread id) at the points that bound the host's critical sections — between
# "R is known" and "backward is launched", and between "backward is launched" and "next preprocess is
# launched".  Off by default: one `is not None` test per mark.
_TRACE = None


def trace_host(on):
    """Start (True) / stop (False) the host trace; returns the list of marks collected so far."""
    global _TRACE
    old = _TRACE
    _TRACE = [] if on else None
    return old


def _mark(tag):
    if _TRACE is not None:
        _TRACE.append((tag, time.perf_counter_ns(), threading.get_ident()))


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool
    # extensions (keyword-only in practice) for the multi-GPU tile-band partition (SURVEY §8e):
    # tile_rows = [begin, end) tile-row band, None = whole frame; out_buffers = (color, allmap) views to
    # render INTO — shapes (3,H,W) / (7,H,W), rows contiguous, both with the same plane stride (e.g. slices
    # of one frame padded to equal bands, which an in-place all-gather then completes).
    tile_rows: Optional[Tuple[int, int]] = None
    out_buffers: Optional[Tuple[torch.Tensor, torch.Tensor]] = None
    # out_replicas = device addresses (ints) of replicated 10-plane frames laid out like out_buffers (peer
    # mappings of every GPU's frame, or one NVSwitch multicast address): the forward's output stores go to each of
    # them instead of to out_buffers — the tile-band exchange fused into the render kernel (surfel_parallel).
    out_replicas: Optional[Tuple[int, ...]] = None


def _dev_f32(t, name, align=4):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError(f"diff_surfel_rasterization: `{name}` must be a CUDA tensor (no CPU path)")
    if t.dtype != torch.float32:
        t = t.float()
    t = t.contiguous()
    if t.data_ptr() % align:
        t = t.clone()
    return t


def _ptr(t):
    return None if t is None or t.numel() == 0 else t.data_ptr()


def _settings_struct(rs: GaussianRasterizationSettings, keep, out_plane=0, grad_plane=0, out_replicas=None, defer_sh=False):
    """ctypes view of the settings.  Built on every call: the reference's world_view_transform /
    full_proj_transform are transposed views, so contiguous copies are made here and must see the
    caller's current values (a long-lived GaussianRasterizer whose camera tensors are updated in place
    would otherwise render with stale matrices); the four tiny copies cost microseconds."""
    bg = _dev_f32(rs.bg, "bg")
    vm = _dev_f32(rs.viewmatrix, "viewmatrix")
    pm = _dev_f32(rs.projmatrix, "projmatrix")
    cp = _dev_f32(rs.campos, "campos")
    keep.extend([bg, vm, pm, cp])
    rows = rs.tile_rows if len(rs) > 12 and rs.tile_rows is not None else (0, 0)
    reps = tuple(int(a) for a in (out_replicas or ()))
    if len(reps) > 8:
        raise RuntimeError("diff_surfel_rasterization: at most 8 output replicas")
    return _cabi.SurfelSettings(
        int(rs.image_height), int(rs.image_width), float(rs.tanfovx), float(rs.tanfovy),
        float(rs.scale_modifier), int(rs.sh_degree), int(bool(rs.prefiltered)), int(bool(rs.debug)),
        int(rows[0]), int(rows[1]), bg.data_ptr(), vm.data_ptr(), pm.data_ptr(), cp.data_ptr(),
        int(out_plane), int(grad_plane), len(reps), int(bool(defer_sh)), (ctypes.c_uint64 * 8)(*reps))


def _plane_stride(t, C, H, W):
    """Plane stride (in elements) of a (C,H,W) float32 CUDA tensor whose rows are contiguous, or None."""
    if t is None or not t.is_cuda or t.dtype != torch.float32 or tuple(t.shape) != (C, H, W):
        return None
    st = t.stride()
    if st[2] != 1 or st[1] != W or st[0] < H * W or t.data_ptr() % 4:
        return None
    return st[0]


_pinned_counter = {}
_last = {"num_rendered": 0}


def last_num_rendered():
    """Instance count R (splat-tile pairs) of the most recent forward in this process."""
    return _last["num_rendered"]



_capacity = {}               # (device, P, W, H, band) -> instance capacity seen last; bounded (oldest evicted)
_CAPACITY_ENTRIES = 64
# SURFEL_SPECULATIVE=0 restores upstream's launch order (block on R, then launch binning + render)
_SPECULATIVE = bool(int(os.environ.get("SURFEL_SPECULATIVE", "1")))


def _pinned_u32(device):
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    ent = _pinned_counter.get(key)
    if ent is None:
        ent = (torch.zeros(1, dtype=torch.int32).pin_memory(), torch.cuda.Event())
        _pinned_counter[key] = ent
    return ent


def _grad_buffers(lib, dev, P, M, has_sh, has_colors, has_scales, has_cov, defer_sh=False):
    """Every gradient the backward writes, carved out of ONE flat allocation (offsets are multiples of four
    floats, so the 128-bit stores of the kernels stay aligned): a caller that has to reduce the gradients
    across ranks (surfel_parallel) reduces `bucket` in place instead of concatenating eight tensors."""
    # defer_sh (multi-GPU band mode): the bucket carries the 3-float colour gradient instead of the (M,3) SH
    # gradient, which is its rank-1 expansion and is produced AFTER the bucket has been reduced across ranks
    defer_sh = bool(defer_sh and has_sh)
    parts = [("d_means3D", (P, 3), True), ("d_means2D", (P, 3), True), ("d_opacity", (P, 1), True),
             ("d_sh", (P, M, 3), has_sh and not defer_sh), ("d_scales", (P, 2), has_scales), ("d_rot", (P, 4), has_scales),
             ("d_colors", (P, 3), has_colors or defer_sh), ("d_cov", (P, 9), has_cov)]
    off, plan = 0, []
    for name, shape, on in parts:
        n = 1
        for d in shape:
            n *= d
        if on:
            plan.append((name, shape, off, n))
            off += (n + 3) // 4 * 4
    bucket = torch.empty((max(off, 4),), dtype=torch.float32, device=dev)
    out = {name: None for name, _, _ in parts}
    for name, shape, o, n in plan:
        out[name] = bucket[o:o + n].view(shape)
    out["bucket"] = bucket
    if defer_sh:
        out["d_sh"] = torch.empty((P, M, 3), dtype=torch.float32, device=dev)
    out["defer_sh"] = defer_sh
    out["scratch"] = torch.empty((max(P, 1), lib.surfel_grad_scratch_floats()), dtype=torch.float32, device=dev)
    return out


class _RasterizeGaussians(torch.autograd.Function):
    """Autograd node around the C ABI (upstream: _RasterizeGaussians, SURVEY §8a row a3)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                cov3Ds_precomp, raster_settings):
        _mark("fwd_enter")
        lib = _cabi.load()
        rs = raster_settings
        if means3D.dim() != 2 or means3D.shape[1] != 3:
            raise RuntimeError("means3D must have dimensions (num_points, 3)")
        P = means3D.shape[0]
        dev = means3D.device
        H, W = int(rs.image_height), int(rs.image_width)
        keep = []
        outb = rs.out_buffers if len(rs) > 13 else None
        out_plane = 0
        if outb is not None:
            out_plane = _plane_stride(outb[0], 3, H, W)
            if out_plane is None or _plane_stride(outb[1], 7, H, W) != out_plane or outb[0].device != dev:
                raise RuntimeError("out_buffers must be float32 CUDA views of shape (3,H,W) and (7,H,W) with "
                                   "contiguous rows and one common plane stride")
        reps = rs.out_replicas if len(rs) > 14 else None
        if reps and (outb is None or outb[1].data_ptr() != outb[0].data_ptr() + 12 * out_plane):
            raise RuntimeError("out_replicas needs out_buffers that are the color / allmap planes of ONE 10-plane frame")
        cs = _settings_struct(rs, keep, out_plane=out_plane, out_replicas=reps)
        means3D = _dev_f32(means3D, "means3D")
        opacities = _dev_f32(opacities, "opacities")
        sh = _dev_f32(sh, "shs", 16) if sh is not None and sh.numel() else None
        colors_precomp = _dev_f32(colors_precomp, "colors_precomp") if colors_precomp is not None and colors_precomp.numel() else None
        scales = _dev_f32(scales, "scales", 8) if scales is not None and scales.numel() else None
        rotations = _dev_f32(rotations, "rotations", 16) if rotations is not None and rotations.numel() else None
        cov3Ds_precomp = _dev_f32(cov3Ds_precomp, "cov3D_precomp") if cov3Ds_precomp is not None and cov3Ds_precomp.numel() else None
        M = 0 if sh is None else sh.shape[1]

        stream = torch.cuda.current_stream(dev).cuda_stream
        band = cs.tile_row_begin != 0 or cs.tile_row_end != 0
        alloc = torch.zeros if band else torch.empty
        if outb is not None:
            color, allmap = outb            # the caller owns what lies outside the band
        else:
            color = alloc((3, H, W), dtype=torch.float32, device=dev)
            allmap = alloc((7, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        geom = torch.empty((lib.surfel_geom_bytes(P),), dtype=torch.uint8, device=dev)
        img = torch.empty((lib.surfel_image_bytes(W, H),), dtype=torch.uint8, device=dev)
        R = cap = 0
        with torch.cuda.device(dev):
            if P > 0:
                host_R, ev = _pinned_u32(dev)
                _cabi.check(lib.surfel_forward_preprocess(
                    ctypes.byref(cs), P, M, _ptr(means3D), _ptr(opacities), _ptr(scales),
                    _ptr(rotations), _ptr(cov3Ds_precomp), _ptr(sh), _ptr(colors_precomp),
                    radii.data_ptr(), geom.data_ptr(), img.data_ptr(), host_R.data_ptr(), stream))
                ev.record(torch.cuda.current_stream(dev))
                _mark("preprocess_launched")
                # The instance count R sizes the binning workspace, so upstream blocks here until the
                # device has produced it.  We launch binning + render SPECULATIVELY with the capacity
                # remembered from earlier calls of the same shape (every kernel clamps to it), and only
                # then wait for R: the device keeps working while the host waits, and the wait ends as
                # soon as preprocess is done.  A too-small guess costs one re-launch.
                key = (dev.index, P, W, H, cs.tile_row_begin, cs.tile_row_end)
                spec = _SPECULATIVE and lib.surfel_accepts_capacity()
                cap = _capacity.get(key, 0) if spec else 0
                if cap:
                    binning = torch.empty((lib.surfel_binning_bytes(cap, W, H),), dtype=torch.uint8, device=dev)
                    _cabi.check(lib.surfel_forward_render(
                        ctypes.byref(cs), P, cap, radii.data_ptr(), geom.data_ptr(), binning.data_ptr(),
                        img.data_ptr(), 1, color.data_ptr(), allmap.data_ptr(), stream))
                # Everything the backward will need is allocated NOW, while the device is busy and before
                # the host blocks: after the wait, the host's critical path to the backward launch (which
                # must land before the queued forward kernels drain) is as short as possible.
                if any(ctx.needs_input_grad[:8]):
                    ctx.bwd_bufs = _grad_buffers(lib, dev, P, M, sh is not None, colors_precomp is not None,
                                                 scales is not None, cov3Ds_precomp is not None,
                                                 defer_sh=getattr(ctx, "defer_sh", False))
                _mark("speculative_work_launched")
                ev.synchronize()
                _mark("R_known")
                R = int(host_R.item()) & 0xFFFFFFFF
                if R > cap or not cap:
                    cap = R if not spec else int(R * 1.25) + 4096
                    if spec:
                        _capacity.pop(key, None)
                        while len(_capacity) >= _CAPACITY_ENTRIES:
                            _capacity.pop(next(iter(_capacity)))
                        _capacity[key] = cap
                    binning = None
            if P == 0 or binning is None:
                binning = torch.empty((lib.surfel_binning_bytes(cap, W, H),), dtype=torch.uint8, device=dev)
                _cabi.check(lib.surfel_forward_render(
                    ctypes.byref(cs), P, cap, radii.data_ptr(), geom.data_ptr(), binning.data_ptr(),
                    img.data_ptr(), int(P > 0), color.data_ptr(), allmap.data_ptr(), stream))

        _last["num_rendered"] = R
        # NOT the caller's out_buffers: they are this node's outputs, and an output held by its own grad_fn's
        # context is a reference cycle — the frame (and everything else the context holds: workspaces, the
        # gradient bucket) would live until the cyclic garbage collector happens to run (measured: +1.8 GB of
        # reserved device memory and two cudaMalloc calls per config-5 step, profiles/r2_band_probe.md)
        ctx.raster_settings = rs._replace(out_buffers=None, out_replicas=None) if outb is not None else rs
        ctx.num_rendered = cap        # the workspace layout was carved for `cap` instance slots
        ctx.M = M
        ctx.flags = (sh is not None, colors_precomp is not None, scales is not None, cov3Ds_precomp is not None)
        none = torch.empty(0, device=dev)
        ctx.out_plane = out_plane
        ctx.save_for_backward(means3D, none if scales is None else scales,
                              none if rotations is None else rotations,
                              none if cov3Ds_precomp is None else cov3Ds_precomp,
                              none if sh is None else sh, radii, geom, binning, img)
        ctx.mark_non_differentiable(radii)
        _mark("fwd_exit")
        return color, radii, allmap

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_allmap):
        grads, _ = _backward(ctx, grad_color, grad_allmap, camera=False)
        return grads + (None,)


def _backward(ctx, grad_color, grad_allmap, camera, camera_sums=False):
    """The backward of both autograd nodes: the eight splat gradients in the order of the node's splat inputs, and,
    when `camera` is set, (dL_dviewmatrix (16), dL_dprojmatrix (16), dL_dcampos (3)) from surfel_camera_backward.
    camera_sums (tile-row bands, surfel_parallel): the camera gradient is instead the (35,) float64 tensor of
    surfel_camera_backward_sums, the band's sums before rounding, in the same order."""
    _mark("bwd_enter")
    lib = _cabi.load()
    rs = ctx.raster_settings
    means3D, scales, rotations, cov3Ds, sh, radii, geom, binning, img = ctx.saved_tensors
    has_sh, has_colors, has_scales, has_cov = ctx.flags
    P, M, R = means3D.shape[0], ctx.M, ctx.num_rendered
    dev = means3D.device
    H, W = int(rs.image_height), int(rs.image_width)
    keep = []
    if grad_color is None:
        grad_color = torch.zeros((3, H, W), device=dev)
    if grad_allmap is None:
        grad_allmap = torch.zeros((7, H, W), device=dev)
    # cotangents are read in place when they are plane-strided views with contiguous rows (e.g. slices of a
    # padded frame); anything else is made contiguous first
    gp = _plane_stride(grad_color, 3, H, W)
    if gp is None or _plane_stride(grad_allmap, 7, H, W) != gp:
        gp = 0
        g_color, g_all = _dev_f32(grad_color, "grad_color"), _dev_f32(grad_allmap, "grad_allmap")
    else:
        g_color, g_all = grad_color, grad_allmap
    b = getattr(ctx, "bwd_bufs", None)
    if b is None:      # P == 0, or backward called twice (retain_graph): allocate here
        b = _grad_buffers(lib, dev, P, M, has_sh, has_colors, has_scales, has_cov, defer_sh=getattr(ctx, "defer_sh", False))
    ctx.bwd_bufs = None
    ctx.grad_bucket = b["bucket"]
    defer = b["defer_sh"]
    cs = _settings_struct(rs, keep, out_plane=getattr(ctx, "out_plane", 0), grad_plane=gp, defer_sh=defer)
    # deferred SH gradient: the caller (surfel_parallel._BandFrame) reduces the bucket and then calls expand()
    ctx.sh_expand = None
    if defer:
        d_col_t, d_sh_t, campos_t = b["d_colors"], b["d_sh"], keep[3]

        def expand():
            with torch.cuda.device(dev):
                _cabi.check(lib.surfel_sh_grad_expand(P, M, int(rs.sh_degree), means3D.data_ptr(), campos_t.data_ptr(),
                                                      d_col_t.data_ptr(), d_sh_t.data_ptr(),
                                                      torch.cuda.current_stream(dev).cuda_stream))
        ctx.sh_expand = expand
    d_means2D, d_opacity, d_means3D = b["d_means2D"], b["d_opacity"], b["d_means3D"]
    d_colors, d_cov, d_sh, d_scales, d_rot, scratch = b["d_colors"], b["d_cov"], b["d_sh"], b["d_scales"], b["d_rot"], b["scratch"]
    stream = torch.cuda.current_stream(dev).cuda_stream
    # the camera gradient needs the full dL_dT that preprocess backward forms anyway: on the scales+rotations path it
    # is requested into a buffer of its own (with transMat_precomp it is d_cov, and the camera step does not read it)
    d_tmat = d_cov
    if camera and d_tmat is None and has_scales:
        d_tmat = torch.empty((P, 9), dtype=torch.float32, device=dev)
    cam = None
    with torch.cuda.device(dev):
        _cabi.check(lib.surfel_backward(
            ctypes.byref(cs), P, M, R, _ptr(means3D), _ptr(scales), _ptr(rotations), _ptr(cov3Ds),
            _ptr(sh), int(has_colors), radii.data_ptr(), geom.data_ptr(), binning.data_ptr(),
            img.data_ptr(), g_color.data_ptr(), g_all.data_ptr(), scratch.data_ptr(),
            d_means2D.data_ptr(), _ptr(d_colors), d_opacity.data_ptr(), d_means3D.data_ptr(),
            _ptr(d_tmat), _ptr(d_sh), _ptr(d_scales), _ptr(d_rot), int(LOWPASS_DEPTH_QUIRK), stream))
        if camera:
            partials = torch.empty((lib.surfel_camera_partials_bytes(P) // 8,), dtype=torch.float64, device=dev)
            out = torch.empty((35,), dtype=torch.float64 if camera_sums else torch.float32, device=dev)
            entry = lib.surfel_camera_backward_sums if camera_sums else lib.surfel_camera_backward
            _cabi.check(entry(
                ctypes.byref(cs), P, M, _ptr(means3D), _ptr(scales), _ptr(rotations), _ptr(cov3Ds), _ptr(sh),
                int(has_colors), radii.data_ptr(), geom.data_ptr(), scratch.data_ptr(), _ptr(d_tmat),
                partials.data_ptr(), out[0:16].data_ptr(), out[16:32].data_ptr(), out[32:35].data_ptr(), stream))
            cam = out if camera_sums else (out[0:16], out[16:32], out[32:35])
    _mark("bwd_launched")
    # (means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
    return (d_means3D, d_means2D, d_sh, (d_colors if has_colors else None), d_opacity, d_scales, d_rot, d_cov), cam


class _RasterizeGaussiansCamera(torch.autograd.Function):
    """The same op with the camera as three more differentiable inputs: viewmatrix (4,4), projmatrix (4,4) and campos
    (3), in the row-vector layout of GaussianRasterizationSettings.  rasterize_gaussians routes here only when one of
    them requires grad; the splat gradients are those of _RasterizeGaussians, the camera gradients come from
    surfel_camera_backward (DESIGN.md §7p).  The whole frame only: a tile-row band gives per-rank partial sums, which
    surfel_parallel.rasterize_tile_band adds across the ranks (DESIGN.md §7r)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                viewmatrix, projmatrix, campos, raster_settings):
        rs = raster_settings
        if any(getattr(rs, k, None) is not None for k in ("tile_rows", "out_buffers", "out_replicas")):
            raise RuntimeError("diff_surfel_rasterization: camera gradients are not available with tile_rows, "
                               "out_buffers or out_replicas (a tile-row band holds only part of the frame); "
                               "surfel_parallel.rasterize_tile_band sums the bands' camera gradients")
        ctx.cam_meta = tuple((t.shape, t.dtype) for t in (viewmatrix, projmatrix, campos))
        rs = rs._replace(viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos)
        return _RasterizeGaussians.forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                           cov3Ds_precomp, rs)

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_allmap):
        grads, cam = _backward(ctx, grad_color, grad_allmap, camera=True)
        cam = tuple(g.reshape(shape).to(dtype) for g, (shape, dtype) in zip(cam, ctx.cam_meta))
        return grads + cam + (None,)


def _wants_camera_grad(rs):
    return torch.is_grad_enabled() and any(
        torch.is_tensor(t) and t.requires_grad for t in (rs.viewmatrix, rs.projmatrix, rs.campos))




def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                        cov3Ds_precomp, raster_settings):
    """The op.  When grad mode is on and raster_settings.viewmatrix, projmatrix or campos requires grad, the
    rasterizer also differentiates in the camera (_RasterizeGaussiansCamera); otherwise the camera is a constant, as
    upstream treats it."""
    if _wants_camera_grad(raster_settings):
        rs = raster_settings
        return _RasterizeGaussiansCamera.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                               cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.campos, rs)
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales,
                                     rotations, cov3Ds_precomp, raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """Near-plane visibility of (P,3) positions -> bool (P,) (upstream mark_visible)."""
        lib = _cabi.load()
        rs = self.raster_settings
        with torch.no_grad():
            pos = _dev_f32(positions, "positions")
            vm = _dev_f32(rs.viewmatrix, "viewmatrix")
            pm = _dev_f32(rs.projmatrix, "projmatrix")
            out = torch.empty((pos.shape[0],), dtype=torch.uint8, device=pos.device)
            with torch.cuda.device(pos.device):
                _cabi.check(lib.surfel_mark_visible(pos.shape[0], _ptr(pos), vm.data_ptr(), pm.data_ptr(),
                                                    _ptr(out), torch.cuda.current_stream(pos.device).cuda_stream))
        return out.bool()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                rotations=None, cov3D_precomp=None):
        rs = self.raster_settings
        if (shs is None) == (colors_precomp is None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        geometric = scales is not None or rotations is not None
        if ((scales is None or rotations is None) and cov3D_precomp is None) or (geometric and cov3D_precomp is not None):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        empty = torch.Tensor([])
        shs = empty if shs is None else shs
        colors_precomp = empty if colors_precomp is None else colors_precomp
        scales = empty if scales is None else scales
        rotations = empty if rotations is None else rotations
        cov3D_precomp = empty if cov3D_precomp is None else cov3D_precomp
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales,
                                   rotations, cov3D_precomp, rs)
