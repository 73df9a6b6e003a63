"""Multi-GPU sharding of the rasterizer hot path (SURVEY.md §8(e)).  One process per GPU.

The reference has no multi-device code at all (SURVEY §2.3); the two modes below are the ones
BASELINE.json's configs 4 and 5 name.

1. View-parallel (config 4, and bench.py --gpus N): independent camera views are dealt out one per
   rank; every rank holds the full splat set and runs the whole pipeline for its own views.  There
   is NO collective on the data path.  `allreduce_gradients` is only needed when the ranks train one
   shared model.

2. Tile-band partition of ONE oversized frame (config 5): rank r owns a band of tile rows (equal bands of
   ceil(gy/n) rows for the copy-free path `rasterize_tile_band`; the floor(gy*r/n) split of SURVEY §8e
   for the helper functions below, which the CPU tests exercise).  Every rank preprocesses all splats
   but clips each splat's tile rect to its band (C ABI: surfel_settings.tile_row_begin/end), so only its
   own instances are emitted, sorted and blended; sort keys stay bit-identical to the single-GPU run
   restricted to the band.  The one exchange step is an all-gather of the band outputs (10 planes), done
   IN PLACE in a frame padded to equal bands; in the backward the per-pixel cotangents are read in place
   (no communication) and the per-splat gradients, which are partial sums over the band's pixels, are
   summed with one all-reduce of the op's flat gradient bucket.  When the camera requires grad, each rank's
   camera step gives its band's share as 35 float64 sums, which one float64 all-reduce adds before a single
   rounding to float32 (DESIGN §7r).

Collectives go through torch.distributed (NCCL over NVLink on GPUs; gloo in the CPU tests).
"""
from typing import Dict, List, Sequence, Tuple

import torch
import torch.distributed as dist

TILE = 16


def shard_views(num_views: int, rank: int, world: int) -> List[int]:
    """Round-robin assignment of independent views to ranks."""
    return list(range(rank, num_views, world))


def tile_rows(H: int) -> int:
    return (H + TILE - 1) // TILE


def tile_row_band(H: int, rank: int, world: int) -> Tuple[int, int]:
    """Tile rows [begin, end) owned by `rank` (SURVEY §8e: floor(gy*r/n) .. floor(gy*(r+1)/n))."""
    gy = tile_rows(H)
    return (gy * rank) // world, (gy * (rank + 1)) // world


def band_pixel_rows(H: int, band: Tuple[int, int]) -> Tuple[int, int]:
    return min(H, band[0] * TILE), min(H, band[1] * TILE)


def gather_band_outputs(planes: torch.Tensor, H: int, rank: int, world: int, group=None) -> torch.Tensor:
    """All-gather of band outputs.  `planes` is this rank's (C,H,W) tensor in which only the rows of
    its own band are meaningful; returns the stitched full (C,H,W) frame on every rank.  Bands differ
    by at most one tile row, so each contribution is padded to the largest band and sent with ONE
    equal-sized all_gather (the natural NCCL collective for this split)."""
    C, H_, W = planes.shape
    assert H_ == H
    bands = [tile_row_band(H, r, world) for r in range(world)]
    rows = [band_pixel_rows(H, b) for b in bands]
    max_rows = max(e - s for s, e in rows)
    s, e = rows[rank]
    send = planes.new_zeros((C, max_rows, W))
    send[:, : e - s] = planes[:, s:e]
    recv = planes.new_empty((world * C, max_rows, W))       # concatenation along dim 0
    if world > 1:
        dist.all_gather_into_tensor(recv, send.contiguous(), group=group)
    else:
        recv.copy_(send)
    recv = recv.view(world, C, max_rows, W)
    out = planes.new_empty((C, H, W))
    for r, (rs, re) in enumerate(rows):
        out[:, rs:re] = recv[r, :, : re - rs]
    return out


def slice_band_cotangent(grad: torch.Tensor, H: int, rank: int, world: int) -> torch.Tensor:
    """Backward of gather_band_outputs for this rank: keep its own rows, zero elsewhere (no comms)."""
    s, e = band_pixel_rows(H, tile_row_band(H, rank, world))
    out = torch.zeros_like(grad)
    out[:, s:e] = grad[:, s:e]
    return out


def allreduce_gradients(grads: Sequence[torch.Tensor], group=None) -> None:
    """Sum per-splat gradients across ranks in place (tile-band backward, or shared-model training in
    view-parallel mode).  Tensors are flattened into one bucket: launch latency, not link count, is
    what matters on NVSwitch."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    off = 0
    for g in grads:
        n = g.numel()
        g.copy_(flat[off:off + n].view_as(g))
        off += n


# ---------------------------------------------------------------------------------------------------
# Tile-band frame, copy-free exchange.
#
# The frame is allocated PADDED to `world` equal bands of ceil(gy / world) tile rows, planar (10, H_pad, W).
# Every rank renders its band straight into that tensor (the op takes the output views and their plane
# stride), then ONE in-place all-gather per plane completes it: rank r's chunk of plane c is the contiguous
# block of rows [r * rows, (r + 1) * rows), i.e. exactly the send buffer NCCL's in-place all-gather expects
# (sendbuff == recvbuff + rank * count).  No pad / stitch / cat copies; the returned render and allmap are
# views of the padded tensor.  In the backward the cotangents are read in place (the band kernels only
# touch their own rows) and the per-splat gradients, which the op writes into one flat bucket, are summed by
# one in-place all-reduce of that bucket.
# ---------------------------------------------------------------------------------------------------
def equal_band_rows(H: int, world: int) -> int:
    """Tile rows per rank of the equal-band partition (the last ranks may own fewer real rows)."""
    return (tile_rows(H) + world - 1) // world


def equal_band(H: int, rank: int, world: int) -> Tuple[int, int]:
    gy, rp = tile_rows(H), equal_band_rows(H, world)
    return min(gy, rank * rp), min(gy, (rank + 1) * rp)


def padded_frame(C: int, H: int, W: int, world: int, device, dtype=torch.float32) -> torch.Tensor:
    return torch.empty((C, equal_band_rows(H, world) * world * TILE, W), device=device, dtype=dtype)


def allgather_frame_inplace(buf: torch.Tensor, H: int, rank: int, world: int, group=None, async_op: bool = False):
    """Completes a padded frame (C, H_pad, W) in which this rank has written its own band.  With async_op the
    collectives are only enqueued (on the backend's own stream, ordered after the work already queued on the
    current stream) and the list of work handles is returned: the caller's stream does not wait for them."""
    if world == 1 or not dist.is_initialized():
        return []
    C, Hp, W = buf.shape
    rows = Hp // world
    works = []
    for c in range(C):
        plane = buf[c]
        send = plane[rank * rows:(rank + 1) * rows].reshape(-1)
        if not buf.is_cuda:
            send = send.clone()          # gloo (CPU tests) does not take an aliased send buffer
        w = dist.all_gather_into_tensor(plane.reshape(-1), send, group=group, async_op=async_op)
        if async_op:
            works.append(w)
    return works


# ---------------------------------------------------------------------------------------------------
# Exchange fused into the render kernel (gather="fused").
#
# The padded frame lives in SYMMETRIC memory (torch.distributed._symmetric_memory: every rank allocates the same
# buffer and maps all peers' buffers over NVLink; with an NVSwitch the group also gets one multicast address
# whose stores the switch fans out to every GPU).  The op is handed those addresses (`out_replicas`) and its
# render kernel stores each output pixel of the band to every replica — the all-gather is done by the stores of
# the kernel that produces the data, overlapped with the blending of the CTAs still running, and the only
# collective left is a cross-GPU barrier (`handle.barrier`) before anyone reads rows outside its own band.
# Frames come from a ring of two symmetric buffers per (shape, group): a rank can only start overwriting a
# buffer after the barrier of the NEXT frame, which every rank enters after the work it queued on the previous
# contents (same stream).  Outputs are therefore views that stay valid until the second-next fused call.
# ---------------------------------------------------------------------------------------------------
_sym_frames = {}


def symmetric_frame(H: int, W: int, world: int, device, group=None, multicast: bool = False):
    """(frame (10, H_pad, W), replica addresses, handle) — the next buffer of the ring for this shape."""
    import torch.distributed._symmetric_memory as symm
    g = group if group is not None else dist.group.WORLD
    key = (H, W, world, torch.device(device).index, g.group_name)
    ent = _sym_frames.get(key)
    if ent is None:
        bufs, hdls = [], []
        for _ in range(2):
            t = symm.empty((10, equal_band_rows(H, world) * world * TILE, W), dtype=torch.float32, device=device)
            hdls.append(symm.rendezvous(t, g))
            bufs.append(t)
        ent = _sym_frames[key] = {"bufs": bufs, "hdls": hdls, "turn": 0}
    i = ent["turn"]
    ent["turn"] ^= 1
    buf, hdl = ent["bufs"][i], ent["hdls"][i]
    off = buf.data_ptr() - int(hdl.buffer_ptrs[hdl.rank])       # the tensor's offset inside the symmetric allocation
    if off < 0 or off + buf.numel() * 4 > int(hdl.buffer_size):
        raise RuntimeError("symmetric frame is not inside this rank's symmetric allocation")
    mc = int(hdl.multicast_ptr) if multicast and hdl.has_multicast_support else 0
    reps = (mc + off,) if mc else tuple(int(a) + off for a in hdl.buffer_ptrs)
    return buf, reps, hdl


def release_symmetric_frames() -> None:
    """Drops the cached symmetric frames (two per frame shape and group; 2 x 1.3 GB for an 8K frame).  Collective in
    effect: every rank should call it at the same point, after its last use of a fused frame."""
    _sym_frames.clear()


_last = {"grad_bucket": None, "frame": None, "works": [], "fused_via": None}


def last_sh_expand():
    """Callable that fills shs.grad from the (reduced) colour gradients of the most recent tile-band backward,
    or None when the SH gradient was not deferred."""
    return _last.get("sh_expand")


def last_exchange_buffers():
    """(padded frame, flat gradient bucket) of the most recent tile-band step in this process — for
    measurement code that wants to time the collectives on the real buffers."""
    return _last["frame"], _last["grad_bucket"]


def reduce_camera_sums(sums: torch.Tensor, world: int, group=None, grad_reduce: str = "all_reduce") -> torch.Tensor:
    """The camera gradient of a tile-band frame, (35,) float32 in surfel_camera_backward's order (viewmatrix 16,
    projmatrix 16, campos 3), from this rank's band sums `sums` ((35,) float64, surfel_camera_backward_sums).  The
    sums are added over the ranks by one in-place float64 all-reduce and rounded to float32 once, so the result is
    one rounding of the whole frame's sum, the same on every rank.  grad_reduce="none" rounds this rank's partial
    instead.  "defer" reduces like "all_reduce": what it defers is the splat bucket, and the camera sums never go
    into that bucket.  Without a process group, or at world 1, nothing is communicated."""
    if grad_reduce != "none" and world > 1 and dist.is_initialized():
        dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=group)
    return sums.to(torch.float32)


class _BandFrame(torch.autograd.Function):
    """One oversized frame rendered cooperatively: this rank's band by the CUDA op, the rest by the in-place
    all-gather.  Wraps the op's own autograd node (same forward / backward code) and adds the exchange.  With the
    camera tensors given (viewmatrix, projmatrix, campos: they replace the settings' own), they are differentiable
    inputs too, as in _RasterizeGaussiansCamera, and their gradients are the bands' sums (reduce_camera_sums)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                settings, rank, world, group, grad_reduce, gather="sync", viewmatrix=None, projmatrix=None,
                campos=None):
        from diff_surfel_rasterization import _RasterizeGaussians, _mark
        H, W = int(settings.image_height), int(settings.image_width)
        _mark("band_enter")
        ctx.cam_meta = None
        if viewmatrix is not None:
            ctx.cam_meta = tuple((t.shape, t.dtype) for t in (viewmatrix, projmatrix, campos))
            settings = settings._replace(viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos)
        band = equal_band(H, rank, world)
        # the SH gradient (48 of the 61 floats per splat) is a rank-1 expansion of 3 numbers: the backward leaves
        # it unexpanded, the 16-float bucket is reduced, and the expansion runs once on the sum
        ctx.defer_sh = world > 1 and dist.is_initialized()
        fused = gather in ("fused", "fused_multicast") and world > 1 and dist.is_initialized()
        if fused:
            buf, reps, hdl = symmetric_frame(H, W, world, means3D.device, group, multicast=(gather == "fused_multicast"))
            if gather == "fused_multicast" and len(reps) != 1:
                raise RuntimeError("gather='fused_multicast': this process group has no multicast address (no NVSwitch?)")
            _last["fused_via"] = "multicast" if len(reps) == 1 else "peer stores"
            rs = settings._replace(tile_rows=band, out_buffers=(buf[:3, :H], buf[3:, :H]), out_replicas=reps)
        else:
            buf = padded_frame(10, H, W, world, means3D.device)
            rs = settings._replace(tile_rows=band, out_buffers=(buf[:3, :H], buf[3:, :H]))
        _mark("band_frame_allocated")
        color, radii, allmap = _RasterizeGaussians.forward(ctx, means3D, means2D, sh, colors_precomp, opacities,
                                                           scales, rotations, cov3Ds_precomp, rs)
        if world > 1 and dist.is_initialized():
            # radii (and so visibility_filter / max_radii2D downstream) are per-band partials: a splat's tile
            # rect is clipped to the band before it is counted.  The MAX over the ranks goes into a COPY: the
            # backward must keep seeing the band's own radii (its preprocess backward skips splats the band
            # culled, whose forward records were never written).  Reduced BEFORE the frame exchange is enqueued:
            # the backend runs its collectives in order, so a blocking collective queued behind asynchronous
            # gathers would make the current stream wait for them.
            radii = radii.clone()          # the context keeps the band's own tensor (saved by the op's forward)
            dist.all_reduce(radii, op=dist.ReduceOp.MAX, group=group)
            ctx.mark_non_differentiable(radii)
        if fused:
            hdl.barrier(channel=0)          # every rank's band has landed in every replica
            _last["works"] = []
        else:
            _last["works"] = allgather_frame_inplace(buf, H, rank, world, group, async_op=(gather == "async"))
        _mark("band_gather_enqueued")
        _last["frame"] = buf
        _mark("band_exit")
        ctx.band_meta = (world, group, grad_reduce)
        return color, radii, allmap

    @staticmethod
    def backward(ctx, g_color, g_radii, g_allmap):
        from diff_surfel_rasterization import _backward
        world, group, grad_reduce = ctx.band_meta
        camera = ctx.cam_meta is not None
        # the camera step runs right after the band backward, on its record, before any collective
        grads, sums = _backward(ctx, g_color, g_allmap, camera=camera, camera_sums=True)
        _last["grad_bucket"] = ctx.grad_bucket
        _last["sh_expand"] = ctx.sh_expand
        if grad_reduce == "all_reduce" and world > 1 and dist.is_initialized():
            dist.all_reduce(ctx.grad_bucket, op=dist.ReduceOp.SUM, group=group)   # every gradient, one collective, in place
        if ctx.sh_expand is not None and grad_reduce != "defer":
            ctx.sh_expand()                  # dL_dsh = basis (x) colour gradient (summed over the ranks after "all_reduce")
        # grad_reduce == "defer": the caller reduces last_exchange_buffers()[1] itself and then calls
        # last_sh_expand()() — until then dL_dsh (shs.grad) is unwritten
        cam = (None, None, None)
        if camera:
            g = reduce_camera_sums(sums, world, group, grad_reduce)
            cam = tuple(t.reshape(shape).to(dtype) for t, (shape, dtype) in zip((g[0:16], g[16:32], g[32:35]), ctx.cam_meta))
        return grads + (None, None, None, None, None, None) + cam


def rasterize_tile_band(rasterizer_cls, settings, rank: int, world: int, group=None, grad_reduce: str = "all_reduce",
                        gather: str = "sync", **inputs) -> Dict[str, torch.Tensor]:
    """One oversized frame split over `world` GPUs (SURVEY §8e, BASELINE config 5).  Returns the COMPLETE
    frame on every rank ("render" (3,H,W), "allmap" (7,H,W): views of one padded tensor), "radii" reduced
    with MAX over the ranks, and the band this rank rendered.  Differentiable; with grad_reduce="all_reduce"
    (default) the gradients that reach the inputs are already summed over the ranks; "none" leaves this
    band's partial sums; "defer" additionally leaves shs.grad UNWRITTEN: the caller reduces the flat bucket
    `last_exchange_buffers()[1]` itself (e.g. with a reduce-scatter for a sharded optimizer) and then runs
    `last_sh_expand()()` to produce shs.grad from the reduced colour gradients.
    The bucket holds 16 floats per splat, not 61: the SH gradient is the rank-1 expansion basis(dir) (x) dL_dcolor
    and is expanded AFTER the reduction (C ABI: sh_grad_deferred / surfel_sh_grad_expand).

    gather="async" only ENQUEUES the all-gathers: the rows of this rank's own band (result["band"]) are valid on
    the current stream at once, the other ranks' rows after result["wait"]() — so a loss that is local to the
    band (per-pixel terms; SSIM with a 5-row halo inside the band) can run its backward, which reads nothing
    but this band's cotangent rows, while the exchange is still in flight.

    gather="fused" has no all-gather at all: the frame lives in symmetric memory and the render kernel itself
    stores the band's pixels into every GPU's copy over NVLink (one store per peer and value; measured at N = 2:
    forward + exchange 3.1 ms against 3.9 ms for forward + NCCL all-gather); a cross-GPU barrier follows.
    "fused_multicast" sends ONE store per value to the group's NVSwitch multicast address instead (measured
    slower at N = 2 — 7.6 ms — the switch handles 32-byte multicast writes poorly; kept for comparison).  The
    returned views belong to a ring of two frames and stay valid until the second-next fused call.

    Camera gradients: when grad mode is on and settings.viewmatrix, projmatrix or campos requires grad (the test of
    rasterize_gaussians), the frame is also differentiable in the camera, in every gather mode.  Each rank forms its
    band's share of the rasterizer's camera gradient as float64 sums; "all_reduce" and "defer" add them over the ranks
    with one float64 all-reduce and round once, "none" rounds this rank's share.  Compose any camera-dependent tail
    (postprocess.surface_outputs / surface_regularizers) on the gathered frame and do NOT reduce its camera gradient:
    every rank already holds the whole frame, so that part is whole-frame on every rank (DESIGN §7r).
    `rasterizer_cls` is accepted for symmetry with the single-GPU call and is not used."""
    del rasterizer_cls
    if grad_reduce not in ("all_reduce", "none", "defer"):
        raise ValueError("grad_reduce must be 'all_reduce', 'none' or 'defer'")
    if gather not in ("sync", "async", "fused", "fused_multicast"):
        raise ValueError("gather must be 'sync', 'async', 'fused' or 'fused_multicast'")
    empty = torch.Tensor([])
    g = lambda k: inputs.get(k) if inputs.get(k) is not None else empty
    if (inputs.get("shs") is None) == (inputs.get("colors_precomp") is None):
        raise Exception("Please provide excatly one of either SHs or precomputed colors!")
    from diff_surfel_rasterization import _wants_camera_grad
    cam = (settings.viewmatrix, settings.projmatrix, settings.campos) if _wants_camera_grad(settings) else ()
    color, radii, allmap = _BandFrame.apply(inputs["means3D"], inputs["means2D"], g("shs"), g("colors_precomp"),
                                            inputs["opacities"], g("scales"), g("rotations"), g("cov3D_precomp"),
                                            settings, rank, world, group, grad_reduce, gather, *cam)
    works = _last["works"]

    def wait():
        for w in works:
            w.wait()
        del works[:]

    return {"render": color, "allmap": allmap, "radii": radii, "band": equal_band(int(settings.image_height), rank, world),
            "wait": wait}
