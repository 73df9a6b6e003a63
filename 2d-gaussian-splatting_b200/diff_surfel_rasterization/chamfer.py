"""DTU Chamfer evaluation of a mesh or point cloud on the device: the body of the reference's
scripts/eval_dtu/eval.py (lines 48-158), the score `scripts/dtu_eval.py` reports, computed from CUDA tensors
(csrc/chamfer.cu):

    pcd = sample_mesh(verts, faces, density=0.2)                 # eval.py:48-71, `--mode mesh`
    r = dtu_chamfer(pcd, stl, obs_mask, bb, res, plane)          # eval.py:79-158 (`--mode pcd`: pass the cloud)
    r.mean_d2s, r.mean_s2d, r.overall

Every step is float64 and reproduces the reference's evaluation order bit for bit; the rules (sampling, the greedy
radius downsampling, the float32 box, the observation grid, the plane, the colours) are in DESIGN.md §7m.  The only
randomness is the shuffle: pass `perm` for the reference's order, or it is drawn on the device from `generator`.
No CPU path.

The step before it, the DTU mask culling of scripts/eval_dtu/evaluate_single_scene.py (cull_scan, lines 19-101), is
here too (csrc/cull.cu, DESIGN.md §7n):

    v, f, c = cull_scan(verts, faces, masks, world_mats, scale_mats, colors=None)   # then sample_mesh(v, f)
"""
import ctypes
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _cabi


@dataclass
class ChamferResult:
    """What eval.py prints and writes.  mean_d2s, mean_s2d, overall: Python floats, NaN where the reference's mean
    of an empty selection is NaN.  data_down (K,3) and data_color (K,3): the cloud and colours of vis_XXX_d2s.ply;
    stl_color (S,3): the colours of vis_XXX_s2d.ply (whose points are `stl`).  dist_d2s: per data_in_obs row,
    dist_s2d: per stl_above row, +inf where the distance is at least max_dist.  rounds: greedy downsampling rounds."""
    mean_d2s: float
    mean_s2d: float
    overall: float
    data_down: torch.Tensor
    data_color: torch.Tensor
    stl_color: torch.Tensor
    dist_d2s: torch.Tensor
    dist_s2d: torch.Tensor
    rounds: int


def _cuda(who, name, t):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError(f"{who}: {name} must be a CUDA tensor (there is no CPU path)")


def _points(who, name, t, dev=None):
    _cuda(who, name, t)
    if t.dtype not in (torch.float32, torch.float64) or t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{who}: {name} must be (N,3) float32 or float64, got {tuple(t.shape)} {t.dtype}")
    if dev is not None and t.device != dev:
        raise ValueError(f"{who}: {name} is on {t.device}, expected {dev}")
    return t.to(torch.float64).contiguous()      # float32 widens exactly


def _host(x, dtype):
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    return np.asarray(x).astype(dtype)


@torch.no_grad()
def sample_mesh(verts, faces, density=0.2):
    """The reference's mesh sampling (eval.py:48-71): (M + T, 3) float64 on the mesh's device, all M vertices (also
    unreferenced ones) then the T samples of every triangle of positive area, in triangle order.  verts (M,3) float32
    or float64, faces (F,3) int32 or int64.  ValueError on a face index outside [0, M), a non-finite vertex, a mesh
    with no triangle of positive area (the reference's np.concatenate([])) or more points than the device supports."""
    who = "sample_mesh"
    v = _points(who, "verts", verts)
    _cuda(who, "faces", faces)
    if faces.dtype not in (torch.int32, torch.int64) or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"{who}: faces must be (F,3) int32 or int64, got {tuple(faces.shape)} {faces.dtype}")
    if faces.device != verts.device:
        raise ValueError(f"{who}: faces are on {faces.device}, verts on {verts.device}")
    density = float(density)
    if not (density > 0 and math.isfinite(density)):
        raise ValueError(f"{who}: density must be positive and finite, got {density}")
    dev = v.device
    lib = _cabi.load()
    M, F = v.shape[0], faces.shape[0]
    limit = lib.surfel_chamfer_max_points()
    if M > limit or F > limit:
        raise ValueError(f"{who}: {M} vertices and {F} faces; at most {limit} of each are supported")
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        f = faces.to(torch.int64).contiguous()
        ws_bytes = lib.surfel_chamfer_sample_workspace_bytes(F)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        info = torch.empty(4, dtype=torch.int64, device=dev)
        _cabi.check(lib.surfel_chamfer_sample_count(M, F, v.data_ptr(), f.data_ptr(), density, ws.data_ptr(),
                                                    ws_bytes, info.data_ptr(), stream))
        total, bad, nonfinite, positive = info.tolist()
        if bad:
            raise ValueError(f"{who}: a face index lies outside [0, {M})")
        if nonfinite:
            raise ValueError(f"{who}: verts contain NaN or infinity")
        if positive == 0:
            raise ValueError(f"{who}: no triangle of positive area, nothing to concatenate")
        if M + total > limit:
            raise ValueError(f"{who}: {M} vertices and {total} samples; at most {limit} points are supported")
        out = torch.empty((M + total, 3), dtype=torch.float64, device=dev)
        out[:M].copy_(v)
        _cabi.check(lib.surfel_chamfer_sample_emit(M, F, v.data_ptr(), f.data_ptr(), density, ws.data_ptr(), ws_bytes,
                                                   total, out.data_ptr(), stream))
        return out


@torch.no_grad()
def dtu_chamfer(pcd, stl, obs_mask, bb, res, plane, perm=None, generator=None, downsample_density=0.2,
                patch_size=60.0, max_dist=20.0, visualize_threshold=10.0):
    """The reference's evaluation (eval.py:79-158) of the cloud `pcd` (N,3) against the STL cloud `stl` (S,3), both
    float32 or float64 on one CUDA device.  obs_mask: (X,Y,Z) bool or uint8 there; bb (2,3), res and plane (4): the
    ObsMask and Plane .mat values (host arrays or tensors).  perm: (N,) integer permutation, the order the reference's
    shuffle gives; None draws one on the device from `generator`.  Returns a ChamferResult.  The inputs are not
    changed.  ValueError where the reference's sklearn or numpy raises one: non-finite coordinates, an empty cloud or
    STL, no inbound or no observed point, no STL point above the plane; also for a perm that is not a permutation."""
    who = "dtu_chamfer"
    p = _points(who, "pcd", pcd)
    dev = p.device
    s = _points(who, "stl", stl, dev)
    _cuda(who, "obs_mask", obs_mask)
    if obs_mask.dtype not in (torch.bool, torch.uint8) or obs_mask.dim() != 3 or obs_mask.device != dev:
        raise ValueError(f"{who}: obs_mask must be (X,Y,Z) bool or uint8 on {dev}, got {tuple(obs_mask.shape)} "
                         f"{obs_mask.dtype} on {obs_mask.device}")
    if min(obs_mask.shape) < 1:
        raise ValueError(f"{who}: obs_mask of shape {tuple(obs_mask.shape)}")
    bb32 = _host(bb, np.float32)                 # eval.py:100, BB.astype(np.float32)
    if bb32.shape != (2, 3):
        raise ValueError(f"{who}: bb must be (2,3), got {bb32.shape}")
    res_a = _host(res, np.float64)
    if res_a.size != 1:
        raise ValueError(f"{who}: res must be a scalar, got shape {res_a.shape}")
    plane_a = _host(plane, np.float64)
    if plane_a.size != 4:
        raise ValueError(f"{who}: plane must hold 4 values, got shape {plane_a.shape}")
    patch = float(patch_size)
    # eval.py:103 in float32: numpy 2 keeps the Python float weak, so it is rounded to float32 before the operation
    lo = (bb32[:1] - patch)[0].astype(np.float64)
    hi = (bb32[1:] + patch * 2)[0].astype(np.float64)
    thresh, md, vis = float(downsample_density), float(max_dist), float(visualize_threshold)
    N, S = p.shape[0], s.shape[0]
    if N == 0 or S == 0:
        raise ValueError(f"{who}: {N} points and {S} STL points; sklearn fits no empty set")
    lib = _cabi.load()
    limit = lib.surfel_chamfer_max_points()
    if N > limit or S > limit:
        raise ValueError(f"{who}: {N} points and {S} STL points; at most {limit} of each are supported")
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        if perm is None:
            order = torch.randperm(N, generator=generator, device=dev)
            bad_perm = torch.zeros((), dtype=torch.bool, device=dev)
        else:
            _cuda(who, "perm", perm)
            if perm.dtype not in (torch.int32, torch.int64) or perm.shape != (N,) or perm.device != dev:
                raise ValueError(f"{who}: perm must be ({N},) int32 or int64 on {dev}, got {tuple(perm.shape)} "
                                 f"{perm.dtype} on {perm.device}")
            q = perm.to(torch.int64)
            inside = (q >= 0) & (q < N)
            order = q.clamp(0, N - 1)
            seen = torch.zeros(N, dtype=torch.bool, device=dev)
            seen[order] = True
            bad_perm = ~(inside.all() & seen.all())
        shuffled = p.index_select(0, order).contiguous()
        flags = torch.stack([bad_perm, ~torch.isfinite(p).all(), ~torch.isfinite(s).all()]).tolist()
        if flags[0]:
            raise ValueError(f"{who}: perm is not a permutation of range({N})")
        if flags[1] or flags[2]:
            raise ValueError(f"{who}: {'pcd' if flags[1] else 'stl'} contains NaN or infinity")
        ws_bytes = lib.surfel_chamfer_workspace_bytes(N, S)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        rounds = ctypes.c_int(0)
        _cabi.check(lib.surfel_chamfer_downsample(N, S, shuffled.data_ptr(), thresh, ws.data_ptr(), ws_bytes,
                                                  ctypes.byref(rounds), stream))
        mask = obs_mask.contiguous().view(torch.uint8)
        down = torch.empty((N, 3), dtype=torch.float64, device=dev)
        d_in = torch.empty((N, 3), dtype=torch.float64, device=dev)
        d_obs = torch.empty((N, 3), dtype=torch.float64, device=dev)
        obs_down = torch.empty(N, dtype=torch.int32, device=dev)
        above = torch.empty((S, 3), dtype=torch.float64, device=dev)
        above_idx = torch.empty(S, dtype=torch.int32, device=dev)
        info = torch.empty(4, dtype=torch.int64, device=dev)
        dv = lambda a: (ctypes.c_double * len(a))(*[float(x) for x in a])   # noqa: E731
        _cabi.check(lib.surfel_chamfer_select(
            N, S, shuffled.data_ptr(), s.data_ptr(), dv(lo), dv(hi), dv(bb32[0].astype(np.float64)),
            float(res_a.reshape(())), mask.data_ptr(), (ctypes.c_int * 3)(*mask.shape), dv(plane_a.reshape(4)),
            ws.data_ptr(), ws_bytes, down.data_ptr(), d_in.data_ptr(), d_obs.data_ptr(), obs_down.data_ptr(),
            above.data_ptr(), above_idx.data_ptr(), info.data_ptr(), stream))
        n_down, n_in, n_obs, n_above = info.tolist()
        if n_obs == 0:
            raise ValueError(f"{who}: no point inside the box and the observation mask "
                             f"({n_down} kept, {n_in} inside the box); sklearn queries no empty set")
        if n_above == 0:
            raise ValueError(f"{who}: no STL point above the plane; sklearn queries no empty set")
        dist_d2s = torch.empty(n_obs, dtype=torch.float64, device=dev)
        dist_s2d = torch.empty(n_above, dtype=torch.float64, device=dev)
        data_color = torch.empty((n_down, 3), dtype=torch.float64, device=dev)
        stl_color = torch.empty((S, 3), dtype=torch.float64, device=dev)
        sums = torch.empty(4, dtype=torch.float64, device=dev)
        _cabi.check(lib.surfel_chamfer_distances(
            N, S, s.data_ptr(), n_down, n_in, d_in.data_ptr(), n_obs, d_obs.data_ptr(), obs_down.data_ptr(), n_above,
            above.data_ptr(), above_idx.data_ptr(), md, vis, ws.data_ptr(), ws_bytes, dist_d2s.data_ptr(),
            dist_s2d.data_ptr(), data_color.data_ptr(), stl_color.data_ptr(), sums.data_ptr(), stream))
        del ws, d_in, d_obs, obs_down, above, above_idx
        s_d2s, c_d2s, s_s2d, c_s2d = sums.tolist()
        mean_d2s = s_d2s / c_d2s if c_d2s else math.nan
        mean_s2d = s_s2d / c_s2d if c_s2d else math.nan
        return ChamferResult(mean_d2s, mean_s2d, (mean_d2s + mean_s2d) / 2, down[:n_down], data_color, stl_color,
                             dist_d2s, dist_s2d, rounds.value)


def dtu_projections(world_mats, scale_mats):
    """The projection cull_scan uses for each DTU view (DESIGN.md §7n, rule 1): (N,3,4) float32 host array, rows 0-2
    of intrinsics @ inverse(pose) as the reference's evaluate_single_scene.py builds them from P = (world_mat @
    scale_mat)[:3, :4] with cv2.decomposeProjectionMatrix.  That product is sign(det P[:, :3]) * P / |P[2, :3]|, which
    is evaluated here in float64 and rounded once.  world_mats, scale_mats: the (N,4,4) matrices of cameras.npz, as
    host arrays or tensors.  ValueError on other shapes, non-finite entries or a singular P[:, :3]."""
    who = "dtu_projections"
    wm, sm = _host(world_mats, np.float32), _host(scale_mats, np.float32)
    if wm.ndim != 3 or wm.shape[1:] != (4, 4) or sm.shape != wm.shape:
        raise ValueError(f"{who}: world_mats and scale_mats must both be (N,4,4), got {wm.shape} and {sm.shape}")
    # world_mat @ scale_mat in float32, one view at a time, as the reference forms it
    P = np.stack([w @ s for w, s in zip(wm, sm)])[:, :3, :4].astype(np.float64) if len(wm) else np.zeros((0, 3, 4))
    det = np.linalg.det(P[:, :, :3]) if len(P) else np.zeros(0)
    norm = np.sqrt((P[:, 2, :3] ** 2).sum(1))
    if not (np.isfinite(P).all() and np.isfinite(det).all() and (det != 0).all() and (norm > 0).all()):
        raise ValueError(f"{who}: a camera matrix is not finite or P[:, :3] is singular")
    return (np.sign(det)[:, None, None] * P / norm[:, None, None]).astype(np.float32)


def _cull(who, verts, faces, masks, proj, scale_mats, colors, image_size, radius):
    """cull_scan with the projections given: dict of the outputs, the bit-packed dilated masks and the keep flags."""
    _cuda(who, "masks", masks)
    if masks.dtype not in (torch.uint8, torch.bool) or masks.dim() != 3:
        raise ValueError(f"{who}: masks must be (N,H,W) uint8 or bool, got {tuple(masks.shape)} {masks.dtype}")
    dev = masks.device
    v = _points(who, "verts", verts, dev)
    _cuda(who, "faces", faces)
    if faces.dtype not in (torch.int32, torch.int64) or faces.dim() != 2 or faces.shape[1] != 3 or faces.device != dev:
        raise ValueError(f"{who}: faces must be (F,3) int32 or int64 on {dev}, got {tuple(faces.shape)} "
                         f"{faces.dtype} on {faces.device}")
    M, F = v.shape[0], faces.shape[0]
    if colors is not None:
        _cuda(who, "colors", colors)
        if colors.dim() != 2 or colors.shape[0] != M or colors.device != dev:
            raise ValueError(f"{who}: colors must be ({M},C) on {dev}, got {tuple(colors.shape)} on {colors.device}")
    size = tuple(int(s) for s in image_size)
    if len(size) != 2 or min(size) < 1:
        raise ValueError(f"{who}: image_size must be (W, H) with positive sides, got {image_size}")
    lib = _cabi.load()
    if isinstance(radius, bool) or int(radius) != radius or not 0 <= radius <= lib.surfel_cull_max_radius():
        raise ValueError(f"{who}: radius must be an integer in [0, {lib.surfel_cull_max_radius()}], got {radius}")
    radius = int(radius)
    N, H, W = masks.shape
    if proj.shape != (N, 3, 4):
        raise ValueError(f"{who}: {N} masks and {proj.shape[0]} cameras")
    if not 1 <= N <= lib.surfel_cull_max_views():
        raise ValueError(f"{who}: {N} views; 1 to {lib.surfel_cull_max_views()} are supported")
    sm0 = _host(scale_mats, np.float32).reshape(-1, 4, 4)[0]
    world = (ctypes.c_double * 4)(float(sm0[0, 0]), float(sm0[0, 3]), float(sm0[1, 3]), float(sm0[2, 3]))
    ws_bytes = lib.surfel_cull_workspace_bytes(N, H, W, M, F)
    if ws_bytes == 0:
        raise ValueError(f"{who}: {N} masks of {W} x {H}, {M} vertices and {F} faces; sides up to 32768 and up to "
                         f"2^31 - 1 vertices and faces are supported")
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        m8 = masks.contiguous().view(torch.uint8)
        f = faces.to(torch.int64).contiguous()
        A = torch.from_numpy(np.ascontiguousarray(proj, np.float32)).to(dev)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        dilated = torch.empty((N, H, (W + 31) // 32), dtype=torch.int32, device=dev)
        keep = torch.empty(M, dtype=torch.uint8, device=dev)
        info = torch.empty(4, dtype=torch.int64, device=dev)
        _cabi.check(lib.surfel_cull_dilate(N, H, W, radius, m8.data_ptr(), ws.data_ptr(), ws_bytes,
                                           dilated.data_ptr(), stream))
        _cabi.check(lib.surfel_cull_vertices(M, v.data_ptr(), F, f.data_ptr(), N, A.data_ptr(), size[0], size[1], H,
                                             W, dilated.data_ptr(), ws.data_ptr(), ws_bytes, keep.data_ptr(),
                                             info.data_ptr(), stream))
        bad, nonfinite, n_verts, n_faces = info.tolist()
        if bad:
            raise ValueError(f"{who}: a face index lies outside [0, {M})")
        if nonfinite:
            raise ValueError(f"{who}: verts contain a coordinate that is not finite in float32")
        out_v = torch.empty((n_verts, 3), dtype=torch.float64, device=dev)
        out_f = torch.empty((n_faces, 3), dtype=torch.int64, device=dev)
        c = None if colors is None else colors.contiguous()
        out_c = None if c is None else torch.empty((n_verts, c.shape[1]), dtype=c.dtype, device=dev)
        row_bytes = 0 if c is None else c.shape[1] * c.element_size()
        _cabi.check(lib.surfel_cull_emit(M, v.data_ptr(), F, f.data_ptr(), world, 0 if c is None else c.data_ptr(),
                                         row_bytes, ws.data_ptr(), ws_bytes, n_verts, n_faces, out_v.data_ptr(),
                                         out_f.data_ptr(),
                                         0 if out_c is None else out_c.data_ptr(), stream))
        return dict(verts=out_v, faces=out_f, colors=out_c, dilated=dilated, keep=keep.bool())


@torch.no_grad()
def cull_scan(verts, faces, masks, world_mats, scale_mats, colors=None, image_size=(1600, 1200), radius=24):
    """The reference's DTU mask culling (cull_scan of scripts/eval_dtu/evaluate_single_scene.py, DESIGN.md §7n), the
    step before eval.py scores a mesh: drops every vertex that some view projects inside the image_size (W, H) frame
    onto a pixel outside that view's mask dilated by disk(radius), drops every face that lost a vertex and maps the
    rest to world units with scale_mats[0].

    verts (M,3) float32 or float64, faces (F,3) int32 or int64, colors None or (M,C), masks (N,H,W) uint8 or bool
    (channel 0 of each mask image; nonzero is set), all on one CUDA device; world_mats and scale_mats: the (N,4,4)
    matrices of cameras.npz.  Returns (verts (M',3) float64, faces (F',3) int64, colours (M',C) or None): kept
    vertices in order (unreferenced ones included) and kept faces renumbered.  Runs on the current stream; the inputs
    are not changed.  ValueError on a face index outside [0, M), a vertex that is not finite in float32, masks and
    cameras that disagree in N, or sizes beyond the supported counts."""
    r = _cull("cull_scan", verts, faces, masks, dtu_projections(world_mats, scale_mats), scale_mats, colors,
              image_size, radius)
    return r["verts"], r["faces"], r["colors"]
