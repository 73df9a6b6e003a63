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
