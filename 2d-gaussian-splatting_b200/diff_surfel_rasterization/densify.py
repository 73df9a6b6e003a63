"""Fused densification: `densify_and_prune(gaussians, max_grad, min_opacity, extent, max_screen_size)` does what the
reference's `GaussianModel.densify_and_prune` (scene/gaussian_model.py:348-403, called at train.py:132) does to the
model and its optimizer, with three CUDA launches (csrc/densify.cu: a plan, then an apply for f_rest and one for the
other five groups) and one device-to-host copy:

    densify_and_prune(gaussians, opt.densify_grad_threshold, 0.005, scene.cameras_extent, size_threshold)

`gaussians` is any object with the reference GaussianModel's attributes: `_xyz`, `_features_dc`,
`_features_rest`, `_opacity`, `_scaling`, `_rotation`, `xyz_gradient_accum`, `denom`, `max_radii2D`,
`percent_dense` and `optimizer` (a `torch.optim.Adam` or `FusedAdam` whose groups are named "xyz", "f_dc",
"f_rest", "opacity", "scaling" and "rotation", one parameter each).  Afterwards it holds new `nn.Parameter`s
(requires_grad, no .grad) in the same groups, the optimizer state is re-keyed to them (surviving rows keep their
moments, new rows get zeros, `step` is untouched, a group without state stays without), and the statistics are
zeros of the new size.  The split samples are one `normal_` of shape (2S, 3) on the default generator of the
device, the draw the reference makes, so a training run keeps the same random stream.  Rules: DESIGN.md §7h.

Unlike the reference it does not call torch.cuda.empty_cache(); that is left to the caller.  No CPU path.
"""
import math

import torch
from torch import nn

from . import _cabi

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
_ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
         "scaling": "_scaling", "rotation": "_rotation"}
_KIND = {"xyz": _cabi.DENSIFY_XYZ, "scaling": _cabi.DENSIFY_SCALING, "rotation": _cabi.DENSIFY_ROTATION}
_ROW = {"xyz": (3,), "opacity": (1,), "scaling": (2,), "rotation": (4,)}


def draw_split_samples(n, device):
    """The standard normal draw of the split rows: torch.normal(mean, std) is normal_(0, 1) on a tensor of the
    result's shape followed by *std + mean, so this consumes the generator exactly as the reference does."""
    return torch.empty((n, 3), dtype=torch.float32, device=device).normal_()


def _check(name, t, P, device):
    if not isinstance(t, torch.Tensor):
        raise RuntimeError(f"densify_and_prune: {name} is not a tensor")
    if not t.is_cuda:
        raise RuntimeError(f"densify_and_prune: {name} must be a CUDA tensor (there is no CPU path)")
    if t.dtype != torch.float32:
        raise RuntimeError(f"densify_and_prune: {name} must be float32, got {t.dtype}")
    if not t.is_contiguous():
        raise RuntimeError(f"densify_and_prune: {name} must be contiguous")
    if t.device != device or t.dim() == 0 or t.shape[0] != P:
        raise RuntimeError(f"densify_and_prune: {name} must have {P} rows on {device}, got {tuple(t.shape)} on {t.device}")


def _apply(lib, gaussians, entries, phase, P, P_new, n_split, z, ws, nbytes, dev):
    """One apply launch over the groups entries[i], i in phase; then their new parameters replace the old ones in
    the optimizer (re-keyed as the reference's _prune_optimizer / cat_tensors_to_optimizer leave it) and on the
    model, and entries[i] is cleared so that nothing here keeps the old tensors alive."""
    opt = gaussians.optimizer
    stream = torch.cuda.current_stream(dev)
    table = (_cabi.DensifyGroup * len(phase))()
    outs = []
    for g, i in zip(table, phase):
        group, p, st = entries[i]
        new_p = torch.empty((P_new,) + tuple(p.shape[1:]), dtype=torch.float32, device=dev)
        new_m = new_v = None
        olds = [p]
        if st is not None:
            new_m, new_v = torch.empty_like(new_p), torch.empty_like(new_p)
            g.exp_avg, g.exp_avg_sq = st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()
            g.out_exp_avg, g.out_exp_avg_sq = new_m.data_ptr(), new_v.data_ptr()
            olds += [st["exp_avg"], st["exp_avg_sq"]]
        g.param, g.out_param = p.data_ptr(), new_p.data_ptr()
        g.row_floats = math.prod(p.shape[1:])
        g.kind = _KIND.get(group["name"], _cabi.DENSIFY_COPY)
        for t in olds:            # read on this stream: not reusable by another before the launch has run
            t.record_stream(stream)
        outs.append((new_p, new_m, new_v))
    _cabi.check(lib.surfel_densify_apply(P, P_new, n_split, len(phase), table, z.data_ptr(), ws.data_ptr(), nbytes,
                                         stream.cuda_stream))
    for i, (new_p, new_m, new_v) in zip(phase, outs):
        group, p, st = entries[i]
        entries[i] = None
        param = nn.Parameter(new_p.requires_grad_(True))
        if st is not None:
            del opt.state[p]
            st["exp_avg"], st["exp_avg_sq"] = new_m, new_v
            opt.state[param] = st
        group["params"][0] = param
        setattr(gaussians, _ATTR[group["name"]], param)


@torch.no_grad()
def densify_and_prune(gaussians, max_grad, min_opacity, extent, max_screen_size):
    opt = gaussians.optimizer
    by_name = {}
    for group in opt.param_groups:
        name = group.get("name")
        if name in by_name:
            raise RuntimeError(f"densify_and_prune: two parameter groups named {name!r}")
        by_name[name] = group
    for name in GROUPS:
        if name not in by_name:
            raise RuntimeError(f"densify_and_prune: the optimizer has no parameter group named {name!r}")
    for group in opt.param_groups:
        if group.get("name") not in GROUPS:      # the reference has no rows to add to any other group
            raise RuntimeError(f"densify_and_prune: unexpected parameter group {group.get('name')!r}")
        if len(group["params"]) != 1:
            raise RuntimeError(f"densify_and_prune: group {group.get('name')!r} must hold exactly one parameter")

    xyz = by_name["xyz"]["params"][0]
    if not isinstance(xyz, torch.Tensor) or not xyz.is_cuda:
        raise RuntimeError("densify_and_prune: parameters must be CUDA tensors (there is no CPU path)")
    dev, P = xyz.device, xyz.shape[0]
    entries = []                                  # (group, param, state or None), in param_groups order
    for group in opt.param_groups:
        name = group.get("name")
        p = group["params"][0]
        _check(f"parameter {name!r}", p, P, dev)
        if name in _ROW and tuple(p.shape[1:]) != _ROW[name]:
            raise RuntimeError(f"densify_and_prune: parameter {name!r} has shape {tuple(p.shape)}")
        st = opt.state.get(p, None)
        if st is not None:
            if "exp_avg" not in st or "exp_avg_sq" not in st:
                raise RuntimeError(f"densify_and_prune: the state of {name!r} has no exp_avg / exp_avg_sq")
            _check(f"exp_avg of {name!r}", st["exp_avg"], P, dev)
            _check(f"exp_avg_sq of {name!r}", st["exp_avg_sq"], P, dev)
            if st["exp_avg"].shape != p.shape or st["exp_avg_sq"].shape != p.shape:
                raise RuntimeError(f"densify_and_prune: the moments of {name!r} do not match its shape")
        entries.append((group, p, st))
    del p, st                                     # entries alone holds the old tensors (see _apply)
    accum, denom = gaussians.xyz_gradient_accum, gaussians.denom
    _check("xyz_gradient_accum", accum, P, dev)
    _check("denom", denom, P, dev)
    _check("max_radii2D", gaussians.max_radii2D, P, dev)
    if accum.numel() != P or denom.numel() != P:
        raise RuntimeError("densify_and_prune: xyz_gradient_accum and denom must be (P, 1)")
    scaling, opacity = by_name["scaling"]["params"][0], by_name["opacity"]["params"][0]

    lib = _cabi.load()
    # the thresholds as Python forms them, in double; the library rounds each once to float32
    clone_max = gaussians.percent_dense * extent
    prune_max = 0.1 * extent
    use_screen = 1 if max_screen_size else 0
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        nbytes = lib.surfel_densify_workspace_bytes(P)
        if nbytes == 0:
            raise RuntimeError(f"densify_and_prune: {P} rows exceed the supported count (2^30 - 1)")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        totals = torch.empty(4, dtype=torch.int32, device=dev)
        _cabi.check(lib.surfel_densify_plan(
            P, accum.data_ptr(), denom.data_ptr(), scaling.data_ptr(), opacity.data_ptr(), float(max_grad),
            float(min_opacity), float(clone_max), float(prune_max), use_screen,
            float(max_screen_size) if use_screen else 0.0, ws.data_ptr(), nbytes, totals.data_ptr(), stream))
        _, _, n_split, P_new = totals.tolist()    # the one device-to-host copy of the call
        z = draw_split_samples(2 * n_split, dev)
        if z.shape != (2 * n_split, 3) or z.dtype != torch.float32 or not z.is_contiguous() or z.device != dev:
            raise RuntimeError("densify_and_prune: the split samples must be a contiguous (2S, 3) float32 tensor")

        # Two launches: first the group with the most floats per row (f_rest; not one the split arithmetic reads),
        # whose old tensors are released before the other groups' new ones are allocated, then the other five.
        # The call so holds the old model plus one new group at a time, not two whole models (DESIGN.md §7h).
        big = max((i for i, e in enumerate(entries) if e[0]["name"] not in _KIND),
                  key=lambda i: math.prod(entries[i][1].shape[1:]))
        for phase in ([big], [i for i in range(len(entries)) if i != big]):
            _apply(lib, gaussians, entries, phase, P, P_new, n_split, z, ws, nbytes, dev)
        for group in opt.param_groups:            # the state in group order again, as the reference leaves it
            p = group["params"][0]
            if p in opt.state:
                opt.state[p] = opt.state.pop(p)
        gaussians.xyz_gradient_accum = torch.zeros((P_new, 1), device=dev)
        gaussians.denom = torch.zeros((P_new, 1), device=dev)
        gaussians.max_radii2D = torch.zeros((P_new,), device=dev)
