"""Opt-in fused parameter update (SURVEY §8(f) row f3).

`FusedAdam` is a drop-in for the optimizer the reference builds in
/root/reference/scene/gaussian_model.py:148-166 (`torch.optim.Adam(l, lr=0.0, eps=1e-15)`) and steps at
/root/reference/train.py:138-140.  It IS a `torch.optim.Adam` (same param_groups, same per-parameter
state keys `step`, `exp_avg`, `exp_avg_sq`, same state_dict), so the reference's densification code that
edits the optimizer state in place (gaussian_model.py:263-345: replace_tensor_to_optimizer,
_prune_optimizer, cat_tensors_to_optimizer) keeps working; only `.step()` is replaced: every parameter
of every group is updated by ONE CUDA launch (csrc/optim.cu) instead of ~12 elementwise passes per group.

`densification_stats(...)` fuses /root/reference/train.py:125-128 and gaussian_model.py:405-407.

No CPU path: parameters must be CUDA float32 tensors.
"""
import ctypes
import math

import torch

from . import _cabi


class FusedAdam(torch.optim.Adam):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=0, amsgrad=False,
                         foreach=False, fused=False, capturable=False, differentiable=False, maximize=False)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = _cabi.load()
        # Every group and tensor is checked before any state is touched or anything is launched: the kernel
        # addresses p.numel() elements of grad, exp_avg and exp_avg_sq, so a mismatched state must never reach it.
        work = []
        for group in self.param_groups:
            for key in _UNSUPPORTED:
                if group.get(key, False):
                    raise RuntimeError(f"FusedAdam: {key}={group[key]!r} is not supported (the fused step is plain "
                                       "Adam: no weight decay, amsgrad or maximize)")
            for p in group["params"]:
                if p.grad is None:
                    continue
                _check_param(p, self.state.get(p))
                work.append((group, p))
        # one launch per (device, betas, eps) bucket: the reference has exactly one
        buckets = {}
        for group, p in work:
            beta1, beta2 = group["betas"]
            lr = float(group["lr"])
            state = self.state[p]
            if len(state) == 0:                             # same lazy state as torch.optim.Adam
                state["step"] = torch.tensor(0.0, dtype=torch.float32)
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            state["step"] += 1
            step = float(state["step"])
            grad = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
            bc1 = 1.0 - beta1 ** step
            bc2 = 1.0 - beta2 ** step
            entry = (p, grad, state["exp_avg"], state["exp_avg_sq"], lr / bc1, math.sqrt(bc2))
            buckets.setdefault((p.device, float(beta1), float(beta2), float(group["eps"])), []).append(entry)
        for (dev, beta1, beta2, eps), entries in buckets.items():
            with torch.cuda.device(dev):
                stream = torch.cuda.current_stream(dev).cuda_stream
                for i in range(0, len(entries), _cabi.ADAM_MAX_GROUPS):
                    chunk = entries[i:i + _cabi.ADAM_MAX_GROUPS]
                    table = (_cabi.AdamGroup * len(chunk))()
                    for g, (p, grad, m, v, step_size, bc2_sqrt) in zip(table, chunk):
                        g.param, g.grad, g.exp_avg, g.exp_avg_sq = p.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr()
                        g.n, g.step_size, g.bias2_sqrt = p.numel(), step_size, bc2_sqrt
                    _cabi.check(lib.surfel_adam_step(len(chunk), table, beta1, beta2, eps, stream))
        return loss


# per-group options torch.optim.Adam accepts that change the update; the kernel implements none of them
_UNSUPPORTED = ("weight_decay", "amsgrad", "maximize", "decoupled_weight_decay")


def _check_param(p, state):
    """Raise unless p, its gradient and its Adam state (if any) are what the kernel addresses: CUDA float32 tensors
    on one device, p and the moments contiguous, gradient and moments of p's shape."""
    grad = p.grad
    if not p.is_cuda or p.dtype != torch.float32:
        raise RuntimeError("FusedAdam: parameters must be CUDA float32 tensors (no CPU path)")
    if grad.is_sparse:
        raise RuntimeError("FusedAdam does not support sparse gradients")
    if grad.dtype != torch.float32 or grad.device != p.device:
        raise RuntimeError(f"FusedAdam: gradient is {grad.dtype} on {grad.device}, parameter float32 on {p.device}")
    if grad.shape != p.shape:
        raise RuntimeError(f"FusedAdam: gradient shape {tuple(grad.shape)} != parameter shape {tuple(p.shape)}")
    if not p.is_contiguous():
        raise RuntimeError("FusedAdam: parameters must be contiguous")
    if not state:
        return
    for key in ("step", "exp_avg", "exp_avg_sq"):
        if key not in state:
            raise RuntimeError(f"FusedAdam: optimizer state has no {key!r}")
    for key in ("exp_avg", "exp_avg_sq"):
        t = state[key]
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.device != p.device:
            raise RuntimeError(f"FusedAdam: state {key!r} must be a float32 tensor on {p.device}")
        if t.shape != p.shape:
            raise RuntimeError(f"FusedAdam: state {key!r} shape {tuple(t.shape)} != parameter shape {tuple(p.shape)}")
        if not t.is_contiguous():
            raise RuntimeError("FusedAdam: optimizer state must be contiguous")


@torch.no_grad()
def densification_stats(xyz_gradient_accum, denom, max_radii2D, viewspace_grad, radii):
    """In place, where radii > 0:  max_radii2D = max(max_radii2D, radii);
    xyz_gradient_accum += |viewspace_grad|;  denom += 1   (train.py:125-128, gaussian_model.py:405-407)."""
    lib = _cabi.load()
    if not (radii.is_cuda and radii.dtype == torch.int32 and radii.dim() == 1 and radii.is_contiguous()):
        raise RuntimeError("densification_stats: radii must be a contiguous CUDA int32 tensor (P,) (no CPU path)")
    P, dev = radii.shape[0], radii.device
    if not (viewspace_grad.device == dev and viewspace_grad.dtype == torch.float32 and viewspace_grad.shape == (P, 3)
            and viewspace_grad.is_contiguous()):
        raise RuntimeError("densification_stats: viewspace_grad must be float32 (P,3) contiguous on radii's device")
    # the kernel addresses P consecutive floats of each statistic
    for name, t in (("xyz_gradient_accum", xyz_gradient_accum), ("denom", denom), ("max_radii2D", max_radii2D)):
        if t is None and name == "max_radii2D":
            continue
        if not (t.device == dev and t.dtype == torch.float32 and t.numel() == P and t.is_contiguous()):
            raise RuntimeError(f"densification_stats: {name} must be a contiguous float32 tensor of {P} elements on "
                               f"{dev}, got {t.dtype} {tuple(t.shape)} on {t.device}")
    with torch.cuda.device(dev):
        _cabi.check(lib.surfel_densify_stats(
            P, radii.data_ptr(), viewspace_grad.data_ptr(), xyz_gradient_accum.data_ptr(), denom.data_ptr(),
            max_radii2D.data_ptr() if max_radii2D is not None else None, torch.cuda.current_stream(dev).cuda_stream))
