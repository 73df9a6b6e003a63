"""Reads tests/golden/ref_adam.npz (tests/golden/make_golden_adam.py): the reference trainer's optimizer steps,
statistics lines and state surgery, recorded per iteration.

`state_before(d, it)` is the state the reference's optimizer.step() of iteration `it` started from: the state after
iteration it-1 (or the model before, with no optimizer state: zero moments, step 0), put through that iteration's
surgery.  The surgery is restated here as the reference's lines do it: prune_points keeps the rows of the mask in
the parameter and both moments; densification_postfix appends the new rows with zero moments; reset_opacity
replaces the opacity with the recorded reset values and zeroes its moments.  None of them touches the step count.

`Surgery` restates the same three edits on a live torch optimizer (any device), for a free run of the sequence.
"""
import numpy as np
import torch
from torch import nn

from densify_ref import ATTR, GROUPS  # noqa: F401  (re-exported: the group names and model attributes)


def iterations(d):
    return range(1, int(d["iters"]) + 1)


def state_after(d, it, name):
    """(param, exp_avg, exp_avg_sq, step) of group `name` after the step of iteration `it`."""
    pre = f"it{it}_{name}"
    return d[pre], d[pre + "_exp_avg"], d[pre + "_exp_avg_sq"], d[pre + "_step"]


def state_before(d, it):
    """{group: (param, exp_avg, exp_avg_sq, step)} the step of iteration `it` started from."""
    out = {}
    for name in GROUPS:
        if it == 1:
            p = d["in_" + name]
            p, m, v, t = p, np.zeros_like(p), np.zeros_like(p), np.float32(0)
        else:
            p, m, v, t = state_after(d, it - 1, name)
        pre = f"it{it}_"
        if pre + "prune_keep" in d:
            keep = d[pre + "prune_keep"]
            p, m, v = p[keep], m[keep], v[keep]
        if pre + "new_" + name in d:
            new = d[pre + "new_" + name]
            p = np.concatenate([p, new])
            m, v = np.concatenate([m, np.zeros_like(new)]), np.concatenate([v, np.zeros_like(new)])
        if name == "opacity" and pre + "reset_opacity" in d:
            p, m, v = d[pre + "reset_opacity"], np.zeros_like(m), np.zeros_like(v)
        out[name] = (p, m, v, t)
    return out


def stats_before(d, it):
    """(xyz_gradient_accum, denom, max_radii2D) the statistics lines of iteration `it` started from: after the
    previous iteration's statistics lines and surgery (a prune slices them, densification_postfix zeroes them)."""
    if it == 1:
        P = len(d["in_xyz"])
        return np.zeros((P, 1), np.float32), np.zeros((P, 1), np.float32), np.zeros((P,), np.float32)
    pre = f"it{it - 1}_"
    a, n, r = d[pre + "accum"], d[pre + "denom"], d[pre + "max_radii2D"]
    if pre + "prune_keep" in d:
        keep = d[pre + "prune_keep"]
        a, n, r = a[keep], n[keep], r[keep]
    if pre + "new_xyz" in d:
        P = len(a) + len(d[pre + "new_xyz"])
        a, n, r = np.zeros((P, 1), np.float32), np.zeros((P, 1), np.float32), np.zeros((P,), np.float32)
    return a, n, r


class Surgery:
    """The reference's state edits of iteration `it` (if any) on a live optimizer whose groups are named as
    GROUPS, each group holding one parameter; the statistics tensors are edited likewise."""

    def __init__(self, d):
        self.d = d

    @staticmethod
    def _swap(opt, group, new_param, m, v):
        old = group["params"][0]
        st = opt.state.get(old, None)
        new_param = nn.Parameter(new_param.requires_grad_(True))
        group["params"][0] = new_param
        if st is not None:
            del opt.state[old]
            st["exp_avg"], st["exp_avg_sq"] = m, v
            opt.state[new_param] = st
        return new_param

    @torch.no_grad()
    def apply(self, opt, stats, it):
        d, pre = self.d, f"it{it}_"
        for group in opt.param_groups:
            name, p = group["name"], group["params"][0]
            st = opt.state.get(p, None)
            m = st["exp_avg"] if st is not None else None
            v = st["exp_avg_sq"] if st is not None else None
            dev = p.device
            if pre + "prune_keep" in d:
                keep = torch.from_numpy(d[pre + "prune_keep"]).to(dev)
                p = self._swap(opt, group, p.detach()[keep], *((m[keep], v[keep]) if st is not None else (None, None)))
                m, v = (m[keep], v[keep]) if st is not None else (None, None)
            if pre + "new_" + name in d:
                new = torch.from_numpy(d[pre + "new_" + name]).to(dev)
                z = torch.zeros_like(new)
                m2, v2 = (torch.cat((m, z)), torch.cat((v, z))) if st is not None else (None, None)
                p = self._swap(opt, group, torch.cat((p.detach(), new)), m2, v2)
                m, v = m2, v2
            if name == "opacity" and pre + "reset_opacity" in d:
                reset = torch.from_numpy(d[pre + "reset_opacity"]).to(dev)
                p = self._swap(opt, group, reset.clone(), torch.zeros_like(reset), torch.zeros_like(reset))
        a, n, r = stats
        if pre + "prune_keep" in d:
            keep = torch.from_numpy(d[pre + "prune_keep"]).to(a.device)
            a, n, r = a[keep], n[keep], r[keep]
        if pre + "new_xyz" in d:
            P = opt.param_groups[0]["params"][0].shape[0]
            a, n, r = (torch.zeros((P, 1), device=a.device), torch.zeros((P, 1), device=a.device),
                       torch.zeros((P,), device=a.device))
        return a, n, r
