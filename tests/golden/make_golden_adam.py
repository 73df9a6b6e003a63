"""Pins FusedAdam and densification_stats to THE REFERENCE TRAINER'S OWN optimizer calls: GaussianModel.training_setup
(torch.optim.Adam with betas 0.9 / 0.999, eps 1e-15), update_learning_rate's xyz schedule, the statistics lines of
train.py (max_radii2D, add_densification_stats), optimizer.step / zero_grad, and the state surgery of prune_points,
densification_postfix and reset_opacity, which keep each group's step count (reset_opacity zeroes the moments but
keeps the step, so the next update applies late-step bias correction to fresh moments).

The reference runs unmodified on the CPU (make_golden.py's cpu_patches / stub_modules) on a seeded model of P0 rows
(tests/densify_ref.py:scene_arrays, SH degree 3 with the rest coefficients of degree 1 active).  Each of ITERS
iterations does, in train.py's order: update_learning_rate(it); the statistics lines with seeded radii (negative,
zero and positive; NaN / inf view-space gradients on some culled rows); the surgery of that iteration, if any;
seeded gradients (exact zeros on some rows, values near 1e-20 on others), optimizer.step() and zero_grad.

Writes tests/golden/ref_adam.npz (tests/adam_golden.py reads it): the model before (in_*), and per iteration
`it<k>_`: radii, vgrad, the statistics after the statistics lines (accum, denom, max_radii2D), the surgery
(prune_keep, new_<group>, reset_opacity), per group the lr and gradient of the step and the state after it
(<group>, _exp_avg, _exp_avg_sq, _step).  The script checks that adam_golden's decoding of the file reproduces
every state the reference left, bit for bit, before it writes the file.

Usage:  python tests/golden/make_golden_adam.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "2d-gaussian-splatting_b200"))
REF = "/root/reference"

P0, SEED, EXTENT, ITERS = 64, 11, 3.7, 8
PRUNE_AT, POSTFIX_AT, RESET_AT, N_NEW = 3, 5, 6, 9
GRAD_SCALE = {"xyz": 1e-4, "f_dc": 1e-3, "f_rest": 1e-4, "opacity": 1e-2, "scaling": 1e-3, "rotation": 1e-3}


def seeded_grad(gen, shape, scale, name):
    g = torch.randn(shape, generator=gen) * scale
    rows = torch.rand(shape[0], generator=gen)
    g[rows < 0.1] = 0.0                                    # exact zeros (idle rows: moments stay zero)
    g[(rows >= 0.1) & (rows < 0.15)] *= 1e-16 / scale      # near 1e-20: g^2 underflows float32
    if name == "f_rest":
        g[:, 3:] = 0.0                                     # SH degree 1 active
    return g


def main():
    import adam_golden as AG
    import densify_ref as DR
    import make_golden as MG
    from torch import nn
    MG.cpu_patches()
    MG.stub_modules({})
    sys.path.insert(0, REF)
    from scene.gaussian_model import GaussianModel

    params, _, _, _ = DR.scene_arrays(P0, SEED, extent=EXTENT, rest_active=3)
    pc = GaussianModel(3)
    for name in DR.GROUPS:
        setattr(pc, DR.ATTR[name], nn.Parameter(torch.from_numpy(params[name].copy()).requires_grad_(True)))
    pc.max_radii2D = torch.zeros(P0)
    pc.spatial_lr_scale = EXTENT
    pc.training_setup(types.SimpleNamespace(
        percent_dense=0.01, position_lr_init=0.00016, position_lr_final=0.0000016, position_lr_delay_mult=0.01,
        position_lr_max_steps=30_000, feature_lr=0.0025, opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001))
    out = {f"in_{n}": params[n].copy() for n in DR.GROUPS}
    out["iters"] = np.int32(ITERS)
    gen = torch.Generator().manual_seed(SEED)
    states, pre_states, pre_stats = {}, {}, {}
    for it in range(1, ITERS + 1):
        pre = f"it{it}_"
        pre_stats[it] = tuple(t.numpy().copy() for t in (pc.xyz_gradient_accum, pc.denom, pc.max_radii2D))
        pc.update_learning_rate(it)
        P = pc._xyz.shape[0]
        radii = torch.randint(-3, 40, (P,), generator=gen, dtype=torch.int32)
        vgrad = torch.randn((P, 3), generator=gen) * 10.0 ** torch.randint(-8, 0, (P, 1), generator=gen).float()
        culled = torch.nonzero(radii <= 0)[:, 0]
        vgrad[culled[:3]] = torch.tensor([float("nan"), float("inf"), -float("inf")])
        visibility_filter = radii > 0
        viewspace_point_tensor = types.SimpleNamespace(grad=vgrad)
        # train.py:126-128, verbatim
        pc.max_radii2D[visibility_filter] = torch.max(pc.max_radii2D[visibility_filter], radii[visibility_filter])
        pc.add_densification_stats(viewspace_point_tensor, visibility_filter)
        out[pre + "radii"], out[pre + "vgrad"] = radii.numpy(), vgrad.numpy()
        out[pre + "accum"], out[pre + "denom"] = pc.xyz_gradient_accum.numpy().copy(), pc.denom.numpy().copy()
        out[pre + "max_radii2D"] = pc.max_radii2D.numpy().copy()
        if it == PRUNE_AT:
            prune = torch.rand(P, generator=gen) < 0.2
            pc.prune_points(prune)
            out[pre + "prune_keep"] = (~prune).numpy()
        if it == POSTFIX_AT:
            src = torch.randint(0, P, (N_NEW,), generator=gen)
            new = {n: getattr(pc, DR.ATTR[n]).detach()[src] + 0.01 * torch.randn(
                getattr(pc, DR.ATTR[n])[src].shape, generator=gen) for n in DR.GROUPS}
            new["f_rest"][:, 3:] = 0.0
            pc.densification_postfix(*(new[n] for n in DR.GROUPS))
            for n in DR.GROUPS:
                out[pre + "new_" + n] = new[n].numpy()
        if it == RESET_AT:
            pc.reset_opacity()
            out[pre + "reset_opacity"] = pc._opacity.detach().numpy().copy()
        for group in pc.optimizer.param_groups:
            name = group["name"]
            p = group["params"][0]
            p.grad = seeded_grad(gen, p.shape, GRAD_SCALE[name], name)
            out[pre + "lr_" + name] = np.float64(group["lr"])
            out[pre + "grad_" + name] = p.grad.numpy().copy()
            st = pc.optimizer.state.get(p, None)
            pre_states[(it, name)] = (p.detach().numpy().copy(),
                                      st["exp_avg"].numpy().copy() if st else np.zeros(p.shape, np.float32),
                                      st["exp_avg_sq"].numpy().copy() if st else np.zeros(p.shape, np.float32),
                                      np.float32(float(st["step"])) if st else np.float32(0))
        pc.optimizer.step()
        pc.optimizer.zero_grad(set_to_none=True)
        for group in pc.optimizer.param_groups:
            name = group["name"]
            p = group["params"][0]
            assert p is getattr(pc, DR.ATTR[name])
            st = pc.optimizer.state[p]
            assert sorted(st) == ["exp_avg", "exp_avg_sq", "step"] and st["step"].dtype == torch.float32
            states[(it, name)] = (p.detach().numpy().copy(), st["exp_avg"].numpy().copy(),
                                  st["exp_avg_sq"].numpy().copy(), np.float32(float(st["step"])))
            for k, a in zip(("", "_exp_avg", "_exp_avg_sq", "_step"), states[(it, name)]):
                out[pre + name + k] = a
        print(f"it {it}: P {P} -> {pc._xyz.shape[0]}, xyz lr {pc.optimizer.param_groups[0]['lr']:.6g}")
    # the decoding the tests use gives back every state the reference left, bit for bit
    raw = lambda a: np.ascontiguousarray(a).reshape(-1).view(np.uint8)
    for it in range(1, ITERS + 1):
        for name in DR.GROUPS:
            got = AG.state_after(out, it, name)
            for a, b in zip(got, states[(it, name)]):
                assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(raw(a), raw(b)), (it, name)
        before = AG.state_before(out, it)
        for name in DR.GROUPS:
            for a, b in zip(before[name], pre_states[(it, name)]):
                assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(raw(a), raw(b)), (it, name)
        for a, b in zip(AG.stats_before(out, it), pre_stats[it]):
            assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(raw(a), raw(b)), it
    np.savez_compressed(os.path.join(HERE, "ref_adam.npz"), **out)
    print("wrote ref_adam.npz")


if __name__ == "__main__":
    main()
