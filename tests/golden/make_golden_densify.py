"""Pins diff_surfel_rasterization.densify to THE REFERENCE'S OWN GaussianModel.densify_and_prune
(scene/gaussian_model.py:348-403 of the reference trainer, called at train.py:132).

The reference runs unmodified on the CPU (make_golden.py's cpu_patches / stub_modules).  Its model is built by its
own training_setup (the optimizer of gaussian_model.py:148-166) from a seeded scene of 800 rows with the SH
layout of degree 3 (tests/densify_ref.py:scene_arrays: every class, every prune criterion, 0/0 and x/0
gradients, gradients exactly at max_grad, max_radii2D above 20), then given three steps of real Adam with seeded
gradients (multiples of 2^-12, which keeps the file small; the SH rest coefficients get gradients on degree 1
only, as early in training).  torch.normal is stubbed to draw its standard normal samples from a seeded
generator and record them; the values it returns are what torch.normal(mean, std) computes from them
(normal_(0, 1), then * std + mean).

Two calls from the same state: max_screen_size = 20 and None.  Writes tests/golden/ref_densify.npz: the state
before (in_*), and per call the draw (<tag>_z) and the state after, with max_grad, min_opacity, extent and
percent_dense.  Most of the state after is rows of the state before, so it is stored losslessly as: the xyz and
scaling after (<tag>_xyz, <tag>_scaling, every row); for every row after, the row before that its other
parameters are a bit-for-bit copy of (<tag>_src); whether its moments are that row's or zero
(<tag>_moments_kept); and each group's step.  The script checks that this reproduces what the reference left,
bit for bit, before it writes the file; tests/densify_ref.py:golden_after decodes it.

Usage:  python tests/golden/make_golden_densify.py
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

P, SEED = 800, 7
MAX_GRAD, MIN_OPACITY, EXTENT, PERCENT_DENSE = 0.0002, 0.005, 3.7, 0.01
GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
        "scaling": "_scaling", "rotation": "_rotation"}


def build_model(GaussianModel, arrays):
    from torch import nn
    params, accum, denom, radii = arrays
    pc = GaussianModel(3)
    for name in GROUPS:
        setattr(pc, ATTR[name], nn.Parameter(torch.from_numpy(params[name].copy()).requires_grad_(True)))
    pc.spatial_lr_scale = EXTENT
    pc.training_setup(types.SimpleNamespace(
        percent_dense=PERCENT_DENSE, position_lr_init=0.00016, position_lr_final=0.0000016, position_lr_delay_mult=0.01,
        position_lr_max_steps=30_000, feature_lr=0.0025, opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001))
    gen = torch.Generator().manual_seed(SEED)
    for _ in range(3):
        for name in GROUPS:
            p = getattr(pc, ATTR[name])
            g = torch.round(torch.randn(p.shape, generator=gen) * 4) * 2.0 ** -12
            if name == "f_rest":
                g[:, 3:] = 0.0
            p.grad = g
        pc.optimizer.step()
    pc.optimizer.zero_grad(set_to_none=True)
    pc.xyz_gradient_accum = torch.from_numpy(accum.copy())
    pc.denom = torch.from_numpy(denom.copy())
    pc.max_radii2D = torch.from_numpy(radii.copy())
    return pc


def dump(pc, prefix, out):
    for group in pc.optimizer.param_groups:
        name = group["name"]
        p = group["params"][0]
        assert p is getattr(pc, ATTR[name])
        st = pc.optimizer.state[p]
        out[prefix + name] = p.detach().numpy().copy()
        out[prefix + name + "_exp_avg"] = st["exp_avg"].numpy().copy()
        out[prefix + name + "_exp_avg_sq"] = st["exp_avg_sq"].numpy().copy()
        out[prefix + name + "_step"] = np.float32(float(st["step"]))
    out[prefix + "accum"] = pc.xyz_gradient_accum.numpy().copy()
    out[prefix + "denom"] = pc.denom.numpy().copy()
    out[prefix + "max_radii2D"] = pc.max_radii2D.numpy().copy()


def encode(out, after, tag, DR):
    """Store the state after (`after`, as dump() writes it) in the form the module docstring describes, and check
    that decoding it gives back every array bit for bit."""
    key = lambda prefix, d, i: b"".join(d[prefix + n][i].tobytes() for n in DR.COPIED)
    before = {key("in_", out, i): i for i in range(len(out["in_xyz"]))}
    assert len(before) == len(out["in_xyz"]), "rows before are not distinguishable"
    n = len(after[tag + "_xyz"])
    src = np.array([before[key(tag + "_", after, r)] for r in range(n)], dtype=np.int32)
    kept = np.array([all(np.array_equal(after[f"{tag}_{g}_{k}"][r], out[f"in_{g}_{k}"][s])
                         for g in DR.GROUPS for k in ("exp_avg", "exp_avg_sq")) for r, s in enumerate(src)], dtype=bool)
    out[tag + "_src"], out[tag + "_moments_kept"] = src, kept
    out[tag + "_xyz"], out[tag + "_scaling"] = after[tag + "_xyz"], after[tag + "_scaling"]
    for g in DR.GROUPS:
        out[f"{tag}_{g}_step"] = after[f"{tag}_{g}_step"]
    decoded = DR.golden_after(out, tag)
    assert sorted(decoded) == sorted(after)
    raw = lambda a: np.ascontiguousarray(a).reshape(-1).view(np.uint8)
    for k, v in after.items():
        assert np.shape(decoded[k]) == np.shape(v) and decoded[k].dtype == v.dtype, k
        assert np.array_equal(raw(decoded[k]), raw(v)), k


def main():
    import densify_ref as DR
    import make_golden as MG
    MG.cpu_patches()
    MG.stub_modules({})
    sys.path.insert(0, REF)
    from scene.gaussian_model import GaussianModel

    arrays = DR.scene_arrays(P, SEED, extent=EXTENT, rest_active=3)
    out = {"max_grad": np.float64(MAX_GRAD), "min_opacity": np.float64(MIN_OPACITY), "extent": np.float64(EXTENT),
           "percent_dense": np.float64(PERCENT_DENSE)}
    orig_normal = torch.normal
    for tag, mss in (("screen20", 20), ("screen_none", None)):
        pc = build_model(GaussianModel, arrays)
        if tag == "screen20":
            dump(pc, "in_", out)
        gen = torch.Generator().manual_seed(SEED + 1)
        drawn = []

        def normal(mean, std, *a, _gen=gen, _drawn=drawn, **k):
            z = torch.empty(mean.shape).normal_(generator=_gen)
            _drawn.append(z.clone())
            return z * std + mean
        torch.normal = normal
        pc.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, mss)
        torch.normal = orig_normal
        assert len(drawn) == 1
        out[tag + "_z"] = drawn[0].numpy()
        after = {}
        dump(pc, tag + "_", after)
        encode(out, after, tag, DR)
        print(f"{tag}: P {P} -> {pc._xyz.shape[0]}, {drawn[0].shape[0] // 2} split rows")
    np.savez_compressed(os.path.join(HERE, "ref_densify.npz"), **out)
    print("wrote ref_densify.npz")


if __name__ == "__main__":
    main()
