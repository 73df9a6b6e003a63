"""Device-agnostic torch restatement of the densification rules of DESIGN.md §7h (the reference trainer's
GaussianModel.densify_and_prune, scene/gaussian_model.py:348-403), and the model scenes the densification tests use.

`densify_and_prune(model, max_grad, min_opacity, extent, max_screen_size, draw=...)` edits `model` and its optimizer
in place as the reference does, but states the result directly: every row's fate is decided first from the source
row alone, and the output is one gather in the order  kept originals | kept clones | kept split copies A | kept split
copies B.  Each float operation is the torch operation the reference uses for it, so on a given device the values
are the reference's bit for bit (on CUDA, `tensor / 1.6` is a multiply by the float reciprocal, on the CPU a
division: the restatement inherits whichever the device does).
"""
import types

import numpy as np
import torch
from torch import nn

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
        "scaling": "_scaling", "rotation": "_rotation"}


def draw_normal(n, device):
    return torch.empty((n, 3), dtype=torch.float32, device=device).normal_()


def rotation_matrices(q):
    """R(q) of the raw quaternion (w, x, y, z) after dividing by its norm, entry by entry as
    utils/general_utils.py:78-99 evaluates it (each product and sum rounded on its own)."""
    n = torch.sqrt(q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3])
    u = q / n[:, None]
    w, x, y, z = u[:, 0], u[:, 1], u[:, 2], u[:, 3]
    rows = [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
            [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
            [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]
    return torch.stack([torch.stack(r, dim=-1) for r in rows], dim=-2)


def decide(model, max_grad, min_opacity, extent, max_screen_size):
    """Per-row decisions of rules 1-3 and 7-8: (clone, split, keep_original, keep_clone, keep_split) as bool (P,)
    tensors, and the new raw scaling of every split row's copies (rows in split order)."""
    g = model.xyz_gradient_accum / model.denom
    g = torch.where(torch.isnan(g), torch.zeros_like(g), g)
    s = torch.exp(model._scaling)
    smax = s.max(dim=1).values
    clone_max = model.percent_dense * extent           # a Python double; torch rounds it to float32 to compare
    clone = (torch.norm(g, dim=-1) >= max_grad) & (smax <= clone_max)
    split = (g[:, 0] >= max_grad) & (smax > clone_max)
    split_scaling = torch.log(s[split] / (0.8 * 2))
    low = (torch.sigmoid(model._opacity) < min_opacity)[:, 0]
    big, big_split = torch.zeros_like(low), torch.zeros(int(split.sum()), dtype=torch.bool, device=low.device)
    if max_screen_size:
        # max_radii2D is all zeros by the time the reference tests it against max_screen_size (rule 8)
        vs = torch.zeros_like(model.max_radii2D) > max_screen_size
        big = vs | (smax > 0.1 * extent)
        big_split = vs[split] | (torch.exp(split_scaling).max(dim=1).values > 0.1 * extent)
    keep_original = ~split & ~(low | big)
    keep_clone = clone & keep_original
    keep_split = ~(low[split] | big_split)
    return clone, split, keep_original, keep_clone, keep_split, split_scaling


@torch.no_grad()
def densify_and_prune(model, max_grad, min_opacity, extent, max_screen_size, draw=draw_normal):
    opt = model.optimizer
    dev = model._xyz.device
    clone, split, keep_original, keep_clone, keep_split, split_scaling = decide(
        model, max_grad, min_opacity, extent, max_screen_size)
    S = int(split.sum())
    z = draw(2 * S, dev)                                   # drawn for every split row, pruned or not (rule 10)
    src = torch.nonzero(split)[:, 0]
    std = torch.cat([torch.exp(model._scaling)[src], torch.zeros((S, 1), device=dev)], dim=1).repeat(2, 1)
    samples = z * std + torch.zeros_like(std)              # torch.normal(mean=0, std): normal_(0,1) * std + mean
    offset = torch.bmm(rotation_matrices(model._rotation[src]).repeat(2, 1, 1), samples[:, :, None])[:, :, 0]
    split_values = {"xyz": offset + model._xyz[src].repeat(2, 1), "scaling": split_scaling.repeat(2, 1)}

    orig_rows = torch.nonzero(keep_original)[:, 0]
    clone_rows = torch.nonzero(keep_clone)[:, 0]
    split_keep = keep_split.repeat(2)                      # copies A then B of the split rows, in split order
    for group in opt.param_groups:
        name = group["name"]
        p = group["params"][0]
        reps = (2,) + (1,) * (p.dim() - 1)
        split_part = split_values[name] if name in split_values else p[src].repeat(*reps)
        new_p = torch.cat([p[orig_rows], p[clone_rows], split_part[split_keep]], dim=0)
        param = nn.Parameter(new_p.requires_grad_(True))
        st = opt.state.get(p, None)
        if st is not None:
            n_new = len(clone_rows) + int(split_keep.sum())
            for key in ("exp_avg", "exp_avg_sq"):
                m = st[key]
                st[key] = torch.cat([m[orig_rows], torch.zeros((n_new,) + tuple(m.shape[1:]), device=dev)], dim=0)
            del opt.state[p]
            opt.state[param] = st
        group["params"][0] = param
        setattr(model, ATTR[name], param)
    P_new = model._xyz.shape[0]
    model.xyz_gradient_accum = torch.zeros((P_new, 1), device=dev)
    model.denom = torch.zeros((P_new, 1), device=dev)
    model.max_radii2D = torch.zeros((P_new,), device=dev)


# ---- model scenes -----------------------------------------------------------------------------------------------

LRS = {"xyz": 0.00016, "f_dc": 0.0025, "f_rest": 0.0025 / 20.0, "opacity": 0.05, "scaling": 0.005, "rotation": 0.001}


def make_model(params, accum, denom, max_radii2D, percent_dense=0.01, optimizer=torch.optim.Adam, adam_steps=3,
               stateless=(), seed=0):
    """A model object with the reference GaussianModel's attributes from host arrays (name -> array) on the
    arrays' target device, its optimizer built as training_setup builds it and stepped `adam_steps` times with
    seeded gradients; groups named in `stateless` are left without optimizer state."""
    dev = params["xyz"].device
    m = types.SimpleNamespace()
    for name in GROUPS:
        setattr(m, ATTR[name], nn.Parameter(params[name].clone().requires_grad_(True)))
    groups = [{"params": [getattr(m, ATTR[n])], "lr": LRS[n], "name": n} for n in GROUPS]
    m.optimizer = optimizer(groups, lr=0.0, eps=1e-15)
    gen = torch.Generator(device="cpu").manual_seed(seed)
    for _ in range(adam_steps):
        for n in GROUPS:
            p = getattr(m, ATTR[n])
            p.grad = None if n in stateless else (torch.randn(p.shape, generator=gen) * 1e-3).to(dev)
        m.optimizer.step()
    for n in GROUPS:
        getattr(m, ATTR[n]).grad = None
    m.xyz_gradient_accum, m.denom, m.max_radii2D = accum.clone(), denom.clone(), max_radii2D.clone()
    m.percent_dense = percent_dense
    return m


def scene_arrays(P, seed, sh_rest=15, extent=4.0, max_grad=0.0002, split_frac=None, clone_frac=None, none=False,
                 rest_active=None):
    """Host arrays of a scene whose rows cover every class and prune criterion.  Scales are spread across the clone
    bound (percent_dense * extent), the split copies' prune bound and the world-size bound; opacities across
    min_opacity; gradients across max_grad, with 0/0 rows, x/0 rows and rows exactly at max_grad.  `none` makes
    every gradient zero (nothing selected); split_frac / clone_frac, if given, set the fractions of rows that are
    split / cloned (the rest get gradients below max_grad) and put 3 % of the rows below min_opacity.
    rest_active = k keeps only the first k SH rest coefficients non-zero, as while the trainer's active SH degree
    is low."""
    rng = np.random.default_rng(seed)
    f32 = np.float32
    xyz = rng.uniform(-2, 2, (P, 3)).astype(f32)
    scale = np.exp(rng.uniform(np.log(0.005), np.log(1.0), (P, 2))).astype(f32)
    scaling = np.log(scale).astype(f32)
    rotation = rng.normal(size=(P, 4)).astype(f32)
    u = rng.uniform(0.001, 0.99, (P, 1))
    opacity = np.log(u / (1 - u)).astype(f32)
    f_dc = (rng.normal(size=(P, 1, 3)) * 0.5).astype(f32)
    f_rest = (rng.normal(size=(P, sh_rest, 3)) * 0.1).astype(f32)
    if rest_active is not None:
        f_rest[:, rest_active:] = 0.0
    denom = rng.integers(0, 50, (P, 1)).astype(f32)
    g = np.exp(rng.uniform(np.log(2e-5), np.log(2e-3), (P, 1)))
    accum = (g * denom).astype(f32)
    if P >= 40:
        accum[:5], denom[:5] = 0.0, 0.0                   # 0/0 -> NaN -> 0
        accum[5:7], denom[5:7] = 1e-3, 0.0                # x/0 -> inf
        accum[7:17], denom[7:17] = f32(max_grad), 1.0     # exactly max_grad
        scaling[7:12] = np.log(0.01)                      # ... cloned
        scaling[12:17] = np.log(0.3)                      # ... split
        accum[17:26], denom[17:26] = 1e-3, 1.0
        scaling[17:20], opacity[17:20] = np.log(0.01), -7.0   # cloned, clone and source below min_opacity
        scaling[20:23], opacity[20:23] = np.log(0.3), -7.0    # split, both copies below min_opacity
        scaling[23:26] = np.log(0.8)                          # split, copies above 0.1 * extent
    if split_frac is not None:
        r = rng.uniform(size=P)
        is_split, is_clone = r < split_frac, (r >= split_frac) & (r < split_frac + clone_frac)
        scaling[:] = rng.uniform(np.log(0.002), np.log(0.35), (P, 2))
        smax = np.exp(scaling).max(1)
        bound = f32(0.01 * extent)
        scaling[is_split & (smax <= bound * 1.5)] = np.log(0.2)
        scaling[is_clone & (smax > bound / 1.5)] = np.log(0.02)
        denom[:] = 1.0
        accum[:, 0] = np.where(is_split | is_clone, 1e-3, 1e-5)
        opacity[:, 0] = np.where(rng.uniform(size=P) < 0.03, -7.0, rng.uniform(-4, 4, P))
    if none:
        accum[:] = 0.0
    max_radii2D = rng.uniform(0, 40, P).astype(f32)
    params = {"xyz": xyz, "f_dc": f_dc, "f_rest": f_rest, "opacity": opacity, "scaling": scaling, "rotation": rotation}
    return params, accum, denom, max_radii2D


COPIED = ("f_dc", "f_rest", "opacity", "rotation")   # groups whose rows after are always copies of rows before


def golden_after(d, tag):
    """The state after call `tag` of tests/golden/ref_densify.npz, decoded (tests/golden/make_golden_densify.py):
    the arrays `<tag>_<name>`, `..._exp_avg`, `..._exp_avg_sq`, `..._step`, `<tag>_accum`, `denom`, `max_radii2D`."""
    src, kept = d[tag + "_src"], d[tag + "_moments_kept"]
    n = len(src)
    out = {}
    for name in GROUPS:
        out[f"{tag}_{name}"] = d[f"in_{name}"][src] if name in COPIED else d[f"{tag}_{name}"]
        for k in ("exp_avg", "exp_avg_sq"):
            m = d[f"in_{name}_{k}"][src]
            m[~kept] = 0.0
            out[f"{tag}_{name}_{k}"] = m
        out[f"{tag}_{name}_step"] = d[f"{tag}_{name}_step"]
    out[tag + "_accum"] = np.zeros((n, 1), np.float32)
    out[tag + "_denom"] = np.zeros((n, 1), np.float32)
    out[tag + "_max_radii2D"] = np.zeros((n,), np.float32)
    return out


def model_from_state(d, prefix, device, optimizer=torch.optim.Adam, percent_dense=0.01):
    """A model object holding a stored state (tests/golden/ref_densify.npz): `<prefix><name>`, `..._exp_avg`,
    `..._exp_avg_sq`, `..._step` per group, `<prefix>accum`, `denom` and `max_radii2D`."""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    m = types.SimpleNamespace()
    for name in GROUPS:
        setattr(m, ATTR[name], nn.Parameter(t(d[prefix + name]).requires_grad_(True)))
    groups = [{"params": [getattr(m, ATTR[n])], "lr": LRS[n], "name": n} for n in GROUPS]
    m.optimizer = optimizer(groups, lr=0.0, eps=1e-15)
    for name in GROUPS:
        m.optimizer.state[getattr(m, ATTR[name])] = {
            "step": torch.tensor(float(d[prefix + name + "_step"]), dtype=torch.float32),
            "exp_avg": t(d[prefix + name + "_exp_avg"]), "exp_avg_sq": t(d[prefix + name + "_exp_avg_sq"])}
    m.xyz_gradient_accum, m.denom, m.max_radii2D = t(d[prefix + "accum"]), t(d[prefix + "denom"]), t(d[prefix + "max_radii2D"])
    m.percent_dense = percent_dense
    return m


def build(arrays, device, **kw):
    params, accum, denom, radii = arrays
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return make_model({k: t(v) for k, v in params.items()}, t(accum), t(denom), t(radii), **kw)


def snapshot(model):
    """Everything densify_and_prune leaves behind, as host tensors: per group (name, param, requires_grad, grad is
    None, state keys, exp_avg, exp_avg_sq, step) and the statistics."""
    out = {"groups": []}
    for group in model.optimizer.param_groups:
        p = group["params"][0]
        assert p is getattr(model, ATTR[group["name"]])
        st = model.optimizer.state.get(p, None)
        out["groups"].append({
            "name": group["name"], "param": p.detach().cpu(), "requires_grad": p.requires_grad, "grad_none": p.grad is None,
            "is_parameter": isinstance(p, nn.Parameter),
            "keys": None if st is None else sorted(st.keys()),
            "exp_avg": None if st is None else st["exp_avg"].cpu(),
            "exp_avg_sq": None if st is None else st["exp_avg_sq"].cpu(),
            "step": None if st is None else float(st["step"])})
    out["accum"], out["denom"], out["max_radii2D"] = (model.xyz_gradient_accum.cpu(), model.denom.cpu(),
                                                      model.max_radii2D.cpu())
    return out
