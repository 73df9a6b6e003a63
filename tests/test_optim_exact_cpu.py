"""The float64 Adam bound of tests/adam_exact.py, checked without a GPU: it accepts every correct float32 evaluation
(a float32 emulation of csrc/optim.cu with and without each contraction, torch's CPU Adam, and every step the
reference trainer took in tests/golden/ref_adam.npz), and it rejects each planted mistake on some element."""
import os

import numpy as np
import pytest
import torch

import adam_exact as AX

F = np.float32
STEPS = (1, 2, 10, 1000, 30000)
LR = 2.5e-3
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_adam.npz")


def torch_adam(p, g, m, v, lr, t, foreach):
    q = torch.nn.Parameter(torch.from_numpy(p.copy()))
    opt = torch.optim.Adam([q], lr=lr, betas=AX.BETAS, eps=AX.EPS, foreach=foreach)
    opt.state[q] = {"step": torch.tensor(float(t - 1)), "exp_avg": torch.from_numpy(m.copy()),
                    "exp_avg_sq": torch.from_numpy(v.copy())}
    q.grad = torch.from_numpy(g.copy())
    opt.step()
    st = opt.state[q]
    assert float(st["step"]) == t
    return q.detach().numpy(), st["exp_avg"].numpy(), st["exp_avg_sq"].numpy()


def assert_within(got, p, g, m, v, lr, t, what, limit=1.0):
    exact, bounds = AX.adam64(p, g, m, v, lr, t)
    for name, a, b, e in zip("pmv", got, exact, bounds):
        r = AX.ratio(a, b, e)
        assert np.all(np.isfinite(b)), (what, name)
        worst = int(np.argmax(r))
        assert r[worst] <= limit, (f"{what}: {name} off by {r[worst]:.3g} x bound at element {worst} "
                                   f"(p {p[worst]!r} g {g[worst]!r} m {m[worst]!r} v {v[worst]!r}, t {t})")
    assert not AX.bitwise_rules(p, g, m, v, lr, *got), what


@pytest.mark.parametrize("t", STEPS)
@pytest.mark.parametrize("contract", [(), ("m",), ("v_beta2",), ("v_grad",), ("p",), ("m", "v_beta2", "p")])
def test_bound_accepts_kernel_emulation(t, contract):
    p, g, m, v = AX.inputs()
    assert_within(AX.emulate(p, g, m, v, LR, t, contract=contract), p, g, m, v, LR, t, f"emulation {contract}")


@pytest.mark.parametrize("t", STEPS)
@pytest.mark.parametrize("foreach", [False, True])
def test_bound_accepts_torch_cpu_adam(t, foreach):
    p, g, m, v = AX.inputs(seed=1)
    assert_within(torch_adam(p, g, m, v, LR, t, foreach), p, g, m, v, LR, t, f"torch foreach={foreach}")


def test_bitwise_rules_hold_at_lr_zero():
    p, g, m, v = AX.inputs(seed=2)
    for t in STEPS:
        got = AX.emulate(p, g, m, v, 0.0, t)
        assert not AX.bitwise_rules(p, g, m, v, 0.0, *got)
        assert_within(got, p, g, m, v, 0.0, t, "lr = 0")


# ---- planted mistakes: each must be rejected on at least one element at some t ---------------------------------

def _mistake(kind, p, g, m, v, lr, t):
    b1, b2 = AX.BETAS
    p, g, m, v = (a.astype(np.float64) for a in (p, g, m, v))
    tb = t - 1 if kind == "bias_t_minus_1" else t
    with np.errstate(all="ignore"):
        bc1, bc2 = 1 - np.float64(b1) ** tb, 1 - np.float64(b2) ** tb      # numpy: 1/0 at t - 1 = 0 is inf
        bc = np.sqrt(bc2) if kind != "bias2_not_sqrt" else bc2
        if kind == "bias2_float32":
            bc = float(np.sqrt(F(1) - F(b2) ** F(t)))
        if kind == "betas_swapped":
            b1, b2 = b2, b1
        w1 = b1 if kind == "lerp_weight_beta1" else 1 - b1
        m1 = m + w1 * (g - m)
        v1 = b2 * v + (1 - b2) * g * g
        den = np.sqrt(v1 / bc ** 2 + AX.EPS) if kind == "eps_in_sqrt" else np.sqrt(v1) / bc + AX.EPS
        p1 = p - lr / bc1 * m1 / den
    if kind == "m_not_written":
        m1 = m
    if kind == "v_not_written":
        v1 = v
    return p1, m1, v1


MISTAKES = ("bias_t_minus_1", "bias2_not_sqrt", "eps_in_sqrt", "lerp_weight_beta1", "betas_swapped", "bias2_float32",
            "m_not_written", "v_not_written")


@pytest.mark.parametrize("kind", MISTAKES)
def test_bound_rejects_planted_mistake(kind):
    p, g, m, v = AX.inputs(seed=3)
    rejected = 0
    for t in STEPS:
        got = _mistake(kind, p, g, m, v, LR, t)
        exact, bounds = AX.adam64(p, g, m, v, LR, t)
        # NaN / inf from a mistake (t - 1 = 0) count as rejections: the comparison fails on them too
        r = np.concatenate([np.where(np.isfinite(a), AX.ratio(a, b, e), np.inf) for a, b, e in zip(got, exact, bounds)])
        rejected += int((r > 1).sum())
    assert rejected > 0, kind


def test_bias2_in_float32_is_far_outside_the_bound_at_t1():
    """1 - beta2 formed in float32 is off by about 1.3e-5 relative (6.4e-6 after the square root): several bounds on
    every p the step moves by about lr."""
    p, g, m, v = AX.inputs(seed=4)
    got = _mistake("bias2_float32", p, g, m, v, LR, 1)
    exact, bounds = AX.adam64(p, g, m, v, LR, 1)
    assert np.nanmax(AX.ratio(got[0], exact[0], bounds[0])) > 5


# ---- densification statistics -----------------------------------------------------------------------------------

def test_stats_bound_accepts_float32_and_keeps_culled_rows():
    rng = np.random.default_rng(5)
    P = 4099
    radii = rng.integers(-3, 40, P).astype(np.int32)
    grad = (rng.normal(size=(P, 3)) * 10.0 ** rng.uniform(-30, 3, (P, 1))).astype(F)
    grad[(radii <= 0) & (rng.uniform(size=P) < 0.3)] = np.array([np.nan, np.inf, -np.inf], F)
    accum = np.where(rng.uniform(size=P) < 0.5, 1e4, rng.uniform(0, 1, P)).astype(F)[:, None]
    denom = rng.integers(0, 9, (P, 1)).astype(F)
    maxr = rng.uniform(0, 50, P).astype(F)
    a1, e_a, d1, m1 = AX.stats64(accum, denom, maxr, grad, radii)
    vis = radii > 0
    # torch.norm and a plain float32 sum of squares, as the reference lines and the kernel compute them
    for n in (torch.norm(torch.from_numpy(grad[vis]), dim=-1).numpy(),
              np.sqrt((grad[vis, 0] * grad[vis, 0] + grad[vis, 1] * grad[vis, 1]) + grad[vis, 2] * grad[vis, 2])):
        got = accum[:, 0].copy()
        got[vis] += n
        assert AX.ratio(got, a1, e_a).max() <= 1
    assert np.array_equal(a1[~vis], accum[~vis, 0].astype(np.float64)) and np.all(e_a[~vis] == 0)
    assert np.array_equal(d1[vis], denom[vis, 0] + 1) and np.array_equal(d1[~vis], denom[~vis, 0])
    # a norm that skips one component, or a squared norm, is rejected
    got = accum[:, 0].copy()
    got[vis] += np.sqrt(grad[vis, 0] ** 2 + grad[vis, 1] ** 2)
    assert AX.ratio(got, a1, e_a).max() > 1
    got = accum[:, 0].copy()
    got[vis] += grad[vis, 0] ** 2 + grad[vis, 1] ** 2 + grad[vis, 2] ** 2
    assert AX.ratio(got, a1, e_a).max() > 1


# ---- the reference trainer's own optimizer calls (tests/golden/ref_adam.npz) -------------------------------------

def test_golden_every_step_within_bound_of_recorded_state():
    import adam_golden as AG
    d = np.load(GOLDEN)
    worst = {"p": 0.0, "m": 0.0, "v": 0.0, "accum": 0.0}
    for it in AG.iterations(d):
        before = AG.state_before(d, it)
        for name in AG.GROUPS:
            p, m, v, t = before[name]
            g, lr = d[f"it{it}_grad_{name}"], float(d[f"it{it}_lr_{name}"])
            after = AG.state_after(d, it, name)
            assert float(after[3]) == t + 1, (it, name)           # the step counter runs through all surgery
            exact, bounds = AX.adam64(p, g, m, v, lr, t + 1)
            for q, a, b, e in zip("pmv", after[:3], exact, bounds):
                worst[q] = max(worst[q], float(AX.ratio(a, b, e).max(initial=0)))
            assert not AX.bitwise_rules(p, g, m, v, lr, *after[:3])
        a1, e_a, d1, m1 = AX.stats64(*AG.stats_before(d, it), d[f"it{it}_vgrad"], d[f"it{it}_radii"])
        worst["accum"] = max(worst["accum"], float(AX.ratio(d[f"it{it}_accum"].reshape(-1), a1, e_a).max(initial=0)))
        assert np.array_equal(d[f"it{it}_denom"].reshape(-1), d1)
        assert np.array_equal(d[f"it{it}_max_radii2D"].reshape(-1), m1)
    assert max(worst.values()) <= 1, worst
