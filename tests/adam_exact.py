"""Float64 evaluation of the Adam step and of the densification statistics, with a first-order bound on what a
float32 evaluation can change (csrc/optim.cu, torch.optim.Adam in any of its implementations).

The reference is torch's published Adam in the configuration the reference trainer builds (betas 0.9 / 0.999,
eps 1e-15, no weight decay, no amsgrad), evaluated in float64 on the float32 inputs of one step: p, g, m, v, the
step count t and the group's lr.  The scalars come from t in double, as torch and the fused wrapper form them:
step_size = lr / (1 - beta1^t), bias2_sqrt = sqrt(1 - beta2^t).

    m' = m + (1 - beta1) (g - m)                 (also beta1 m + (1 - beta1) g: the same value)
    v' = beta2 v + (1 - beta2) g^2
    p' = p - step_size * m' / (sqrt(v') / bias2_sqrt + eps)

The bound (`adam64`) follows tsdf_ref.evaluate64 and preprocess_exact: each rounded float32 operation adds
U |result| + ETA (ETA covers the subnormal range), each error is carried through the later operations, and the
rounding of 1-beta1, beta1, beta2, 1-beta2, eps, step_size and bias2_sqrt to float32 is included, because the ABI
(and torch's kernels) carry them as floats.  It is written for any order of evaluation, with or without FMA: the
lerp or the two-product form of m', a division or a multiply by the reciprocal of bias2_sqrt, (step_size * m') /
den or step_size * (m' / den).  The error of m' is bounded in absolute terms, so cancellation in m + w1 (g - m) is
covered.  Square roots use |sqrt(a) - sqrt(b)| <= min(|a - b| / sqrt(b), sqrt(|a - b|)), which holds at v' = 0.

`emulate` is a numpy float32 restatement of optim.cu's adam_one, op for op, uncontracted or with any of the
contractions nvcc may make.
"""
import math

import numpy as np

F = np.float32
U = 2.0 ** -24          # unit roundoff of float32
ETA = 2.0 ** -150       # half the smallest float32 subnormal: the absolute rounding error in the subnormal range

BETAS, EPS = (0.9, 0.999), 1e-15   # the reference trainer's optimizer (torch.optim.Adam(l, lr=0.0, eps=1e-15))


def scalars(lr, t, beta1=BETAS[0], beta2=BETAS[1]):
    """(step_size, bias2_sqrt) in double, as FusedAdam.step and torch's single-tensor Adam form them from t."""
    t = float(t)            # a numpy float32 step count would make beta ** t a float32
    return lr / (1.0 - beta1 ** t), math.sqrt(1.0 - beta2 ** t)


def adam64(p, g, m, v, lr, t, beta1=BETAS[0], beta2=BETAS[1], eps=EPS):
    """One Adam step in float64 on float32 inputs.  Returns ((p', m', v'), (e_p, e_m, e_v)): the exact values and
    per-element bounds on the absolute error of any float32 evaluation."""
    p, g, m, v = (np.asarray(a, F).astype(np.float64) for a in (p, g, m, v))
    ss, bc = scalars(lr, t, beta1, beta2)
    w1, w2 = 1.0 - beta1, 1.0 - beta2
    with np.errstate(all="ignore"):
        m1 = m + w1 * (g - m)
        # lerp: g - m, * w1 (w1 rounded), + m; two-product form: beta1 m and w1 g (each constant rounded), +
        e_m = U * (3.0 * (np.abs(m) + np.abs(g)) + np.abs(m1)) + 3 * ETA
        v1 = beta2 * v + w2 * (g * g)
        # beta2 v: constant + product; w2 g g: constant + two products; the sum (no cancellation: both terms >= 0)
        e_v = U * (2 * beta2 * np.abs(v) + 3 * w2 * g * g + v1) + ETA * (3 + np.abs(g))
        s = np.sqrt(v1)
        e_s = np.where(s > 0, np.minimum(e_v / np.where(s > 0, s, 1.0), np.sqrt(e_v)), np.sqrt(e_v)) + U * s + ETA
        q = s / bc
        e_q = e_s / bc + 3 * U * q + ETA            # bias2_sqrt rounded, its reciprocal, the product
        den = q + eps
        e_den = e_q + U * eps + U * den + ETA      # eps rounded, the sum
        r = m1 / den
        upd = ss * r
        den_lo = den - e_den
        e_upd = (ss * (e_m + np.abs(r) * e_den) / den_lo + 3 * U * np.abs(upd)
                 + ETA * (1 + ss + 1.0 / den_lo))     # step_size rounded; two rounded products / quotients
        p1 = p - upd
        e_p = e_upd + U * np.abs(p1) + ETA
    return (p1, m1, v1), (e_p, e_m, e_v)


def fma32(a, b, c):
    """float32 fma(a, b, c): the product of two floats is exact in double; one rounding of the sum to float
    (through double: a double rounding, which can differ from a true fma only at exact float32 ties)."""
    return (np.asarray(a, F).astype(np.float64) * np.asarray(b, F).astype(np.float64)
            + np.asarray(c, F).astype(np.float64)).astype(F)


CONTRACTIONS = ("m", "v_beta2", "v_grad", "p")   # each fma nvcc may form from adam_one's expressions


def emulate(p, g, m, v, lr, t, beta1=BETAS[0], beta2=BETAS[1], eps=EPS, contract=()):
    """optim.cu's adam_one in numpy float32, with the constants formed as surfel_adam_step and FusedAdam.step form
    them.  `contract` names the contractions to apply (CONTRACTIONS)."""
    p, g, m, v = (np.asarray(a, F).copy() for a in (p, g, m, v))
    ss, bc = scalars(lr, t, beta1, beta2)
    w1, w2, b2, ep, ssf, bcf = F(1.0 - beta1), F(1.0 - beta2), F(beta2), F(eps), F(ss), F(bc)
    with np.errstate(all="ignore"):
        d = g - m
        m = fma32(w1, d, m) if "m" in contract else m + w1 * d
        wg = w2 * g
        if "v_beta2" in contract:
            v = fma32(v, b2, wg * g)
        elif "v_grad" in contract:
            v = fma32(wg, g, v * b2)
        else:
            v = v * b2 + wg * g
        den = np.sqrt(v) / bcf + ep
        r = m / den
        p = fma32(-ssf, r, p) if "p" in contract else p - ssf * r
    return p, m, v


def inputs(n=4096, seed=0):
    """p, g, m, v float32: gradients log-uniform over 1e-30..1e4 with both signs, exact +-0, moments of every
    magnitude down to subnormal and zero, idle elements (g = +-0, m = v = +0)."""
    rng = np.random.default_rng(seed)
    sign = lambda k: np.where(rng.uniform(size=k) < 0.5, -1.0, 1.0)
    g = sign(n) * 10.0 ** rng.uniform(-30, 4, n)
    m = sign(n) * 10.0 ** rng.uniform(-42, 3, n)
    v = 10.0 ** rng.uniform(-44, 8, n)
    p = rng.normal(size=n)
    g[:16], g[16:32] = 0.0, -0.0
    m[:24], v[:24] = 0.0, 0.0                       # idle: g = +-0, m = v = +0
    m[32:40], v[32:40] = 1e-44, 1e-45               # subnormal moments
    g[40:48] = 1e-20 * sign(8)                      # g^2 below the float32 range
    m[48:56] = g[48:56]                             # g - m = 0: the lerp cancels exactly
    p[56:60] = 0.0
    return tuple(a.astype(F) for a in (p, g, m, v))


def ratio(got, want, bound):
    """Per-element |got - want| / bound (0 where both are equal, inf where they differ by more than nothing
    against a zero bound)."""
    got, want, bound = (np.asarray(a, np.float64) for a in (got, want, bound))
    diff = np.abs(got - want)
    with np.errstate(all="ignore"):
        return np.where(diff == 0, 0.0, diff / bound)


def worst(state_got, exact, bounds):
    """Worst ratio of (p, m, v) got against the float64 values and their bounds: a tuple of three floats."""
    return tuple(float(ratio(a, b, e).max(initial=0.0)) for a, b, e in zip(state_got, exact, bounds))


def bitwise_rules(p, g, m, v, lr, p_new, m_new, v_new):
    """The rules checked exactly, not within the bound: an element with g = +-0 and m = v = +0 keeps p, m and v
    bit-unchanged; with lr = 0, every non-zero p keeps its bits (a zero p may come out with the other sign, in
    torch as here: p - 0 * r).  Returns the names of the rules broken."""
    bits = lambda a: np.asarray(a, F).view(np.uint32)
    g, m, v = (np.asarray(a, F) for a in (g, m, v))
    idle = (g == 0) & (bits(m) == 0) & (bits(v) == 0)
    broken = []
    for name, old, new in (("p", p, p_new), ("m", m, m_new), ("v", v, v_new)):
        if not np.array_equal(bits(old)[idle], bits(new)[idle]):
            broken.append(f"idle element changed {name}")
    if lr == 0:
        nz = np.asarray(p, F) != 0
        if not np.array_equal(bits(p)[nz], bits(p_new)[nz]):
            broken.append("lr = 0 changed p")
    return broken


def stats64(accum, denom, max_radii, grad, radii):
    """densification_stats in float64: where radii > 0, accum += |grad|_2, denom += 1, max_radii = max(max_radii,
    radii).  Returns (accum', bound, denom', max_radii'); denom' and max_radii' are float32 and must match bit for
    bit, and rows with radii <= 0 keep every bit of their statistics (accum' = accum there, with a zero bound)."""
    a = np.asarray(accum, F).reshape(-1).astype(np.float64)
    gg = np.asarray(grad, F).astype(np.float64)
    vis = np.asarray(radii) > 0
    with np.errstate(all="ignore"):
        sq = np.where(vis, (gg * gg).sum(1), 0.0)
        n = np.sqrt(sq)
        e_sq = 3 * U * sq + 5 * ETA                  # three rounded squares, two rounded sums, any order
        e_n = np.where(n > 0, np.minimum(e_sq / np.where(n > 0, n, 1.0), np.sqrt(e_sq)), np.sqrt(e_sq)) + U * n + ETA
        a1 = np.where(vis, a + n, a)
        e_a = np.where(vis, e_n + U * np.abs(a1) + ETA, 0.0)
    d = np.asarray(denom, F).reshape(-1).copy()
    d[vis] += F(1)
    mr = None
    if max_radii is not None:
        mr = np.asarray(max_radii, F).reshape(-1).copy()
        mr[vis] = np.maximum(mr[vis], np.asarray(radii)[vis].astype(F))
    return a1, e_a, d, mr
