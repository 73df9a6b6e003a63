"""FusedAdam (csrc/optim.cu) and densification_stats held to the float64 evaluation of tests/adam_exact.py: every
element of every step lies within the bound evaluated on the GPU's own previous state, with no budget.  Covered: the
reference trainer's recorded steps (tests/golden/ref_adam.npz) one by one and as a free run with the surgery
restated, the kernel's float4 lane, 1024-element blocks and 1-3-element tails, misaligned views (scalar path),
zero-size groups, more than SURFEL_ADAM_MAX_GROUPS tensors, several params per group and grad=None, two betas/eps
buckets, lr changes and lr = 0, late steps, non-contiguous gradients and a side stream.  torch.optim.Adam on CUDA
(foreach) must pass the same bound, which checks the bound itself.  Mismatched states are refused before
anything is launched."""
import os

import numpy as np
import pytest
import torch
from torch import nn

import adam_exact as AX

gpu = pytest.mark.gpu
F = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_adam.npz")
WORST = {"p": 0.0, "m": 0.0, "v": 0.0, "accum": 0.0}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nworst |error| / bound:", {k: round(v, 4) for k, v in WORST.items()})


def host(t):
    return t.detach().cpu().numpy().reshape(-1).copy()


def check(before, after, lr, t, what, betas=AX.BETAS, eps=AX.EPS, record=True):
    """before = (p, g, m, v), after = (p', m', v') host arrays: within the bound, and the bitwise rules hold.
    `record` adds the worst ratios to those the module reports for FusedAdam."""
    p, g, m, v = before
    exact, bounds = AX.adam64(p, g, m, v, lr, t, betas[0], betas[1], eps)
    for q, a, b, e in zip("pmv", after, exact, bounds):
        r = AX.ratio(a, b, e)
        if r.size:
            i = int(np.argmax(r))
            if record:
                WORST[q] = max(WORST[q], float(r[i]))
            assert r[i] <= 1, (f"{what}: {q} off by {r[i]:.3g} x bound at {i} (p {p[i]!r} g {g[i]!r} m {m[i]!r} "
                                   f"v {v[i]!r} t {t} lr {lr})")
    assert not AX.bitwise_rules(p, g, m, v, lr, *after), what


def adam_case(n, t, seed, dev="cuda"):
    """A parameter of n elements with gradient and state at step t - 1 (moments from AX.inputs)."""
    reps = -(-max(n, 1) // 4096)
    arrs = [np.tile(a, reps)[:n] for a in AX.inputs(4096, seed)]
    p, g, m, v = (torch.from_numpy(a.copy()).to(dev) for a in arrs)
    return p, g, m, v, tuple(arrs)


def fused_step(specs, lr=2.5e-3, t=7, betas=AX.BETAS, eps=AX.EPS):
    """One FusedAdam step over parameters given as (n, seed) in one group each; checks every element."""
    from diff_surfel_rasterization.optim import FusedAdam
    params, cases = [], []
    for n, seed in specs:
        p, g, m, v, arrs = adam_case(n, t, seed)
        q = nn.Parameter(p)
        q.grad = g
        params.append((q, m, v))
        cases.append(arrs)
    opt = FusedAdam([{"params": [q], "lr": lr} for q, _, _ in params], lr=lr, betas=betas, eps=eps)
    for q, m, v in params:
        opt.state[q] = {"step": torch.tensor(float(t - 1)), "exp_avg": m, "exp_avg_sq": v}
    opt.step()
    torch.cuda.synchronize()
    for (q, m, v), arrs, (n, _) in zip(params, cases, specs):
        assert float(opt.state[q]["step"]) == t
        check(arrs, (host(q), host(m), host(v)), lr, t, f"n={n}", betas, eps)


# ---- the reference trainer's steps ---------------------------------------------------------------------------------

@gpu
def test_golden_each_recorded_step():
    """From each state the reference's step started from, one FusedAdam step: within 1x the bound of float64 and
    within 2x of the reference's own result."""
    import adam_golden as AG
    from diff_surfel_rasterization.optim import FusedAdam
    d = np.load(GOLDEN)
    dev = torch.device("cuda")
    for it in AG.iterations(d):
        before = AG.state_before(d, it)
        params = {n: nn.Parameter(torch.from_numpy(before[n][0].copy()).to(dev)) for n in AG.GROUPS}
        opt = FusedAdam([{"params": [params[n]], "lr": float(d[f"it{it}_lr_{n}"]), "name": n} for n in AG.GROUPS],
                        lr=0.0, eps=1e-15)
        for n in AG.GROUPS:
            p, m, v, t = before[n]
            if t > 0:
                opt.state[params[n]] = {"step": torch.tensor(float(t)), "exp_avg": torch.from_numpy(m.copy()).to(dev),
                                        "exp_avg_sq": torch.from_numpy(v.copy()).to(dev)}
            params[n].grad = torch.from_numpy(d[f"it{it}_grad_{n}"]).to(dev)
        opt.step()
        for n in AG.GROUPS:
            p, m, v, t = before[n]
            st = opt.state[params[n]]
            got = (host(params[n]), host(st["exp_avg"]), host(st["exp_avg_sq"]))
            lr = float(d[f"it{it}_lr_{n}"])
            ins = (p.reshape(-1), d[f"it{it}_grad_{n}"].reshape(-1), m.reshape(-1), v.reshape(-1))
            check(ins, got, lr, float(t) + 1, f"it {it} {n}")
            ref = AG.state_after(d, it, n)
            assert float(st["step"]) == float(ref[3]) and st["step"].dtype == torch.float32
            assert sorted(st) == ["exp_avg", "exp_avg_sq", "step"]
            _, bounds = AX.adam64(*ins, lr, float(t) + 1)
            for a, b, e in zip(got, ref[:3], bounds):
                assert np.all(np.abs(a.astype(np.float64) - b.reshape(-1)) <= 2 * e), (it, n)


@gpu
def test_golden_free_run():
    """The recorded sequence run freely on the device: recorded lr, radii, gradients and surgery, each step checked
    against the bound on the GPU's own previous state, the statistics likewise."""
    import adam_golden as AG
    from diff_surfel_rasterization.optim import FusedAdam, densification_stats
    d = np.load(GOLDEN)
    dev = torch.device("cuda")
    params = {n: nn.Parameter(torch.from_numpy(d["in_" + n].copy()).to(dev)) for n in AG.GROUPS}
    opt = FusedAdam([{"params": [params[n]], "lr": float(d[f"it1_lr_{n}"]), "name": n} for n in AG.GROUPS],
                    lr=0.0, eps=1e-15)
    P = len(d["in_xyz"])
    stats = (torch.zeros((P, 1), device=dev), torch.zeros((P, 1), device=dev), torch.zeros((P,), device=dev))
    surgery = AG.Surgery(d)
    for it in AG.iterations(d):
        for group in opt.param_groups:                       # update_learning_rate: only the xyz lr moves
            group["lr"] = float(d[f"it{it}_lr_{group['name']}"])
        a0, n0, r0 = (host(s) for s in stats)
        radii = torch.from_numpy(d[f"it{it}_radii"]).to(dev)
        vgrad = torch.from_numpy(d[f"it{it}_vgrad"]).to(dev)
        densification_stats(*stats, vgrad, radii)
        a1, e_a, dn1, mr1 = AX.stats64(a0, n0, r0, d[f"it{it}_vgrad"], d[f"it{it}_radii"])
        assert AX.ratio(host(stats[0]), a1, e_a).max() <= 1
        assert np.array_equal(host(stats[1]), dn1) and np.array_equal(host(stats[2]), mr1)
        stats = surgery.apply(opt, stats, it)
        before = {}
        for group in opt.param_groups:
            n, q = group["name"], group["params"][0]
            q.grad = torch.from_numpy(d[f"it{it}_grad_{n}"]).to(dev)
            st = opt.state.get(q, None)
            t = float(st["step"]) if st else 0.0
            zero = np.zeros(q.numel(), F)
            before[n] = ((host(q), host(q.grad), host(st["exp_avg"]) if st else zero,
                          host(st["exp_avg_sq"]) if st else zero), t)
        opt.step()
        opt.zero_grad(set_to_none=True)
        for group in opt.param_groups:
            n, q = group["name"], group["params"][0]
            st = opt.state[q]
            ins, t = before[n]
            check(ins, (host(q), host(st["exp_avg"]), host(st["exp_avg_sq"])), group["lr"], t + 1, f"free it {it} {n}")
            ref = AG.state_after(d, it, n)
            assert float(st["step"]) == float(ref[3]) and tuple(q.shape) == ref[0].shape


@gpu
def test_golden_densification_stats():
    import adam_golden as AG
    from diff_surfel_rasterization.optim import densification_stats
    d = np.load(GOLDEN)
    for it in AG.iterations(d):
        a0, n0, r0 = AG.stats_before(d, it)
        stats = [torch.from_numpy(x.copy()).cuda() for x in (a0, n0, r0)]
        densification_stats(*stats, torch.from_numpy(d[f"it{it}_vgrad"]).cuda(), torch.from_numpy(d[f"it{it}_radii"]).cuda())
        a1, e_a, dn1, mr1 = AX.stats64(a0, n0, r0, d[f"it{it}_vgrad"], d[f"it{it}_radii"])
        r = AX.ratio(host(stats[0]), a1, e_a)
        WORST["accum"] = max(WORST["accum"], float(r.max()))
        assert r.max() <= 1
        assert AX.ratio(d[f"it{it}_accum"].reshape(-1), a1, e_a).max() <= 1
        assert np.array_equal(host(stats[1]), dn1) and np.array_equal(host(stats[1]), d[f"it{it}_denom"].reshape(-1))
        assert np.array_equal(host(stats[2]), mr1) and np.array_equal(host(stats[2]), d[f"it{it}_max_radii2D"])


# ---- kernel paths ---------------------------------------------------------------------------------------------------

SIZES = (0, 1, 2, 3, 4, 5, 1023, 1024, 1025, 1027, 4097, 59 * 100_003)


@gpu
@pytest.mark.parametrize("t", [1, 2, 10, 1000, 30000])
def test_group_sizes(t):
    """Float4 lanes, 1024-element blocks and 1-3-element tails; 12 groups, so the table is split into two launches,
    with zero-size groups first."""
    fused_step([(n, i) for i, n in enumerate(SIZES)], t=t)


@gpu
@pytest.mark.parametrize("order", ["first", "middle", "last"])
def test_zero_size_groups(order):
    sizes = {"first": (0, 0, 1025, 7), "middle": (1025, 0, 0, 7), "last": (1025, 7, 0, 0)}[order]
    fused_step([(n, i + 20) for i, n in enumerate(sizes)])


@gpu
@pytest.mark.parametrize("count", [8, 9, 16, 17])
def test_tensor_counts(count):
    fused_step([(1000 + 37 * i, 40 + i) for i in range(count)])


@gpu
@pytest.mark.parametrize("which", ["param", "grad", "exp_avg", "exp_avg_sq"])
@pytest.mark.parametrize("offset", [1, 2, 3])
def test_misaligned_views(which, offset):
    """One array 4, 8 or 12 bytes off 16-byte alignment (a view into a larger buffer, whose guard words must keep
    their bits), next to an aligned group in the same launch."""
    from diff_surfel_rasterization.optim import FusedAdam
    n, t, lr = 1031, 5, 2.5e-3
    p, g, m, v, arrs = adam_case(n, t, 60 + offset)
    arrays = {"param": p, "grad": g, "exp_avg": m, "exp_avg_sq": v}
    buf = torch.full((n + 8,), float("nan"), device="cuda")
    buf.view(torch.int32)[:] = 0x7fc0dead
    buf[offset:offset + n] = arrays[which]
    arrays[which] = buf[offset:offset + n]
    assert arrays[which].data_ptr() % 16 == 4 * offset
    q = nn.Parameter(arrays["param"])
    q.grad = arrays["grad"]
    p2, g2, m2, v2, arrs2 = adam_case(2048, t, 70)
    q2 = nn.Parameter(p2)
    q2.grad = g2
    opt = FusedAdam([{"params": [q], "lr": lr}, {"params": [q2], "lr": lr}], lr=lr, eps=AX.EPS)
    opt.state[q] = {"step": torch.tensor(float(t - 1)), "exp_avg": arrays["exp_avg"], "exp_avg_sq": arrays["exp_avg_sq"]}
    opt.state[q2] = {"step": torch.tensor(float(t - 1)), "exp_avg": m2, "exp_avg_sq": v2}
    opt.step()
    torch.cuda.synchronize()
    if which == "param":
        assert q.data_ptr() == arrays["param"].data_ptr()
    check(arrs, (host(q), host(arrays["exp_avg"]), host(arrays["exp_avg_sq"])), lr, t, f"{which}+{offset}")
    check(arrs2, (host(q2), host(m2), host(v2)), lr, t, "aligned neighbour")
    guards = buf.view(torch.int32).cpu().numpy()
    assert np.all(guards[:offset] == 0x7fc0dead) and np.all(guards[offset + n:] == 0x7fc0dead)


@gpu
def test_several_params_per_group_and_grad_none():
    """A group of four params, two without a gradient: their state (one stored, one never created) is untouched."""
    from diff_surfel_rasterization.optim import FusedAdam
    t, lr = 3, 1e-2
    cases = [adam_case(n, t, 80 + i) for i, n in enumerate((1000, 513, 9, 4100))]
    qs = [nn.Parameter(c[0]) for c in cases]
    opt = FusedAdam([{"params": qs, "lr": lr}], lr=lr, eps=AX.EPS)
    for i, (q, c) in enumerate(zip(qs, cases)):
        if i != 3:
            opt.state[q] = {"step": torch.tensor(float(t - 1)), "exp_avg": c[2], "exp_avg_sq": c[3]}
        q.grad = c[1] if i in (0, 2) else None
    opt.step()
    torch.cuda.synchronize()
    for i in (0, 2):
        check(cases[i][4], (host(qs[i]), host(cases[i][2]), host(cases[i][3])), lr, t, f"param {i}")
    st = opt.state[qs[1]]
    assert float(st["step"]) == t - 1
    for a, b in zip((host(qs[1]), host(st["exp_avg"]), host(st["exp_avg_sq"])), (cases[1][4][0], cases[1][4][2], cases[1][4][3])):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert len(opt.state.get(qs[3], {})) == 0 and np.array_equal(host(qs[3]), cases[3][4][0])


@gpu
def test_two_betas_eps_buckets():
    from diff_surfel_rasterization.optim import FusedAdam
    t, lr = 4, 2.5e-3
    a, b = adam_case(3000, t, 90), adam_case(2001, t, 91)
    qa, qb = nn.Parameter(a[0]), nn.Parameter(b[0])
    qa.grad, qb.grad = a[1], b[1]
    opt = FusedAdam([{"params": [qa], "lr": lr}, {"params": [qb], "lr": lr, "betas": (0.8, 0.99), "eps": 1e-8}],
                    lr=lr, eps=AX.EPS)
    for q, c in ((qa, a), (qb, b)):
        opt.state[q] = {"step": torch.tensor(float(t - 1)), "exp_avg": c[2], "exp_avg_sq": c[3]}
    opt.step()
    torch.cuda.synchronize()
    check(a[4], (host(qa), host(a[2]), host(a[3])), lr, t, "bucket 1")
    check(b[4], (host(qb), host(b[2]), host(b[3])), lr, t, "bucket 2", betas=(0.8, 0.99), eps=1e-8)


@gpu
def test_lr_change_lr_zero_and_late_steps():
    """Three steps from a state loaded at step 29 999: one group's lr changes after the first, one group has lr = 0
    (its non-zero params keep their bits)."""
    from diff_surfel_rasterization.optim import FusedAdam
    t0 = 29_999
    a, b = adam_case(5000, t0 + 1, 100), adam_case(1500, t0 + 1, 101)
    qa, qb = nn.Parameter(a[0]), nn.Parameter(b[0])
    opt = FusedAdam([{"params": [qa], "lr": 1.6e-4}, {"params": [qb], "lr": 0.0}], lr=0.0, eps=AX.EPS)
    for q, c in ((qa, a), (qb, b)):
        opt.state[q] = {"step": torch.tensor(float(t0)), "exp_avg": c[2], "exp_avg_sq": c[3]}
    gen = torch.Generator().manual_seed(5)
    for k in range(3):
        if k == 1:
            opt.param_groups[0]["lr"] = 3.1e-5
        before = []
        for q, c in ((qa, a), (qb, b)):
            q.grad = (torch.randn(q.shape, generator=gen) * 10.0 ** -k).cuda()
            before.append((host(q), host(q.grad), host(c[2]), host(c[3])))
        opt.step()
        torch.cuda.synchronize()
        for (q, c), ins, grp in zip(((qa, a), (qb, b)), before, opt.param_groups):
            check(ins, (host(q), host(c[2]), host(c[3])), grp["lr"], t0 + 1 + k, f"step {k}")
            assert float(opt.state[q]["step"]) == t0 + 1 + k


@gpu
def test_non_contiguous_grad():
    from diff_surfel_rasterization.optim import FusedAdam
    t, lr = 6, 5e-2
    p, g, m, v, arrs = adam_case(3 * 1001, t, 110)
    q = nn.Parameter(p.reshape(1001, 3))
    wide = torch.zeros((1001, 6), device="cuda")
    wide[:, ::2] = g.reshape(1001, 3)
    q.grad = wide[:, ::2]
    assert not q.grad.is_contiguous()
    opt = FusedAdam([{"params": [q], "lr": lr}], lr=lr, eps=AX.EPS)
    opt.state[q] = {"step": torch.tensor(float(t - 1)), "exp_avg": m.reshape(1001, 3), "exp_avg_sq": v.reshape(1001, 3)}
    opt.step()
    torch.cuda.synchronize()
    check(arrs, (host(q), host(m), host(v)), lr, t, "non-contiguous grad")


@gpu
def test_side_stream():
    """The step runs on the caller's current stream: gradients written on a side stream behind a delay are the ones
    it reads, with only that stream synchronised."""
    from diff_surfel_rasterization.optim import FusedAdam
    t, lr = 2, 2.5e-3
    p, g, m, v, arrs = adam_case(1 << 20, t, 120)
    q = nn.Parameter(p)
    q.grad = torch.zeros_like(p)
    opt = FusedAdam([{"params": [q], "lr": lr}], lr=lr, eps=AX.EPS)
    opt.state[q] = {"step": torch.tensor(float(t - 1)), "exp_avg": m, "exp_avg_sq": v}
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)
        q.grad.copy_(g)
        opt.step()
    side.synchronize()
    check(arrs, (host(q), host(m), host(v)), lr, t, "side stream")


@gpu
@pytest.mark.parametrize("t", [1, 2, 10, 1000, 30000])
def test_torch_cuda_adam_passes_the_same_bound(t):
    """The bound is a statement about every float32 evaluation of the published formula: torch's CUDA foreach Adam
    must pass it.  (torch's fused=True kernel is not such an evaluation: it forms 1 - beta2^t and 1 - beta2 in
    float32 from a float32 beta2, which is off by about 1.3e-5 relative, and lies up to 11x outside the bound.)"""
    lr = 2.5e-3
    p, g, m, v, arrs = adam_case(4097, t, 130)
    q = nn.Parameter(p)
    q.grad = g
    opt = torch.optim.Adam([q], lr=lr, eps=AX.EPS, foreach=True)
    opt.state[q] = {"step": torch.tensor(float(t - 1)), "exp_avg": m, "exp_avg_sq": v}
    opt.step()
    torch.cuda.synchronize()
    check(arrs, (host(q), host(m), host(v)), lr, t, "torch foreach", record=False)


# ---- densification statistics ---------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("P", [0, 1, 255, 256, 257, 100_003])
@pytest.mark.parametrize("with_max", [True, False])
def test_densification_stats_exact(P, with_max):
    from diff_surfel_rasterization.optim import densification_stats
    rng = np.random.default_rng(P + 7)
    radii = rng.integers(-3, 40, P).astype(np.int32)
    grad = (rng.normal(size=(P, 3)) * 10.0 ** rng.integers(-30, 3, (P, 1))).astype(F)
    culled = np.nonzero(radii <= 0)[0]
    grad[culled[::2]] = np.array([np.nan, np.inf, -np.inf], F)
    accum = np.where(rng.uniform(size=P) < 0.5, F(1e4), rng.uniform(0, 1, P)).astype(F)[:, None]
    denom = rng.integers(0, 9, (P, 1)).astype(F)
    maxr = rng.uniform(0, 50, P).astype(F)
    ts = [torch.from_numpy(x.copy()).cuda() for x in (accum, denom, maxr)]
    densification_stats(ts[0], ts[1], ts[2] if with_max else None, torch.from_numpy(grad).cuda(),
                        torch.from_numpy(radii).cuda())
    a1, e_a, d1, m1 = AX.stats64(accum, denom, maxr, grad, radii)
    got = [host(x) for x in ts]
    r = AX.ratio(got[0], a1, e_a)
    WORST["accum"] = max(WORST["accum"], float(r.max(initial=0)))
    assert r.max(initial=0) <= 1
    vis = radii > 0
    assert np.array_equal(got[0][~vis].view(np.uint32), accum[~vis, 0].view(np.uint32))
    assert np.array_equal(got[1], d1)
    assert np.array_equal(got[2], m1 if with_max else maxr)


# ---- rejections: nothing is launched on a mismatched state ---------------------------------------------------------

class _Recorder:
    """Stands in for the native library: any launch fails the test."""

    def __getattr__(self, name):
        def launch(*a, **k):
            pytest.fail(f"{name} was launched on a state it must refuse")
        return launch


@pytest.fixture
def no_launch(monkeypatch):
    from diff_surfel_rasterization import _cabi
    monkeypatch.setattr(_cabi, "load", lambda: _Recorder())


def _opt_with(state_edit=None, group_extra=None, grad=None):
    from diff_surfel_rasterization.optim import FusedAdam
    q = nn.Parameter(torch.ones(12, 3, device="cuda"))
    group = {"params": [q], "lr": 1e-2, **(group_extra or {})}
    opt = FusedAdam([group], lr=1e-2, eps=AX.EPS)
    opt.state[q] = {"step": torch.tensor(4.0), "exp_avg": torch.zeros(12, 3, device="cuda"),
                    "exp_avg_sq": torch.zeros(12, 3, device="cuda")}
    if state_edit:
        state_edit(opt.state[q])
    q.grad = torch.ones(12, 3, device="cuda") if grad is None else grad
    return opt, q


def _assert_refused(opt, q):
    st = opt.state[q]
    snap = [host(q), host(q.grad)] + [host(st[k]) if isinstance(st[k], torch.Tensor) else st[k]
                                      for k in ("exp_avg", "exp_avg_sq")]
    with pytest.raises(RuntimeError):
        opt.step()
    assert float(st["step"]) == 4.0
    after = [host(q), host(q.grad)] + [host(st[k]) for k in ("exp_avg", "exp_avg_sq")]
    assert all(np.array_equal(a, b) for a, b in zip(snap, after))


@gpu
@pytest.mark.parametrize("option", [("weight_decay", 0.01), ("amsgrad", True), ("maximize", True),
                                    ("decoupled_weight_decay", True)])
def test_refuses_unsupported_group_options(no_launch, option):
    _assert_refused(*_opt_with(group_extra=dict([option])))


@gpu
@pytest.mark.parametrize("edit", ["short_exp_avg", "short_exp_avg_sq", "float64_exp_avg", "cpu_exp_avg_sq",
                                  "flat_exp_avg", "strided_exp_avg_sq"])
def test_refuses_mismatched_state(no_launch, edit):
    edits = {
        "short_exp_avg": lambda s: s.update(exp_avg=torch.zeros(11, 3, device="cuda")),
        "short_exp_avg_sq": lambda s: s.update(exp_avg_sq=torch.zeros(11, 3, device="cuda")),
        "float64_exp_avg": lambda s: s.update(exp_avg=torch.zeros(12, 3, device="cuda", dtype=torch.float64)),
        "cpu_exp_avg_sq": lambda s: s.update(exp_avg_sq=torch.zeros(12, 3)),
        "flat_exp_avg": lambda s: s.update(exp_avg=torch.zeros(35, device="cuda")),
        "strided_exp_avg_sq": lambda s: s.update(exp_avg_sq=torch.zeros(12, 6, device="cuda")[:, ::2]),
    }
    _assert_refused(*_opt_with(state_edit=edits[edit]))


@gpu
def test_refuses_short_grad(no_launch):
    opt, q = _opt_with()
    q.grad.data = torch.ones(11, 3, device="cuda")          # a shape the autograd setter would refuse
    _assert_refused(opt, q)


@gpu
def test_refuses_grad_on_another_device(no_launch):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    opt, q = _opt_with()
    q.grad.data = torch.ones(12, 3, device="cuda:1")
    _assert_refused(opt, q)


@gpu
@pytest.mark.parametrize("which", ["accum", "denom", "max_radii2D"])
@pytest.mark.parametrize("bad", ["float64", "short", "strided"])
def test_densification_stats_refuses_bad_statistics(no_launch, which, bad):
    from diff_surfel_rasterization.optim import densification_stats
    P = 100
    good = {"accum": torch.zeros(P, 1, device="cuda"), "denom": torch.zeros(P, 1, device="cuda"),
            "max_radii2D": torch.zeros(P, device="cuda")}
    shape = good[which].shape
    good[which] = {"float64": torch.zeros(shape, device="cuda", dtype=torch.float64),
                   "short": torch.zeros((P - 1,) + tuple(shape[1:]), device="cuda"),
                   "strided": torch.zeros((P, 2), device="cuda")[:, :1].reshape(shape) if len(shape) == 2
                   else torch.zeros(2 * P, device="cuda")[::2]}[bad]
    if bad == "strided":
        assert not good[which].is_contiguous()
    snap = {k: host(v) for k, v in good.items()}
    with pytest.raises(RuntimeError):
        densification_stats(good["accum"], good["denom"], good["max_radii2D"], torch.ones(P, 3, device="cuda"),
                             torch.ones(P, dtype=torch.int32, device="cuda"))
    assert all(np.array_equal(host(good[k]), snap[k]) for k in good)
