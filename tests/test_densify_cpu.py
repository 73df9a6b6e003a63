"""Densification without a GPU: the torch restatement (tests/densify_ref.py) against the reference's own
densify_and_prune (tests/golden/ref_densify.npz), each rule of DESIGN.md §7h on a hand-built model, the Python
entry point's argument checks and the C ABI's."""
import os

import numpy as np
import pytest
import torch
from torch import nn

import densify_ref as DR

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32
GOLDEN = os.path.join(HERE, "golden", "ref_densify.npz")


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("tag,mss", [("screen20", 20), ("screen_none", None)])
def test_restatement_reproduces_reference_bit_for_bit(tag, mss):
    d = np.load(GOLDEN)
    m = DR.model_from_state(d, "in_", "cpu", percent_dense=float(d["percent_dense"]))
    z = torch.from_numpy(d[tag + "_z"])
    DR.densify_and_prune(m, float(d["max_grad"]), float(d["min_opacity"]), float(d["extent"]), mss,
                         draw=lambda n, dev: z if n == len(z) else pytest.fail(f"drew {n} rows, the reference {len(z)}"))
    snap = DR.snapshot(m)
    after = DR.golden_after(d, tag)
    for g in snap["groups"]:
        name = g["name"]
        assert g["is_parameter"] and g["requires_grad"] and g["grad_none"]
        assert same_bits(g["param"].numpy(), after[f"{tag}_{name}"]), name
        assert same_bits(g["exp_avg"].numpy(), after[f"{tag}_{name}_exp_avg"]), name
        assert same_bits(g["exp_avg_sq"].numpy(), after[f"{tag}_{name}_exp_avg_sq"]), name
        assert g["step"] == float(after[f"{tag}_{name}_step"]) == float(d[f"in_{name}_step"]) == 3.0
        assert g["keys"] == ["exp_avg", "exp_avg_sq", "step"]
    for k in ("accum", "denom", "max_radii2D"):
        assert same_bits(snap[k].numpy(), after[f"{tag}_{k}"]), k


def test_golden_covers_every_case():
    """The stored call exercises every class and criterion the rules name."""
    d = np.load(GOLDEN)
    m = DR.model_from_state(d, "in_", "cpu", percent_dense=float(d["percent_dense"]))
    args = float(d["max_grad"]), float(d["min_opacity"]), float(d["extent"])
    clone, split, keep_o, keep_c, keep_s, _ = DR.decide(m, *args, 20)
    g = (m.xyz_gradient_accum / m.denom)[:, 0]
    low = (torch.sigmoid(m._opacity) < args[1])[:, 0]
    assert clone.sum() >= 50 and split.sum() >= 50 and (~clone & ~split).sum() >= 50
    assert (clone & ~keep_c).any() and (split & ~keep_s[torch.cumsum(split.long(), 0) - 1]).any()
    assert (~split & low).any() and (split & low).any()
    smax = torch.exp(m._scaling).max(1).values
    assert (~split & ~low & (smax > 0.1 * args[2])).any()                    # world-size prune of an original
    _, _, _, _, keep_s_none, sc = DR.decide(m, *args, None)
    assert (keep_s_none & ~keep_s).any()                                     # split copies pruned by their new scale
    assert (torch.isnan(g) & (m.denom[:, 0] == 0)).any() and torch.isinf(g).any()
    assert (g == torch.tensor(args[0], dtype=torch.float32)).sum() >= 10
    assert (m.max_radii2D > 20).sum() >= 100


# ---- hand-built cases, one rule each -----------------------------------------------------------------------------

def tiny(rows, percent_dense=0.01, stateless=()):
    """rows: list of dicts with g (accum with denom 1, or a (accum, denom) pair), s (scale pair), o (opacity raw)."""
    P = len(rows)
    f = lambda a: torch.tensor(np.asarray(a, F32))
    params = {"xyz": f([[i, 2 * i, 3 * i] for i in range(P)]).reshape(P, 3),
              "f_dc": f(np.arange(P * 3).reshape(P, 1, 3)), "f_rest": f(np.arange(P * 45).reshape(P, 15, 3) * 0.5),
              "opacity": f([[r.get("o", 2.0)] for r in rows]).reshape(P, 1),
              "scaling": f([np.log(r["s"]) for r in rows]).reshape(P, 2),
              "rotation": f([[1, 0, 0, 0]] * P).reshape(P, 4)}
    acc = [r["g"] if isinstance(r["g"], tuple) else (r["g"], 1.0) for r in rows]
    accum, denom = f([[a] for a, _ in acc]).reshape(P, 1), f([[b] for _, b in acc]).reshape(P, 1)
    return DR.make_model(params, accum, denom, torch.full((P,), 100.0), percent_dense=percent_dense,
                         stateless=stateless)


def run(m, mss=None, max_grad=0.0002, min_opacity=0.005, extent=4.0, z=None):
    drawn = []

    def draw(n, dev):
        out = DR.draw_normal(n, dev) if z is None else z[:n]
        drawn.append(out)
        return out
    before = {n: getattr(m, DR.ATTR[n]).detach().clone() for n in DR.GROUPS}
    DR.densify_and_prune(m, max_grad, min_opacity, extent, mss, draw=draw)
    return before, drawn[0]


def test_rule_1_thresholds_round_once_to_float32():
    # percent_dense * extent = 0.01 * 3.7 in double; a row whose scale is that value rounded to float32 lies above
    # the double: compared in double it would split, compared in float32 (as torch does) it clones
    t = np.float32(0.01 * 3.7)
    assert float(t) > 0.01 * 3.7
    raw = [r for r in (np.float32(np.log(t)) + np.float32(k) * np.spacing(np.float32(np.log(t))) for k in range(-8, 9))
           if torch.exp(torch.tensor(r)).item() == float(t)]
    assert raw, "no float32 whose exp is t"
    m = tiny([{"g": 1e-3, "s": (0.001, 0.001)}, {"g": 1e-3, "s": (0.001, 0.001)}])
    m._scaling.data[:, 0] = float(raw[0])
    clone, split, *_ = DR.decide(m, 0.0002, 0.005, 3.7, None)
    assert clone.tolist() == [True, True] and split.tolist() == [False, False]
    # max_grad = 0.0002 in double lies above its float32 rounding: a gradient of exactly that float32 is selected
    assert float(np.float32(0.0002)) < 0.0002
    m = tiny([{"g": float(np.float32(0.0002)), "s": (0.01, 0.01)}])
    clone, *_ = DR.decide(m, 0.0002, 0.005, 4.0, None)
    assert clone.tolist() == [True]


def test_rule_2_3_gradient_exactly_at_max_grad_and_nan():
    mg = float(np.float32(0.0002))
    below = float(np.nextafter(np.float32(mg), np.float32(0)))
    m = tiny([{"g": mg, "s": (0.01, 0.01)}, {"g": mg, "s": (0.3, 0.01)}, {"g": below, "s": (0.01, 0.01)},
              {"g": below, "s": (0.3, 0.3)}, {"g": (0.0, 0.0), "s": (0.3, 0.3)}, {"g": (1.0, 0.0), "s": (0.3, 0.3)}])
    clone, split, *_ = DR.decide(m, 0.0002, 0.005, 4.0, None)
    assert clone.tolist() == [True, False, False, False, False, False]
    assert split.tolist() == [False, True, False, False, False, True]     # 0/0 -> 0 is not selected, 1/0 = inf is


def test_rule_4_5_6_row_order_values_and_moments():
    m = tiny([{"g": 1e-3, "s": (0.3, 0.2)}, {"g": 0.0, "s": (0.01, 0.01)}, {"g": 1e-3, "s": (0.01, 0.02)},
              {"g": 1e-3, "s": (0.5, 0.1)}, {"g": 1e-3, "s": (0.02, 0.01)}])
    m._rotation.data[3] = torch.tensor([0.5, 0.5, -0.5, 0.5])
    m_before = {n: m.optimizer.state[getattr(m, DR.ATTR[n])]["exp_avg"].clone() for n in DR.GROUPS}
    z = torch.tensor([[0.5, -1.0, 3.0], [1.5, 0.25, -2.0], [-0.5, 2.0, 1.0], [0.75, -0.125, 0.5]])
    before, drawn = run(m, z=z)
    assert drawn.shape == (4, 3)
    # originals 1, 2, 4 | clones of 2, 4 | split A of 0, 3 | split B of 0, 3
    src = [1, 2, 4, 2, 4, 0, 3, 0, 3]
    for n in ("f_dc", "f_rest", "opacity", "rotation"):
        assert torch.equal(getattr(m, DR.ATTR[n]).detach(), before[n][src]), n
    assert torch.equal(m._xyz.detach()[:5], before["xyz"][src[:5]])
    assert torch.equal(m._scaling.detach()[:5], before["scaling"][src[:5]])
    s = torch.exp(before["scaling"][[0, 3, 0, 3]])
    assert torch.equal(m._scaling.detach()[5:], torch.log(s / 1.6))
    R = DR.rotation_matrices(before["rotation"][[0, 3, 0, 3]])
    samples = z * torch.cat([s, torch.zeros(4, 1)], 1) + 0.0
    want = torch.bmm(R, samples[:, :, None])[:, :, 0] + before["xyz"][[0, 3, 0, 3]]
    assert torch.equal(m._xyz.detach()[5:], want)
    assert torch.allclose(R[1] @ R[1].T, torch.eye(3), atol=1e-6)
    for n in DR.GROUPS:
        st = m.optimizer.state[getattr(m, DR.ATTR[n])]
        assert torch.equal(st["exp_avg"][:3], m_before[n][[1, 2, 4]])
        assert not st["exp_avg"][3:].any() and not st["exp_avg_sq"][3:].any()
        assert float(st["step"]) == 3.0


def test_rule_6_group_without_state():
    m = tiny([{"g": 1e-3, "s": (0.3, 0.2)}, {"g": 1e-3, "s": (0.01, 0.01)}], stateless=("f_rest", "opacity"))
    run(m)
    for n in DR.GROUPS:
        p = getattr(m, DR.ATTR[n])
        assert p.shape[0] == 4 and isinstance(p, nn.Parameter) and p.requires_grad and p.grad is None
        assert (p in m.optimizer.state) == (n not in ("f_rest", "opacity"))


def test_rule_7_8_prune_criteria():
    rows = [{"g": 0.0, "s": (0.01, 0.01), "o": -6.0},     # sigmoid < 0.005: pruned
            {"g": 0.0, "s": (0.5, 0.01)},                 # world-size: pruned only with a screen size
            {"g": 1e-3, "s": (0.5, 0.1)},                 # split; copies 0.3125 <= 0.4 survive
            {"g": 1e-3, "s": (0.7, 0.1)},                 # split; copies 0.4375 > 0.4 pruned with a screen size
            {"g": 1e-3, "s": (0.01, 0.01), "o": -6.0},    # clone of a pruned row: pruned with it
            {"g": 0.0, "s": (0.01, 0.01)}]                # max_radii2D = 100 > 20 but kept (rule 8)
    m = tiny(rows)
    before, _ = run(m, mss=20)
    assert torch.equal(m._opacity.detach()[:1], before["opacity"][[5]])
    assert m._xyz.shape[0] == 1 + 2
    m = tiny(rows)
    run(m, mss=None)
    assert m._xyz.shape[0] == 2 + 4                       # rows 1, 5 and both copies of rows 2, 3
    m = tiny(rows)
    run(m, mss=-1)                                        # zeros > -1: every row pruned
    assert m._xyz.shape[0] == 0


def test_rule_9_statistics_and_edges():
    m = tiny([{"g": 1e-3, "s": (0.3, 0.2)}, {"g": 1e-3, "s": (0.01, 0.01)}, {"g": 0.0, "s": (0.01, 0.01)}])
    run(m, mss=20)
    assert m.xyz_gradient_accum.shape == (5, 1) and m.denom.shape == (5, 1) and m.max_radii2D.shape == (5,)
    assert not m.xyz_gradient_accum.any() and not m.denom.any() and not m.max_radii2D.any()
    # nothing selected: the model is the model, the draw is empty
    m = tiny([{"g": 0.0, "s": (0.3, 0.2)}, {"g": 1e-5, "s": (0.01, 0.01)}])
    before, drawn = run(m)
    assert drawn.shape == (0, 3)
    for n in DR.GROUPS:
        assert torch.equal(getattr(m, DR.ATTR[n]).detach(), before[n])
    # P = 0
    m = tiny([{"g": 0.0, "s": (0.3, 0.2)}])
    run(m, mss=-1)
    assert m._xyz.shape == (0, 3)
    before, drawn = run(m, mss=20)
    assert m._xyz.shape == (0, 3) and m._features_rest.shape == (0, 15, 3) and drawn.shape == (0, 3)


def test_rule_10_one_draw_of_2S_rows_including_pruned_splits():
    rows = [{"g": 1e-3, "s": (0.7, 0.1)}, {"g": 1e-3, "s": (0.3, 0.1), "o": -6.0}, {"g": 1e-3, "s": (0.3, 0.1)}]
    m = tiny(rows)
    torch.manual_seed(3)
    _, drawn = run(m, mss=20)
    assert drawn.shape == (6, 3) and m._xyz.shape[0] == 2
    after = torch.randn(1)
    torch.manual_seed(3)
    torch.empty(6, 3).normal_()
    assert torch.equal(after, torch.randn(1))


# ---- the entry point and the C ABI without a device ---------------------------------------------------------------

def test_python_entry_rejects_bad_models():
    from diff_surfel_rasterization.densify import densify_and_prune
    m = tiny([{"g": 1e-3, "s": (0.3, 0.2)}])
    with pytest.raises(RuntimeError, match="CUDA"):
        densify_and_prune(m, 0.0002, 0.005, 4.0, None)
    m.optimizer.param_groups[2]["name"] = "sh_rest"
    with pytest.raises(RuntimeError, match="f_rest"):
        densify_and_prune(m, 0.0002, 0.005, 4.0, None)


def test_cabi_rejects_bad_arguments_without_a_device():
    import ctypes
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    err = lambda: lib.surfel_last_error().decode()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    n = lib.surfel_densify_workspace_bytes(1000)
    assert n >= 1000 * 16
    assert lib.surfel_densify_workspace_bytes(-1) == 0 and lib.surfel_densify_workspace_bytes(1 << 30) == 0
    plan = lambda P, a=p, d=p, s=p, o=p, ws=p, nb=n, tot=p: lib.surfel_densify_plan(
        P, a, d, s, o, 0.0002, 0.005, 0.04, 0.4, 1, 20.0, ws, nb, tot, None)
    assert plan(-1) != 0 and "P < 0" in err()
    assert plan(1 << 30) != 0 and "exceeds" in err()
    assert plan(5, a=None) != 0 and "NULL" in err()
    assert plan(5, o=None) != 0 and "NULL" in err()
    assert plan(5, ws=None) != 0 and "NULL" in err()
    assert plan(5, tot=None) != 0 and "NULL" in err()
    assert plan(5, nb=lib.surfel_densify_workspace_bytes(5) - 1) != 0 and "workspace" in err()

    def table(**over):
        t = (_cabi.DensifyGroup * 6)()
        for g, (name, rf, kind) in zip(t, [("xyz", 3, 1), ("f_dc", 3, 0), ("f_rest", 45, 0), ("opacity", 1, 0),
                                          ("scaling", 2, 2), ("rotation", 4, 3)]):
            g.param = g.exp_avg = g.exp_avg_sq = g.out_param = g.out_exp_avg = g.out_exp_avg_sq = p
            g.row_floats, g.kind = rf, kind
            for k, v in over.get(name, {}).items():
                setattr(g, k, v)
        return t
    apply = lambda P, P_out, S, t, z=p, ng=6, ws=p, nb=n: lib.surfel_densify_apply(P, P_out, S, ng, t, z, ws, nb, None)
    assert apply(-1, 0, 0, table()) != 0 and "P < 0" in err()
    assert apply(5, 11, 0, table()) != 0 and "inconsistent" in err()
    assert apply(5, 5, 6, table()) != 0 and "inconsistent" in err()
    assert apply(5, 5, 0, table(), ng=0) != 0 and "n_groups" in err()
    assert apply(5, 5, 0, table(), ng=9) != 0 and "n_groups" in err()
    assert apply(5, 5, 0, table(), ws=None) != 0 and "NULL" in err()
    assert apply(5, 5, 2, table(), z=None) != 0 and "NULL z" in err()
    assert apply(5, 5, 0, table(), nb=lib.surfel_densify_workspace_bytes(5) - 1) != 0 and "workspace" in err()
    assert apply(5, 5, 0, table(xyz={"row_floats": 4})) != 0 and "floats per row" in err()
    assert apply(5, 5, 0, table(f_dc={"kind": 7})) != 0 and "unknown kind" in err()
    assert apply(5, 5, 0, table(f_dc={"kind": 1, "row_floats": 3})) != 0 and "two groups" in err()
    assert apply(5, 5, 0, table(rotation={"kind": 0})) != 0 and "rotation" in err()
    assert apply(5, 5, 0, table(opacity={"param": None})) != 0 and "NULL parameter" in err()
    assert apply(5, 5, 0, table(opacity={"out_param": None})) != 0 and "NULL parameter" in err()
    assert apply(5, 5, 0, table(opacity={"exp_avg_sq": None})) != 0 and "one of its two moments" in err()
    assert apply(5, 5, 0, table(opacity={"out_exp_avg": None, "out_exp_avg_sq": None})) != 0 and "disagree" in err()
