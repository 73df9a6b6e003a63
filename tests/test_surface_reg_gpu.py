"""postprocess.surface_regularizers (SURVEY §8f row f2, DESIGN §7l) held, entry by entry and with no budget, to the
float64 evaluation of train.py's regularisers in tests/surface_reg_exact.py, replayed against the reference's own
stored values and gradients, and composed with the rasterizer and the fused photometric loss.  Where the
reference's gradient is NaN (D/alpha not finite), the fused one is 0."""
import types

import numpy as np
import pytest
import torch

import surface_reg_exact as R
import surfel_scenes as S
import tail_loss_scenes as TS
from parity_bars import record_stats
from test_postprocess_gpu import reference_tail

pytestmark = pytest.mark.gpu

PAIRS = ((0.05, 0.0), (0.05, 100.0), (0.05, 1000.0), (0.0, 100.0), (0.0, 0.0))

# Tolerances: |fused - exact| <= TOL * bound for both values and every gradient entry (bounds of
# surface_reg_exact.reg_f64, in which the float32 emulation of the kernels reaches 0.50).  Cut at about 4x the worst
# value observed on an H100 80GB HBM3 (700 W power limit) over every scene, depth ratio and lambda pair below.
VALUE_TOL = 2.0         # worst observed 0.50 (holes, depth ratio 0, dist_loss: its float32 rounding)
GRAD_TOL = 1.4          # worst observed 0.33 (f33x9, depth ratio 0.3, (0.05, 100))
# fused against the eager float32 compositions through the rasterizer: |a - b| over the leaf's largest entry; worst
# observed 2.4e-5 (allmap.grad against the eager tail), 2.5e-7 against surface_outputs + train.py's lines
COMPOSE_TOL = 1e-4


def _fused(scene, ratio, ln, ld, dev="cuda"):
    from diff_surfel_rasterization.postprocess import surface_regularizers
    a = torch.from_numpy(scene["allmap"]).to(dev).requires_grad_(True)
    n, d = surface_regularizers(a, R.view_of(scene, dev), ratio, ln, ld)
    (n + d).backward()
    return (n.detach(), d.detach()), a.grad


def _exact(scene, ratio, ln, ld):
    return R.reg_f64(scene["allmap"], scene["view"], scene["proj"], ratio, ln, ld, dev="cuda")


def _tag(ratio, ln, ld):
    return f"r{ratio:g}_n{ln:g}_d{ld:g}".replace(".", "p")


@pytest.mark.parametrize("ratio", (0.0, 1.0))
@pytest.mark.parametrize("ln,ld", PAIRS)
def test_golden_replay(cuda_lib, ratio, ln, ld):
    """Against the reference's own float32 values and gradient: each is within its bound of the exact value, so the
    two are within (TOL + 1) x bound of each other; the reference's NaN entries are 0 here."""
    g = np.load(R.X.__file__.replace("tail_loss_exact.py", "golden/ref_surface_reg.npz"))
    scene = TS.golden()
    t = _tag(ratio, ln, ld)
    (n, d), grad = _fused(scene, ratio, ln, ld)
    assert n.dtype == torch.float32 and n.dim() == 0 and n.is_cuda and d.dtype == torch.float32 and d.dim() == 0
    values, eg, vb, gb, hole = _exact(scene, ratio, ln, ld)
    for got, ref, b, tol in ((n, g[t + "_normal_loss"], vb[0], VALUE_TOL), (d, g[t + "_dist_loss"], vb[1], VALUE_TOL)):
        assert abs(float(got) - float(ref)) <= R.U * b * (tol + 1), (float(got), float(ref))
    ref = torch.from_numpy(g[t + "_grad_allmap"]).cuda().double()
    nan = torch.isnan(ref)
    assert int(nan.sum()) == 400 and torch.isfinite(grad).all()
    assert bool((grad[nan] == 0).all())
    err = (grad.double() - ref).abs()[~nan]
    b = R.U * gb[~nan] * (GRAD_TOL + 1)
    assert bool((err <= b).all()), float((err / b.clamp_min(1e-300)).max())


@pytest.mark.parametrize("ln,ld", PAIRS)
@pytest.mark.parametrize("name,ratio", TS.ALLMAP_CASES)
def test_every_scene_is_within_its_bound(cuda_lib, name, ratio, ln, ld):
    scene = TS.ALLMAPS[name][0]()
    values, grad = _fused(scene, ratio, ln, ld)
    ex = _exact(scene, ratio, ln, ld)
    worst, r = R.worst_ratios(values, grad, ex, "hole")
    record_stats(f"surface_reg {name} r{ratio} n{ln} d{ld} grad", r.cpu().numpy())
    record_stats(f"surface_reg {name} r{ratio} n{ln} d{ld} values", np.array([worst["normal"], worst["dist"]]))
    assert worst["normal"] <= VALUE_TOL and worst["dist"] <= VALUE_TOL, worst
    assert worst["grad"] <= GRAD_TOL, worst


@pytest.mark.parametrize("name", ["golden", "holes", "nan_medians", "f1920x1080"])
def test_zero_lambdas_give_exact_zeros(cuda_lib, name):
    scene = TS.ALLMAPS[name][0]()
    (n, d), g = _fused(scene, 0.3, 0.0, 100.0)
    assert float(n) == 0.0 and float(d) != 0.0 and bool((g[:6] == 0).all()) and bool((g[6] != 0).all())
    (n, d), g = _fused(scene, 0.3, 0.05, 0.0)
    assert float(d) == 0.0 and float(n) != 0.0 and bool((g[6] == 0).all())
    (n, d), g = _fused(scene, 0.3, 0.0, 0.0)
    assert float(n) == 0.0 and float(d) == 0.0 and bool((g == 0).all())


@pytest.mark.parametrize("W,H", [(1, 1), (2, 2), (1, 64), (64, 1), (2, 40), (40, 2)])
def test_frames_without_interior(cuda_lib, W, H):
    """No pixel has a 3x3 stencil: surf_normal is 0 everywhere, so each normal error is exactly 1."""
    scene = TS.frame(W, H)
    for ratio in (0.0, 1.0):
        (n, d), g = _fused(scene, ratio, 0.05, 100.0)
        assert float(n) == float(np.float32(0.05)) and bool((g[:6] == 0).all())


def test_run_to_run_and_side_stream_are_bit_identical(cuda_lib):
    scene = TS.frame(1920, 1080)
    (n0, d0), g0 = _fused(scene, 0.3, 0.05, 1000.0)
    for _ in range(2):
        (n1, d1), g1 = _fused(scene, 0.3, 0.05, 1000.0)
        assert torch.equal(n0, n1) and torch.equal(d0, d1) and torch.equal(g0, g1)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        (n1, d1), g1 = _fused(scene, 0.3, 0.05, 1000.0)
    s.synchronize()
    assert torch.equal(n0, n1) and torch.equal(d0, d1) and torch.equal(g0, g1)


def test_only_one_output_used(cuda_lib):
    from diff_surfel_rasterization.postprocess import surface_regularizers
    scene = TS.holes()
    _, g_both = _fused(scene, 0.3, 0.05, 100.0)
    for k in (0, 1):
        a = torch.from_numpy(scene["allmap"]).cuda().requires_grad_(True)
        out = surface_regularizers(a, R.view_of(scene, "cuda"), 0.3, 0.05, 100.0)
        out[k].backward()
        if k == 0:
            assert torch.equal(a.grad[:6], g_both[:6]) and bool((a.grad[6] == 0).all())
        else:
            assert bool((a.grad[:6] == 0).all()) and torch.equal(a.grad[6], g_both[6])


def test_sparse_scene_composes_with_the_rasterizer_and_the_loss(cuda_lib):
    """Rasterize the sparse scene with the CUDA rasterizer and run train.py's objective three ways: the fused
    regularisers + fused loss, surface_outputs + train.py's lines + fused loss, and the eager restatements.  Leaf
    gradients agree; allmap.grad agrees where the eager one is finite and is 0 where it is NaN."""
    from diff_surfel_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from diff_surfel_rasterization.loss import l1_ssim_loss
    from diff_surfel_rasterization.postprocess import surface_outputs, surface_regularizers
    from test_loss_gpu import reference_loss
    dev = "cuda"
    W, H, P = 320, 200, 60
    ln, ld = 0.05, 1000.0
    cam = S.make_camera(W, H, R=S.look_at_rotation(15, -8), t=[0.2, -0.1, 0.3])
    scene = S.make_scene(P, W, H, 7, depth_complexity=6)
    m = torch.cat([scene["means3D"], torch.ones(P, 1)], 1) @ cam["viewmatrix"].inverse()
    scene["means3D"] = m[:, :3].contiguous()
    rs = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=dev),
        scale_modifier=1.0, viewmatrix=cam["viewmatrix"].to(dev), projmatrix=cam["projmatrix"].to(dev), sh_degree=3,
        campos=cam["campos"].to(dev), prefiltered=False, debug=False)
    view = types.SimpleNamespace(world_view_transform=cam["viewmatrix"].to(dev), full_proj_transform=cam["projmatrix"].to(dev),
                                 image_width=W, image_height=H)
    gt = TS.image_pair((3, H, W), "noisy")[1].to(dev)

    def lines(out):
        normal_error = (1 - (out["rend_normal"] * out["surf_normal"]).sum(dim=0))[None]
        return ln * normal_error.mean(), ld * out["rend_dist"].mean()

    paths = {"fused": (lambda a: surface_regularizers(a, view, 0.0, ln, ld), l1_ssim_loss),
             "outputs": (lambda a: lines(surface_outputs(a, view, 0.0)), l1_ssim_loss),
             "eager": (lambda a: lines(reference_tail(a, view, 0.0)), reference_loss)}
    res = {}
    for name, (reg, loss) in paths.items():
        leaf = {k: v.to(dev).requires_grad_(True) for k, v in scene.items()}
        color, _, allmap = GaussianRasterizer(rs)(means3D=leaf["means3D"], means2D=torch.zeros(P, 3, device=dev),
                                                  shs=leaf["shs"], opacities=leaf["opacities"], scales=leaf["scales"],
                                                  rotations=leaf["rotations"])
        allmap.retain_grad()
        n, d = reg(allmap)
        (loss(color, gt, 0.2) + d + n).backward()
        res[name] = ({k: v.grad for k, v in leaf.items()}, allmap.grad, allmap.detach(), (float(n), float(d)))
    assert float((res["fused"][2][1] == 0).float().mean()) >= 0.10
    ga = res["fused"][1]
    assert torch.isfinite(ga).all()
    for other in ("outputs", "eager"):
        for k in (0, 1):
            assert abs(res["fused"][3][k] - res[other][3][k]) <= 1e-5 * abs(res[other][3][k]), (other, k)
        gb_ = res[other][1]
        nan = torch.isnan(gb_)
        assert bool((ga[nan] == 0).all())
        scale = ga.abs().flatten(1).max(1).values[:, None, None].clamp_min(1e-30)
        err = ((ga - gb_.nan_to_num()).abs() / scale)[~nan]
        record_stats(f"surface_reg compose vs {other} allmap.grad", err.cpu().numpy())
        assert float(err.max()) < COMPOSE_TOL, (other, float(err.max()))
        for k, gf in res["fused"][0].items():
            ge = res[other][0][k]
            fin = torch.isfinite(ge)
            assert torch.isfinite(gf).all(), k
            e = float((gf - ge).abs()[fin].max() / ge[fin].abs().max().clamp_min(1e-30))
            record_stats(f"surface_reg compose vs {other} {k}", np.array([e]))
            assert e < COMPOSE_TOL, (other, k, e)


def test_rejects_bad_inputs_before_launching(cuda_lib):
    from diff_surfel_rasterization import _cabi
    from diff_surfel_rasterization.postprocess import surface_regularizers
    lib = _cabi.load()
    scene = TS.holes()
    a = torch.from_numpy(scene["allmap"])
    view = R.view_of(scene, "cuda")
    before = lib.surfel_launch_count()
    with pytest.raises(RuntimeError, match="surface_regularizers: allmap must be a CUDA tensor"):
        surface_regularizers(a, view, 0.0, 0.05, 100.0)
    with pytest.raises(RuntimeError, match="allmap must be"):
        surface_regularizers(a[:6].cuda(), view, 0.0, 0.05, 100.0)
    with pytest.raises(RuntimeError, match="allmap must be"):
        surface_regularizers(a[:, 1:].cuda(), view, 0.0, 0.05, 100.0)
    with pytest.raises(RuntimeError, match="camera world_view_transform"):
        surface_regularizers(a.cuda(), R.view_of(scene, "cpu"), 0.0, 0.05, 100.0)
    v = R.view_of(scene, "cuda")
    v.full_proj_transform = v.full_proj_transform.cpu()
    with pytest.raises(RuntimeError, match="camera full_proj_transform"):
        surface_regularizers(a.cuda(), v, 0.0, 0.05, 100.0)
    v = R.view_of(scene, "cuda")
    v.world_view_transform = v.world_view_transform[:3]
    with pytest.raises(RuntimeError, match="camera world_view_transform"):
        surface_regularizers(a.cuda(), v, 0.0, 0.05, 100.0)
    if torch.cuda.device_count() > 1:
        with pytest.raises(RuntimeError, match="camera world_view_transform"):
            surface_regularizers(a.to("cuda:1"), view, 0.0, 0.05, 100.0)
    assert lib.surfel_launch_count() == before


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="one device")
def test_second_device(cuda_lib):
    scene = TS.holes()
    (n0, d0), g0 = _fused(scene, 0.3, 0.05, 100.0)
    (n1, d1), g1 = _fused(scene, 0.3, 0.05, 100.0, dev="cuda:1")
    assert n1.device == torch.device("cuda:1") and g1.device == torch.device("cuda:1")
    assert torch.equal(n0.cpu(), n1.cpu()) and torch.equal(d0.cpu(), d1.cpu()) and torch.equal(g0.cpu(), g1.cpu())
