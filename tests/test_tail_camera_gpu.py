"""Camera gradients of the fused render() tail and of the 2DGS regularisers (csrc/postprocess.cu,
surfel_post_camera_backward / surfel_post_reg_camera_backward, DESIGN.md §7q) on the GPU.

  1. exact pass: on the device's own inputs (allmap, rays, cotangents, the saved surf_depth and the tmp6 the backward
     left), each of the 21 outputs is within TOL x its first-order bound (tests/tail_camera_exact.sums_from, with
     tail_loss_exact's bounds for the recomputed surf_depth and surf_normal) plus the final cast;
  2. end to end: the camera gradients of surface_outputs and surface_regularizers agree with float64 autograd of the
     reference's tail within 2 x the float32 torch tail's own distance (or float32 rounding of the sums' magnitude);
  3. the bug: rasterizer -> fused tail gives the camera gradients of rasterizer -> reference torch tail;
  4. nothing else changes: allmap.grad is bit-identical with camera gradients requested, the launch count is the old
     one without them, +2 with them and +0 at lambda_normal == 0, and the pass writes only its own outputs;
  5. repeat calls and a side stream give bit-identical results;
  6. the user story: pose refinement with L1 + surface_regularizers.
"""
import math
import types

import numpy as np
import pytest
import torch

import camera_pose as CP
import surfel_scenes as S
import tail_camera_exact as C
import tail_loss_exact as X
import tail_loss_scenes as TS
from parity_bars import record_stats

pytestmark = pytest.mark.gpu

# x the bound of tail_camera_exact.sums_from, fixed before the first device run
TOL = 2.0
CAST = 2.0 ** -24
E2E_FACTOR = 2.0
SCENES = [("dense_raster", 0.0), ("sparse_raster", 0.3), ("golden", 1.0), ("holes", 0.3), ("nan_medians", 1.0),
          ("far_camera", 0.3), ("f33x9", 0.3), ("f1920x1080", 0.3)]


def _dev(x):
    return torch.as_tensor(np.asarray(x)).float().cuda().contiguous()


def _matrices(s, W, H):
    from diff_surfel_rasterization.postprocess import _view_matrices
    return _view_matrices(_dev(s["view"]), _dev(s["proj"]), W, H)


def outputs_pass(s, ratio, cot, stream=None, poison=False):
    """surfel_post_forward, surfel_post_backward and the camera pass on the device; returns the pass's inputs and its
    21 outputs (g_rot9 then g_rays12), all device tensors."""
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    a = _dev(s["allmap"])
    _, H, W = a.shape
    rot, rays = _matrices(s, W, H)
    g_rn, g_sd, g_sn = (None if cot.get(k) is None else _dev(cot[k]) for k in ("rend_normal", "surf_depth", "surf_normal"))
    p = lambda t: None if t is None else t.data_ptr()
    rn, sd, sn = torch.empty(3, H, W, device="cuda"), torch.empty(1, H, W, device="cuda"), torch.empty(3, H, W, device="cuda")
    tmp, g_allmap = torch.empty(6, H, W, device="cuda"), torch.empty(7, H, W, device="cuda")
    partials = torch.full((lib.surfel_post_camera_partials_bytes(W, H) // 8,), float("nan"), dtype=torch.float64, device="cuda")
    out = torch.full((21,), float("nan"), device="cuda")
    st = torch.cuda.current_stream() if stream is None else stream
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        _cabi.check(lib.surfel_post_forward(W, H, ratio, a.data_ptr(), rot.data_ptr(), rays.data_ptr(), rn.data_ptr(),
                                            sd.data_ptr(), sn.data_ptr(), st.cuda_stream))
        _cabi.check(lib.surfel_post_backward(W, H, ratio, a.data_ptr(), rot.data_ptr(), rays.data_ptr(), sd.data_ptr(),
                                             p(g_rn), p(g_sd), p(g_sn), tmp.data_ptr(), g_allmap.data_ptr(), st.cuda_stream))
        ins = dict(allmap=a, rot=rot, rays=rays, surf_depth=sd, tmp=tmp, g_allmap=g_allmap,
                   **{k: v for k, v in (("g_rn", g_rn), ("g_sd", g_sd), ("g_sn", g_sn)) if v is not None})
        before = {k: v.clone() for k, v in ins.items()} if poison else None
        _cabi.check(lib.surfel_post_camera_backward(W, H, ratio, a.data_ptr(), rot.data_ptr(), rays.data_ptr(),
                                                    sd.data_ptr(), p(g_rn), p(g_sd), p(g_sn), tmp.data_ptr(),
                                                    partials.data_ptr(), out[:9].data_ptr(), out[9:].data_ptr(),
                                                    st.cuda_stream))
    st.synchronize()
    if poison:
        for k, v in before.items():
            assert torch.equal(v, ins[k]), f"the camera pass wrote its input {k}"
    return ins, out


def reg_pass(s, ratio, ln, ld, g_normal=1.0, stream=None, poison=False):
    """surfel_post_reg_backward and the camera pass on the device; returns the pass's inputs and its 21 outputs."""
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    a = _dev(s["allmap"])
    _, H, W = a.shape
    rot, rays = _matrices(s, W, H)
    n = float(W * H)
    gscale = torch.tensor([g_normal * (ln / n), ld / n], dtype=torch.float32, device="cuda")
    tmp, g_allmap = torch.empty(6, H, W, device="cuda"), torch.empty(7, H, W, device="cuda")
    partials = torch.full((lib.surfel_post_camera_partials_bytes(W, H) // 8,), float("nan"), dtype=torch.float64, device="cuda")
    out = torch.full((21,), float("nan"), device="cuda")
    st = torch.cuda.current_stream() if stream is None else stream
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        _cabi.check(lib.surfel_post_reg_backward(W, H, ratio, ln, ld, a.data_ptr(), rot.data_ptr(), rays.data_ptr(),
                                                 gscale.data_ptr(), tmp.data_ptr(), g_allmap.data_ptr(), st.cuda_stream))
        ins = dict(allmap=a, rot=rot, rays=rays, gscale=gscale, tmp=tmp, g_allmap=g_allmap)
        before = {k: v.clone() for k, v in ins.items()} if poison else None
        _cabi.check(lib.surfel_post_reg_camera_backward(W, H, ratio, ln, ld, a.data_ptr(), rot.data_ptr(),
                                                        rays.data_ptr(), gscale.data_ptr(), tmp.data_ptr(),
                                                        partials.data_ptr(), out[:9].data_ptr(), out[9:].data_ptr(),
                                                        st.cuda_stream))
    st.synchronize()
    if poison:
        for k, v in before.items():
            assert torch.equal(v, ins[k]), f"the camera pass wrote its input {k}"
    return ins, out


def _ratio(got, G, B):
    """Worst (|got - G| - cast) / (u B) over the 21 outputs; inf where the bound is 0 and got differs."""
    got = got.double().cpu()
    err = ((got - G).abs() - CAST * G.abs()).clamp_min(0)
    b = X.U * B
    r = torch.where(b > 0, err / b.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    assert bool(torch.isfinite(got).all()), got
    return float(r.max())


# ---------------------------------------------------------------------------------------------- 1. exact pass
@pytest.mark.parametrize("name,ratio", SCENES)
def test_outputs_pass_matches_exact(cuda_lib, name, ratio):
    s = TS.ALLMAPS[name][0]()
    H, W = s["allmap"].shape[1:]
    worst = 0.0
    for kind in ("random", "train"):
        if kind == "train":
            out, *_ = X.tail_f64(s["allmap"], s["view"], s["proj"], ratio)
            cot = TS.cotangents(H, W, "train", out)
        else:
            cot = TS.cotangents(H, W, "random")
        ins, got = outputs_pass(s, ratio, cot)
        a = ins["allmap"].double().cpu()
        tmp = ins["tmp"].double().cpu()
        d = ins["surf_depth"][0].double().cpu()
        g_rn = torch.as_tensor(cot["rend_normal"]).double()
        G, B = C.sums_from(a[2:5], g_rn, d, C.gather(tmp), e_dP=3 * C.gather(tmp, absolute=True))
        r = _ratio(got, G, B)
        worst = max(worst, r)
        assert r <= TOL, (kind, r)
    record_stats("tail camera pass (outputs) error / bound", np.array([worst]), dict(tol=TOL, scene=name, ratio=ratio))


@pytest.mark.parametrize("name,ratio", SCENES)
def test_regularizer_pass_matches_exact(cuda_lib, name, ratio):
    s = TS.ALLMAPS[name][0]()
    worst = 0.0
    for ln, ld, gn in ((0.05, 100.0, 1.0), (0.05, 0.0, -3.0)):
        ins, got = reg_pass(s, ratio, ln, ld, gn)
        a = ins["allmap"].double().cpu()
        rays = ins["rays"].double().cpu()
        tmp = ins["tmp"].double().cpu()
        sc = float(ins["gscale"][0])
        d = C.surf_depth(a, ratio)
        sn = C.surf_normal(a, d, rays)
        _, _, ob, _, _ = X.tail_f64(s["allmap"], s["view"], s["proj"], ratio)
        e_gw = abs(sc) * (ob["surf_normal"] + 2 * sn.abs())      # sn's own error, and the product with s
        G, B = C.sums_from(a[2:5], -sc * sn, d, C.gather(tmp), e_gw=e_gw, e_d=ob["surf_depth"][0],
                           e_dP=3 * C.gather(tmp, absolute=True))
        r = _ratio(got, G, B)
        worst = max(worst, r)
        assert r <= TOL, (ln, ld, gn, r)
    record_stats("tail camera pass (regularisers) error / bound", np.array([worst]), dict(tol=TOL, scene=name, ratio=ratio))


# ---------------------------------------------------------------------------------------------- 2. end to end
def _cam_leaves(s, dtype=torch.float32):
    H, W = s["allmap"].shape[1:]
    return types.SimpleNamespace(world_view_transform=torch.as_tensor(s["view"]).cuda().to(dtype).requires_grad_(True),
                                 full_proj_transform=torch.as_tensor(s["proj"]).cuda().to(dtype).requires_grad_(True),
                                 image_width=W, image_height=H)


def fused_camera_grads(s, ratio, loss_kind, cot=None, ln=0.05, ld=100.0):
    from diff_surfel_rasterization.postprocess import surface_outputs, surface_regularizers
    cam = _cam_leaves(s)
    a = _dev(s["allmap"]).requires_grad_(True)
    if loss_kind == "outputs":
        out = surface_outputs(a, cam, ratio)
        loss = C.outputs_loss(cot)(out)
    else:
        nl, dl = surface_regularizers(a, cam, ratio, ln, ld)
        loss = nl + dl
    loss.backward()
    return cam.world_view_transform.grad.double().cpu(), cam.full_proj_transform.grad.double().cpu(), a.grad


@pytest.mark.parametrize("name,ratio", [("dense_raster", 0.0), ("sparse_raster", 1.0), ("golden", 0.3), ("holes", 0.3),
                                        ("far_camera", 0.3)])
@pytest.mark.parametrize("loss_kind", ["outputs", "regularizers"])
def test_end_to_end_against_float64_autograd(cuda_lib, name, ratio, loss_kind):
    s = TS.ALLMAPS[name][0]()
    H, W = s["allmap"].shape[1:]
    rot, rays = C.view_matrices(torch.from_numpy(s["view"]), torch.from_numpy(s["proj"]), W, H)
    if loss_kind == "outputs":
        cot = TS.cotangents(H, W, "random")
        loss = C.outputs_loss(cot)
        _, B = C.outputs_sums(s["allmap"], rot, rays, ratio, cot)
    else:
        cot, loss = None, C.reg_loss(0.05, 100.0)
        _, B = C.reg_sums(s["allmap"], rot, rays, ratio, 0.05)
    gv, gp, _ = fused_camera_grads(s, ratio, loss_kind, cot)
    r64 = C.reference_camera_grads(s["allmap"], s["view"], s["proj"], ratio, loss, torch.float64, "cuda")
    r32 = C.reference_camera_grads(s["allmap"], s["view"], s["proj"], ratio, loss, torch.float32, "cuda")
    floors = C.chain_bound(B, s["view"], s["proj"], W, H)
    for key, g, a64, a32, fl in zip(("world_view_transform", "full_proj_transform"), (gv, gp), r64, r32, floors):
        a64, a32 = a64.double().cpu(), a32.double().cpu()
        d_dev, d_32 = float((g - a64).abs().max()), float((a32 - a64).abs().max())
        bar = max(E2E_FACTOR * d_32, X.U * float(fl.max()))
        record_stats(f"tail camera e2e {key}: max|device - f64| / max|f32 - f64|", np.array([d_dev / max(d_32, 1e-300)]),
                     dict(scene=name, loss=loss_kind, device=d_dev, torch_f32=d_32, scale=float(a64.abs().max())))
        assert d_dev <= bar, f"{key}: max|device - f64| {d_dev:.3e} > {bar:.3e} (torch f32 {d_32:.3e})"


# ---------------------------------------------------------------------------------------------- 3. the bug
def _raster_then_tail(case, tail, seed):
    """The public op with camera gradients, then `tail` ('fused', 'torch', or 'constant': the torch tail with the camera
    detached, what the fused tail computed before it had camera gradients) and train.py's regularisers plus a colour
    term; returns the camera gradients (viewmatrix, projmatrix, campos)."""
    from diff_surfel_rasterization import GaussianRasterizer
    from diff_surfel_rasterization.postprocess import surface_regularizers
    from test_camera_grad_gpu import parity_scene, settings
    from test_postprocess_gpu import reference_tail
    scene, cam = parity_scene(case)
    dev = torch.device("cuda")
    rs = settings(cam, dev)
    leaf = {k: torch.as_tensor(np.asarray(v)).to(dev) for k, v in scene.items()}
    color, _, allmap = GaussianRasterizer(rs)(means3D=leaf["means3D"], means2D=torch.zeros_like(leaf["means3D"]),
                                              shs=leaf["shs"], opacities=leaf["opacities"], scales=leaf["scales"],
                                              rotations=leaf["rotations"])
    vm, pm = (rs.viewmatrix.detach(), rs.projmatrix.detach()) if tail == "constant" else (rs.viewmatrix, rs.projmatrix)
    view = types.SimpleNamespace(world_view_transform=vm, full_proj_transform=pm, image_width=int(cam["W"]),
                                 image_height=int(cam["H"]))
    if tail == "fused":
        nl, dl = surface_regularizers(allmap, view, 0.0, 0.05, 100.0)
        loss = nl + dl
    else:
        loss = C.reg_loss(0.05, 100.0)(reference_tail(allmap, view, 0.0))
    gc, _ = S.make_cotangents(int(cam["W"]), int(cam["H"]), seed)
    (loss + 1e-3 * (color * gc.to(dev)).mean()).backward()
    return [getattr(rs, k).grad.double().cpu() for k in ("viewmatrix", "projmatrix", "campos")]


@pytest.mark.parametrize("ci", range(3))
def test_rasterizer_then_fused_tail_gives_the_torch_tails_camera_gradients(cuda_lib, ci):
    from test_camera_grad_gpu import parity_cases
    case = parity_cases()[ci]
    ref = _raster_then_tail(case, "torch", 5)
    ref2 = _raster_then_tail(case, "torch", 5)
    got = _raster_then_tail(case, "fused", 5)
    const = _raster_then_tail(case, "constant", 5)
    missed = {}
    for key, r, r2, g, c in zip(("viewmatrix", "projmatrix", "campos"), ref, ref2, got, const):
        scale, spread, diff = float(r.abs().max()), float((r2 - r).abs().max()), float((g - r).abs().max())
        missed[key] = float((c - r).abs().max()) / max(2 * spread, 1e-3 * scale)
        print(f"{key}: max|fused - torch| {diff:.3e}, torch run-to-run {spread:.3e}, scale {scale:.3e}; "
              f"a constant tail misses by {missed[key]:.3g} x the bar")
        record_stats(f"tail camera bug {key}: max|fused - torch| / scale", np.array([diff / max(scale, 1e-300)]), dict(case=ci))
        assert scale > 0
        assert diff <= max(2 * spread, 1e-3 * scale), key
    # the bar separates: a tail that treats the camera as a constant fails it
    assert missed["viewmatrix"] > 1.0 and missed["projmatrix"] > 1.0, missed


# ---------------------------------------------------------------------------------------------- 4. nothing else
@pytest.mark.parametrize("loss_kind", ["outputs", "regularizers"])
def test_camera_gradients_change_nothing_else(cuda_lib, loss_kind):
    from diff_surfel_rasterization.postprocess import surface_outputs, surface_regularizers
    lib = cuda_lib
    s = TS.holes()
    H, W = s["allmap"].shape[1:]
    cot = TS.cotangents(H, W, "random")

    def run(camera_grad, ln=0.05):
        cam = _cam_leaves(s)
        if not camera_grad:
            cam.world_view_transform.requires_grad_(False)
            cam.full_proj_transform.requires_grad_(False)
        a = _dev(s["allmap"]).requires_grad_(True)
        n0 = lib.surfel_launch_count()
        if loss_kind == "outputs":
            C.outputs_loss(cot)(surface_outputs(a, cam, 0.3)).backward()
        else:
            sum(surface_regularizers(a, cam, 0.3, ln, 100.0)).backward()
        torch.cuda.synchronize()
        return a.grad.clone(), lib.surfel_launch_count() - n0, cam

    g_plain, n_plain, _ = run(False)
    g_cam, n_cam, cam = run(True)
    assert torch.equal(g_plain, g_cam)
    assert n_cam == n_plain + 2
    assert cam.world_view_transform.grad is not None and cam.full_proj_transform.grad is not None
    if loss_kind == "regularizers":
        g0, n0_plain, _ = run(False, 0.0)
        g0c, n0_cam, cam0 = run(True, 0.0)
        assert torch.equal(g0, g0c) and n0_cam == n0_plain
        assert not cam0.world_view_transform.grad.any() and not cam0.full_proj_transform.grad.any()


def test_camera_pass_writes_only_its_outputs(cuda_lib):
    s = TS.holes()
    H, W = s["allmap"].shape[1:]
    _, out = outputs_pass(s, 0.3, TS.cotangents(H, W, "random"), poison=True)
    assert bool(torch.isfinite(out).all())
    _, out = reg_pass(s, 0.3, 0.05, 100.0, poison=True)
    assert bool(torch.isfinite(out).all())
    _, out = reg_pass(s, 0.3, 0.0, 100.0)
    assert not out.any()


# ---------------------------------------------------------------------------------------------- 5. repeatable
def test_repeat_calls_and_side_stream_are_bit_identical(cuda_lib):
    s = TS.ALLMAPS["f1920x1080"][0]()
    H, W = s["allmap"].shape[1:]
    cot = TS.cotangents(H, W, "random")
    first_o = outputs_pass(s, 0.3, cot)[1].cpu()
    first_r = reg_pass(s, 0.3, 0.05, 100.0)[1].cpu()
    side = torch.cuda.Stream()
    for stream in (None, side):
        assert torch.equal(first_o.view(torch.int32), outputs_pass(s, 0.3, cot, stream)[1].cpu().view(torch.int32))
        assert torch.equal(first_r.view(torch.int32), reg_pass(s, 0.3, 0.05, 100.0, stream=stream)[1].cpu().view(torch.int32))


# ---------------------------------------------------------------------------------------------- 6. user story
LAMBDA_NORMAL, LAMBDA_DIST = 0.05, 100.0


def refine_with_regularizers(tail, steps, W=CP.W_GPU, H=CP.H_GPU, P=CP.P_GPU):
    """camera_pose.refine's loop on the public op, with L1 + train.py's two regularisers through `tail` ('fused':
    surface_regularizers, 'torch': the reference's torch tail); returns the errors, losses and first-step gradient."""
    from diff_surfel_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from diff_surfel_rasterization.postprocess import surface_regularizers
    from test_postprocess_gpu import reference_tail
    scene = {k: v.cuda() for k, v in CP.make_scene(P, W, H).items()}
    cam = S.make_camera(W, H, fovy_deg=CP.FOVY)
    proj_T = torch.linalg.solve(cam["viewmatrix"].double(), cam["projmatrix"].double())
    tanfovy = math.tan(math.radians(CP.FOVY) / 2)

    def render(vm, pm, cp):
        rs = GaussianRasterizationSettings(H, W, tanfovy * W / H, tanfovy, torch.zeros(3, device="cuda"), 1.0, vm, pm, 1,
                                           cp, False, False)
        color, _, allmap = GaussianRasterizer(rs)(means3D=scene["means3D"], means2D=torch.zeros_like(scene["means3D"]),
                                                  opacities=scene["opacities"], shs=scene["shs"], scales=scene["scales"],
                                                  rotations=scene["rotations"])
        return color, allmap

    R_true, t_true = np.eye(3), np.zeros(3)
    with torch.no_grad():
        vm, pm, cp = (x.float().cuda() for x in CP.camera_tensors(torch.tensor(R_true), torch.tensor(t_true), proj_T))
        target = render(vm, pm, cp)[0]
    w0, d0 = CP.perturbation()
    R0t = CP.so3_exp(torch.tensor(w0)) @ torch.tensor(R_true)
    t0t = torch.tensor(t_true + d0)
    omega = torch.zeros(3, dtype=torch.float64, requires_grad=True)
    tau = torch.zeros(3, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([dict(params=[omega], lr=CP.LR_ROT), dict(params=[tau], lr=CP.LR_TRANS)])
    rot_err, trans_err, losses, first = [], [], [], None
    for it in range(steps + 1):
        E = CP.so3_exp(omega)
        R, t = E @ R0t, E @ t0t + tau
        e = CP.pose_errors(R.detach().numpy(), t.detach().numpy(), R_true, t_true)
        rot_err.append(e[0]); trans_err.append(e[1])
        if it == steps:
            break
        vm, pm, cp = (x.float().cuda() for x in CP.camera_tensors(R, t, proj_T))
        color, allmap = render(vm, pm, cp)
        view = types.SimpleNamespace(world_view_transform=vm, full_proj_transform=pm, image_width=W, image_height=H)
        if tail == "fused":
            nl, dl = surface_regularizers(allmap, view, 0.0, LAMBDA_NORMAL, LAMBDA_DIST)
        else:
            out = reference_tail(allmap, view, 0.0)
            nl = LAMBDA_NORMAL * (1 - (out["rend_normal"] * out["surf_normal"]).sum(dim=0)).mean()
            dl = LAMBDA_DIST * out["rend_dist"].mean()
        loss = (color - target).abs().mean() + nl + dl
        losses.append(loss.item())
        opt.zero_grad()
        loss.backward()
        if first is None:
            first = torch.cat([omega.grad, tau.grad]).clone()
        opt.step()
    return dict(rot_err=rot_err, trans_err=trans_err, losses=losses, first=first)


def test_pose_refinement_with_regularizers(cuda_lib):
    fused = refine_with_regularizers("fused", CP.STEPS)
    torch_tail = refine_with_regularizers("torch", 1)
    g, r = fused["first"], torch_tail["first"]
    diff = float((g - r).abs().max() / r.abs().max())
    r0, r1, t0, t1 = fused["rot_err"][0], fused["rot_err"][-1], fused["trans_err"][0], fused["trans_err"][-1]
    print(f"first-step gradient: fused {g.numpy()}, torch tail {r.numpy()}, max rel diff {diff:.3e}")
    print(f"rotation {np.degrees(r0):.4f} -> {np.degrees(r1):.4f} deg, centre {t0:.4e} -> {t1:.4e}, "
          f"loss {fused['losses'][0]:.4e} -> {fused['losses'][-1]:.4e}")
    record_stats("pose refinement with regularisers final / initial error", np.array([r1 / r0, t1 / t0]),
                 dict(first_step_rel_diff=diff))
    assert diff <= 1e-3
    assert r1 < 0.25 * r0 and t1 < 0.25 * t0
