"""diff_surfel_rasterization.metrics on the device (DESIGN.md §7o): PSNR equal to its float64 value rounded once,
SSIM inside the fused loss's bound, each TF32 conv layer inside its per-output bound, exact pools, the tap kernel
inside its bound, and LPIPS end to end within twice the error cuDNN's TF32 convolutions make against float64."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import metrics_ref as R
import tail_loss_exact as X

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_metrics.npz")
M360 = ((822, 1237), (1039, 1558))            # (H, W): outdoor images_4, indoor images_2


@pytest.fixture(scope="module")
def weights():
    return R.vgg_weights(), R.lin_weights()


@pytest.fixture(scope="module")
def lpips(cuda_lib, weights):
    from diff_surfel_rasterization.metrics import LPIPS
    return LPIPS(*weights)


def _pairs(H, W, seed):
    """Random 8-bit pair and a blurred-and-noised pair of a smooth 8-bit image, (1,3,H,W) float32 on the GPU."""
    g = torch.Generator().manual_seed(seed)
    q = lambda t: (t.clamp(0, 1) * 255).round() / 255
    a, b = q(torch.rand((1, 3, H, W), generator=g)), q(torch.rand((1, 3, H, W), generator=g))
    gt = q(F.interpolate(torch.rand((1, 3, H // 16 + 2, W // 16 + 2), generator=g), size=(H, W), mode="bilinear",
                         align_corners=False))
    r = q(F.avg_pool2d(gt, 5, 1, 2, count_include_pad=False) + 0.03 * torch.randn(gt.shape, generator=g))
    return [(a.cuda(), b.cuda()), (r.cuda(), gt.cuda())]


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def _conv(lib, layer, x):
    cin, cout, packed, bias = layer
    n, _, h, w = x.shape
    out = torch.empty((n, h, w, cout), device="cuda")
    xin = _nhwc(x.float())
    assert lib.surfel_metrics_conv3x3(n, h, w, cin, cout, xin.data_ptr(), packed.data_ptr(), bias.data_ptr(),
                                      out.data_ptr(), None) == 0, lib.surfel_last_error()
    return _nchw(out)


def _pool(lib, x):
    n, c, h, w = x.shape
    out = torch.empty((n, h // 2, w // 2, c), device="cuda")
    xin = _nhwc(x)
    assert lib.surfel_metrics_maxpool(n, h, w, c, xin.data_ptr(), out.data_ptr(), None) == 0
    return _nchw(out)


def _cudnn_lpips(x, y, weights, tf32):
    """The restatement in float32 through cuDNN, with TF32 convolutions (torch's default) or without."""
    vgg, lin = weights
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        layers = R.conv_layers(vgg, torch.float32, "cuda")
        fx, fy = R.trunk(R.zscore(x), layers), R.trunk(R.zscore(y), layers)
        return float(R.tap_values(fx, fy, lin).sum())
    finally:
        torch.backends.cudnn.allow_tf32 = old


# ---- PSNR ----

@pytest.mark.parametrize("shape", [(1, 3, 37, 53), (2, 3, 20, 16), (1, 3) + M360[0], (1, 3) + M360[1]])
def test_psnr_is_f64_rounded_once(cuda_lib, shape):
    from diff_surfel_rasterization.metrics import psnr
    g = torch.Generator().manual_seed(sum(shape))
    a = (torch.randint(0, 256, shape, generator=g).float() / 255).cuda()
    b = ((a.cpu() * 255 + torch.randint(-6, 7, shape, generator=g)).clamp(0, 255) / 255).float().cuda()
    got = psnr(a, b)
    assert got.shape == (shape[0], 1) and got.dtype == torch.float32
    d = a.cpu().double().numpy().reshape(shape[0], -1) - b.cpu().double().numpy().reshape(shape[0], -1)
    want = (20 * np.log10(1.0 / np.sqrt((d * d).sum(1) / d.shape[1]))).astype(np.float32)
    assert np.array_equal(got.cpu().numpy()[:, 0], want)
    ref = 20 * torch.log10(1.0 / torch.sqrt(((a - b) ** 2).view(shape[0], -1).mean(1, keepdim=True)))
    err = (got.double() - ref.double()).abs().max().item()
    assert err <= 10 / math.log(10) * 64 * 2.0 ** -24 + 4 * 2.0 ** -24 * float(ref.abs().max()), err


def test_psnr_identical_is_inf(cuda_lib):
    from diff_surfel_rasterization.metrics import psnr
    a = torch.rand((1, 3, 20, 20), device="cuda")
    assert torch.isinf(psnr(a, a.clone())).all()


# ---- SSIM ----

@pytest.mark.parametrize("shape", [(1, 3, 37, 53), (3, 64, 48), (1, 3) + M360[0]])
def test_ssim_within_fused_loss_bound(cuda_lib, shape):
    from diff_surfel_rasterization.loss import l1_ssim_loss
    from diff_surfel_rasterization.metrics import ssim
    g = torch.Generator().manual_seed(7)
    gt = torch.rand(shape, generator=g)
    img = (gt + 0.1 * torch.randn(shape, generator=g)).clamp(0, 1)
    s = ssim(img.cuda(), gt.cuda())
    assert s.dim() == 0 and s.dtype == torch.float32
    ev, _, vb, _, _, _ = X.loss_f64(img, gt, 1.0, dev="cuda")           # 1 - mean SSIM and its bound (units of u)
    assert abs((1.0 - float(s)) - ev) <= vb * X.U + 2.0 ** -24
    loss = float(l1_ssim_loss(img.cuda(), gt.cuda(), 1.0))             # its SSIM term, from the same double sum
    assert abs(loss - (1.0 - float(s))) <= 2.0 ** -23


# ---- layers ----

def _layer_check(lib, lpips, weights, x, label):
    """Every conv layer fed the float64 activation rounded to float32, against its per-output bound; pools exact."""
    vgg, _ = weights
    layers64 = R.conv_layers(vgg, torch.float64, "cuda")
    cur = R.zscore(x.double())
    worst, li = [], 0
    for k, n in enumerate(R.BLOCKS):
        for _ in range(n):
            w32, b32 = vgg[f"features.{R.CONV_INDICES[li]}.weight"].cuda(), vgg[f"features.{R.CONV_INDICES[li]}.bias"].cuda()
            xin = cur.float()
            got = _conv(lib, lpips.layers[li], xin).double()
            want, bound = R.conv_bound(xin, w32, b32)
            ratio = ((got - want).abs() / bound.clamp_min(1e-300)).max().item()
            worst.append(ratio)
            assert ratio <= 1.0, f"{label} conv{li}: error/bound {ratio}"
            w64, b64 = layers64[li]
            cur = F.relu(F.conv2d(cur, w64, b64, padding=1))
            li += 1
        if k + 1 < len(R.BLOCKS):
            c32 = cur.float()
            assert torch.equal(_pool(lib, c32), F.max_pool2d(c32, 2, 2)), f"{label} pool{k}"
            cur = F.max_pool2d(cur, 2, 2)
    print(f"\n{label}: per-layer worst error/bound " + " ".join(f"{r:.3f}" for r in worst))
    return worst


@pytest.mark.parametrize("hw", [(37, 53), (16, 16), (35, 17), M360[0]])
def test_conv_layers_within_bound(cuda_lib, lpips, weights, hw):
    x = torch.cat(_pairs(*hw, seed=hw[0])[1], 0)          # render and gt as the batch of two
    _layer_check(cuda_lib, lpips, weights, x, f"{hw[0]}x{hw[1]}")


def test_tap_kernel_within_bound(cuda_lib, lpips, weights):
    lib = cuda_lib
    _, lin = weights
    u = 2.0 ** -24
    for k, (c, (h, w)) in enumerate(zip(R.TAP_CHANNELS, ((61, 45), (30, 22), (15, 11), (7, 5), (3, 2)))):
        g = torch.Generator().manual_seed(k)
        f = F.relu(torch.randn((2, c, h, w), generator=g)).cuda()
        f[0, :, 0, 0] = 0                                # a zero-norm pixel: the eps path
        f[1, :, 0, 0] = 0
        partials = torch.empty(lib.surfel_metrics_partials_count(1), dtype=torch.float64, device="cuda")
        fn = _nhwc(f)
        for t in range(5):                               # every slot holds this tap; taps[0] below is its mean
            assert lib.surfel_metrics_lpips_tap(t, h, w, c, fn.data_ptr(), lpips.lin[k].data_ptr(),
                                                partials.data_ptr(), None) == 0
        taps = torch.empty(5, device="cuda")
        out = torch.empty(1, device="cuda")
        pix = (ctypes.c_longlong * 5)(*([h * w] * 5))
        assert lib.surfel_metrics_lpips_finish(pix, partials.data_ptr(), out.data_ptr(), taps.data_ptr(), None) == 0
        f64 = f.double()
        a, b = R.normalize(f64[:1]), R.normalize(f64[1:])
        wl = lin[f"lin{k}.model.1.weight"].double().cuda()
        want = float(((a - b) ** 2 * wl).sum(1).mean())
        e = (c + 8) * u
        bound = float((wl * (2 * (a - b).abs() * e * (a.abs() + b.abs()) + e * (a - b) ** 2)).sum(1).mean()) \
            + u * abs(want)
        assert abs(float(taps[0]) - want) <= bound, (k, float(taps[0]), want, bound)


# ---- end to end ----

def _e2e(lpips, weights, pairs):
    rows = []
    for x, y in pairs:
        f64 = R.lpips_f64(x, y, *weights, device="cuda")[0]
        dev = float(lpips(x, y))
        tf32 = _cudnn_lpips(x, y, weights, True)
        fp32 = _cudnn_lpips(x, y, weights, False)
        rows.append((tuple(x.shape[-2:]), f64, dev - f64, tf32 - f64, fp32 - f64))
    print("\n  H x W        lpips f64    device-f64   cudnnTF32-f64  cudnnFP32-f64")
    for hw, f64, d, t, s in rows:
        print(f"  {hw[0]:4d}x{hw[1]:<5d}  {f64:.8f}  {d:+.3e}   {t:+.3e}     {s:+.3e}")
    dmax = max(abs(r[2]) for r in rows)
    tmax = max(abs(r[3]) for r in rows)
    print(f"  max |device - f64| = {dmax:.3e}, max |cuDNN TF32 - f64| = {tmax:.3e}")
    return dmax, tmax


def test_lpips_m360_within_twice_cudnn_tf32(cuda_lib, lpips, weights):
    pairs = [p for i, hw in enumerate(M360) for p in _pairs(*hw, seed=100 + i)]
    dmax, tmax = _e2e(lpips, weights, pairs)
    assert dmax <= 2 * tmax


def test_lpips_golden(cuda_lib, lpips, weights):
    z = np.load(GOLDEN)
    names = [str(n) for n in z["names"]]
    pairs, f64s = [], []
    for n in names:
        x = torch.from_numpy(z[f"{n}/render"]).cuda()
        y = torch.from_numpy(z[f"{n}/gt"]).cuda()
        got = lpips(x, y)
        assert got.shape == (1, 1, 1, 1) and got.dtype == torch.float32
        if n.startswith("identical"):
            assert float(got) == 0.0
        else:
            pairs.append((x, y))
            f64s.append(float(z[f"{n}/lpips_f64"]))
    dmax, tmax = _e2e(lpips, weights, pairs)
    for (x, y), want in zip(pairs, f64s):                 # the golden's float64 module agrees with the restatement
        assert abs(R.lpips_f64(x, y, *weights)[0] - want) <= 1e-12
    assert dmax <= 2 * tmax


def test_lpips_identical_is_zero(cuda_lib, lpips):
    x = torch.rand((1, 3, 40, 33), device="cuda")
    assert float(lpips(x, x.clone())) == 0.0


def test_lpips_repeatable_stream_shape_and_inputs(cuda_lib, lpips):
    (x, y), = _pairs(96, 80, seed=5)[1:]
    x0, y0 = x.clone(), y.clone()
    a = lpips(x, y)
    b = lpips(x[0], y[0])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        c = lpips(x, y)
    s.synchronize()
    assert torch.equal(a, b) and torch.equal(a, c) and torch.equal(a, lpips(x, y))
    assert torch.equal(x, x0) and torch.equal(y, y0)


def test_rejects_bad_arguments(cuda_lib, lpips):
    from diff_surfel_rasterization.metrics import LPIPS, psnr, ssim
    x = torch.rand((1, 3, 32, 32), device="cuda")
    with pytest.raises(ValueError):
        lpips(x[:, :, :15], x[:, :, :15])
    with pytest.raises(ValueError):
        lpips(x.repeat(2, 1, 1, 1), x.repeat(2, 1, 1, 1))
    with pytest.raises(ValueError):
        lpips(x[:, :2], x[:, :2])
    with pytest.raises(TypeError):
        lpips(x.cpu(), x.cpu())
    with pytest.raises(TypeError):
        lpips(x.double(), x.double())
    with pytest.raises(ValueError):
        psnr(x, x[:, :, :5])
    with pytest.raises(TypeError):
        ssim(x.cpu(), x)
    with pytest.raises(KeyError):
        LPIPS({}, {})
