"""Restatement of the reference's novel-view metrics (metrics.py: utils/image_utils.psnr and lpipsPyTorch's
LPIPS('vgg')) for diff_surfel_rasterization.metrics (DESIGN.md §7o), and the seeded weights that stand in for the
real VGG-16 and LPIPS lin weights in the tests and in tests/golden/make_golden_metrics.py.

  * vgg_weights / lin_weights: the seeded weights under the original key names.  The conv weights are He-scaled
    normals with each filter's spatial mean removed (He init alone answers mostly to the flat z-score offset, so
    all images look alike and LPIPS lands near 1e-3); the lin weights are non-negative like LPIPS's.  Perturbed
    pairs then score in the range real LPIPS values take (about 0.05 to 0.5).
  * trunk / lpips_f64: torchvision's vgg16().features to relu5_3 in whatever dtype is given, and the tap formula
    written out: f / (sqrt(sum_c f^2) + 1e-10), (fx - fy)^2, the 1x1 lin conv without bias, the spatial mean, the
    five taps summed.
  * conv_bound: the first-order bound of one TF32 conv layer at every output, in float64.
"""
import hashlib

import numpy as np
import torch
import torch.nn.functional as F

SEED = 20261018
CONV_INDICES = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
CONV_CHANNELS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256),
                 (256, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512))
BLOCKS = (2, 2, 3, 3, 3)
TAP_CHANNELS = (64, 128, 256, 512, 512)
TARGET_MODULES = (4, 9, 16, 23, 30)            # 1-based modules of vgg16().features whose outputs are the taps
MEAN = (-.030, -.088, -.188)
STD = (.458, .448, .450)
MIN_SIDE = 16
U_TF32 = 2.0 ** -11                            # a TF32 operand rounded to nearest (10 stored bits)
U_F32 = 2.0 ** -23                             # one float32 addition, truncating


def vgg_weights(seed=SEED):
    """features.{i}.weight / .bias of the 13 convolutions, float32, from a fixed-seed CPU generator."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for idx, (cin, cout) in zip(CONV_INDICES, CONV_CHANNELS):
        w = torch.randn((cout, cin, 3, 3), generator=g, dtype=torch.float32)
        w = (w - w.mean((2, 3), keepdim=True)) * (2.0 / (9 * cin)) ** 0.5    # no response to a flat patch
        b = torch.randn((cout,), generator=g, dtype=torch.float32) * 0.05
        sd[f"features.{idx}.weight"], sd[f"features.{idx}.bias"] = w, b
    return sd


def lin_weights(seed=SEED + 1):
    """lin{k}.model.1.weight (1, C_k, 1, 1), non-negative float32, from a fixed-seed CPU generator."""
    g = torch.Generator().manual_seed(seed)
    return {f"lin{k}.model.1.weight": (torch.rand((1, c, 1, 1), generator=g, dtype=torch.float32) * (20.0 / c))
            for k, c in enumerate(TAP_CHANNELS)}


def weights_sha256(vgg, lin):
    h = hashlib.sha256()
    for sd in (vgg, lin):
        for k in sorted(sd):
            h.update(k.encode())
            h.update(np.ascontiguousarray(sd[k].numpy()).tobytes())
    return h.hexdigest()


def zscore(x):
    """(x - mean) / std with the reference's float32 buffers, in x's dtype (the buffers are float32 values)."""
    m = torch.tensor(MEAN, dtype=torch.float32).to(x)[None, :, None, None]
    s = torch.tensor(STD, dtype=torch.float32).to(x)[None, :, None, None]
    return (x - m) / s


def conv_layers(vgg, dtype, device):
    return [(vgg[f"features.{i}.weight"].to(device, dtype), vgg[f"features.{i}.bias"].to(device, dtype))
            for i in CONV_INDICES]


def trunk(x, layers):
    """vgg16().features up to relu5_3 on a z-scored (N,3,H,W) input: the five tap activations (before the norm)."""
    out, it = [], iter(layers)
    for k, n in enumerate(BLOCKS):
        for _ in range(n):
            w, b = next(it)
            x = F.relu(F.conv2d(x, w, b, padding=1))
        out.append(x)
        if k + 1 < len(BLOCKS):
            x = F.max_pool2d(x, 2, 2)
    return out


def normalize(f):
    return f / (torch.sqrt(torch.sum(f ** 2, dim=1, keepdim=True)) + 1e-10)


def tap_values(fx, fy, lin):
    """Per tap: the lin-weighted squared difference of the normalized features, averaged over pixels."""
    vals = []
    for k, (a, b) in enumerate(zip(fx, fy)):
        w = lin[f"lin{k}.model.1.weight"].to(a)
        d = (normalize(a) - normalize(b)) ** 2
        vals.append((d * w).sum(1).mean((1, 2)))
    return torch.stack(vals, 0)                   # (5, N)


def lpips_f64(x, y, vgg, lin, device="cpu"):
    """LPIPS of (1,3,H,W) images in float64: (value, five tap values, five x-tap features, five y-tap features)."""
    layers = conv_layers(vgg, torch.float64, device)
    x = zscore(x.to(device, torch.float64))
    y = zscore(y.to(device, torch.float64))
    fx, fy = trunk(x, layers), trunk(y, layers)
    taps = tap_values(fx, fy, lin)[:, 0]
    return float(taps.sum()), taps, fx, fy


def psnr_f64(a, b):
    """(N,) float64: 20 log10(1 / sqrt(mse)) with the mean squared error in float64."""
    a, b = a.double(), b.double()
    n = a.shape[0]
    mse = ((a - b) ** 2).reshape(n, -1).mean(1)
    return 20 * torch.log10(1.0 / torch.sqrt(mse))


def tf32_rna(w):
    """float32 -> TF32, to nearest with ties away from zero (cvt.rna.tf32.f32), as the packed weights are."""
    u = w.float().contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    u = (u + 0x1000) & 0xFFFFE000
    u = torch.where(u >= 2 ** 31, u - 2 ** 32, u).to(torch.int32)
    return u.view(torch.float32)


def conv_bound(x, w, b):
    """Per output of relu(conv3x3(x, w) + b) (x: float32 input as float64, w: float32 weights), in float64:
    the reference value from the TF32-rounded weights and the bound around it, 2 u_tf32 sum|w x| for the operand
    roundings to nearest (the weights' is exact in the reference value, so this over-covers), (K + 1) u_f32 (sum|w x|
    + |b|) for a truncating float32 accumulation over K = 9 Cin products and the bias, plus the rounding of the
    output.  ReLU is 1-Lipschitz, so the bound carries through it."""
    x = x.double()
    wr = tf32_rna(w).double() if w.shape[1] % 32 == 0 else w.double()
    exact = F.conv2d(x, wr, b.double(), padding=1)
    mag = F.conv2d(x.abs(), wr.abs(), None, padding=1)
    K = 9 * w.shape[1]
    tc = w.shape[1] % 32 == 0
    bound = (2 * U_TF32 * mag if tc else 0) + (K + 1) * U_F32 * (mag + b.double().abs()[None, :, None, None]) \
        + U_F32 * exact.abs()
    return F.relu(exact), bound
