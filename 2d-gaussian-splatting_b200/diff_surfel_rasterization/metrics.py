"""Novel-view metrics of the reference's metrics.py on the device (csrc/metrics.cu, DESIGN.md §7o):

    psnr(render, gt)          # utils/image_utils.psnr: (N,1) float32
    ssim(render, gt)          # utils/loss_utils.ssim: scalar float32 (the fused loss kernel's SSIM sum)
    lpips = LPIPS.load()      # lpipsPyTorch's LPIPS('vgg'): VGG-16 trunk to relu5_3, packed to the device once
    lpips(render, gt)         # (1,1,1,1) float32

Inputs are CUDA float32 images in [0,1], (1,3,H,W) or (3,H,W), taken as given: LPIPS z-scores them with the
constants built for [-1,1] input, as metrics.py does.  The convolutions run on TF32 tensor cores, the precision the
reference's cuDNN convolutions use on an H100 at torch's defaults.  Forward only; no CPU path.
"""
import ctypes
import os

import torch

from . import _cabi

# torchvision vgg16().features: conv layers by module index, (cin, cout); a tap ends each block
CONV_INDICES = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
CONV_CHANNELS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256),
                 (256, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512))
BLOCKS = (2, 2, 3, 3, 3)                        # convs per block; a 2x2 pool follows every block but the last
TAP_CHANNELS = (64, 128, 256, 512, 512)
VGG_FILE = "vgg16-397923af.pth"                 # torchvision's VGG16_Weights.IMAGENET1K_V1
LIN_FILE = "vgg.pth"                            # LPIPS v0.1 lin weights, as lpipsPyTorch caches them


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _images(who, a, b):
    for name, t in (("img1", a), ("img2", b)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise TypeError(f"{who}: {name} must be a CUDA tensor (there is no CPU path)")
        if t.dtype != torch.float32:
            raise TypeError(f"{who}: {name} must be float32, got {t.dtype}")
    if a.shape != b.shape or a.device != b.device:
        raise ValueError(f"{who}: shapes {tuple(a.shape)} and {tuple(b.shape)} on {a.device}, {b.device} differ")
    if a.dim() < 1 or a.numel() == 0:
        raise ValueError(f"{who}: empty input {tuple(a.shape)}")
    return a.contiguous(), b.contiguous()


def psnr(img1, img2):
    """20 log10(1 / sqrt(mse)) per leading index: (N,1) float32, the mean squared error summed in double."""
    a, b = _images("psnr", img1, img2)
    lib = _cabi.load()
    n = a.shape[0]
    dev = a.device
    partials = torch.empty(lib.surfel_metrics_partials_count(n), dtype=torch.float64, device=dev)
    out = torch.empty((n, 1), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _cabi.check(lib.surfel_metrics_psnr(n, a.numel() // n, a.data_ptr(), b.data_ptr(), partials.data_ptr(),
                                            out.data_ptr(), _stream(dev)))
    return out


def ssim(img1, img2):
    """Mean SSIM (11x11 Gaussian, sigma 1.5, zero padding, per channel) over every element: a 0-d float32 tensor.
    (C,H,W) or (..., C,H,W); leading dimensions fold into the channels."""
    a, b = _images("ssim", img1, img2)
    if a.dim() < 3:
        raise ValueError(f"ssim: expected (..., C, H, W), got {tuple(a.shape)}")
    lib = _cabi.load()
    H, W = a.shape[-2:]
    C = a.numel() // (H * W)
    dev = a.device
    maps = torch.empty((3, C, H, W), device=dev)
    sums = torch.empty(2, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _cabi.check(lib.surfel_l1_ssim_forward(C, H, W, a.data_ptr(), b.data_ptr(), maps[0].data_ptr(),
                                               maps[1].data_ptr(), maps[2].data_ptr(), sums.data_ptr(), _stream(dev)))
    return (sums[1] / float(a.numel())).float()


class LPIPS:
    """LPIPS v0.1 with the VGG-16 trunk.  vgg_state_dict: torchvision's keys `features.{i}.weight` / `.bias` for
    the 13 convolutions; lin_state_dict: LPIPS's keys `lin{k}.model.1.weight` (1, C_k, 1, 1).  Both are packed to
    `device` (default: the current CUDA device) once."""

    def __init__(self, vgg_state_dict, lin_state_dict, device=None):
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise TypeError("LPIPS: device must be a CUDA device (there is no CPU path)")
        lib = _cabi.load()
        self.layers = []
        with torch.no_grad(), torch.cuda.device(self.device):
            for idx, (cin, cout) in zip(CONV_INDICES, CONV_CHANNELS):
                w = _param(vgg_state_dict, f"features.{idx}.weight", (cout, cin, 3, 3)).to(self.device)
                b = _param(vgg_state_dict, f"features.{idx}.bias", (cout,)).to(self.device).contiguous()
                packed = torch.empty((cout, 3, 3, cin), dtype=torch.float32, device=self.device)
                _cabi.check(lib.surfel_metrics_pack_conv(cout, cin, w.contiguous().data_ptr(), packed.data_ptr(),
                                                         _stream(self.device)))
                self.layers.append((cin, cout, packed, b))
            self.lin = [_param(lin_state_dict, f"lin{k}.model.1.weight", (1, c, 1, 1)).reshape(c)
                        .to(self.device).contiguous() for k, c in enumerate(TAP_CHANNELS)]
        torch.cuda.current_stream(self.device).synchronize()   # the state dicts' tensors may be freed after this

    @classmethod
    def load(cls, vgg_path=None, lin_path=None, device=None):
        """Read torchvision's vgg16-397923af.pth and LPIPS's vgg.pth (default: under torch.hub.get_dir()/checkpoints,
        where the reference's metrics.py leaves them).  Never downloads."""
        ckpt = os.path.join(torch.hub.get_dir(), "checkpoints")
        paths = [vgg_path or os.path.join(ckpt, VGG_FILE), lin_path or os.path.join(ckpt, LIN_FILE)]
        for p in paths:
            if not os.path.isfile(p):
                raise FileNotFoundError(f"LPIPS.load: weights file {p} not found (it is never downloaded)")
        vgg, lin = (torch.load(p, map_location="cpu", weights_only=True) for p in paths)
        return cls(vgg, lin, device)

    def __call__(self, x, y):
        """LPIPS(x, y) of one image pair, (1,3,H,W) or (3,H,W) float32 in [0,1]: a (1,1,1,1) float32 tensor."""
        x, y = _images("LPIPS", x, y)
        if x.device != self.device:
            raise ValueError(f"LPIPS: input on {x.device}, weights on {self.device}")
        if x.dim() == 4:
            if x.shape[0] != 1:
                raise ValueError(f"LPIPS: batch of {x.shape[0]} images; pass one pair at a time")
            x, y = x[0], y[0]
        if x.dim() != 3 or x.shape[0] != 3:
            raise ValueError(f"LPIPS: expected (1,3,H,W) or (3,H,W), got {tuple(x.shape)}")
        lib = _cabi.load()
        H, W = x.shape[1:]
        lo, hi = lib.surfel_metrics_min_side(), lib.surfel_metrics_max_side()
        if not (lo <= H <= hi and lo <= W <= hi):
            raise ValueError(f"LPIPS: image {H}x{W}: each side must be in [{lo}, {hi}] (the four pools before "
                             f"conv5 need a side of at least {lo})")
        dev, st = self.device, _stream(self.device)
        out = torch.empty((1, 1, 1, 1), dtype=torch.float32, device=dev)
        with torch.no_grad(), torch.cuda.device(dev):
            cur = torch.empty((2, H, W, 3), device=dev)
            _cabi.check(lib.surfel_metrics_lpips_input(1, 3, H, W, x.data_ptr(), y.data_ptr(), cur.data_ptr(), st))
            big = 2 * H * W * 64                                # the largest activation: conv1 at full size
            bufs = [torch.empty(big, device=dev), torch.empty(big, device=dev)]
            partials = torch.empty(lib.surfel_metrics_partials_count(1), dtype=torch.float64, device=dev)
            pixels = (ctypes.c_longlong * 5)()
            layers = iter(self.layers)
            h, w, which = H, W, 0
            for k, nconv in enumerate(BLOCKS):
                for _ in range(nconv):
                    cin, cout, packed, bias = next(layers)
                    nxt = bufs[which][:2 * h * w * cout]
                    _cabi.check(lib.surfel_metrics_conv3x3(2, h, w, cin, cout, cur.data_ptr(), packed.data_ptr(),
                                                           bias.data_ptr(), nxt.data_ptr(), st))
                    cur, which = nxt, 1 - which
                _cabi.check(lib.surfel_metrics_lpips_tap(k, h, w, cout, cur.data_ptr(), self.lin[k].data_ptr(),
                                                         partials.data_ptr(), st))
                pixels[k] = h * w
                if k + 1 < len(BLOCKS):
                    nxt = bufs[which][:2 * (h // 2) * (w // 2) * cout]
                    _cabi.check(lib.surfel_metrics_maxpool(2, h, w, cout, cur.data_ptr(), nxt.data_ptr(), st))
                    cur, which, h, w = nxt, 1 - which, h // 2, w // 2
            _cabi.check(lib.surfel_metrics_lpips_finish(pixels, partials.data_ptr(), out.data_ptr(), None, st))
        return out


def _param(sd, key, shape):
    if key not in sd:
        raise KeyError(f"LPIPS: state dict has no {key}")
    t = sd[key]
    if tuple(t.shape) != shape:
        raise ValueError(f"LPIPS: {key} has shape {tuple(t.shape)}, expected {shape}")
    return t.detach().float()
