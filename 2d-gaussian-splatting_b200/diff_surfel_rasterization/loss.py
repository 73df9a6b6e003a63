"""Opt-in fused photometric loss (SURVEY §8(f) row f2).

`l1_ssim_loss(image, gt, lambda_dssim)` == (1 - l) * l1_loss(image, gt) + l * (1 - ssim(image, gt))
of the reference (/root/reference/train.py:73-74, /root/reference/utils/loss_utils.py:6-7, :43-73),
computed by one CUDA kernel forward and one backward (csrc/loss.cu) instead of 5 grouped conv2d and
~15 elementwise kernels each way.  Gradient flows to `image` only (gt is data).

Like the reference's l1_loss and ssim, it takes (C,H,W) or batched (..., C,H,W) input: every leading
dimension is folded into the channels (SSIM is per channel either way) and both means run over all
elements.
"""
import torch

from . import _cabi


class _L1SSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt, lam):
        lib = _cabi.load()
        if not image.is_cuda:
            raise RuntimeError("l1_ssim_loss: image must be a CUDA tensor (no CPU path)")
        if not torch.is_tensor(gt) or not gt.is_cuda or gt.device != image.device:
            raise RuntimeError(f"l1_ssim_loss: gt must be a CUDA tensor on {image.device}")
        if gt.shape != image.shape:
            raise RuntimeError(f"l1_ssim_loss: gt shape {tuple(gt.shape)} != image shape {tuple(image.shape)}")
        if image.dim() < 3 or image.numel() == 0:
            raise RuntimeError(f"l1_ssim_loss: expected a non-empty (..., C, H, W) image, got {tuple(image.shape)}")
        image, gt = image.contiguous().float(), gt.contiguous().float()
        H, W = image.shape[-2:]
        C = image.numel() // (H * W)                     # leading dimensions fold into the channels
        dev = image.device
        maps = torch.empty((3, C, H, W), device=dev)
        sums = torch.empty(2, dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            _cabi.check(lib.surfel_l1_ssim_forward(C, H, W, image.data_ptr(), gt.data_ptr(), maps[0].data_ptr(),
                                                   maps[1].data_ptr(), maps[2].data_ptr(), sums.data_ptr(),
                                                   torch.cuda.current_stream(dev).cuda_stream))
        n = float(image.numel())
        ctx.save_for_backward(image, gt, maps)
        ctx.consts = (float(lam), n)
        return ((1.0 - lam) * sums[0] / n + lam * (1.0 - sums[1] / n)).float()

    @staticmethod
    def backward(ctx, g):
        lib = _cabi.load()
        image, gt, maps = ctx.saved_tensors
        lam, n = ctx.consts
        H, W = image.shape[-2:]
        C = image.numel() // (H * W)
        dev = image.device
        gscale = torch.stack([g * ((1.0 - lam) / n), g * (-lam / n)]).float().contiguous()
        g_img = torch.empty_like(image)
        with torch.cuda.device(dev):
            _cabi.check(lib.surfel_l1_ssim_backward(C, H, W, image.data_ptr(), gt.data_ptr(), maps[0].data_ptr(),
                                                    maps[1].data_ptr(), maps[2].data_ptr(), gscale.data_ptr(),
                                                    g_img.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        return g_img, None, None


def l1_ssim_loss(image, gt, lambda_dssim=0.2):
    """image, gt: (C,H,W) or (..., C,H,W) CUDA float tensors of one shape, in [0,1] -> scalar loss."""
    return _L1SSIM.apply(image, gt, float(lambda_dssim))
