"""Photometric losses on the fused sm_90a kernels.

`ssim` is a drop-in for the reference's `ssim` (gaussian-splatting utils/loss_utils.py, copied into ManiGaussian's
agents/manigaussian_bc/loss.py) for images already rendered, e.g. by the single-view `render()`; `render_views(...,
ssim=True)` evaluates the same loss behind each view's blend instead.  The tiled forward and backward kernels are
manigaussian_b200/csrc/ssim.cu (C ABI mgs_ssim / mgs_ssim_backward); the definitions are in include/mgs_rasterizer.h.
"""
import torch

from . import _binding as _b


class _SSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, g):
        V, C, H, W = x.shape
        terms = torch.empty((V, 3 * C, H, W), dtype=torch.float32, device=x.device)
        acc = torch.empty((V, 2), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            stream = torch.cuda.current_stream(x.device).cuda_stream
            _b.check(_b.lib().mgs_ssim(V, C, H, W, x.data_ptr(), g.data_ptr(), terms.data_ptr(), acc.data_ptr(), stream), "mgs_ssim")
        ctx.save_for_backward(x, g, terms)
        return acc[:, 1].sum() / float(V * C * H * W)

    @staticmethod
    def backward(ctx, grad):
        x, g, terms = ctx.saved_tensors
        V, C, H, W = x.shape
        # the kernel's d ssim_v / dx is per image (mean over its C H W entries); the result is the mean over the V images
        gs = (grad.to(torch.float32) / V).expand(V)
        scale = torch.stack([torch.zeros_like(gs), gs], 1).contiguous()
        cot = torch.empty_like(x)
        with torch.cuda.device(x.device):
            stream = torch.cuda.current_stream(x.device).cuda_stream
            _b.check(_b.lib().mgs_ssim_backward(V, C, H, W, x.data_ptr(), g.data_ptr(), terms.data_ptr(), scale.data_ptr(), None,
                                                cot.data_ptr(), stream), "mgs_ssim_backward")
        return cot, None


def ssim(img1, img2, window_size=11, size_average=True):
    """SSIM of img1 against img2, [C,H,W] or [B,C,H,W], as the reference's ssim(img1, img2) with its defaults: every
    channel on its own, 11x11 Gaussian window (sigma 1.5), zero padding, mean over all entries.  The result is SSIM itself
    (the 3DGS objective uses 1 - ssim).  Differentiable with respect to img1 only; img2 is the target."""
    if window_size != 11:
        raise ValueError("ssim: only window_size=11 is implemented")
    if size_average is not True:
        raise ValueError("ssim: only size_average=True is implemented")
    if img2.requires_grad:
        raise ValueError("ssim: img2 is the target and must not require grad (no gradient flows to it)")
    if img1.shape != img2.shape or img1.dim() not in (3, 4):
        raise ValueError("ssim: img1 and img2 must both be [C,H,W] or [B,C,H,W] of one shape")
    if not img1.is_cuda or img2.device != img1.device:
        raise ValueError("ssim: both images must be on the same CUDA device (there is no CPU path)")
    x = img1.to(torch.float32).contiguous()
    g = img2.to(torch.float32).contiguous()
    if x.dim() == 3:
        x, g = x.unsqueeze(0), g.unsqueeze(0)
    return _SSIM.apply(x, g)
