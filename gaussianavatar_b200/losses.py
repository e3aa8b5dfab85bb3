"""Image losses with the reference's names and semantics (/root/reference utils/loss_utils.py:7-8,23-53) over the fused
sm_90a kernel, plus the combined form train.py:74-77 uses, and the masked L1 depth loss (`depth_loss`)."""
from __future__ import annotations

import torch

from . import _lib
from ._lib import ptr


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _ImageLoss(torch.autograd.Function):
    """w_l1 * L1 + w_ssim * (1 - SSIM) in one forward and one backward kernel."""

    @staticmethod
    def forward(ctx, image, gt, w_l1, w_ssim):
        if not image.is_cuda:
            raise RuntimeError("gaussianavatar_b200 losses need CUDA tensors (no CPU fallback)")
        img = image.float().contiguous()
        gtc = gt.float().contiguous()
        if img.dim() == 3:
            img, gtc = img[None], gtc[None]
        B, C, H, W = img.shape
        assert C == 3, "the fused loss is built for 3-channel images"
        L = _lib.lib()
        ws = torch.empty(L.ga_loss_workspace_bytes(B, H, W), dtype=torch.uint8, device=img.device)
        out = torch.empty(3, dtype=torch.float32, device=img.device)
        _lib.check(L.ga_loss_forward(B, H, W, ptr(img), ptr(gtc), float(w_l1), float(w_ssim), ptr(ws), ptr(out), _stream()),
                   "ga_loss_forward")
        ctx.save_for_backward(img, gtc, ws)
        ctx.w = (float(w_l1), float(w_ssim))
        ctx.in_shape = image.shape
        ctx.mark_non_differentiable(out)
        return out[0].clone(), out

    @staticmethod
    def backward(ctx, g, _g_aux):
        img, gtc, ws = ctx.saved_tensors
        B, C, H, W = img.shape
        d_img = torch.empty_like(img)
        g = g.float().contiguous()
        _lib.check(_lib.lib().ga_loss_backward(B, H, W, ptr(img), ptr(gtc), ctx.w[0], ctx.w[1], ptr(g), ptr(ws), ptr(d_img), _stream()),
                   "ga_loss_backward")
        return d_img.reshape(ctx.in_shape), None, None, None


def image_loss(image, gt, lambda_dssim: float = 0.2):
    """(1 - lambda) * l1_loss_w(image, gt) + lambda * (1 - ssim(image, gt))   (train.py:74-75), fused."""
    return _ImageLoss.apply(image, gt, 1.0 - lambda_dssim, lambda_dssim)[0]


def l1_loss_w(network_output, gt):
    """utils/loss_utils.py:7-8."""
    return _ImageLoss.apply(network_output, gt, 1.0, 0.0)[0]


def ssim(img1, img2, window_size=11, size_average=True):
    """utils/loss_utils.py:23-53 (window 11, size_average=True: the only form the reference calls)."""
    if window_size != 11 or not size_average:
        raise NotImplementedError("only ssim(window_size=11, size_average=True) is on the reference's path (train.py:75)")
    # w_l1 = 0, w_ssim = -1  ->  out = -(1 - ssim) = ssim - 1 ; add 1 back
    return _ImageLoss.apply(img1, img2, 0.0, -1.0)[0] + 1.0


class _DepthLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, target, lam):
        if not depth.is_cuda:
            raise RuntimeError("gaussianavatar_b200 losses need CUDA tensors (no CPU fallback)")
        d = depth.float().contiguous()
        if d.dim() != 4 or d.shape[1] != 2:
            raise ValueError(f"depth must be [B,2,H,W] (mean, median), got {tuple(depth.shape)}")
        B, _, H, W = d.shape
        t = target.to(device=d.device, dtype=torch.float32).reshape(B, H, W).contiguous()
        L = _lib.lib()
        ws = torch.empty(L.ga_depth_loss_workspace_bytes(B, H, W), dtype=torch.uint8, device=d.device)
        out = torch.empty(2, dtype=torch.float32, device=d.device)
        _lib.check(L.ga_depth_loss_forward(B, H, W, ptr(d), ptr(t), float(lam), ptr(ws), ws.numel(), ptr(out), _stream()),
                   "ga_depth_loss_forward")
        ctx.save_for_backward(d, t, ws)
        ctx.mark_non_differentiable(out)
        return out[0].clone(), out

    @staticmethod
    def backward(ctx, g, _g_aux):
        d, t, ws = ctx.saved_tensors
        B, _, H, W = d.shape
        d_m = torch.empty(B, H, W, dtype=torch.float32, device=d.device)
        g = g.float().contiguous()
        _lib.check(_lib.lib().ga_depth_loss_backward(B, H, W, ptr(d), ptr(t), ptr(g), ptr(ws), ws.numel(), ptr(d_m), _stream()),
                   "ga_depth_loss_backward")
        grad = torch.zeros_like(d)
        grad[:, 0] = d_m
        return grad, None, None


def depth_loss(depth, target, lam: float = 1.0, return_count: bool = False):
    """lam / N * sum |m - target| over the pixels where target > 0 and the render is at least half opaque (plane 1 non-zero),
    N their number over the batch (0 when N = 0).  depth [B,2,H,W] from `rasterizer.rasterize_batch_with_depth` (differentiable in
    plane 0, the mean view-space z), target [B,H,W] in the same units (metres for metric captures; 0 = no measurement).  One fused
    kernel pair; N stays on the device.  return_count: also the device tensor N (float)."""
    loss, out = _DepthLoss.apply(depth, target, lam)
    return (loss, out[1]) if return_count else loss
