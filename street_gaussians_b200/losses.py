"""Image-space losses of the training step (SURVEY.md §8 row f2) over sgr_image_loss / sgr_sky_loss / sgr_obj_acc_loss /
sgr_lidar_depth_loss (include/sgr.h).

Same signatures as the reference's lib/utils/loss_utils.py so `from street_gaussians_b200.losses import l1_loss, ssim` replaces
`from lib.utils.loss_utils import l1_loss, ssim` (train.py:16) unchanged:
    l1_loss(network_output, gt, mask=None)                                   loss_utils.py:21-37
    ssim(img1, img2, window_size=11, size_average=True, mask=None)            loss_utils.py:91-126
and the fused form of train.py:101-104,
    photometric_loss(image, gt, mask, lambda_l1, lambda_dssim) = (1 - l) * l1w * L1 + l * (1 - SSIM),
which produces the value and dL/dimage in two kernels; `sky_loss(acc, sky_mask, weight)` is train.py:107-113,
`obj_acc_loss(acc_obj, obj_bound, weight)` is train.py:114-122 and `lidar_depth_loss(depth, acc, lidar_depth, mask, weight, keep)`
is train.py:124-132.
The gradient image is computed in the forward call (it costs one more kernel) and handed to autograd in backward, so the
rasterizer's backward receives it without replaying ~20 PyTorch kernels.  CUDA tensors only: there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _capi
from .rasterizer import _ptr, _stream


def _prep(img: torch.Tensor) -> torch.Tensor:
    if not img.is_cuda:
        raise _capi.SgrError("street_gaussians_b200.losses needs CUDA tensors (there is no CPU fallback)")
    return img if (img.dtype == torch.float32 and img.is_contiguous()) else img.to(torch.float32).contiguous()


class _ImageLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt, mask, w_l1: float, w_ssim: float, which: int):
        L = _capi.lib()
        img, g = _prep(image), _prep(gt.detach())
        if img.dim() != 3 or img.shape != g.shape:
            raise ValueError(f"image / gt must both be [C, H, W], got {tuple(image.shape)} and {tuple(gt.shape)}")
        Cn, H, W = (int(v) for v in img.shape)
        dev = img.device
        m = None
        if mask is not None:
            m = mask.reshape(-1).to(device=dev, dtype=torch.uint8).contiguous()
            if m.numel() != H * W:
                raise ValueError("mask must be [1, H, W]")
        need_grad = image.requires_grad
        grad = torch.empty_like(img) if need_grad else None
        scalars = torch.empty(4, device=dev, dtype=torch.float32)
        nbytes = int(L.sgr_image_loss_scratch_bytes(Cn, H, W))
        scratch = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            rc = L.sgr_image_loss(Cn, H, W, _ptr(img), _ptr(g), _ptr(m), float(w_l1), float(w_ssim), _ptr(grad), _ptr(scalars), _ptr(scratch),
                                  nbytes, _stream(dev))
        _capi.check(rc, "sgr_image_loss")
        ctx.save_for_backward(grad) if need_grad else None
        ctx.has_grad, ctx.in_dtype = need_grad, image.dtype
        return scalars[which]

    @staticmethod
    def backward(ctx, g_out):
        if not ctx.has_grad:
            return None, None, None, None, None, None
        (grad,) = ctx.saved_tensors
        return (grad * g_out).to(ctx.in_dtype), None, None, None, None, None


def l1_loss(network_output, gt, mask=None):
    """mean |network_output - gt| over the masked pixels (all pixels without a mask); inputs [C, H, W], mask [1, H, W] bool."""
    return _ImageLoss.apply(network_output, gt, mask, 1.0, 0.0, 0)


def l2_loss(network_output, gt, mask=None):
    """Not on the hot path (the reference's train.py never calls it); plain torch like the reference."""
    a, b = network_output.permute(1, 2, 0), gt.permute(1, 2, 0)
    if mask is not None:
        a, b = a[mask.squeeze(0)], b[mask.squeeze(0)]
    return ((a - b) ** 2).mean()


def ssim(img1, img2, window_size=11, size_average=True, mask=None):
    """Mean SSIM with the reference's 11x11 / sigma 1.5 Gaussian window, zero padding and masking convention."""
    if window_size != 11 or not size_average:
        raise _capi.SgrError("the fused SSIM implements the configuration the reference trains with: window_size=11, size_average=True")
    return _ImageLoss.apply(img1, img2, mask, 0.0, 1.0, 0)


def photometric_loss(image, gt, mask=None, lambda_l1: float = 1.0, lambda_dssim: float = 0.2):
    """(1 - lambda_dssim) * lambda_l1 * L1 + lambda_dssim * (1 - SSIM)   (train.py:101-104), one fused evaluation."""
    return _ImageLoss.apply(image, gt, mask, (1.0 - lambda_dssim) * lambda_l1, -lambda_dssim, 0) + lambda_dssim


class _AccLoss(torch.autograd.Function):
    """A per-pixel loss of an accumulation map selected by a bool mask: sgr_sky_loss or sgr_obj_acc_loss (same C signature)."""
    @staticmethod
    def forward(ctx, acc, flag_mask, weight: float, entry: str):
        L = _capi.lib()
        a = _prep(acc)
        dev = a.device
        m = flag_mask.reshape(-1).to(device=dev, dtype=torch.uint8).contiguous()
        if m.numel() != a.numel():
            raise ValueError(f"the mask of {entry} must have the shape of acc")
        need_grad = acc.requires_grad
        grad = torch.empty_like(a) if need_grad else None
        scalars = torch.empty(2, device=dev, dtype=torch.float32)
        scratch = torch.empty(64, device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            rc = getattr(L, entry)(a.numel(), _ptr(a), _ptr(m), float(weight), _ptr(grad), _ptr(scalars), _ptr(scratch), _stream(dev))
        _capi.check(rc, entry)
        ctx.save_for_backward(grad) if need_grad else None
        ctx.has_grad, ctx.in_dtype = need_grad, acc.dtype
        return scalars[0]

    @staticmethod
    def backward(ctx, g_out):
        if not ctx.has_grad:
            return None, None, None, None
        (grad,) = ctx.saved_tensors
        return (grad * g_out).to(ctx.in_dtype), None, None, None


def sky_loss(acc, sky_mask, weight: float = 1.0):
    """weight * mean( sky ? -log(1 - acc) : -log(acc) ) with acc clamped to [1e-6, 1 - 1e-6]   (train.py:107-113)."""
    return _AccLoss.apply(acc, sky_mask, weight, "sgr_sky_loss")


def obj_acc_loss(acc_obj, obj_bound, weight: float = 1.0):
    """weight * mean( obj_bound ? -(a log a + (1 - a) log(1 - a)) : -log(1 - a) ), a = acc_obj clamped to [1e-6, 1 - 1e-6]
    (train.py:114-122).  acc_obj is the accumulation of the objects-only render (render_object), [1, H, W]; obj_bound bool [1, H, W]."""
    return _AccLoss.apply(acc_obj, obj_bound, weight, "sgr_obj_acc_loss")


class _LidarDepthLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, acc, lidar_depth, mask, weight: float, keep: float):
        L = _capi.lib()
        d, a, ld = _prep(depth), _prep(acc), _prep(lidar_depth.detach())
        N = d.numel()
        if a.numel() != N or ld.numel() != N:
            raise ValueError(f"depth, acc and lidar_depth must have one shape, got {tuple(depth.shape)}, {tuple(acc.shape)}, "
                             f"{tuple(lidar_depth.shape)}")
        dev = d.device
        m = None
        if mask is not None:
            m = mask.reshape(-1).to(device=dev, dtype=torch.uint8).contiguous()
            if m.numel() != N:
                raise ValueError("mask must have the shape of depth")
        need_d, need_a = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        g_depth = torch.empty_like(d) if need_d else None
        g_acc = torch.empty_like(a) if need_a else None
        scalars = torch.empty(4, device=dev, dtype=torch.float32)
        nbytes = int(L.sgr_lidar_depth_loss_scratch_bytes(N))
        scratch = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            rc = L.sgr_lidar_depth_loss(N, _ptr(d), _ptr(a), _ptr(ld), _ptr(m), float(keep), float(weight), _ptr(g_depth), _ptr(g_acc),
                                        _ptr(scalars), _ptr(scratch), nbytes, _stream(dev))
        _capi.check(rc, "sgr_lidar_depth_loss")
        ctx.save_for_backward(g_depth, g_acc)
        ctx.dtypes = (depth.dtype, acc.dtype)
        return scalars[0]

    @staticmethod
    def backward(ctx, g_out):
        g_depth, g_acc = ctx.saved_tensors
        gd = (g_depth * g_out).to(ctx.dtypes[0]) if g_depth is not None else None
        ga = (g_acc * g_out).to(ctx.dtypes[1]) if g_acc is not None else None
        return gd, ga, None, None, None, None


def lidar_depth_loss(depth, acc, lidar_depth, mask=None, weight: float = 1.0, keep: float = 0.95):
    """weight * mean of the int(keep * n) smallest |depth / (acc + 1e-10) - lidar_depth| over the n pixels with lidar_depth > 0 and
    mask (train.py:124-132); depth, acc, lidar_depth [1, H, W], mask bool [1, H, W] or None.

    Pass the UNCLAMPED accumulation, render_pkg['acc'], as the reference does at train.py:127 - not the copy the sky loss clamped at
    :107.  The selection runs on the device: no boolean index, no host-side k, no synchronisation, so the call can be captured in a
    CUDA graph.  Differentiable w.r.t. depth and acc; of the pixels tied at the k-th error, the lowest flat indices are taken.  With
    k == 0 (fewer than two valid pixels at keep = 0.95) the value is NaN and both gradients are zero, like the reference."""
    return _LidarDepthLoss.apply(depth, acc, lidar_depth, mask, weight, keep)
