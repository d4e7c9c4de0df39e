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
from ._capi import ptr


def _check_cuda(*ts: torch.Tensor) -> None:
    if not all(t.is_cuda for t in ts):
        raise _capi.SgrError("street_gaussians_b200.losses needs CUDA tensors (there is no CPU fallback)")


class _ImageLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, gt, mask, w_l1: float, w_ssim: float, which: int):
        L = _capi.lib()
        _check_cuda(image, gt)
        img, g = _capi.f32(image), _capi.f32(gt.detach())
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
        _capi.call("sgr_image_loss", dev, Cn, H, W, ptr(img), ptr(g), ptr(m), float(w_l1), float(w_ssim), ptr(grad), ptr(scalars),
                   ptr(scratch), nbytes)
        ctx.save_for_backward(grad) if need_grad else None
        ctx.has_grad, ctx.in_dtype = need_grad, image.dtype
        return scalars[which]

    @staticmethod
    def backward(ctx, g_out):
        if not ctx.has_grad:
            return None, None, None, None, None, None
        (grad,) = ctx.saved_tensors
        return (grad * g_out).to(ctx.in_dtype), None, None, None, None, None


def _band_image(image, gt, mask, w_l1: float, w_ssim: float, band, group, rasterizer):
    from . import band_losses
    return band_losses._frame(image, gt, mask, w_l1, w_ssim, None, None, 0.0, None, None, 0.0, band, group, rasterizer)[0]


def l1_loss(network_output, gt, mask=None, *, band=None, group=None, rasterizer=None):
    """mean |network_output - gt| over the masked pixels (all pixels without a mask); inputs [C, H, W], mask [1, H, W] bool.

    band= / group=: network_output holds the rendered rows of this rank's TileRowBand (sharded.py); COLLECTIVE over `group`, the value
    is the whole frame's on every rank and the gradient covers the band's rows (band_losses.py).  rasterizer= (the
    GaussianShardedRasterizer that rendered the rows): its band, and with exchange="p2p" the halo and the sums over its peer workspace
    (band_losses.resolve)."""
    if band is not None or rasterizer is not None:
        return _band_image(network_output, gt, mask, 1.0, 0.0, band, group, rasterizer)
    return _ImageLoss.apply(network_output, gt, mask, 1.0, 0.0, 0)


def l2_loss(network_output, gt, mask=None):
    """Not on the hot path (the reference's train.py never calls it); plain torch like the reference."""
    a, b = network_output.permute(1, 2, 0), gt.permute(1, 2, 0)
    if mask is not None:
        a, b = a[mask.squeeze(0)], b[mask.squeeze(0)]
    return ((a - b) ** 2).mean()


def ssim(img1, img2, window_size=11, size_average=True, mask=None, *, band=None, group=None, rasterizer=None):
    """Mean SSIM with the reference's 11x11 / sigma 1.5 Gaussian window, zero padding and masking convention.  band= / group= as l1_loss's
    (img1 is the rendered image: its halo rows come from the ranks owning them); rasterizer= as l1_loss's."""
    if window_size != 11 or not size_average:
        raise _capi.SgrError("the fused SSIM implements the configuration the reference trains with: window_size=11, size_average=True")
    if band is not None or rasterizer is not None:
        return _band_image(img1, img2, mask, 0.0, 1.0, band, group, rasterizer)
    return _ImageLoss.apply(img1, img2, mask, 0.0, 1.0, 0)


def photometric_loss(image, gt, mask=None, lambda_l1: float = 1.0, lambda_dssim: float = 0.2, *, band=None, group=None, rasterizer=None):
    """(1 - lambda_dssim) * lambda_l1 * L1 + lambda_dssim * (1 - SSIM)   (train.py:101-104), one fused evaluation.  band= / group= as
    l1_loss's (and rasterizer=); band_losses.frame_losses evaluates it with the sky and object-accumulation losses under one all-reduce."""
    if band is not None or rasterizer is not None:
        return _band_image(image, gt, mask, (1.0 - lambda_dssim) * lambda_l1, -lambda_dssim, band, group, rasterizer) + lambda_dssim
    return _ImageLoss.apply(image, gt, mask, (1.0 - lambda_dssim) * lambda_l1, -lambda_dssim, 0) + lambda_dssim


class _AccLoss(torch.autograd.Function):
    """A per-pixel loss of an accumulation map selected by a bool mask: sgr_sky_loss or sgr_obj_acc_loss (same C signature)."""
    @staticmethod
    def forward(ctx, acc, flag_mask, weight: float, entry: str):
        _check_cuda(acc)
        a = _capi.f32(acc)
        dev = a.device
        m = flag_mask.reshape(-1).to(device=dev, dtype=torch.uint8).contiguous()
        if m.numel() != a.numel():
            raise ValueError(f"the mask of {entry} must have the shape of acc")
        need_grad = acc.requires_grad
        grad = torch.empty_like(a) if need_grad else None
        scalars = torch.empty(2, device=dev, dtype=torch.float32)
        scratch = torch.empty(64, device=dev, dtype=torch.uint8)
        _capi.call(entry, dev, a.numel(), ptr(a), ptr(m), float(weight), ptr(grad), ptr(scalars), ptr(scratch))
        ctx.save_for_backward(grad) if need_grad else None
        ctx.has_grad, ctx.in_dtype = need_grad, acc.dtype
        return scalars[0]

    @staticmethod
    def backward(ctx, g_out):
        if not ctx.has_grad:
            return None, None, None, None
        (grad,) = ctx.saved_tensors
        return (grad * g_out).to(ctx.in_dtype), None, None, None


def sky_loss(acc, sky_mask, weight: float = 1.0, *, band=None, group=None, rasterizer=None):
    """weight * mean( sky ? -log(1 - acc) : -log(acc) ) with acc clamped to [1e-6, 1 - 1e-6]   (train.py:107-113).  band= / group= as
    l1_loss's (and rasterizer=), acc [1, H, W]."""
    if band is not None or rasterizer is not None:
        from . import band_losses
        return band_losses.frame_losses(acc=acc, sky_mask=sky_mask, sky_weight=weight, band=band, group=group, rasterizer=rasterizer)["sky"]
    return _AccLoss.apply(acc, sky_mask, weight, "sgr_sky_loss")


def obj_acc_loss(acc_obj, obj_bound, weight: float = 1.0, *, band=None, group=None, rasterizer=None):
    """weight * mean( obj_bound ? -(a log a + (1 - a) log(1 - a)) : -log(1 - a) ), a = acc_obj clamped to [1e-6, 1 - 1e-6]
    (train.py:114-122).  acc_obj is the accumulation of the objects-only render (render_object), [1, H, W]; obj_bound bool [1, H, W].
    band= / group= / rasterizer= as l1_loss's."""
    if band is not None or rasterizer is not None:
        from . import band_losses
        return band_losses.frame_losses(acc_obj=acc_obj, obj_bound=obj_bound, obj_weight=weight, band=band, group=group,
                                        rasterizer=rasterizer)["obj_acc"]
    return _AccLoss.apply(acc_obj, obj_bound, weight, "sgr_obj_acc_loss")


class _LidarDepthLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, acc, lidar_depth, mask, weight: float, keep: float):
        L = _capi.lib()
        _check_cuda(depth, acc, lidar_depth)
        d, a, ld = _capi.f32(depth), _capi.f32(acc), _capi.f32(lidar_depth.detach())
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
        _capi.call("sgr_lidar_depth_loss", dev, N, ptr(d), ptr(a), ptr(ld), ptr(m), float(keep), float(weight), ptr(g_depth), ptr(g_acc),
                   ptr(scalars), ptr(scratch), nbytes)
        ctx.save_for_backward(g_depth, g_acc)
        ctx.dtypes = (depth.dtype, acc.dtype)
        return scalars[0]

    @staticmethod
    def backward(ctx, g_out):
        g_depth, g_acc = ctx.saved_tensors
        gd = (g_depth * g_out).to(ctx.dtypes[0]) if g_depth is not None else None
        ga = (g_acc * g_out).to(ctx.dtypes[1]) if g_acc is not None else None
        return gd, ga, None, None, None, None


def lidar_depth_loss(depth, acc, lidar_depth, mask=None, weight: float = 1.0, keep: float = 0.95, *, band=None, group=None,
                     rasterizer=None):
    """weight * mean of the int(keep * n) smallest |depth / (acc + 1e-10) - lidar_depth| over the n pixels with lidar_depth > 0 and
    mask (train.py:124-132); depth, acc, lidar_depth [1, H, W], mask bool [1, H, W] or None.

    Pass the UNCLAMPED accumulation, render_pkg['acc'], as the reference does at train.py:127 - not the copy the sky loss clamped at
    :107.  The selection runs on the device: no boolean index, no host-side k, no synchronisation, so the call can be captured in a
    CUDA graph.  Differentiable w.r.t. depth and acc; of the pixels tied at the k-th error, the lowest flat indices are taken.  With
    k == 0 (fewer than two valid pixels at keep = 0.95) the value is NaN and both gradients are zero, like the reference.

    band= / group=: depth and acc hold the rendered rows of this rank's TileRowBand; COLLECTIVE over `group` (four small all-reduces of
    the select's histograms and sums), the selected pixels and the value are the whole frame's (band_losses.py).  rasterizer= as
    l1_loss's: with exchange="p2p" the four sums go over its peer workspace."""
    if band is not None or rasterizer is not None:
        from . import band_losses
        return band_losses.lidar_depth_loss(depth, acc, lidar_depth, mask, weight, keep, band=band, group=group, rasterizer=rasterizer)
    return _LidarDepthLoss.apply(depth, acc, lidar_depth, mask, weight, keep)
