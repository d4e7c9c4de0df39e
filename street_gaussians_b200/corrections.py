"""The per-camera colour correction of the reference (lib/models/color_correction.py, cfg.model.use_color_correction) over
sgr_color_correct_forward / sgr_color_correct_backward / sgr_color_correction_reg (include/sgr.h).

    color_correct(image, affine)                          color_correction.py:129-132, street_gaussian_renderer.py:113-114
    color_correction_reg_loss(affine, affine_sky, weight)  color_correction.py:134-140 as train.py:135-138 adds it

`affine` is the [3, 4] matrix ColorCorrection.get_affine_trans(camera) returns, in its embedding or its MLP mode (the MLP stays the
caller's torch module; its output is differentiable like any other tensor).  The background pose correction is not here: pass its
two rows to `compose(..., pose_correction=...)`.  CUDA tensors only: there is no CPU fallback.

color_correct's band= / group= (keyword-only, as in losses.py): the image holds the rendered rows of this rank's TileRowBand
(sharded.py); the band's rows are corrected (sgr_band_color_correct_*), and the backward all-reduces the band's 12 fp64 sums of
dL/daffine over `group` before rounding them, so every rank's affine gradient is the whole frame's.  rasterizer= (a
sharded.GaussianShardedRasterizer) supplies the band and the transport as in sky.py: with exchange="p2p" the 12 sums are added over
peer memory (band_losses.peer_sum on the loss section), in ascending rank order, with no NCCL call and no host read-back.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _capi
from ._capi import ptr


def _check_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise _capi.SgrError(f"street_gaussians_b200.corrections needs CUDA tensors ({what} is on {t.device}; there is no CPU fallback)")


def _affine(a: torch.Tensor, what: str, dev) -> torch.Tensor:
    if tuple(a.shape) != (3, 4):
        raise ValueError(f"{what} must be [3, 4], got {tuple(a.shape)}")
    _check_cuda(a, what)
    a = _capi.f32(a)
    if a.device != dev:
        raise ValueError(f"{what} is on {a.device}, the image on {dev}")
    return a


class _ColorCorrect(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, affine, band, xfer):
        _check_cuda(image, "image")
        img = _capi.f32(image)
        if img.dim() != 3 or img.shape[0] != 3:
            raise ValueError(f"image must be [3, H, W], got {tuple(image.shape)}")
        A = _affine(affine, "affine", img.device)
        H, W = int(img.shape[1]), int(img.shape[2])
        if band is None:
            rows = None
            out = torch.empty_like(img)
            _capi.call("sgr_color_correct_forward", img.device, H, W, ptr(img), ptr(A), ptr(out))
        else:
            from .band_losses import check_band
            rows = check_band(band, H)
            out = torch.zeros_like(img)
            _capi.call("sgr_band_color_correct_forward", img.device, H, W, *rows, ptr(img), ptr(A), ptr(out))
        ctx.save_for_backward(img, A)
        ctx.dtypes = (image.dtype, affine.dtype)
        ctx.band, ctx.xfer = rows, xfer
        return out

    @staticmethod
    def backward(ctx, g_out):
        L = _capi.lib()
        img, A = ctx.saved_tensors
        dev = img.device
        H, W = int(img.shape[1]), int(img.shape[2])
        _check_cuda(g_out, "dL/dout")
        g = _capi.f32(g_out)
        g_A = torch.empty((3, 4), device=dev, dtype=torch.float32)
        if ctx.band is None:
            g_img = torch.empty_like(img) if ctx.needs_input_grad[0] else None
            nbytes = int(L.sgr_color_correct_scratch_bytes(H, W))
            scratch = torch.empty(nbytes, device=dev, dtype=torch.uint8)
            _capi.call("sgr_color_correct_backward", dev, H, W, ptr(img), ptr(A), ptr(g), ptr(g_img), ptr(g_A), ptr(scratch), nbytes)
        else:
            g_img = torch.zeros_like(img) if ctx.needs_input_grad[0] else None
            sums = torch.empty(12, device=dev, dtype=torch.float64)
            nbytes = int(L.sgr_band_color_correct_scratch_bytes(H, W))
            scratch = torch.empty(nbytes, device=dev, dtype=torch.uint8)
            _capi.call("sgr_band_color_correct_backward", dev, H, W, *ctx.band, ptr(img), ptr(A), ptr(g), ptr(g_img), ptr(sums), ptr(scratch), nbytes)
            if ctx.needs_input_grad[1]:  # COLLECTIVE: the band's 12 sums -> the frame's, rounded once to fp32
                ctx.xfer.sum(sums)
                _capi.call("sgr_band_color_correct_affine_grad", dev, ptr(sums), ptr(g_A))
        return ((g_img.to(ctx.dtypes[0]) if g_img is not None else None), (g_A.to(ctx.dtypes[1]) if ctx.needs_input_grad[1] else None), None,
                None)


def color_correct(image: torch.Tensor, affine: torch.Tensor, *, band=None, group=None, rasterizer=None) -> torch.Tensor:
    """einsum('ij,jhw->ihw', affine[:3, :3], image) + affine[:3, 3, None, None] for image [3, H, W]; differentiable in both.

    band= / group=: image holds the rendered rows of this rank's TileRowBand (sharded.py).  The output and dL/dimage have the band's
    rows, zeros elsewhere, equal bit for bit to the whole-frame call's rows.  COLLECTIVE in the backward: the 12 fp64 sums of
    dL/daffine are all-reduced over `group` (every rank must run its backward), then rounded once, so dL/daffine is the frame's on
    every rank and does not depend on how the rows are split (it may differ from the whole-frame call's fp32-accumulated sums by
    their rounding).  An affine from the MLP mode works unchanged: its gradient flows back into the module as usual.

    rasterizer= (the GaussianShardedRasterizer that rendered the rows, whose forward must have run): its band, the whole frame at world
    1; a band= or group= that differs from its own raises ValueError.  exchange="nccl": the all-reduce above over its group.
    exchange="p2p": COLLECTIVE in the backward over its peer memory (no NCCL call, no host synchronisation); dL/daffine is the
    ascending-rank fp64 sum of the 12 partials, rounded once, the same on every rank."""
    from .sky import _resolve
    rows, xfer = _resolve(band, group, rasterizer, int(image.shape[-2]))  # a bad or mismatched band fails before anything else
    return _ColorCorrect.apply(image, affine, rows, xfer)


class _Reg(torch.autograd.Function):
    @staticmethod
    def forward(ctx, affine, affine_sky, weight: float):
        A = _affine(affine, "affine", affine.device)
        S = _affine(affine_sky, "affine_sky", A.device) if affine_sky is not None else None
        dev = A.device
        value = torch.empty((), device=dev, dtype=torch.float32)
        gA = torch.empty((3, 4), device=dev, dtype=torch.float32)
        gS = torch.empty((3, 4), device=dev, dtype=torch.float32) if S is not None else None
        _capi.call("sgr_color_correction_reg", dev, ptr(A), ptr(S), float(weight), ptr(value), ptr(gA), ptr(gS))
        ctx.save_for_backward(gA, gS if gS is not None else gA)
        ctx.has_sky = S is not None
        ctx.dtypes = (affine.dtype, affine_sky.dtype if affine_sky is not None else None)
        return value

    @staticmethod
    def backward(ctx, g_out):
        gA, gS = ctx.saved_tensors
        g_sky = (gS * g_out).to(ctx.dtypes[1]) if ctx.has_sky else None
        return (gA * g_out).to(ctx.dtypes[0]), g_sky, None


def color_correction_reg_loss(affine: torch.Tensor, affine_sky: Optional[torch.Tensor] = None, weight: float = 1.0) -> torch.Tensor:
    """weight * mean(|affine - I| + |affine_sky - I|) over the 12 entries (only |affine - I| without affine_sky): the regularisation
    train.py:135-138 adds with weight = lambda_color_correction.  Returns a 0-dim CUDA tensor; gradients reach both matrices."""
    return _Reg.apply(affine, affine_sky, weight)
