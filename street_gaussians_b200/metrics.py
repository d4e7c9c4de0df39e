"""Scoring rendered views on the device: masked PSNR, SSIM and L1 per view (include/sgr.h, "Evaluation metrics").

The reference scores views with torch lines that synchronise with the host on every view: training_report (train.py:274-303) adds
`l1_loss(...).mean().double()` and `psnr(...).mean().double()` of the clamped render to Python floats, each after a boolean-index
`nonzero`, and metrics.py:76-81 takes ssim and psnr of the saved 8-bit PNGs one by one.  Here each view is three kernels that add its sums to
a device slot, and `ViewMetrics.result()` turns every slot into values with ONE host read:

    vm = ViewMetrics()                                   # training_report: clamp, masked L1 / PSNR (and SSIM of the masked images)
    for cam in cameras:
        vm.add(render(cam)["rgb"], cam.original_image, cam.original_mask)
    r = vm.result()                                      # r["mean"]["psnr"], r["psnr"][i], ...

    ViewMetrics(quantize8=True, ssim_masked=False)       # metrics.py: the save_image PNG round trip, unmasked SSIM and PSNR

On a tile-row band (the multi-GPU rasterizers return images whose rows outside the rank's band are zero), `band=` / `group=` make each
`add` fetch the rows within the SSIM window's reach from the neighbouring ranks (band_losses.exchange_halo) and `result()` sum every
slot over the ranks with one all-reduce; every rank gets the whole frame's numbers, without gathering a frame.  `rasterizer=` (the
GaussianShardedRasterizer that rendered the rows) takes its band and transport as the band losses do (band_losses.resolve): with
exchange="p2p" the halo and the sum go over the loss section of its peer workspace (sgr_band_halo_exchange_peers, sgr_band_peer_sum),
with no NCCL call.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _capi, band_losses
from ._capi import ptr


def _check_cuda(*ts) -> None:
    if not all(t.is_cuda for t in ts if t is not None):
        raise _capi.SgrError("street_gaussians_b200.metrics needs CUDA tensors (there is no CPU fallback)")


def _flags(clamp: bool, quantize8: bool, ssim_masked: bool) -> int:
    if quantize8 and not clamp:
        raise ValueError("quantize8 scores the 8-bit PNG round trip of the clamped image: it needs clamp=True")
    return (_capi.EVAL_CLAMP if clamp else 0) | (_capi.EVAL_QUANT8 if quantize8 else 0) | (_capi.EVAL_SSIM_MASKED if ssim_masked else 0)


def _mask_u8(mask, H: int, W: int, device) -> Optional[torch.Tensor]:
    """A [1, H, W] or [H, W] bool / uint8 mask (the reference's convention) as uint8 [H W] on `device`."""
    if mask is None:
        return None
    if mask.dtype not in (torch.bool, torch.uint8) or tuple(mask.shape[-2:]) != (H, W) or mask.numel() != H * W:
        raise ValueError(f"mask must be a [1, H, W] or [H, W] bool / uint8 tensor of {H}x{W}, got {mask.dtype} {tuple(mask.shape)}")
    return mask.reshape(-1).to(device=device, dtype=torch.uint8).contiguous()


def accumulate(image: torch.Tensor, gt: torch.Tensor, mask, sums: torch.Tensor, flags: int, band=None) -> None:
    """sgr_eval_metrics_accumulate / sgr_band_eval_metrics_accumulate: add the sums of the V views of image, gt [V, C, H, W] (mask
    uint8 [V, H W] or None) to sums [V, 5] float64, in place.  With a band, image holds its rows and their halo."""
    V, Cn, H, W = (int(v) for v in image.shape)
    dev = image.device
    nbytes = int(_capi.lib().sgr_eval_metrics_scratch_bytes(V, Cn, H, W))
    if nbytes == 0:
        raise ValueError(f"bad view batch {V}x{Cn}x{H}x{W} for the evaluation metrics")
    if tuple(gt.shape) != (V, Cn, H, W) or tuple(sums.shape) != (V, _capi.EVAL_SUMS) or sums.dtype != torch.float64:
        raise ValueError(f"gt {tuple(gt.shape)} / sums {tuple(sums.shape)} do not fit {V} views of {Cn}x{H}x{W}")
    if mask is not None and mask.numel() != V * H * W:
        raise ValueError(f"mask must have {V * H * W} bytes, got {mask.numel()}")
    scratch = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    if band is None:
        _capi.call("sgr_eval_metrics_accumulate", dev, V, Cn, H, W, int(flags), ptr(image), ptr(gt), ptr(mask), ptr(sums), ptr(scratch), nbytes)
    else:
        b, e, s = band_losses.check_band(band, H)
        _capi.call("sgr_band_eval_metrics_accumulate", dev, V, Cn, H, W, b, e, s, int(flags), ptr(image), ptr(gt), ptr(mask), ptr(sums),
                   ptr(scratch), nbytes)


def finish(sums: torch.Tensor) -> torch.Tensor:
    """sgr_eval_metrics_finish: [V + 1, 4] float32 on the device, rows {psnr, ssim, l1, n} per view, then {the means, V}."""
    V = int(sums.shape[0])
    out = torch.empty((V + 1, 4), device=sums.device, dtype=torch.float32)
    _capi.call("sgr_eval_metrics_finish", sums.device, V, ptr(sums), ptr(out))
    return out


@torch.no_grad()
def psnr(img1: torch.Tensor, img2: torch.Tensor, mask=None) -> torch.Tensor:
    """loss_utils.psnr on the device: img1, img2 [C, H, W], mask [1, H, W] or [H, W] (the masked pixels' elements count), no clamp.
    A 0-dim float32 tensor; +inf for identical images, NaN for an empty mask, as the reference.  No gradient."""
    _check_cuda(img1, img2)
    if img1.dim() != 3 or img1.shape != img2.shape:
        raise ValueError(f"img1 / img2 must both be [C, H, W], got {tuple(img1.shape)} and {tuple(img2.shape)}")
    dev = img1.device
    Cn, H, W = (int(v) for v in img1.shape)
    sums = torch.zeros((1, _capi.EVAL_SUMS), device=dev, dtype=torch.float64)
    accumulate(_capi.f32(img1.detach())[None], _capi.f32(img2.detach(), dev)[None], _mask_u8(mask, H, W, dev), sums, _capi.EVAL_NO_SSIM)
    return finish(sums)[0, 0]


class ViewMetrics:
    """Scores views on the device and reads them back once.

    clamp        clamp image and gt to [0, 1] first (training_report);
    quantize8    then score what a PNG written by torchvision.utils.save_image and read back by to_tensor holds (the nearest of the
                 256 levels, halves up, computed in fp32 as save_image does), the files metrics.py scores (needs clamp);
    ssim_masked  with a mask, SSIM of the images zeroed outside it (ssim(mask=)); otherwise SSIM of the whole images, as metrics.py;
    band, group  the rank's TileRowBand and process group of a multi-GPU renderer: `add` is then COLLECTIVE (a halo exchange with the
                 neighbouring ranks) and `result` COLLECTIVE (one all-reduce of every slot).
    rasterizer   the sharded.GaussianShardedRasterizer that rendered the rows instead: its band (the whole image at world 1), and with
                 exchange="p2p" the halo and the sum of the slots over the loss section of the workspace its forward set up, which
                 must hold the [V, 5] fp64 slots of `result` (ValueError otherwise); a band= or group= that differs from it raises.

    L1 and PSNR average over the masked pixels' elements (every pixel without a mask); SSIM over all pixels."""

    def __init__(self, clamp: bool = True, quantize8: bool = False, ssim_masked: bool = True, band=None, group=None, rasterizer=None):
        self.flags = _flags(clamp, quantize8, ssim_masked)
        self.band, self.group, self.rasterizer = band, group, rasterizer
        self._sums: Optional[torch.Tensor] = None
        self._n = 0
        self._H = 0  # image height of the views added (band_losses.resolve takes it for the rasterizer's band)

    def __len__(self) -> int:
        return self._n

    def _slot(self, device) -> torch.Tensor:
        if self._sums is None or self._sums.device != device:
            if self._n:
                raise ValueError("all views of one ViewMetrics must be on one device")
            self._sums = torch.zeros((16, _capi.EVAL_SUMS), device=device, dtype=torch.float64)
        if self._n == self._sums.shape[0]:  # grow by doubling; the filled slots are copied once on the device
            self._sums = torch.cat([self._sums, torch.zeros_like(self._sums)])
        self._n += 1
        return self._sums[self._n - 1:self._n]

    @torch.no_grad()
    def add(self, image: torch.Tensor, gt: torch.Tensor, mask=None) -> None:
        """Enqueue one view: image, gt [C, H, W] (with a band, image holds the rank's rows; gt and mask are whole frames), mask
        [1, H, W] / [H, W] bool or uint8 or None.  Nothing is read back."""
        _check_cuda(image, gt)
        if image.dim() != 3 or image.shape != gt.shape:
            raise ValueError(f"image / gt must both be [C, H, W], got {tuple(image.shape)} and {tuple(gt.shape)}")
        dev = image.device
        Cn, H, W = (int(v) for v in image.shape)
        band = self.band
        self._H = H
        if self.rasterizer is not None:
            band, xfer = band_losses.resolve(self.band, self.group, self.rasterizer, H)
            band_losses.check_band(band, H)
            img = xfer.halo(image.detach(), band)
        elif band is not None:
            band_losses.check_band(band, H)
            img = band_losses.exchange_halo(image.detach(), band, self.group)
        else:
            img = _capi.f32(image.detach())
        accumulate(img[None], _capi.f32(gt.detach(), dev)[None], _mask_u8(mask, H, W, dev), self._slot(dev), self.flags, band)

    @torch.no_grad()
    def result(self) -> dict:
        """The scores of the views added so far, and a fresh start: {"psnr", "ssim", "l1": float32 [V], "n": int64 [V] (masked elements),
        "mean": {"psnr", "ssim", "l1"}}, on the host after one read.  With a band, COLLECTIVE: one all-reduce of the slots (with a p2p
        rasterizer, one peer-memory sum)."""
        V, sums = self._n, self._sums
        xfer = None
        if V and self.rasterizer is not None:
            _, xfer = band_losses.resolve(self.band, self.group, self.rasterizer, self._H)
            if xfer.kind == "p2p" and V * _capi.EVAL_SUMS * 8 > xfer.ws.loss_bytes:
                raise ValueError(f"the sums of {V} views ({V * _capi.EVAL_SUMS * 8} bytes) do not fit the peer workspace's loss section of "
                                 f"{xfer.ws.loss_bytes} bytes: call result() after fewer views")
        self._sums, self._n = None, 0
        if V == 0:
            nan = float("nan")
            empty = torch.empty(0, dtype=torch.float32)
            return {"psnr": empty, "ssim": empty, "l1": empty, "n": torch.empty(0, dtype=torch.int64),
                    "mean": {"psnr": nan, "ssim": nan, "l1": nan}}
        sums = sums[:V]
        if xfer is not None:
            xfer.sum(sums)
        elif self.band is not None:
            band_losses.all_reduce_sum(sums, self.group)
        # one transfer: the fp32 values and the exact fp64 counts
        both = torch.cat([finish(sums).double().reshape(-1), sums[:, 3]]).cpu()
        out, n = both[:4 * (V + 1)].reshape(V + 1, 4).float(), both[4 * (V + 1):]
        return {"psnr": out[:V, 0], "ssim": out[:V, 1], "l1": out[:V, 2], "n": n.to(torch.int64),
                "mean": {"psnr": float(out[V, 0]), "ssim": float(out[V, 1]), "l1": float(out[V, 2])}}
