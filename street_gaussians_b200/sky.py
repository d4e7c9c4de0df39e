"""The sky cube map of the reference (lib/models/sky_cubemap.py:77-123, model.nsg.include_sky) composited onto the rendered frame
(street_gaussian_renderer.py:107-111) over sgr_sky_composite_forward / sgr_sky_composite_backward (include/sgr.h).

    sky_composite(rgb, acc, cube_map, K, w2c, sky_mask=..., perturb=..., white_background=...)
        == rgb + SkyCubeMap(camera, acc.detach()) * (1 - acc)

`cube_map` is SkyCubeMap.sky_cube_map [6, R, R, 3]; `w2c` is camera.world_view_transform.transpose(0, 1).  With `sky_mask` (training
with the guidance mask) the cube is sampled where the mask is set and on rows 0-49; without it, where 1 - acc > 1e-3.  The caller's
mask is only read: the reference sets its rows 0-49 in place, which the sky loss then sees, so a caller who wants that loss input
sets those rows itself.  `perturb` jitters each pixel's sample point as get_rays_torch(perturb=True) does, with two torch.rand(H, W)
draws on the current CUDA generator.  CUDA tensors only: there is no CPU fallback.

band= / group= (keyword-only, as in losses.py): rgb and acc hold the rendered rows of this rank's TileRowBand (sharded.py); the
composite runs on the band's pixels only (sgr_band_sky_composite_*), the output is zero outside the band, and the backward gives
dL/dacc on the band's rows and all-reduces the cube map's gradient over `group`, so every rank's cube_map.grad is the whole frame's.

rasterizer= (a sharded.GaussianShardedRasterizer, resolved like the band losses' band_losses.resolve): its band (the whole-frame
entries at world 1) and its transport.  With exchange="nccl" the all-reduce above over its group.  With exchange="p2p" the backward
marks the 32 x 32-texel blocks of the cube its band touched (sgr_band_sky_composite_backward_marked) and sums only those over peer
memory (sgr_sky_grad_peer_sum, through the rasterizer's sky_workspace): no NCCL call, no host read-back, and every rank's
cube_map.grad holds the same bytes, the ascending-rank fp32 sum of the ranks' partials block by block.

blocks= (keyword-only, with block_map(R, device)): the 32 x 32-texel blocks of the cube this call's backward adds gradient into are
OR-ed into `blocks` (set to 1; other bytes kept), for training.CubeMapSparseAdam, which steps only those blocks and clears the map.  In
every mode `blocks` ends up with the union over the ranks, the same bytes on every rank: the whole frame marks through
sgr_band_sky_composite_backward_or_marks over every tile row; band= / group= sums the band's marks over the group after the gradient's
all-reduce; rasterizer= with exchange="p2p" takes the union the peer-memory sum already forms (sgr_sky_grad_peer_sum_union).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _capi
from ._capi import ptr


def _check(rgb, acc, cube_map, K, w2c, sky_mask):
    if rgb.dim() != 3 or rgb.shape[0] != 3:
        raise ValueError(f"rgb must be [3, H, W], got {tuple(rgb.shape)}")
    H, W = int(rgb.shape[1]), int(rgb.shape[2])
    if tuple(acc.shape) != (1, H, W):
        raise ValueError(f"acc must be [1, {H}, {W}], got {tuple(acc.shape)}")
    if cube_map.dim() != 4 or cube_map.shape[0] != 6 or cube_map.shape[3] != 3:
        raise ValueError(f"cube_map must be [6, R, R, 3], got {tuple(cube_map.shape)}")
    if cube_map.shape[1] != cube_map.shape[2]:
        raise ValueError(f"cube_map faces must be square, got {cube_map.shape[1]} x {cube_map.shape[2]}")
    if tuple(K.shape) != (3, 3) or tuple(w2c.shape) != (4, 4):
        raise ValueError(f"K must be [3, 3] and w2c [4, 4], got {tuple(K.shape)} and {tuple(w2c.shape)}")
    if sky_mask is not None:
        if tuple(sky_mask.shape) not in ((1, H, W), (H, W)) or sky_mask.dtype != torch.bool:
            raise ValueError(f"sky_mask must be a bool [1, {H}, {W}] or [{H}, {W}], got {sky_mask.dtype} {tuple(sky_mask.shape)}")
    named = dict(rgb=rgb, acc=acc, cube_map=cube_map, K=K, w2c=w2c)
    for what, t in named.items():
        if t.dtype != torch.float32:
            raise ValueError(f"{what} must be float32, got {t.dtype}")
    if sky_mask is not None:
        named["sky_mask"] = sky_mask
    for what, t in named.items():
        if not t.is_cuda:
            raise _capi.SgrError(f"street_gaussians_b200.sky needs CUDA tensors ({what} is on {t.device}; there is no CPU fallback)")
        if t.device != rgb.device:
            raise ValueError(f"{what} is on {t.device}, rgb on {rgb.device}")
    return H, W, int(cube_map.shape[1])


def _band_rows(band, H: int):
    """(begin, end, step) of the band, or None for the whole frame."""
    if band is None:
        return None
    from .band_losses import check_band
    return check_band(band, H)


def _resolve(band, group, rasterizer, H: int):
    """(rows or None, band_losses.Transport) of a call: band= / group= as given without a rasterizer; with one, its band and transport
    (band_losses.resolve, which refuses a band= or group= that differs from the rasterizer's), the whole frame at world 1."""
    from .band_losses import Transport, resolve
    if rasterizer is None:
        return _band_rows(band, H), Transport(group)
    own, xfer = resolve(band, group, rasterizer, H)
    if rasterizer.band is None:
        return None, Transport()
    return _band_rows(own, H), xfer


def block_map(R: int, device=None) -> torch.Tensor:
    """A zeroed block map of a [6, R, R, 3] cube: sgr_sky_grad_blocks(R) = 6 ceil(R / 32)^2 uint8 bytes, one per 32 x 32-texel block,
    for sky_composite(blocks=) and training.CubeMapSparseAdam.step."""
    n = int(_capi.lib().sgr_sky_grad_blocks(int(R)))
    if n <= 0:
        raise ValueError(f"no cube block map for R={R} (0 < R <= 16384)")
    return torch.zeros(n, dtype=torch.uint8, device=device)


def _check_blocks(blocks, R: int, device):
    n = int(_capi.lib().sgr_sky_grad_blocks(R))
    if blocks.dtype != torch.uint8 or blocks.dim() != 1 or blocks.numel() != n or not blocks.is_contiguous():
        raise ValueError(f"blocks must be a contiguous uint8 tensor of sgr_sky_grad_blocks({R}) = {n} bytes, got {blocks.dtype} "
                         f"{tuple(blocks.shape)}")
    if blocks.device != device:
        raise ValueError(f"blocks is on {blocks.device}, rgb on {device}")


def sky_grad_peer_sum(ws, sky_ws, g_cube: torch.Tensor, union: Optional[torch.Tensor] = None) -> torch.Tensor:
    """COLLECTIVE over the ranks of the peer workspace `ws` (sgr_sky_grad_peer_sum, on the device): in place on this rank's partial
    g_cube [6, R, R, 3], zero outside the blocks sky_ws.block_map marks (sgr_band_sky_composite_backward_marked on a zeroed g_cube),
    every rank ends with the marked blocks' ascending-rank sum and zeros elsewhere.  Three barriers on ws's pad.  union: a block map
    (block_map) into which every block some rank marked is OR-ed, the same bytes on every rank (sgr_sky_grad_peer_sum_union)."""
    ws.next_epochs(3)
    if union is None:
        _capi.call("sgr_sky_grad_peer_sum", g_cube.device, C.byref(ws.peers), C.byref(sky_ws.peers), int(g_cube.shape[1]),
                   ptr(sky_ws.block_map), ptr(g_cube))
    else:
        _capi.call("sgr_sky_grad_peer_sum_union", g_cube.device, C.byref(ws.peers), C.byref(sky_ws.peers), int(g_cube.shape[1]),
                   ptr(sky_ws.block_map), ptr(g_cube), ptr(union))
    return g_cube


class _SkyComposite(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rgb, acc, cube_map, K, w2c, sky_mask, perturb: bool, fill: float, rows, xfer, rasterizer, blocks):
        H, W, R = _check(rgb, acc, cube_map, K, w2c, sky_mask)
        dev = rgb.device
        if blocks is not None:
            _check_blocks(blocks, R, dev)
        rgb_c, acc_c, cube = rgb.contiguous(), acc.contiguous(), cube_map.contiguous()
        Kc, Tc = K.contiguous(), w2c.contiguous()
        mask = sky_mask.contiguous() if sky_mask is not None else None
        mode = _capi.SKY_MASK_GIVEN if mask is not None else _capi.SKY_MASK_ACC
        if perturb:  # graphics_utils.py:195-196, in that order
            jx = torch.rand(H, W, device=dev)
            jy = torch.rand(H, W, device=dev)
        else:
            jx = jy = None
        if rows is None:
            out = torch.empty_like(rgb_c)
            _capi.call("sgr_sky_composite_forward", dev, H, W, R, mode, float(fill), ptr(rgb_c), ptr(acc_c), ptr(mask), ptr(cube), ptr(Kc),
                       ptr(Tc), ptr(jx), ptr(jy), ptr(out))
        else:
            out = torch.zeros_like(rgb_c)
            _capi.call("sgr_band_sky_composite_forward", dev, H, W, *rows, R, mode, float(fill), ptr(rgb_c), ptr(acc_c), ptr(mask), ptr(cube),
                       ptr(Kc), ptr(Tc), ptr(jx), ptr(jy), ptr(out))
        ctx.save_for_backward(acc_c, cube, Kc, Tc, mask, jx, jy)
        ctx.args = (H, W, R, mode, float(fill))
        ctx.band, ctx.xfer, ctx.blocks = rows, xfer, blocks
        # exchange="p2p": the sky section is collective on first use, so it is allocated here, where every rank runs
        ctx.sky_ws = rasterizer.sky_workspace(R, dev) if rows is not None and xfer.kind == "p2p" else None
        return out

    @staticmethod
    def backward(ctx, g_out):
        acc, cube, Kc, Tc, mask, jx, jy = ctx.saved_tensors
        H, W, R, mode, fill = ctx.args
        dev = acc.device
        g = g_out.contiguous()
        need_rgb, need_acc, need_cube = ctx.needs_input_grad[:3]
        g_cube = torch.zeros_like(cube) if need_cube else None
        blocks = ctx.blocks if need_cube else None
        if ctx.band is None and blocks is not None:  # the band of every tile row: the whole-frame gradient, with the blocks marked
            g_acc = torch.empty_like(acc) if need_acc else None
            _capi.call("sgr_band_sky_composite_backward_or_marks", dev, H, W, 0, (H + 15) // 16, 1, R, mode, fill, ptr(acc), ptr(mask),
                       ptr(cube), ptr(Kc), ptr(Tc), ptr(jx), ptr(jy), ptr(g), ptr(g_acc), ptr(g_cube), ptr(blocks))
        elif ctx.band is None:
            g_acc = torch.empty_like(acc) if need_acc else None
            _capi.call("sgr_sky_composite_backward", dev, H, W, R, mode, fill, ptr(acc), ptr(mask), ptr(cube), ptr(Kc), ptr(Tc), ptr(jx),
                       ptr(jy), ptr(g), ptr(g_acc), ptr(g_cube))
        elif ctx.sky_ws is not None and need_cube:  # COLLECTIVE over peer memory: only the blocks some band touched are exchanged
            g_acc = torch.zeros_like(acc) if need_acc else None
            _capi.call("sgr_band_sky_composite_backward_marked", dev, H, W, *ctx.band, R, mode, fill, ptr(acc), ptr(mask), ptr(cube), ptr(Kc),
                       ptr(Tc), ptr(jx), ptr(jy), ptr(g), ptr(g_acc), ptr(g_cube), ptr(ctx.sky_ws.block_map))
            if blocks is None:
                sky_grad_peer_sum(ctx.xfer.ws, ctx.sky_ws, g_cube)
            else:
                sky_grad_peer_sum(ctx.xfer.ws, ctx.sky_ws, g_cube, blocks)
        elif blocks is not None:  # COLLECTIVE: as below, then the ranks' marks summed the same way; non-zero counts are the union
            g_acc = torch.zeros_like(acc) if need_acc else None
            local = torch.empty_like(blocks)
            _capi.call("sgr_band_sky_composite_backward_marked", dev, H, W, *ctx.band, R, mode, fill, ptr(acc), ptr(mask), ptr(cube), ptr(Kc),
                       ptr(Tc), ptr(jx), ptr(jy), ptr(g), ptr(g_acc), ptr(g_cube), ptr(local))
            ctx.xfer.sum(g_cube)
            counts = local.to(torch.int32)
            ctx.xfer.sum(counts)
            blocks.logical_or_(counts)
        else:
            g_acc = torch.zeros_like(acc) if need_acc else None
            _capi.call("sgr_band_sky_composite_backward", dev, H, W, *ctx.band, R, mode, fill, ptr(acc), ptr(mask), ptr(cube), ptr(Kc), ptr(Tc),
                       ptr(jx), ptr(jy), ptr(g), ptr(g_acc), ptr(g_cube))
            if need_cube:  # COLLECTIVE: this band's partial dL/dcube -> the whole frame's, on every rank
                ctx.xfer.sum(g_cube)
        return (g_out if need_rgb else None), g_acc, g_cube, None, None, None, None, None, None, None, None, None


def sky_composite(rgb: torch.Tensor, acc: torch.Tensor, cube_map: torch.Tensor, K: torch.Tensor, w2c: torch.Tensor, *,
                  sky_mask: Optional[torch.Tensor] = None, perturb: bool = False, white_background: bool = True, band=None,
                  group=None, rasterizer=None, blocks: Optional[torch.Tensor] = None) -> torch.Tensor:
    """rgb [3, H, W] + sky * (1 - acc [1, H, W]) with the sky sampled from cube_map [6, R, R, 3] along the rays of K [3, 3] and
    w2c [4, 4], clamped to [0, 1]; pixels the mask rule leaves out take 1 (white_background) or 0.  Differentiable in rgb, acc and
    cube_map.  sky_mask: bool [1, H, W] or [H, W] (training with the guidance mask), None for the acc rule.  All fp32 CUDA tensors.

    band= / group=: rgb and acc hold the rendered rows of this rank's TileRowBand (sharded.py); sky_mask is the whole frame's.  The
    output has the band's rows, zeros elsewhere, equal bit for bit to the whole-frame call's rows; dL/dacc covers the band's rows.
    COLLECTIVE in the backward: the cube map's gradient is all-reduced over `group` (every rank must run its backward).  perturb=True
    draws the same full-frame [H, W] jitter pair, in the same order, as the whole-frame call, so a rank's rows equal the single-GPU
    call's whenever the ranks' CUDA generators are in the same state.

    rasterizer= (the GaussianShardedRasterizer that rendered the rows, whose forward must have run): its band, the whole frame at world
    1; a band= or group= that differs from its own raises ValueError.  exchange="nccl": the all-reduce above over its group.
    exchange="p2p": COLLECTIVE in the backward over its peer memory, no NCCL call and no host synchronisation; cube_map.grad is the
    ascending-rank fp32 sum of the ranks' partials, block by block, and the same bytes on every rank.  Every rank must ask for the cube
    map's gradient alike.

    blocks= (block_map(R, device)): when the backward forms the cube map's gradient, it also OR-s into `blocks` the 32 x 32-texel blocks
    that gradient touched (set to 1, other bytes kept), over every rank in the multi-GPU modes, so that marks accumulate over backward
    passes until training.CubeMapSparseAdam.step consumes them; with several ranks, every rank must pass a map holding the same bytes.
    The gradients are those of the call without blocks= (dL/dcube up to the order of its texels' float atomics)."""
    rows, xfer = _resolve(band, group, rasterizer, int(rgb.shape[-2]))  # a bad or mismatched band fails before anything else
    return _SkyComposite.apply(rgb, acc, cube_map, K, w2c, sky_mask, bool(perturb), 1.0 if white_background else 0.0, rows, xfer, rasterizer,
                               blocks)
