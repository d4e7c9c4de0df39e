"""The training losses of losses.py on a tile-row band (include/sgr.h, "The same four losses on a tile-row band").

The multi-GPU rasterizers (sharded.py) return full-size images of which only the rows of the rank's band hold the render.  The reference's
losses are not band-local: the 11x11 SSIM window of a pixel near a band edge reads the neighbouring rows, the L1 / SSIM / sky /
object-accumulation means divide by the frame's count, and the LiDAR loss keeps the int(0.95 n) smallest errors of the frame.  Here
every loss runs in stages around one collective each, and every rank ends with the loss of the whole frame and the gradient rows of
its band, bit-identical to the single-GPU call's:

  photometric  halo exchange of the image rows within 10 px of the band (batch_isend_irecv with the ranks owning the neighbouring tile
               rows) -> stats kernel -> sum of 3 doubles -> gradient kernel;
  sky, obj     per-pixel kernel -> sum of 1 double -> value;
  LiDAR        keys + level-0 histogram -> sum -> select, level-1 histogram -> sum -> select, level-2 histogram -> sum -> select, the
               sums below the k-th error and the ties per tile row -> sum -> gradient kernel.

The low-level steps below are one C-ABI call each; the tests drive them directly to emulate N ranks on one GPU.  `frame_losses` is the
autograd entry that runs the photometric, sky and object-accumulation losses of one frame with ONE all-reduce of their partial sums
(the reference adds them); `losses.py`'s functions take the same `band=` / `group=` keywords.

Two transports carry the halo and the sums; the stages, their order and the autograd functions are the same for both.  With band= /
group= (or rasterizer= of a GaussianShardedRasterizer with exchange="nccl") they are NCCL's batch_isend_irecv and all_reduce.  With
rasterizer= of one with exchange="p2p" they are the library's peer-memory calls over the loss section of the workspace that rasterizer's
forward set up (sgr_band_halo_exchange_peers, sgr_band_peer_sum): device-side barriers, no NCCL call, no host read-back; the fp64 sums add
the ranks in ascending order, so every rank holds the same bytes.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist

from . import _capi
from ._capi import ptr
from .rasterizer import TileRowBand

HALO = 10  # image rows past a band edge the photometric loss reads: 5 for the SSIM window, 5 for the derivative maps it convolves
SEND_UP, SEND_DOWN, RECV_UP, RECV_DOWN = _capi.HALO_SEND_UP, _capi.HALO_SEND_DOWN, _capi.HALO_RECV_UP, _capi.HALO_RECV_DOWN
LIDAR_STATE_BYTES = C.sizeof(_capi.SgrLidarState)


def check_band(band, image_height: int) -> Tuple[int, int, int]:
    """(begin, end, step) of a TileRowBand for an image of `image_height` rows; raises ValueError for a band the kernels cannot run."""
    if band is None:
        raise ValueError("band must be a TileRowBand")
    b, e, s = (int(v) for v in band)
    rows = (int(image_height) + 15) // 16
    if s < 1 or b < 0 or e > rows or b > e:
        raise ValueError(f"bad tile-row band [{b},{e}) step {s} for {rows} tile rows (image height {image_height})")
    return b, e, s


def _owned_tiles(b: int, e: int, s: int) -> List[int]:
    return list(range(b, e, s))


def halo_strips(image_height: int, band, side: int) -> List[int]:
    """First pixel row of each strip of HALO rows (the last one clipped at the image height) of a halo message; the sides as in
    include/sgr.h.  The same rule as the kernels': a tile row has a halo edge where its neighbour is another rank's."""
    H = int(image_height)
    b, e, s = check_band(band, H)
    rows = (H + 15) // 16
    own = _owned_tiles(b, e, s)
    if side in (SEND_UP, RECV_UP):
        tiles = [t for t in own if t >= 1 and (t - 1) not in own]
        off = 0 if side == SEND_UP else -HALO
    else:
        tiles = [t for t in own if t + 1 < rows and (t + 1) not in own]
        off = 16 - HALO if side == SEND_DOWN else 16
    return [16 * t + off for t in tiles]


def halo_row_indices(image_height: int, band, side: int) -> torch.Tensor:
    """Pixel rows of a halo message, in buffer order."""
    H = int(image_height)
    out = [r for base in halo_strips(H, band, side) for r in range(base, min(base + HALO, H))]
    return torch.tensor(out, dtype=torch.long)


def halo_peers(rank: int, world: int) -> Tuple[int, int]:
    """(owner of the tile rows above the band's, owner of those below) for cyclic_band and contiguous_band: the neighbouring ranks."""
    return (rank - 1) % world, (rank + 1) % world


def halo_of_rows(image_height: int, rank: int, world: int, layout: str = "cyclic"):
    """The band_of_rows counterpart of the halo: [(source rank, pixel rows)] that `rank` needs from the others for the photometric
    loss, the rows within HALO of its band that other ranks own."""
    from .sharded import contiguous_band, cyclic_band
    band = (cyclic_band if layout == "cyclic" else contiguous_band)(image_height, rank, world)
    up, down = halo_peers(rank, world)
    out = []
    for peer, side in ((up, RECV_UP), (down, RECV_DOWN)):
        rows = halo_row_indices(image_height, band, side)
        if rows.numel():
            out.append((peer, rows))
    return out


def halo_rows(image_height: int, band, side: int) -> int:
    """Rows of one halo message (sgr_band_halo_rows); a buffer is [C, rows, W] fp32."""
    b, e, s = check_band(band, image_height)
    n = int(_capi.lib().sgr_band_halo_rows(int(image_height), b, e, s, int(side)))
    if n < 0:
        raise ValueError(f"bad halo side {side}")
    return n


def halo_pack(image: torch.Tensor, band, side: int) -> torch.Tensor:
    """The rows of `image` [C, H, W] that the neighbour on `side` (SEND_UP / SEND_DOWN) needs, as a [C, rows, W] buffer."""
    Cn, H, W = (int(v) for v in image.shape)
    b, e, s = check_band(band, H)
    buf = torch.empty((Cn, halo_rows(H, band, side), W), device=image.device, dtype=torch.float32)
    _capi.call("sgr_band_halo_pack", image.device, Cn, H, W, b, e, s, int(side), ptr(image), ptr(buf))
    return buf


def halo_unpack(image: torch.Tensor, band, side: int, buf: torch.Tensor) -> None:
    """Write a received [C, rows, W] buffer (RECV_UP / RECV_DOWN) into its rows of `image` [C, H, W], in place."""
    Cn, H, W = (int(v) for v in image.shape)
    b, e, s = check_band(band, H)
    if tuple(buf.shape) != (Cn, halo_rows(H, band, side), W):
        raise ValueError(f"halo buffer of shape {tuple(buf.shape)} for side {side} of a {Cn}x{H}x{W} image")
    _capi.call("sgr_band_halo_unpack", image.device, Cn, H, W, b, e, s, int(side), ptr(buf), ptr(image))


def exchange_halo(image: torch.Tensor, band, group=None) -> torch.Tensor:
    """COLLECTIVE (the ranks owning the neighbouring tile rows): a copy of `image` [C, H, W] with the halo rows filled in."""
    out = _capi.f32(image).clone()
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    if world == 1:
        return out
    up, down = halo_peers(dist.get_rank(group), world)
    Cn, H, W = (int(v) for v in out.shape)
    peer = (lambda r: dist.get_global_rank(group, r)) if group is not None else (lambda r: r)
    recv = {side: torch.empty((Cn, halo_rows(H, band, side), W), device=out.device) for side in (RECV_UP, RECV_DOWN)}
    # Each rank issues its sends and receives in one order (down before up), so two messages between the same pair of ranks (world 2,
    # cyclic) match: a rank's SEND_DOWN is its lower neighbour's RECV_UP, its SEND_UP the upper neighbour's RECV_DOWN.
    ops = []
    for side, to in ((SEND_DOWN, down), (SEND_UP, up)):
        buf = halo_pack(out, band, side)
        if buf.numel():
            ops.append(dist.P2POp(dist.isend, buf, peer(to), group))
    for side, frm in ((RECV_UP, up), (RECV_DOWN, down)):
        if recv[side].numel():
            ops.append(dist.P2POp(dist.irecv, recv[side], peer(frm), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    for side in (RECV_UP, RECV_DOWN):
        if recv[side].numel():
            halo_unpack(out, band, side, recv[side])
    return out


def all_reduce_sum(t: torch.Tensor, group=None) -> torch.Tensor:
    """COLLECTIVE: in-place SUM over the group (nothing with one rank or no process group)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


def peer_exchange_halo(ws, image: torch.Tensor, band) -> torch.Tensor:
    """exchange_halo over the loss section of a peer workspace (sgr_band_halo_exchange_peers; COLLECTIVE over the workspace's ranks, on
    the device): a copy of `image` [C, H, W] with the halo rows filled in.  C must fit the section (3 for sharded.PeerWorkspace)."""
    out = _capi.f32(image).clone()
    Cn, H, W = (int(v) for v in out.shape)
    b, e, s = check_band(band, H)
    ws.next_epochs(2)
    _capi.call("sgr_band_halo_exchange_peers", out.device, C.byref(ws.peers), Cn, H, W, b, e, s, ptr(out), ptr(out))
    return out


def peer_sum(ws, t: torch.Tensor) -> torch.Tensor:
    """all_reduce_sum over the loss section of a peer workspace (sgr_band_peer_sum; COLLECTIVE over the workspace's ranks, on the
    device): in place, the ranks added from 0 in ascending order.  `t` is a contiguous int32 or float64 tensor."""
    kinds = {torch.int32: _capi.PEER_SUM_INT32, torch.float64: _capi.PEER_SUM_FLOAT64}
    if t.dtype not in kinds or not t.is_contiguous():
        raise ValueError(f"peer_sum takes a contiguous int32 or float64 tensor, got {t.dtype}")
    ws.next_epochs(2)
    _capi.call("sgr_band_peer_sum", t.device, C.byref(ws.peers), kinds[t.dtype], t.numel(), ptr(t), ptr(t))
    return t


class Transport:
    """How a band loss moves its halo and sums its partials: over `group` with NCCL (ws None) or over the loss section of the peer
    workspace `ws`."""

    def __init__(self, group=None, ws=None):
        self.group, self.ws = group, ws

    @property
    def kind(self) -> str:
        return "nccl" if self.ws is None else "p2p"

    def halo(self, image: torch.Tensor, band) -> torch.Tensor:
        return exchange_halo(image, band, self.group) if self.ws is None else peer_exchange_halo(self.ws, image, band)

    def sum(self, t: torch.Tensor) -> torch.Tensor:
        return all_reduce_sum(t, self.group) if self.ws is None else peer_sum(self.ws, t)


def resolve(band, group, rasterizer, image_height: int):
    """(band, Transport) of a band loss call.  Without `rasterizer`, band= / group= as given (NCCL over `group`).  With one (a
    sharded.GaussianShardedRasterizer), its band (the whole image at world 1, where it has none) and, with exchange="p2p", the loss
    section of the workspace its forward set up, else NCCL over its group; a band= or group= that differs from the rasterizer's raises
    ValueError."""
    if rasterizer is None:
        return band, Transport(group)
    if group is not None and group is not rasterizer.group:
        raise ValueError("the band losses: group= differs from the rasterizer's group")
    own = rasterizer.band if rasterizer.band is not None else TileRowBand(0, (int(image_height) + 15) // 16, 1)
    if band is not None and tuple(int(v) for v in band) != tuple(int(v) for v in own):
        raise ValueError(f"the band losses: band= {tuple(band)} differs from the rasterizer's band {tuple(own)}")
    if rasterizer.exchange == "p2p":
        return own, Transport(ws=rasterizer.loss_workspace())
    return own, Transport(rasterizer.group)


# ---- photometric loss ----------------------------------------------------------------------------------------------------------
def _mask_u8(mask, n: int, device, what: str):
    if mask is None:
        return None
    m = mask.reshape(-1).to(device=device, dtype=torch.uint8).contiguous()
    if m.numel() != n:
        raise ValueError(f"{what} must have {n} pixels, got {m.numel()}")
    return m


def image_loss_stats(image: torch.Tensor, gt: torch.Tensor, mask, band, partials: Optional[torch.Tensor] = None):
    """Stage 1 (sgr_band_image_loss_stats): the band's partial sums {SSIM, masked |x - y|, masked pixels} into `partials` (3 float64;
    allocated when None) and the derivative maps into the returned scratch.  `image` holds the band's rows and its halo."""
    Cn, H, W = (int(v) for v in image.shape)
    b, e, s = check_band(band, H)
    dev = image.device
    nbytes = int(_capi.lib().sgr_image_loss_scratch_bytes(Cn, H, W))
    scratch = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    if partials is None:
        partials = torch.empty(3, device=dev, dtype=torch.float64)
    _capi.call("sgr_band_image_loss_stats", dev, Cn, H, W, b, e, s, ptr(image), ptr(gt), ptr(mask), ptr(partials), ptr(scratch), nbytes)
    return partials, scratch


def image_loss_grad(image, gt, mask, band, w_l1: float, w_ssim: float, partials, scratch, need_grad: bool = True):
    """Stage 2 (sgr_band_image_loss_grad), after the partials were summed over the ranks: (dL/dimage with the band's rows, zero
    elsewhere, or None; scalars {value, L1, SSIM, masked pixels} of the frame)."""
    Cn, H, W = (int(v) for v in image.shape)
    b, e, s = check_band(band, H)
    dev = image.device
    grad = torch.zeros_like(image) if need_grad else None
    scalars = torch.empty(4, device=dev, dtype=torch.float32)
    _capi.call("sgr_band_image_loss_grad", dev, Cn, H, W, b, e, s, ptr(image), ptr(gt), ptr(mask), float(w_l1), float(w_ssim), ptr(partials),
               ptr(grad), ptr(scalars), ptr(scratch), scratch.numel())
    return grad, scalars


# ---- sky and object-accumulation losses ---------------------------------------------------------------------------------------
def acc_loss_band(entry: str, acc: torch.Tensor, flag: torch.Tensor, weight: float, band, need_grad: bool = True,
                  partial: Optional[torch.Tensor] = None):
    """sgr_band_sky_loss / sgr_band_obj_acc_loss on acc [1, H, W]: (dL/dacc with the band's rows or None, partial sum [1] float64)."""
    H, W = int(acc.shape[-2]), int(acc.shape[-1])
    b, e, s = check_band(band, H)
    dev = acc.device
    grad = torch.zeros_like(acc) if need_grad else None
    if partial is None:
        partial = torch.empty(1, device=dev, dtype=torch.float64)
    _capi.call(entry, dev, H, W, b, e, s, ptr(acc), ptr(flag), float(weight), ptr(grad), ptr(partial))
    return grad, partial


def acc_loss_value(N: int, weight: float, total: torch.Tensor) -> torch.Tensor:
    """sgr_band_acc_loss_value: {weight * mean, mean} of the frame from the summed partial."""
    scalars = torch.empty(2, device=total.device, dtype=torch.float32)
    _capi.call("sgr_band_acc_loss_value", total.device, int(N), float(weight), ptr(total), ptr(scalars))
    return scalars


# ---- LiDAR depth loss ---------------------------------------------------------------------------------------------------------
def lidar_level_words(state: torch.Tensor, level: int) -> torch.Tensor:
    """The int32 words of the state that the ranks sum before select `level` + 1: level 0 is n, the (zero) select fields and the
    level-0 histogram; levels 1 and 2 their histograms."""
    if level == 0:
        lo, hi = 0, 4 * _capi.LIDAR_LEVEL0_WORDS
    else:
        lo = _capi.SgrLidarState.hist.offset + 4 * _capi.LIDAR_BINS * level
        hi = lo + 4 * _capi.LIDAR_BINS
    return state[lo:hi].view(torch.int32)


def lidar_keys(depth, acc, lidar_depth, mask, band):
    """Stage 1 (sgr_band_lidar_keys): (state [sizeof SgrLidarState] bytes, scratch)."""
    H, W = int(depth.shape[-2]), int(depth.shape[-1])
    b, e, s = check_band(band, H)
    dev = depth.device
    nbytes = int(_capi.lib().sgr_band_lidar_scratch_bytes(H, W))
    if nbytes == 0:
        raise ValueError(f"bad image size {H}x{W} for the LiDAR depth loss")
    scratch = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    state = torch.empty(LIDAR_STATE_BYTES, device=dev, dtype=torch.uint8)
    _capi.call("sgr_band_lidar_keys", dev, H, W, b, e, s, ptr(depth), ptr(acc), ptr(lidar_depth), ptr(mask), ptr(state), ptr(scratch), nbytes)
    return state, scratch


def lidar_select(level: int, keep: float, H: int, W: int, band, state, scratch, sums: Optional[torch.Tensor] = None):
    """Stages 2-4 (sgr_band_lidar_select, level 1, 2, 3) after the previous level's words were summed.  Level 3 returns `sums`
    [1 + ceil(H / 16)] float64: {sum of the errors below the k-th, the ties per tile row}."""
    b, e, s = check_band(band, H)
    dev = state.device
    if level == 3 and sums is None:
        sums = torch.empty(1 + (int(H) + 15) // 16, device=dev, dtype=torch.float64)
    _capi.call("sgr_band_lidar_select", dev, int(level), float(keep), int(H), int(W), b, e, s, ptr(state), ptr(sums) if level == 3 else None,
               ptr(scratch), scratch.numel())
    return sums


def lidar_grad(depth, acc, lidar_depth, weight: float, band, state, sums, scratch, need_depth: bool = True, need_acc: bool = True):
    """Stage 5 (sgr_band_lidar_grad) after `sums` were summed: (dL/ddepth or None, dL/dacc or None, scalars {weight * mean, mean, n, k})."""
    H, W = int(depth.shape[-2]), int(depth.shape[-1])
    b, e, s = check_band(band, H)
    dev = depth.device
    gd = torch.zeros_like(depth) if need_depth else None
    ga = torch.zeros_like(acc) if need_acc else None
    scalars = torch.empty(4, device=dev, dtype=torch.float32)
    _capi.call("sgr_band_lidar_grad", dev, H, W, b, e, s, ptr(depth), ptr(acc), ptr(lidar_depth), float(weight), ptr(state), ptr(sums),
               ptr(gd), ptr(ga), ptr(scalars), ptr(scratch), scratch.numel())
    return gd, ga, scalars


# ---- autograd entries ---------------------------------------------------------------------------------------------------------
def _check_cuda(*ts) -> None:
    if not all(t.is_cuda for t in ts if t is not None):
        raise _capi.SgrError("street_gaussians_b200.band_losses needs CUDA tensors (there is no CPU fallback)")


class _FrameLosses(torch.autograd.Function):
    """Photometric, sky and object-accumulation losses of one frame on a band, with one all-reduce of their partial sums."""
    @staticmethod
    def forward(ctx, image, acc, acc_obj, spec):
        band, xfer = spec["band"], spec["transport"]
        out = []
        dev = next(t for t in (image, acc, acc_obj) if t is not None).device
        partials = torch.empty(5, device=dev, dtype=torch.float64)  # {SSIM, L1, mask count} {sky} {obj}
        grads = [None, None, None]
        if image is not None:
            img = xfer.halo(image, band)
            g = _capi.f32(spec["gt"].detach(), dev)
            if img.dim() != 3 or img.shape != g.shape:
                raise ValueError(f"image / gt must both be [C, H, W], got {tuple(image.shape)} and {tuple(spec['gt'].shape)}")
            m_img = _mask_u8(spec["mask"], img.shape[1] * img.shape[2], dev, "mask")
            _, scratch = image_loss_stats(img, g, m_img, band, partials[0:3])
        accs = []
        for i, (t, key, entry) in enumerate(((acc, "sky_mask", "sgr_band_sky_loss"), (acc_obj, "obj_bound", "sgr_band_obj_acc_loss"))):
            if t is None:
                continue
            a = _capi.f32(t, dev)
            m = _mask_u8(spec[key], a.numel(), dev, key)
            grads[1 + i], _ = acc_loss_band(entry, a, m, spec["weights"][1 + i], band, t.requires_grad, partials[3 + i:4 + i])
            accs.append((i, a))
        xfer.sum(partials)
        if image is not None:
            grads[0], scalars = image_loss_grad(img, g, m_img, band, spec["w_l1"], spec["w_ssim"], partials[0:3], scratch, image.requires_grad)
            out.append(scalars[0])
        for i, a in accs:
            out.append(acc_loss_value(a.numel(), spec["weights"][1 + i], partials[3 + i:4 + i])[0])
        ctx.save_for_backward(*(g if g is not None else torch.empty(0) for g in grads))
        ctx.has = [g is not None for g in grads]
        ctx.dtypes = [t.dtype if t is not None else None for t in (image, acc, acc_obj)]
        return tuple(out)

    @staticmethod
    def backward(ctx, *g_outs):
        saved = ctx.saved_tensors
        res, k = [], 0
        present = [d is not None for d in ctx.dtypes]
        for i in range(3):
            if not present[i]:
                res.append(None)
                continue
            g_out = g_outs[k]
            k += 1
            res.append((saved[i] * g_out).to(ctx.dtypes[i]) if ctx.has[i] else None)
        return res[0], res[1], res[2], None


def _frame(image, gt, mask, w_l1: float, w_ssim: float, acc, sky_mask, sky_weight: float, acc_obj, obj_bound, obj_weight: float, band, group,
           rasterizer=None):
    """Values of the present losses, in the order image, acc, acc_obj; the image's is w_l1 * L1 + w_ssim * SSIM."""
    if band is None and rasterizer is None:
        raise ValueError("the band losses need the rank's band")
    if image is None and acc is None and acc_obj is None:
        raise ValueError("frame_losses needs at least one of image, acc and acc_obj")
    H = int((image if image is not None else acc if acc is not None else acc_obj).shape[-2])
    band, xfer = resolve(band, group, rasterizer, H)
    check_band(band, H)
    if xfer.kind == "p2p" and image is not None and (image.dim() != 3 or int(image.shape[0]) != 3):
        raise ValueError(f"the peer-memory halo carries 3-channel images, got an image of shape {tuple(image.shape)}")
    if image is not None and gt is None:
        raise ValueError("the photometric loss needs gt")
    if acc is not None and sky_mask is None:
        raise ValueError("the sky loss needs sky_mask")
    if acc_obj is not None and obj_bound is None:
        raise ValueError("the object-accumulation loss needs obj_bound")
    _check_cuda(image, gt, acc, acc_obj)
    spec = dict(band=band, transport=xfer, gt=gt, mask=mask, sky_mask=sky_mask, obj_bound=obj_bound, w_l1=w_l1, w_ssim=w_ssim,
                weights=(None, sky_weight, obj_weight))
    return list(_FrameLosses.apply(image, acc, acc_obj, spec))


def frame_losses(image=None, gt=None, mask=None, lambda_l1: float = 1.0, lambda_dssim: float = 0.2, acc=None, sky_mask=None,
                 sky_weight: float = 1.0, acc_obj=None, obj_bound=None, obj_weight: float = 1.0, *, band: Optional[TileRowBand] = None,
                 group=None, rasterizer=None):
    """COLLECTIVE over `group`: the photometric loss of `image` (train.py:101-104), the sky loss of `acc` (:107-113) and the
    object-accumulation loss of `acc_obj` (:114-122) of one frame, each rank holding the rendered rows of its `band`; any of the three
    may be left out.  One halo exchange and ONE all-reduce of the five partial sums.  Returns {"photometric", "sky", "obj_acc"} (the
    present ones) as the frame's values on every rank; their gradients reach the band's rows.
    rasterizer= (the GaussianShardedRasterizer that rendered the rows): its band, and with exchange="p2p" the halo and the sum over its
    peer workspace (resolve); the image must then have 3 channels."""
    vals = _frame(image, gt, mask, (1.0 - lambda_dssim) * lambda_l1, -lambda_dssim, acc, sky_mask, sky_weight, acc_obj, obj_bound, obj_weight,
                  band, group, rasterizer)
    out = {}
    if image is not None:
        out["photometric"] = vals.pop(0) + lambda_dssim
    if acc is not None:
        out["sky"] = vals.pop(0)
    if acc_obj is not None:
        out["obj_acc"] = vals.pop(0)
    return out


class _LidarDepthLossBand(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, acc, lidar_depth, mask, weight: float, keep: float, band, xfer):
        _check_cuda(depth, acc, lidar_depth)
        d, a = _capi.f32(depth), _capi.f32(acc)
        dev = d.device
        ld = _capi.f32(lidar_depth.detach(), dev)
        if d.dim() < 2 or a.shape != d.shape or ld.shape != d.shape:
            raise ValueError(f"depth, acc and lidar_depth must be one [.., H, W] shape, got {tuple(depth.shape)}, {tuple(acc.shape)}, "
                             f"{tuple(lidar_depth.shape)}")
        H, W = int(d.shape[-2]), int(d.shape[-1])
        if d.numel() != H * W:
            raise ValueError("depth must be [1, H, W]")
        m = _mask_u8(mask, H * W, dev, "mask")
        state, scratch = lidar_keys(d, a, ld, m, band)
        for level in (1, 2):
            xfer.sum(lidar_level_words(state, level - 1))
            lidar_select(level, keep, H, W, band, state, scratch)
        xfer.sum(lidar_level_words(state, 2))
        sums = lidar_select(3, keep, H, W, band, state, scratch)
        xfer.sum(sums)
        gd, ga, scalars = lidar_grad(d, a, ld, weight, band, state, sums, scratch, ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        ctx.save_for_backward(gd, ga)
        ctx.dtypes = (depth.dtype, acc.dtype)
        return scalars[0]

    @staticmethod
    def backward(ctx, g_out):
        gd, ga = ctx.saved_tensors
        return ((gd * g_out).to(ctx.dtypes[0]) if gd is not None else None, (ga * g_out).to(ctx.dtypes[1]) if ga is not None else None,
                None, None, None, None, None, None)


def lidar_depth_loss(depth, acc, lidar_depth, mask=None, weight: float = 1.0, keep: float = 0.95, *, band: Optional[TileRowBand] = None,
                     group=None, rasterizer=None):
    """COLLECTIVE over `group` (four small all-reduces): losses.lidar_depth_loss of the frame, each rank holding the rendered rows of
    its `band` of depth and acc; lidar_depth and mask are whole frames.  The selected pixels are the single-GPU call's.  rasterizer= as
    frame_losses' (with exchange="p2p" the four sums go over its peer workspace)."""
    if not (0.0 < float(keep) <= 1.0):
        raise ValueError(f"keep must be in (0, 1], got {keep}")
    band, xfer = resolve(band, group, rasterizer, int(depth.shape[-2]))
    check_band(band, int(depth.shape[-2]))
    return _LidarDepthLossBand.apply(depth, acc, lidar_depth, mask, weight, keep, band, xfer)
