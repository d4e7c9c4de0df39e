"""Tile-row sharding of one frame across the GPUs of a node (SURVEY.md §8e; no counterpart in the reference, which is
single-GPU).  One process per GPU (torch.distributed); Gaussian parameters are replicated, pixels are partitioned:

  forward : every rank preprocesses all P Gaussians (HBM-bound) but bins / sorts / blends only the 16-px tile
            rows it owns -> no collective.  Each rank's output images are zero outside its rows.
  backward: each rank's blend_bwd produces PARTIAL per-Gaussian screen-space sums grad2d[P,12] (+ semantics[P,S]);
            ONE sum-all-reduce over NVLink (NCCL) makes them global, then the cheap per-Gaussian chain rule
            (preprocess_bwd) runs replicated, so every rank ends with the full, identical parameter gradients
            ("Variant B" of SURVEY.md §8e: 48 B/Gaussian on the wire instead of a 248 B/Gaussian all-gather).

Rows are dealt cyclically (row r -> rank r % world) so a horizon-heavy street scene balances without a histogram.

GaussianShardedRasterizer ("variant A" of SURVEY.md §8e) additionally partitions the GAUSSIANS: every rank owns P/N of them
(parameters, optimiser state and gradients stay sharded, as in a ZeRO-style trainer) and a tile-row band.

  forward : project own Gaussians -> 48-B screen-space records; all-gather records + radii (NCCL); count / sort / blend
            the own band from the gathered records.
  backward: blend_bwd over the own band -> partial grad2d[P_total,12]; ONE reduce-scatter hands every rank the summed
            rows of its own Gaussians; the per-Gaussian chain rule then runs on P/N Gaussians only.

Compared with ShardedGaussianRasterizer no per-Gaussian stage is replicated any more (at N = 8 the replicated preprocess
fwd/bwd were about a third of the step) and the 2x91 MB all-reduce becomes a 91 MB all-gather plus a 91 MB reduce-scatter.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from . import _capi
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, InstanceCapacity, TileRowBand, _copy_status, _ForwardState,
                         _backward_blend_impl, _backward_geom_impl, _dev_f32, _fit_grads, _fp32_inputs, _geom_grad_buffers, _image_grads,
                         _input_shapes, _make_frame, _ptr, _reference_inputs, _stream)


def cyclic_band(image_height: int, rank: int, world: int) -> TileRowBand:
    rows = (int(image_height) + 15) // 16
    return TileRowBand(begin=rank, end=rows, step=world) if rank < rows else TileRowBand(begin=0, end=0, step=1)


def contiguous_band(image_height: int, rank: int, world: int) -> TileRowBand:
    rows = (int(image_height) + 15) // 16
    per = (rows + world - 1) // world
    return TileRowBand(begin=min(rows, rank * per), end=min(rows, (rank + 1) * per), step=1)


class ShardedGaussianRasterizer(GaussianRasterizer):
    """GaussianRasterizer whose forward covers this rank's tile rows and whose backward all-reduces the per-Gaussian
    screen-space sums.  With world == 1 it is exactly GaussianRasterizer."""

    def __init__(self, raster_settings: GaussianRasterizationSettings, group: Optional[dist.ProcessGroup] = None,
                 layout: str = "cyclic", capacity=None):
        world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        rank = dist.get_rank(group) if world > 1 else 0
        band = None
        reduce = None
        if world > 1:
            mk = cyclic_band if layout == "cyclic" else contiguous_band
            band = mk(raster_settings.image_height, rank, world)

            def reduce(grad2d: torch.Tensor, g_sem: torch.Tensor):
                dist.all_reduce(grad2d, op=dist.ReduceOp.SUM, group=group)
                if g_sem.numel():
                    dist.all_reduce(g_sem, op=dist.ReduceOp.SUM, group=group)
                return grad2d, g_sem

        super().__init__(raster_settings, band=band, grad_reduce=reduce, capacity=capacity)
        self.group, self.world, self.rank = group, world, rank

    def forward_layers(self, *args, **kwargs):
        raise _capi.SgrError("render layers are single-GPU only: use GaussianRasterizer")

    def gather_images(self, *images: torch.Tensor):
        """Sum the zero-padded per-band images into full frames on every rank (only needed when a full image is wanted
        on one device; the loss can be evaluated band-locally)."""
        if self.world == 1:
            return images
        out = []
        for im in images:
            full = im.detach().clone()
            dist.all_reduce(full, op=dist.ReduceOp.SUM, group=self.group)
            out.append(full)
        return tuple(out)


def band_of_rows(image_height: int, rank: int, world: int, layout: str = "cyclic") -> torch.Tensor:
    """Boolean mask [H] of the pixel rows owned by `rank` (host-side helper for tests and band-local losses)."""
    band = (cyclic_band if layout == "cyclic" else contiguous_band)(image_height, rank, world)
    rows = torch.arange((int(image_height) + 15) // 16)
    own = (rows >= band.begin) & (rows < band.end) & (((rows - band.begin) % max(band.step, 1)) == 0)
    return own.repeat_interleave(16)[: int(image_height)]


# ---------------------------------------------------------------------------------------------------------------------
# Gaussian-sharded mode: low-level steps (each is one C-ABI call; tests drive them directly to emulate N ranks on one GPU)
# ---------------------------------------------------------------------------------------------------------------------
REC_FLOATS = 12  # sgr_record_bytes() / 4


def chunk_size(P_local: int, group=None) -> int:
    """COLLECTIVE: the common slot count per rank (max of the local Gaussian counts; smaller ranks pad with radii == 0)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return int(P_local)
    t = torch.tensor([int(P_local)], dtype=torch.int64, device="cuda" if dist.get_backend(group) == "nccl" else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return int(t.item())


_local_tensors = _fp32_inputs  # step 0: the local Gaussians as the kernels read them


def project_records(tensors, settings: GaussianRasterizationSettings, chunk: int):
    """Step 1 (sgr_project): records[chunk,12] float32 view + radii[chunk] int32 of the local Gaussians; slots past
    P_local are padding (radii == 0)."""
    L = _capi.lib()
    means3D = tensors["means3D"]
    device, P = means3D.device, int(means3D.shape[0])
    if P > chunk:
        raise _capi.SgrError(f"{P} local Gaussians do not fit the per-rank chunk of {chunk}; call repartition()")
    rec = torch.empty((chunk, REC_FLOATS), device=device, dtype=torch.float32)
    radii = (torch.empty if P == chunk else torch.zeros)((chunk,), device=device, dtype=torch.int32)
    M = int(tensors["sh"].shape[1]) if tensors["sh"] is not None else 0
    fr, keep = _make_frame(settings, P, M, 0, device, None)
    with torch.cuda.device(device):
        rc = L.sgr_project(C.byref(fr), _ptr(means3D), _ptr(tensors["sh"]), _ptr(tensors["colors_precomp"]), _ptr(tensors["opacities"]),
                           _ptr(tensors["scales"]), _ptr(tensors["rotations"]), _ptr(tensors["cov3Ds_precomp"]), _ptr(radii), _ptr(rec),
                           _stream(device))
    _capi.check(rc, "sgr_project")
    del keep
    return rec, radii


def alloc_gathered(settings: GaussianRasterizationSettings, P_total: int, S: int, device):
    """Forward state for P_total gathered Gaussians.  Returns (state, records view [P_total,12] float32 into state.geom —
    the all-gather target —, geom_bytes, img_bytes)."""
    L = _capi.lib()
    fr, keep = _make_frame(settings, P_total, 0, S, device, None)
    gb, ib = C.c_size_t(0), C.c_size_t(0)
    _capi.check(L.sgr_state_sizes(C.byref(fr), C.byref(gb), C.byref(ib)), "sgr_state_sizes")
    st = _ForwardState()
    st.geom = torch.empty((gb.value,), device=device, dtype=torch.uint8)
    st.img = torch.empty((ib.value,), device=device, dtype=torch.uint8)
    st.binning, st.num_instances = None, 0
    rec_all = st.geom[: P_total * REC_FLOATS * 4].view(torch.float32).view(P_total, REC_FLOATS)
    del keep
    return st, rec_all, gb.value, ib.value


def forward_records(settings: GaussianRasterizationSettings, band: Optional[TileRowBand], st: _ForwardState, sizes, radii_all,
                    semantics_all, capacity: Optional[InstanceCapacity] = None):
    """Step 3 (sgr_forward_records): bin / sort / blend `band` from the records already gathered into st.geom."""
    L = _capi.lib()
    device, P = radii_all.device, int(radii_all.shape[0])
    H, W = int(settings.image_height), int(settings.image_width)
    S = int(semantics_all.shape[1]) if semantics_all is not None else 0
    f32 = dict(device=device, dtype=torch.float32)
    alloc_img = torch.empty if band is None else torch.zeros
    color, depth, alpha, semantic = alloc_img((3, H, W), **f32), alloc_img((1, H, W), **f32), alloc_img((1, H, W), **f32), alloc_img((S, H, W), **f32)
    fr, keep = _make_frame(settings, P, 0, S, device, band)
    gb, ib = sizes
    if capacity is not None:
        capacity.check()
    bounded = capacity is not None and capacity.capacity is not None
    cap = int(capacity.capacity) if bounded else -1
    nbytes = 0
    if bounded:
        nbytes = int(L.sgr_binning_bytes(cap))
        st.binning = torch.empty((nbytes,), device=device, dtype=torch.uint8)

    def _alloc(_user, n):
        st.binning = torch.empty((int(n),), device=device, dtype=torch.uint8)
        return st.binning.data_ptr()

    cb = _capi.ALLOC_FN() if bounded else _capi.ALLOC_FN(_alloc)
    bin_ptr, n_inst = C.c_void_p(), C.c_int64(0)
    with torch.cuda.device(device):
        rc = L.sgr_forward_records(C.byref(fr), _ptr(radii_all), _ptr(semantics_all), _ptr(color), _ptr(depth), _ptr(alpha), _ptr(semantic),
                                   _ptr(st.geom), gb, _ptr(st.img), ib, cb, None, C.byref(bin_ptr), C.byref(n_inst),
                                   _ptr(st.binning) if bounded else None, nbytes, cap, _stream(device))
        _capi.check(rc, "sgr_forward_records")
        if bounded:
            capacity.record_status(fr, st.geom, device)
            st.num_instances = cap
        else:
            st.num_instances = int(n_inst.value)
            if capacity is not None:
                capacity.observe(st.num_instances)
    del keep
    return color, depth, alpha, semantic


def backward_blend_records(settings, band, st: _ForwardState, P_total: int, semantics_all, alpha, grad_color, grad_depth, grad_alpha,
                           grad_semantic, grad2d_out=None):
    """Step 4: partial grad2d[P_total,12] (+ dL_dsemantics[P_total,S]) of this rank's band."""
    shim = dict(means3D=torch.empty((P_total, 0), device=alpha.device), semantics=semantics_all, sh=None)
    return _backward_blend_impl(settings, band, st, shim, alpha, grad_color, grad_depth, grad_alpha, grad_semantic, grad2d_out)


def backward_geom_local(settings, tensors, rec_local, radii_local, grad2d_local):
    """Step 5: chain rule for the local Gaussians from their own records and their reduced grad2d rows."""
    P = int(tensors["means3D"].shape[0])
    st = _ForwardState()
    st.geom = rec_local  # sgr_backward_geom reads only the record array, which sits at offset 0 of a geom_state
    local = dict(tensors)
    local["semantics"] = None
    return _backward_geom_impl(settings, None, st, local, radii_local[:P], grad2d_local[:P].contiguous())


def _align(n: int, a: int = 256) -> int:
    return (n + a - 1) // a * a


class PeerWorkspace:
    """Per-rank buffer [geom_state | radii_all | grad2d] that every rank of the group can address (include/sgr.h, SgrPeers).

    Real multi-GPU: ONE torch symmetric-memory allocation per rank (CUDA VMM mapped into every process; NVLink loads and
    stores), rendezvous'ed once; `barrier()` is the device-side signal-pad barrier of that allocation (a few microseconds
    over NVLink).  `emulate(...)` builds `world` ordinary buffers on ONE device that point at each other, so the exchange
    kernels can be tested without a second GPU."""

    def __init__(self, settings, chunk: int, world: int, rank: int, device, group=None, _buffers=None):
        self.chunk, self.world, self.rank, self.P_total = int(chunk), int(world), int(rank), int(chunk) * int(world)
        if world > _capi.MAX_PEERS:
            raise _capi.SgrError(f"peer exchange supports at most {_capi.MAX_PEERS} ranks, got {world}")
        self.geom_bytes, self.img_bytes, self.off_radii, self.off_grad, self.off_flags, self.total = self.layout(settings, self.P_total, device)
        self.hdl = None
        self.in_flight = False  # a differentiable forward has used the buffers and its backward has not run yet
        self.epoch = 0          # epoch of the last sgr_peer_barrier issued on this workspace (every rank counts alike)
        self.fwd_pending = False  # the last fused call was a forward: the next forward needs a leading barrier (see sgr.h)
        self._step_bufs = None
        if _buffers is not None:  # single-process emulation: (my buffer, base pointers of all ranks' buffers)
            self.buf, ptrs = _buffers
        else:
            import torch.distributed._symmetric_memory as symm
            self.buf = symm.empty(self.total, dtype=torch.uint8, device=device)
            self.buf[self.off_flags:].zero_()  # barrier pads start at epoch 0
            self.buf[self.off_radii: self.off_grad].zero_()
            self.hdl = symm.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
            ptrs = list(self.hdl.buffer_ptrs)
            self.hdl.barrier(channel=0)  # every pad is zero before any rank can send its first epoch
        self.geom = self.buf[: self.geom_bytes]
        self.radii_all = self.buf[self.off_radii: self.off_radii + 4 * self.P_total].view(torch.int32)
        self.grad2d = self.buf[self.off_grad: self.off_grad + 48 * self.P_total].view(torch.float32).view(self.P_total, 12)
        if _buffers is not None:
            self.buf[self.off_flags:].zero_()
            self.buf[self.off_radii: self.off_grad].zero_()
        self.peers = _capi.SgrPeers()
        self.peers.world, self.peers.rank, self.peers.chunk = self.world, self.rank, self.chunk
        for p in range(self.world):
            self.peers.records[p] = ptrs[p]
            self.peers.radii[p] = ptrs[p] + self.off_radii
            self.peers.grad2d[p] = ptrs[p] + self.off_grad
            self.peers.flags[p] = ptrs[p] + self.off_flags

    @staticmethod
    def layout(settings, P_total: int, device):
        """(geom_bytes, img_bytes, offset of radii_all, offset of grad2d, offset of the barrier pad, total bytes) of the per-rank buffer."""
        L = _capi.lib()
        fr, keep = _make_frame(settings, P_total, 0, 0, device, None)
        gb, ib = C.c_size_t(0), C.c_size_t(0)
        _capi.check(L.sgr_state_sizes(C.byref(fr), C.byref(gb), C.byref(ib)), "sgr_state_sizes")
        del keep
        off_radii = _align(gb.value)
        off_grad = _align(off_radii + 4 * P_total)
        off_flags = _align(off_grad + 48 * P_total)
        return gb.value, ib.value, off_radii, off_grad, off_flags, off_flags + 256

    @classmethod
    def emulate(cls, settings, chunk: int, world: int, device):
        """`world` workspaces on ONE device whose peer tables point at each other (tests; world == 1 module path)."""
        total = cls.layout(settings, int(chunk) * int(world), device)[5]
        bufs = [torch.empty(total, dtype=torch.uint8, device=device) for _ in range(world)]
        ptrs = [b.data_ptr() for b in bufs]
        return [cls(settings, chunk, world, r, device, _buffers=(bufs[r], ptrs)) for r in range(world)]

    def barrier(self):
        """Device-side barrier of the STAGED path (torch symmetric memory's signal pad)."""
        if self.hdl is not None:
            self.hdl.barrier(channel=0)

    def next_epochs(self, n: int = 1) -> int:
        """Reserve `n` consecutive barrier epochs of the fused path; returns the LAST one."""
        self.epoch += n
        return self.epoch

    def step_buffers(self, capacity_bytes: int):
        """Buffers that live from a fused forward to its backward.  One forward is in flight per workspace, so they are
        allocated once (and re-grown with the instance capacity) instead of once per step."""
        dev = self.buf.device
        b = self._step_bufs
        if b is None:
            b = dict(rec=torch.empty((self.chunk, REC_FLOATS), device=dev, dtype=torch.float32),
                     radii=torch.empty((self.chunk,), device=dev, dtype=torch.int32),
                     img=torch.empty((self.img_bytes,), device=dev, dtype=torch.uint8), binning=None)
            self._step_bufs = b
        if b["binning"] is None or b["binning"].numel() < capacity_bytes:
            b["binning"] = torch.empty((capacity_bytes,), device=dev, dtype=torch.uint8)
        return b


def scatter_records(settings, ws: PeerWorkspace, rec_local, radii_local, P_local: int):
    """Step 2 over peer memory (sgr_scatter_records).  The caller issues ws.barrier() afterwards."""
    L = _capi.lib()
    device = rec_local.device
    fr, keep = _make_frame(settings, P_local, 0, 0, device, None)
    with torch.cuda.device(device):
        rc = L.sgr_scatter_records(C.byref(fr), C.byref(ws.peers), _ptr(rec_local), _ptr(radii_local), _stream(device))
    _capi.check(rc, "sgr_scatter_records")
    del keep


def gather_grad2d(settings, ws: PeerWorkspace, rec_local, radii_local, P_local: int):
    """Step 4 over peer memory (sgr_gather_grad2d): summed grad2d rows [chunk,12] of the local Gaussians.  The caller has
    issued ws.barrier() after every rank's backward_blend_records(grad2d_out=ws.grad2d)."""
    L = _capi.lib()
    device = rec_local.device
    out = torch.empty((ws.chunk, 12), device=device, dtype=torch.float32)
    fr, keep = _make_frame(settings, P_local, 0, 0, device, None)
    with torch.cuda.device(device):
        rc = L.sgr_gather_grad2d(C.byref(fr), C.byref(ws.peers), _ptr(rec_local), _ptr(radii_local), _ptr(out), _stream(device))
    _capi.check(rc, "sgr_gather_grad2d")
    del keep
    return out


def peer_forward_state(ws: PeerWorkspace):
    st = _ForwardState()
    st.geom = ws.geom
    st.img = torch.empty((ws.img_bytes,), device=ws.buf.device, dtype=torch.uint8)
    st.binning, st.num_instances = None, 0
    return st


class _GaussianShardedRasterize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp, settings, owner,
                differentiable=True):
        tensors = _local_tensors(means3D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp)
        device, P = means3D.device, int(means3D.shape[0])
        world, chunk, group = owner.world, owner.chunk_for(P), owner.group
        S = int(tensors["semantics"].shape[1]) if tensors["semantics"] is not None else 0
        P_total = chunk * world
        ws = owner.workspace(device) if owner.exchange == "p2p" else None
        sem_all = None
        cap = owner.capacity
        if ws is not None and owner.fused and S == 0 and cap is not None and cap.capacity is not None:
            return _fused_forward(ctx, tensors, settings, owner, ws, P, chunk, differentiable,
                                  (means3D, means2D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp))
        rec, radii = project_records(tensors, settings, chunk)
        if ws is not None:  # records go straight into the peers' gathered arrays over NVLink
            if ws.in_flight:
                raise _capi.SgrError("GaussianShardedRasterizer(exchange='p2p') owns ONE peer workspace: run backward() of the previous "
                                     "forward (or call release_workspace()) before the next forward, or use one rasterizer per camera")
            if ws.fwd_pending:
                # the previous forward on this workspace had no backward (eval / no_grad loop): a peer may still be counting,
                # emitting or blending from the records this scatter overwrites — only the backward barrier orders that
                ws.barrier()
            scatter_records(settings, ws, rec, radii, P)
            ws.barrier()
            ws.fwd_pending = True
            st, radii_all, gb, ib = peer_forward_state(ws), ws.radii_all, ws.geom_bytes, ws.img_bytes
        else:
            st, rec_all, gb, ib = alloc_gathered(settings, P_total, S, device)
            radii_all = torch.empty((P_total,), device=device, dtype=torch.int32)
            if world > 1:
                dist.all_gather_into_tensor(rec_all.view(-1), rec.view(-1), group=group)
                dist.all_gather_into_tensor(radii_all, radii, group=group)
            else:
                rec_all.copy_(rec)
                radii_all.copy_(radii)
        if S > 0:
            sem_local = tensors["semantics"]
            if P < chunk:
                sem_local = torch.cat([sem_local, sem_local.new_zeros((chunk - P, S))])
            sem_all = torch.empty((P_total, S), device=device, dtype=torch.float32)
            if world > 1:
                dist.all_gather_into_tensor(sem_all.view(-1), sem_local.contiguous().view(-1), group=group)
            else:
                sem_all.copy_(sem_local)
        color, depth, alpha, semantic = forward_records(settings, owner.band, st, (gb, ib), radii_all, sem_all, owner.capacity)
        ctx.settings, ctx.owner, ctx.state, ctx.tensors = settings, owner, st, tensors
        ctx.sem_all, ctx.P_total, ctx.chunk, ctx.ws = sem_all, P_total, chunk, ws
        ctx.shapes = _input_shapes(means3D, means2D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp)
        ctx.save_for_backward(rec, radii, alpha)
        radii_out = radii[:P]
        ctx.mark_non_differentiable(radii_out)
        if ws is not None:
            ws.in_flight = bool(differentiable)
        return color, radii_out, depth, alpha, semantic

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha, grad_semantic):
        if getattr(ctx, "fused", False):
            return _fused_backward(ctx, grad_color, grad_depth, grad_alpha)
        rec, radii, alpha = ctx.saved_tensors
        settings, owner, st, tensors, shapes = ctx.settings, ctx.owner, ctx.state, ctx.tensors, ctx.shapes
        dev = alpha.device
        S = int(ctx.sem_all.shape[1]) if ctx.sem_all is not None else 0
        P = int(tensors["means3D"].shape[0])
        grad_color, grad_depth, grad_alpha, grad_semantic = _image_grads(settings, dev, (grad_color, grad_depth, grad_alpha, grad_semantic),
                                                                         (3, 1, 1, S))
        ws = ctx.ws
        grad2d, g_sem = backward_blend_records(settings, owner.band, st, ctx.P_total, ctx.sem_all, alpha, grad_color, grad_depth,
                                               grad_alpha, grad_semantic, grad2d_out=ws.grad2d if ws is not None else None)
        if ws is not None:  # pull the partial rows of the own Gaussians from the ranks that rendered them
            ws.barrier()
            ws.fwd_pending = False
            grad2d = gather_grad2d(settings, ws, rec, radii, P)
            ws.in_flight = False  # stream order protects the buffers from here on: the next forward is enqueued after the gather
            if owner.world > 1 and S > 0:
                gs_local = torch.empty((ctx.chunk, S), device=dev, dtype=torch.float32)
                dist.reduce_scatter_tensor(gs_local.view(-1), g_sem.view(-1), op=dist.ReduceOp.SUM, group=owner.group)
                g_sem = gs_local
        elif owner.world > 1:
            g2_local = torch.empty((ctx.chunk, 12), device=dev, dtype=torch.float32)
            dist.reduce_scatter_tensor(g2_local.view(-1), grad2d.view(-1), op=dist.ReduceOp.SUM, group=owner.group)
            if S > 0:
                gs_local = torch.empty((ctx.chunk, S), device=dev, dtype=torch.float32)
                dist.reduce_scatter_tensor(gs_local.view(-1), g_sem.view(-1), op=dist.ReduceOp.SUM, group=owner.group)
                g_sem = gs_local
            grad2d = g2_local
        if P == 0:
            g = (None,) * 8
        else:
            g = backward_geom_local(settings, tensors, rec, radii, grad2d)
        g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov = g
        return _fit_grads(shapes, (g_means3D, g_means2D, g_sh, g_colors, g_sem[:P] if S > 0 else None, g_opac, g_scales, g_rots,
                                   g_cov)) + (None, None, None)


def sharded_forward_raw(settings, band, ws: "PeerWorkspace", tensors, P: int, capacity: int, gaussian_capacity: int, status_word=None):
    """One sgr_sharded_forward call on the current stream (used by the autograd path and, with emulated workspaces on
    separate streams, by the single-GPU tests).  Returns (color, depth, alpha, step buffers)."""
    L = _capi.lib()
    device = tensors["means3D"].device
    H, W = int(settings.image_height), int(settings.image_width)
    nbytes = int(L.sgr_binning_bytes(capacity))
    bufs = ws.step_buffers(nbytes)
    z = lambda c: torch.zeros((c, H, W), device=device, dtype=torch.float32)  # foreign rows stay zero
    color, depth, alpha = z(3), z(1), z(1)  # (separate tensors: autograd outputs that are views of one base cannot be modified in place)
    M = int(tensors["sh"].shape[1]) if tensors["sh"] is not None else 0
    fr, keep = _make_frame(settings, P, M, 0, device, band)
    pre = 1 if ws.fwd_pending else 0
    ws.next_epochs(1 + pre)  # host-side tally only: the epochs themselves are counted on the device (barrier_epoch = 0)
    epoch = 0
    with torch.cuda.device(device):
        rc = L.sgr_sharded_forward(C.byref(fr), C.byref(ws.peers), _ptr(tensors["means3D"]), _ptr(tensors["sh"]), _ptr(tensors["colors_precomp"]),
                                   _ptr(tensors["opacities"]), _ptr(tensors["scales"]), _ptr(tensors["rotations"]), _ptr(tensors["cov3Ds_precomp"]),
                                   _ptr(color), _ptr(depth), _ptr(alpha), _ptr(bufs["radii"]), _ptr(bufs["rec"]), ws.geom_bytes,
                                   _ptr(bufs["img"]), ws.img_bytes, _ptr(bufs["binning"]), nbytes, capacity, gaussian_capacity, epoch, pre,
                                   _stream(device))
        _capi.check(rc, "sgr_sharded_forward")
        if status_word is not None:  # the status of the gathered frame (P_total slots)
            frt, keep2 = _make_frame(settings, ws.P_total, 0, 0, device, band)
            _copy_status(frt, ws.geom, status_word, device)
            del keep2
    del keep
    ws.fwd_pending = True
    return color, depth, alpha, bufs


def sharded_backward_raw(settings, band, ws: "PeerWorkspace", tensors, P: int, capacity: int, alpha, gc, gd, ga):
    """One sgr_sharded_backward call on the current stream.  Returns the 8 gradients in _backward_geom_impl's order."""
    L = _capi.lib()
    dev = alpha.device
    sh, colors, scales, rots, cov = (tensors[k] for k in ("sh", "colors_precomp", "scales", "rotations", "cov3Ds_precomp"))
    M = int(sh.shape[1]) if sh is not None else 0
    g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov = _geom_grad_buffers(tensors, P, dev)
    bufs = ws.step_buffers(0)
    fr, keep = _make_frame(settings, P, M, 0, dev, band)
    ws.next_epochs(1)
    epoch = 0  # device-side count
    with torch.cuda.device(dev):
        rc = L.sgr_sharded_backward(C.byref(fr), C.byref(ws.peers), capacity, _ptr(tensors["means3D"]), _ptr(sh), _ptr(colors), _ptr(scales),
                                    _ptr(rots), _ptr(cov), _ptr(bufs["radii"]), _ptr(bufs["rec"]), _ptr(bufs["img"]), _ptr(bufs["binning"]),
                                    _ptr(alpha), _ptr(gc), _ptr(gd), _ptr(ga), _ptr(g_means3D), _ptr(g_means2D), _ptr(g_sh), _ptr(g_colors),
                                    _ptr(g_opac), _ptr(g_scales), _ptr(g_rots), _ptr(g_cov), epoch, _stream(dev))
    _capi.check(rc, "sgr_sharded_backward")
    del keep
    ws.fwd_pending = False  # every rank passed the backward barrier after its blend_bwd: the records may be overwritten
    return g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov


def _fused_forward(ctx, tensors, settings, owner, ws: "PeerWorkspace", P: int, chunk: int, differentiable: bool, inputs):
    """sgr_sharded_forward: project + scatter, barrier, bin / sort / blend in ONE C-ABI call (no host work between the ~28 launches)."""
    device = tensors["means3D"].device
    if ws.in_flight:
        raise _capi.SgrError("GaussianShardedRasterizer(exchange='p2p') owns ONE peer workspace: run backward() of the previous "
                             "forward (or call release_workspace()) before the next forward, or use one rasterizer per camera")
    cap = owner.capacity
    if not cap.frozen:
        cap.check()
    H, W = int(settings.image_height), int(settings.image_width)
    capacity = int(cap.capacity)
    # depth-order slots: learnt from the previous frames (status word 4); the first fused frame compacts into all slots
    gcap = int(cap.gaussian_capacity) if cap.gaussian_capacity is not None else ws.P_total
    color, depth, alpha, bufs = sharded_forward_raw(settings, owner.band, ws, tensors, P, capacity, gcap)
    if not cap.frozen:  # the status of the gathered frame (P_total slots)
        frt, keep = _make_frame(settings, ws.P_total, 0, 0, device, owner.band)
        cap.record_status(frt, ws.geom, device)
        del keep
    ws.in_flight = bool(differentiable)
    ctx.fused, ctx.settings, ctx.owner, ctx.ws, ctx.P, ctx.capacity, ctx.tensors = True, settings, owner, ws, P, capacity, tensors
    ctx.shapes = _input_shapes(*inputs)
    ctx.save_for_backward(alpha)
    radii_out = bufs["radii"][:P]
    ctx.mark_non_differentiable(radii_out)
    return color, radii_out, depth, alpha, torch.zeros((0, H, W), device=device, dtype=torch.float32)


def _fused_backward(ctx, grad_color, grad_depth, grad_alpha):
    """sgr_sharded_backward: blend_bwd, barrier, chain rule with the peer gather folded in — ONE C-ABI call."""
    (alpha,) = ctx.saved_tensors
    settings, owner, ws, P, tensors, shapes = ctx.settings, ctx.owner, ctx.ws, ctx.P, ctx.tensors, ctx.shapes
    dev = alpha.device
    gc, gd, ga = (_dev_f32(g, dev) for g in _image_grads(settings, dev, (grad_color, grad_depth, grad_alpha), (3, 1, 1)))
    g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov = sharded_backward_raw(settings, owner.band, ws, tensors, P,
                                                                                                   ctx.capacity, alpha, gc, gd, ga)
    ws.in_flight = False
    return _fit_grads(shapes, (g_means3D, g_means2D, g_sh, g_colors, None, g_opac, g_scales, g_rots, g_cov)) + (None, None, None)


class GaussianShardedRasterizer(nn.Module):
    """Same call signature as GaussianRasterizer.forward, but every argument holds only THIS rank's Gaussians and the
    returned radii / gradients cover only them; the images cover this rank's tile rows (zeros elsewhere).  The gathered
    order is rank-major, so with rank r holding rows [r*chunk, (r+1)*chunk) of a global array the images are
    bit-identical to the single-GPU render of that array."""

    def __init__(self, raster_settings: GaussianRasterizationSettings, group: Optional[dist.ProcessGroup] = None,
                 layout: str = "cyclic", capacity: Optional[InstanceCapacity] = None, chunk: Optional[int] = None,
                 exchange: str = "nccl", fused: bool = True):
        """exchange = "nccl": all-gather of records / reduce-scatter of grad2d.  exchange = "p2p": each record is stored
        over NVLink into the gathered arrays of only the ranks whose band it touches and the grad2d rows are read back
        from them (PeerWorkspace; needs torch symmetric memory and the cyclic layout).  With "p2p" the rasterizer owns ONE
        workspace: a forward's backward must run before the next forward of the same module."""
        super().__init__()
        if exchange not in ("nccl", "p2p"):
            raise ValueError("exchange must be 'nccl' or 'p2p'")
        if exchange == "p2p" and layout != "cyclic":
            raise ValueError("the peer-memory exchange needs the cyclic tile-row layout")
        self.exchange, self._ws = exchange, None
        # exchange="p2p" with a capacity object (sync-free binning) and no feature channels runs the whole forward / backward as
        # ONE C-ABI call each (sgr_sharded_forward / sgr_sharded_backward) once the capacity is known; fused=False keeps the
        # staged calls (one per step of include/sgr.h's list)
        self.fused = bool(fused)
        self.raster_settings, self.group, self.capacity = raster_settings, group, capacity
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        mk = cyclic_band if layout == "cyclic" else contiguous_band
        self.band = mk(raster_settings.image_height, self.rank, self.world) if self.world > 1 else None
        self.chunk = int(chunk) if chunk else None

    def repartition(self, P_local: int) -> int:
        """COLLECTIVE: agree on the per-rank slot count after the local Gaussian count changed (densify / prune)."""
        self.chunk = chunk_size(P_local, self.group)
        return self.chunk

    def workspace(self, device) -> "PeerWorkspace":
        """COLLECTIVE on first use and after repartition(): allocate + rendezvous the peer-mapped buffer."""
        if self._ws is None or self._ws.chunk != self.chunk:
            if self.world > 1:
                self._ws = PeerWorkspace(self.raster_settings, self.chunk, self.world, self.rank, device, self.group)
            else:
                self._ws = PeerWorkspace.emulate(self.raster_settings, self.chunk, 1, device)[0]
        return self._ws

    def release_workspace(self):
        """Declare that the last differentiable forward will never be back-propagated (its graph was dropped)."""
        if self._ws is not None:
            self._ws.in_flight = False

    def chunk_for(self, P_local: int) -> int:
        if self.chunk is None:  # first forward: every rank is here together
            self.repartition(P_local)
        return self.chunk

    def synchronize_capacity(self):
        if self.capacity is not None:
            self.capacity.check(wait=True)

    def forward_layers(self, *args, **kwargs):
        raise _capi.SgrError("render layers are single-GPU only: use GaussianRasterizer")

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None,
                semantics=None):
        shs, colors_precomp, scales, rotations, cov3D_precomp, semantics = _reference_inputs(means3D, shs, colors_precomp, scales, rotations,
                                                                                             cov3D_precomp, semantics)
        args = (means3D, means2D, shs, colors_precomp, semantics, opacities, scales, rotations, cov3D_precomp)
        differentiable = torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in args)
        return _GaussianShardedRasterize.apply(*args, self.raster_settings, self, differentiable)
