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

import contextlib
import ctypes as C
import math
from typing import List, NamedTuple, Optional, Sequence

import torch
import torch.distributed as dist
import torch.nn as nn

from . import _capi
from ._capi import ptr
from .training import ADAM_GROUP_NAMES, PARAM_NAMES, STAT_NAMES, _attr, _has, _install, _param_slots, _segment, _set, _stat_segment
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, InstanceCapacity, TileRowBand, _check_layers, _copy_status,
                         _ForwardState, _backward_blend_impl, _backward_geom_impl, _fit_grads, _fp32_inputs, _geom_grad_buffers, _image_grads,
                         _input_shapes, _make_frame, _reference_inputs)


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
    P_local are padding (radii == 0).  The records are the head of a whole geom state for P_local (sgr_state_sizes bytes,
    132 B per Gaussian + cub temp), which also holds the colour Jacobian that backward_geom_local reads, so the state stays
    alive with the records until the backward; the rows of padding slots may overlap that Jacobian (they are never read)."""
    means3D = tensors["means3D"]
    device, P = means3D.device, int(means3D.shape[0])
    if P > chunk:
        raise _capi.SgrError(f"{P} local Gaussians do not fit the per-rank chunk of {chunk}; call repartition()")
    M = int(tensors["sh"].shape[1]) if tensors["sh"] is not None else 0
    fr, keep = _make_frame(settings, P, M, 0, device, None)
    gb = C.c_size_t(0)
    _capi.call("sgr_state_sizes", None, C.byref(fr), C.byref(gb), None)
    state = torch.empty((max(gb.value, chunk * REC_FLOATS * 4),), device=device, dtype=torch.uint8)
    rec = state[: chunk * REC_FLOATS * 4].view(torch.float32).view(chunk, REC_FLOATS)
    radii = (torch.empty if P == chunk else torch.zeros)((chunk,), device=device, dtype=torch.int32)
    _capi.call("sgr_project", device, C.byref(fr), ptr(means3D), ptr(tensors["sh"]), ptr(tensors["colors_precomp"]), ptr(tensors["opacities"]),
               ptr(tensors["scales"]), ptr(tensors["rotations"]), ptr(tensors["cov3Ds_precomp"]), ptr(radii), ptr(state))
    del keep
    return rec, radii


def alloc_gathered(settings: GaussianRasterizationSettings, P_total: int, S: int, device):
    """Forward state for P_total gathered Gaussians.  Returns (state, records view [P_total,12] float32 into state.geom —
    the all-gather target —, geom_bytes, img_bytes)."""
    fr, keep = _make_frame(settings, P_total, 0, S, device, None)
    gb, ib = C.c_size_t(0), C.c_size_t(0)
    _capi.call("sgr_state_sizes", None, C.byref(fr), C.byref(gb), C.byref(ib))
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
    _capi.call("sgr_forward_records", device, C.byref(fr), ptr(radii_all), ptr(semantics_all), ptr(color), ptr(depth), ptr(alpha), ptr(semantic),
               ptr(st.geom), gb, ptr(st.img), ib, cb, None, C.byref(bin_ptr), C.byref(n_inst), ptr(st.binning) if bounded else None, nbytes, cap)
    st.bounded = bounded
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
    st.geom = rec_local  # the head of project_records' geom state: sgr_backward_geom reads the colour Jacobian sgr_project left there
    local = dict(tensors)
    local["semantics"] = None
    return _backward_geom_impl(settings, None, st, local, radii_local[:P], grad2d_local[:P].contiguous())


def _align(n: int, a: int = 256) -> int:
    return (n + a - 1) // a * a


class PeerWorkspace:
    """Per-rank buffer [geom_state | radii_all | grad2d | sem | gsem | pose_acc | loss | layer_mask | layer_grad2d | barrier pad] that
    every rank of the group can address (include/sgr.h, SgrPeers).  The two layer sections exist with `layers` > 0 (render layers of
    the fused step, GaussianShardedRasterizer.forward_layers).

    Real multi-GPU: ONE torch symmetric-memory allocation per rank (CUDA VMM mapped into every process; NVLink loads and
    stores), rendezvous'ed once; `barrier()` is the device-side signal-pad barrier of that allocation (a few microseconds
    over NVLink).  `emulate(...)` builds `world` ordinary buffers on ONE device that point at each other, so the exchange
    kernels can be tested without a second GPU."""

    def __init__(self, settings, chunk: int, world: int, rank: int, device, group=None, _buffers=None, S: int = 0, layers: int = 0):
        self.chunk, self.world, self.rank, self.P_total = int(chunk), int(world), int(rank), int(chunk) * int(world)
        self.S, self.layers = int(S), int(layers)
        if world > _capi.MAX_PEERS:
            raise _capi.SgrError(f"peer exchange supports at most {_capi.MAX_PEERS} ranks, got {world}")
        self.geom_bytes, self.img_bytes, self.off_radii, self.off_grad, self.off_flags, self.total = self.layout(settings, self.P_total, device,
                                                                                                                 self.S, layers=self.layers)
        self.off_sem, self.off_gsem = self.feature_offsets(self.off_grad, self.P_total, self.S)
        self.off_pose = self.pose_offset(self.off_grad, self.P_total, self.S)
        self.off_loss, self.loss_bytes = self.loss_offset(self.off_grad, self.P_total, self.S), self.loss_section_bytes(settings)
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
            if self.S:
                self.peers.sem[p] = ptrs[p] + self.off_sem
                self.peers.gsem[p] = ptrs[p] + self.off_gsem
            self.peers.pose_acc[p] = ptrs[p] + self.off_pose
            self.peers.loss[p] = ptrs[p] + self.off_loss
        self.peers.loss_bytes = self.loss_bytes
        self.off_layer_mask, self.off_layer_grad = self.layer_offsets(settings, self.off_grad, self.P_total, self.S)
        self.layer_peers = _capi.SgrLayerPeers()
        self.layer_peers.layers = self.layers
        if self.layers:
            for p in range(self.world):
                self.layer_peers.layer_mask[p] = ptrs[p] + self.off_layer_mask
                self.layer_peers.layer_grad2d[p] = ptrs[p] + self.off_layer_grad
        self.layer_mask = self.buf[self.off_layer_mask: self.off_layer_mask + self.P_total * (self.layers > 0)]
        nl = 48 * self.P_total * self.layers
        self.layer_grad2d = self.buf[self.off_layer_grad: self.off_layer_grad + nl].view(torch.float32).view(self.layers, self.P_total, 12)
        self._layer_states = []
        nsem = self.P_total * self.S
        self.sem = self.buf[self.off_sem: self.off_sem + 4 * nsem].view(torch.float32).view(self.P_total, self.S)
        self.gsem = self.buf[self.off_gsem: self.off_gsem + 4 * nsem].view(torch.float32).view(self.P_total, self.S)

    @staticmethod
    def feature_offsets(off_grad: int, P_total: int, S: int):
        """Offsets of the feature sections sem and gsem ([P_total, S] fp32 each, rows by slot), between grad2d and the barrier pad."""
        off_sem = _align(off_grad + 48 * P_total)
        return off_sem, _align(off_sem + 4 * P_total * S)

    @staticmethod
    def pose_offset(off_grad: int, P_total: int, S: int) -> int:
        """Offset of the composer's accumulator section (_capi.POSE_ACC_ROWS rows of 16 fp32, composer.compose's reduction over the
        ranks), after the feature sections and before the barrier pad."""
        return _align(PeerWorkspace.feature_offsets(off_grad, P_total, S)[1] + 4 * P_total * S)

    @staticmethod
    def loss_offset(off_grad: int, P_total: int, S: int) -> int:
        """Offset of the band losses' section (band_losses.py's peer-memory halo and sums), after the composer's accumulator section
        and before the barrier pad."""
        return _align(PeerWorkspace.pose_offset(off_grad, P_total, S) + 64 * _capi.POSE_ACC_ROWS)

    @staticmethod
    def loss_section_bytes(settings) -> int:
        """Bytes of the band losses' section for the settings' image: sgr_band_peer_bytes of a 3-channel image (the largest pair of
        halo messages any band sends, or the largest array the losses sum)."""
        n = int(_capi.lib().sgr_band_peer_bytes(3, int(settings.image_height), int(settings.image_width)))
        if n == 0:
            raise _capi.SgrError(f"bad image size {settings.image_width}x{settings.image_height} for the band losses' section")
        return n

    @staticmethod
    def layer_offsets(settings, off_grad: int, P_total: int, S: int):
        """Offsets of the render layers' sections, after the band losses' section and before the barrier pad: layer_mask (one byte per
        slot, bit k = layer k) and layer_grad2d (rows of 12 fp32 per slot, P_total rows per layer)."""
        off_mask = _align(PeerWorkspace.loss_offset(off_grad, P_total, S) + PeerWorkspace.loss_section_bytes(settings))
        return off_mask, _align(off_mask + P_total)

    @staticmethod
    def layout(settings, P_total: int, device, S: int = 0, layers: int = 0):
        """(geom_bytes, img_bytes, offset of radii_all, offset of grad2d, offset of the barrier pad, total bytes) of the per-rank buffer.
        With S feature channels the sections sem and gsem (feature_offsets) sit before the pad; S = 0 leaves them empty.  The composer's
        accumulator section (pose_offset) follows them, then the band losses' section (loss_offset, loss_section_bytes), then with
        `layers` render layers their mask and gradient sections (layer_offsets)."""
        fr, keep = _make_frame(settings, P_total, 0, 0, device, None)
        gb, ib = C.c_size_t(0), C.c_size_t(0)
        _capi.call("sgr_state_sizes", None, C.byref(fr), C.byref(gb), C.byref(ib))
        del keep
        off_radii = _align(gb.value)
        off_grad = _align(off_radii + 4 * P_total)
        if layers:
            off_flags = _align(PeerWorkspace.layer_offsets(settings, off_grad, P_total, S)[1] + 48 * P_total * int(layers))
        else:
            off_flags = _align(PeerWorkspace.loss_offset(off_grad, P_total, S) + PeerWorkspace.loss_section_bytes(settings))
        return gb.value, ib.value, off_radii, off_grad, off_flags, off_flags + 256

    @classmethod
    def emulate(cls, settings, chunk: int, world: int, device, S: int = 0, layers: int = 0):
        """`world` workspaces on ONE device whose peer tables point at each other (tests; world == 1 module path)."""
        total = cls.layout(settings, int(chunk) * int(world), device, S, layers=layers)[-1]
        bufs = [torch.empty(total, dtype=torch.uint8, device=device) for _ in range(world)]
        ptrs = [b.data_ptr() for b in bufs]
        return [cls(settings, chunk, world, r, device, _buffers=(bufs[r], ptrs), S=S, layers=layers) for r in range(world)]

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

    def layer_states(self, n: int, state_bytes: int):
        """The states of `n` render layers (sgr_sharded_layer_state_sizes bytes each), kept from a fused forward to its backward like
        step_buffers."""
        dev = self.buf.device
        st = self._layer_states
        while len(st) < n:
            st.append(torch.empty((0,), device=dev, dtype=torch.uint8))
        for k in range(n):
            if st[k].numel() < state_bytes:
                st[k] = torch.empty((state_bytes,), device=dev, dtype=torch.uint8)
        return st[:n]


class SkyWorkspace:
    """Per-rank sky section [6 R^2 3 fp32 | block map] that every rank of the group can address (include/sgr.h, SgrSkyPeers), and this
    rank's own block map: the sky cube gradient's exchange over peer memory (sky.sky_composite with rasterizer= of a
    GaussianShardedRasterizer(exchange="p2p"), sgr_sky_grad_peer_sum).

    Its own torch symmetric-memory allocation, keyed on (R, world), so it outlives the rasterizer's PeerWorkspace across repartition();
    it has no barrier pad: the exchange takes its barriers from the rasterizer's current workspace.  `emulate(...)` builds `world`
    ordinary buffers on ONE device that point at each other, as PeerWorkspace.emulate does."""

    def __init__(self, R: int, world: int, rank: int, device, group=None, _buffers=None):
        self.R, self.world, self.rank = int(R), int(world), int(rank)
        if world > _capi.MAX_PEERS:
            raise _capi.SgrError(f"peer exchange supports at most {_capi.MAX_PEERS} ranks, got {world}")
        self.bytes, self.blocks = self.section_bytes(self.R), int(_capi.lib().sgr_sky_grad_blocks(self.R))
        self.hdl = None
        if _buffers is not None:
            self.buf, ptrs = _buffers
        else:
            import torch.distributed._symmetric_memory as symm
            self.buf = symm.empty(self.bytes, dtype=torch.uint8, device=device)
            self.hdl = symm.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
            ptrs = list(self.hdl.buffer_ptrs)
        self.peers = _capi.SgrSkyPeers()
        for p in range(self.world):
            self.peers.sec[p] = ptrs[p]
        self.peers.bytes = self.bytes
        self.block_map = torch.zeros(self.blocks, dtype=torch.uint8, device=device)

    @staticmethod
    def section_bytes(R: int) -> int:
        n = int(_capi.lib().sgr_sky_peer_bytes(int(R)))
        if n == 0:
            raise _capi.SgrError(f"bad cube map resolution R={R} for the sky section")
        return n

    @classmethod
    def emulate(cls, R: int, world: int, device):
        """`world` sky workspaces on ONE device whose section tables point at each other (tests)."""
        bufs = [torch.empty(cls.section_bytes(R), dtype=torch.uint8, device=device) for _ in range(world)]
        ptrs = [b.data_ptr() for b in bufs]
        return [cls(R, world, r, device, _buffers=(bufs[r], ptrs)) for r in range(world)]


def scatter_records(settings, ws: PeerWorkspace, rec_local, radii_local, P_local: int):
    """Step 2 over peer memory (sgr_scatter_records).  The caller issues ws.barrier() afterwards."""
    device = rec_local.device
    fr, keep = _make_frame(settings, P_local, 0, 0, device, None)
    _capi.call("sgr_scatter_records", device, C.byref(fr), C.byref(ws.peers), ptr(rec_local), ptr(radii_local))
    del keep


def gather_grad2d(settings, ws: PeerWorkspace, rec_local, radii_local, P_local: int):
    """Step 4 over peer memory (sgr_gather_grad2d): summed grad2d rows [chunk,12] of the local Gaussians.  The caller has
    issued ws.barrier() after every rank's backward_blend_records(grad2d_out=ws.grad2d)."""
    device = rec_local.device
    out = torch.empty((ws.chunk, 12), device=device, dtype=torch.float32)
    fr, keep = _make_frame(settings, P_local, 0, 0, device, None)
    _capi.call("sgr_gather_grad2d", device, C.byref(fr), C.byref(ws.peers), ptr(rec_local), ptr(radii_local), ptr(out))
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
        cap = owner.capacity
        # feature channels ride the fused step up to the blend backward's limit; more take the staged path (forward only)
        fused = owner.exchange == "p2p" and owner.fused and S <= _capi.MAX_SEMANTIC_BWD and cap is not None and cap.capacity is not None
        ws = owner.workspace(device, S if fused else 0) if owner.exchange == "p2p" else None
        sem_all = None
        if fused:
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
            return _fused_backward(ctx, grad_color, grad_depth, grad_alpha, grad_semantic)
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


def sharded_forward_raw(settings, band, ws: "PeerWorkspace", tensors, P: int, capacity: int, gaussian_capacity: int, status_word=None,
                        semantics=None, layers=None):
    """One sgr_sharded_forward call on the current stream (used by the autograd path and, with emulated workspaces on
    separate streams, by the single-GPU tests).  Returns (color, depth, alpha, step buffers).  semantics [P, S] (this rank's rows,
    S = ws.S): sgr_sharded_forward_features, and the banded feature image [S, H, W] is returned as a fifth value.  layers: (begin, end,
    bg) per render layer in this rank's rows (at most ws.layers): sgr_sharded_forward_layers, and the list of every layer's (color,
    depth, alpha), zero outside the band, is returned as a fifth value; the layer states stay in the workspace for the backward."""
    L = _capi.lib()
    device = tensors["means3D"].device
    H, W = int(settings.image_height), int(settings.image_width)
    nbytes = int(L.sgr_binning_bytes(capacity))
    bufs = ws.step_buffers(nbytes)
    z = lambda c: torch.zeros((c, H, W), device=device, dtype=torch.float32)  # foreign rows stay zero
    color, depth, alpha = z(3), z(1), z(1)  # (separate tensors: autograd outputs that are views of one base cannot be modified in place)
    M = int(tensors["sh"].shape[1]) if tensors["sh"] is not None else 0
    S = 0 if semantics is None else int(semantics.shape[1])
    if S != ws.S:
        raise ValueError(f"the workspace carries {ws.S} feature channels, the call {S}")
    fr, keep = _make_frame(settings, P, M, S, device, band)
    pre = 1 if ws.fwd_pending else 0
    ws.next_epochs(1 + pre)  # host-side tally only: the epochs themselves are counted on the device (barrier_epoch = 0)
    epoch = 0
    args = (C.byref(fr), C.byref(ws.peers), ptr(tensors["means3D"]), ptr(tensors["sh"]), ptr(tensors["colors_precomp"]), ptr(tensors["opacities"]),
            ptr(tensors["scales"]), ptr(tensors["rotations"]), ptr(tensors["cov3Ds_precomp"]), ptr(color), ptr(depth), ptr(alpha), ptr(bufs["radii"]),
            ptr(bufs["rec"]), ws.geom_bytes, ptr(bufs["img"]), ws.img_bytes, ptr(bufs["binning"]), nbytes, capacity, gaussian_capacity, epoch, pre)
    if S:
        sem_in = _capi.f32(semantics, device)
        semantic = z(S)
        _capi.call("sgr_sharded_forward_features", device, *args, ptr(sem_in), ptr(semantic))
    elif layers is not None:
        if not 0 < len(layers) <= ws.layers:
            raise ValueError(f"the workspace carries {ws.layers} render layers, the call {len(layers)}")
        nb = C.c_size_t(0)
        _capi.call("sgr_sharded_layer_state_sizes", None, C.byref(fr), capacity, C.byref(nb))
        states = ws.layer_states(len(layers), nb.value)
        table = (_capi.SgrShardedLayer * len(layers))()
        outs, bgs = [], []
        for k, (b, e, bg) in enumerate(layers):
            bgs.append(_capi.f32(bg, device, align16=True))
            outs.append((z(3), z(1), z(1)))
            table[k] = _capi.SgrShardedLayer(b, e, bgs[-1].data_ptr(), states[k].data_ptr(), states[k].numel(), *(t.data_ptr() for t in outs[-1]))
        _capi.call("sgr_sharded_forward_layers", device, *args, C.byref(ws.layer_peers), table, len(layers))
        semantic = outs
    else:
        _capi.call("sgr_sharded_forward", device, *args)
    if status_word is not None:  # the status of the gathered frame (P_total slots)
        frt, keep2 = _make_frame(settings, ws.P_total, 0, 0, device, band)
        _copy_status(frt, ws.geom, status_word, device)
        del keep2
    del keep
    ws.fwd_pending = True
    return (color, depth, alpha, bufs, semantic) if S or layers is not None else (color, depth, alpha, bufs)


def sharded_backward_raw(settings, band, ws: "PeerWorkspace", tensors, P: int, capacity: int, alpha, gc, gd, ga, gs=None, layers=None):
    """One sgr_sharded_backward call on the current stream.  Returns the 8 gradients in _backward_geom_impl's order.  gs [S, H, W]
    (the feature image's upstream gradient, after a forward with semantics): sgr_sharded_backward_features, and dL/dsemantics [P, S]
    of this rank's own Gaussians is returned as a ninth value.  layers (after a forward with layers, the same table): (begin, end, bg,
    alpha, (g_color, g_depth, g_alpha) or None, means2D sink [end - begin, 3] fp32 or None) per layer: sgr_sharded_backward_layers,
    which writes each layer's own screen-space gradient into its sink."""
    dev = alpha.device
    sh, colors, scales, rots, cov = (tensors[k] for k in ("sh", "colors_precomp", "scales", "rotations", "cov3Ds_precomp"))
    M = int(sh.shape[1]) if sh is not None else 0
    g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov = _geom_grad_buffers(tensors, P, dev)
    bufs = ws.step_buffers(0)
    S = 0 if gs is None else ws.S
    fr, keep = _make_frame(settings, P, M, S, dev, band)
    ws.next_epochs(1)
    epoch = 0  # device-side count
    args = (C.byref(fr), C.byref(ws.peers), capacity, ptr(tensors["means3D"]), ptr(sh), ptr(colors), ptr(scales), ptr(rots), ptr(cov),
            ptr(bufs["radii"]), ptr(bufs["rec"]), ptr(bufs["img"]), ptr(bufs["binning"]), ptr(alpha), ptr(gc), ptr(gd), ptr(ga), ptr(g_means3D),
            ptr(g_means2D), ptr(g_sh), ptr(g_colors), ptr(g_opac), ptr(g_scales), ptr(g_rots), ptr(g_cov), epoch)
    if S:
        g_sem = torch.empty((P, S), device=dev, dtype=torch.float32)
        _capi.call("sgr_sharded_backward_features", dev, *args, ptr(_capi.f32(gs, dev)), ptr(g_sem))
    elif layers is not None:
        frs = _make_frame(settings, P, M, 0, dev, band)
        nb = C.c_size_t(0)
        _capi.call("sgr_sharded_layer_state_sizes", None, C.byref(frs[0]), capacity, C.byref(nb))
        states = ws.layer_states(len(layers), nb.value)
        table = (_capi.SgrShardedLayer * len(layers))()
        keep_alive = []
        for k, (b, e, bg, l_alpha, grads, sink) in enumerate(layers):
            bg = _capi.f32(bg, dev, align16=True)
            gl = (None,) * 3 if grads is None else tuple(_capi.f32(g, dev, align16=True) for g in grads)
            keep_alive += [bg, *gl]
            table[k] = _capi.SgrShardedLayer(b, e, bg.data_ptr(), states[k].data_ptr(), states[k].numel(), None, None, l_alpha.data_ptr(),
                                             *(None if g is None else g.data_ptr() for g in gl), None if sink is None else sink.data_ptr())
        _capi.call("sgr_sharded_backward_layers", dev, *args, C.byref(ws.layer_peers), table, len(layers))
        del keep_alive, frs
    else:
        _capi.call("sgr_sharded_backward", dev, *args)
    del keep
    ws.fwd_pending = False  # every rank passed the backward barrier after its blend_bwd: the records may be overwritten
    grads = (g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov)
    return grads + (g_sem,) if S else grads


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
    S = ws.S
    out = sharded_forward_raw(settings, owner.band, ws, tensors, P, capacity, gcap, semantics=tensors["semantics"] if S else None)
    color, depth, alpha, bufs = out[:4]
    semantic = out[4] if S else torch.zeros((0, H, W), device=device, dtype=torch.float32)
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
    return color, radii_out, depth, alpha, semantic


def _fused_backward(ctx, grad_color, grad_depth, grad_alpha, grad_semantic):
    """sgr_sharded_backward: blend_bwd, barrier, chain rule with the peer gather folded in — ONE C-ABI call."""
    (alpha,) = ctx.saved_tensors
    settings, owner, ws, P, tensors, shapes = ctx.settings, ctx.owner, ctx.ws, ctx.P, ctx.tensors, ctx.shapes
    dev = alpha.device
    S = ws.S
    gc, gd, ga, gs = (_capi.f32(g, dev, align16=True) if g is not None else None
                      for g in _image_grads(settings, dev, (grad_color, grad_depth, grad_alpha, grad_semantic), (3, 1, 1, S)))
    out = sharded_backward_raw(settings, owner.band, ws, tensors, P, ctx.capacity, alpha, gc, gd, ga, gs if S else None)
    g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov = out[:8]
    g_sem = out[8] if S else None
    ws.in_flight = False
    return _fit_grads(shapes, (g_means3D, g_means2D, g_sh, g_colors, g_sem, g_opac, g_scales, g_rots, g_cov)) + (None, None, None)


class _GaussianShardedLayers(torch.autograd.Function):
    """The fused step with render layers (sgr_sharded_forward_layers / sgr_sharded_backward_layers).  Outputs (color, radii, depth,
    alpha, semantic), then (color, depth, alpha) per layer; `layers` holds _check_layers' tuples and `sinks` their means2D tensors."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp, settings, owner,
                differentiable, layers, *sinks):
        # an output without upstream gradient arrives as None, so a layer without one costs nothing in backward
        ctx.set_materialize_grads(False)
        tensors = _local_tensors(means3D, sh, colors_precomp, None, opacities, scales, rotations, cov3Ds_precomp)
        device, P = means3D.device, int(means3D.shape[0])
        owner.chunk_for(P)
        # (checked before workspace() may replace a workspace whose forward still awaits its backward)
        if owner._ws is not None and owner._ws.in_flight:
            raise _capi.SgrError("GaussianShardedRasterizer(exchange='p2p') owns ONE peer workspace: run backward() of the previous "
                                 "forward (or call release_workspace()) before the next forward, or use one rasterizer per camera")
        ws = owner.workspace(device, 0, len(layers))
        cap = owner.capacity
        if not cap.frozen:
            cap.check()
        H, W = int(settings.image_height), int(settings.image_width)
        capacity = int(cap.capacity)
        gcap = int(cap.gaussian_capacity) if cap.gaussian_capacity is not None else ws.P_total
        color, depth, alpha, bufs, louts = sharded_forward_raw(settings, owner.band, ws, tensors, P, capacity, gcap,
                                                               layers=[(b, e, bg) for b, e, bg, _ in layers])
        if not cap.frozen:
            frt, keep = _make_frame(settings, ws.P_total, 0, 0, device, owner.band)
            cap.record_status(frt, ws.geom, device)
            del keep
        ws.in_flight = bool(differentiable)
        ctx.settings, ctx.owner, ctx.ws, ctx.P, ctx.capacity, ctx.tensors, ctx.layers = settings, owner, ws, P, capacity, tensors, layers
        ctx.shapes = _input_shapes(means3D, means2D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp)
        ctx.save_for_backward(alpha, *(a for _, _, a in louts))
        radii_out = bufs["radii"][:P]
        ctx.mark_non_differentiable(radii_out)
        return (color, radii_out, depth, alpha, torch.zeros((0, H, W), device=device, dtype=torch.float32), *(t for o in louts for t in o))

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha, grad_semantic, *grad_layers):
        alpha, *layer_alphas = ctx.saved_tensors
        settings, owner, ws, P, tensors = ctx.settings, ctx.owner, ctx.ws, ctx.P, ctx.tensors
        dev = alpha.device
        gc, gd, ga = (_capi.f32(g, dev, align16=True) for g in _image_grads(settings, dev, (grad_color, grad_depth, grad_alpha), (3, 1, 1)))
        table = []
        for k, (b, e, bg, sink) in enumerate(ctx.layers):
            g3 = grad_layers[3 * k: 3 * k + 3]
            grads = None if all(g is None for g in g3) else _image_grads(settings, dev, g3, (3, 1, 1))
            sg = None
            if grads is not None and sink is not None and ctx.needs_input_grad[13 + k]:
                sg = torch.empty((e - b, 3), device=dev, dtype=torch.float32)
            table.append((b, e, bg, layer_alphas[k], grads, sg))
        out = sharded_backward_raw(settings, owner.band, ws, tensors, P, ctx.capacity, alpha, gc, gd, ga, layers=table)
        ws.in_flight = False
        g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov = out
        return (_fit_grads(ctx.shapes, (g_means3D, g_means2D, g_sh, g_colors, None, g_opac, g_scales, g_rots, g_cov)) + (None,) * 4
                + tuple(None if t[5] is None else t[5].to(dtype=l[3].dtype, device=l[3].device) for t, l in zip(table, ctx.layers)))


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
        self._sky = None  # SkyWorkspace of sky_workspace(R), kept across repartition()
        # exchange="p2p" with a capacity object (sync-free binning) and at most 32 feature channels runs the whole forward / backward as
        # ONE C-ABI call each (sgr_sharded_forward / sgr_sharded_backward) once the capacity is known; fused=False keeps the
        # staged calls (one per step of include/sgr.h's list)
        self.fused = bool(fused)
        self.raster_settings, self.group, self.capacity = raster_settings, group, capacity
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        mk = cyclic_band if layout == "cyclic" else contiguous_band
        self.band = mk(raster_settings.image_height, self.rank, self.world) if self.world > 1 else None
        self.chunk = int(chunk) if chunk else None

    def repartition(self, P_local: int, chunk: Optional[int] = None) -> int:
        """COLLECTIVE: agree on the per-rank slot count after the local Gaussian count changed (densify / prune).  A caller that
        already knows every rank's count (rebalance) passes their maximum as `chunk`, and then no collective is taken."""
        self.chunk = int(chunk) if chunk is not None else chunk_size(P_local, self.group)
        return self.chunk

    def workspace(self, device, S: int = 0, layers: int = 0) -> "PeerWorkspace":
        """COLLECTIVE on first use, after repartition() and when the number of feature channels the fused step carries changes:
        allocate + rendezvous the peer-mapped buffer (keyed on (chunk, S)).  A forward with render layers needs their sections: a
        workspace with fewer is replaced, one with more is kept."""
        if self._ws is None or self._ws.chunk != self.chunk or self._ws.S != S or self._ws.layers < layers:
            layers = max(layers, self._ws.layers if self._ws is not None and self._ws.chunk == self.chunk and self._ws.S == S else 0)
            if self.world > 1:
                self._ws = PeerWorkspace(self.raster_settings, self.chunk, self.world, self.rank, device, self.group, S=S, layers=layers)
            else:
                self._ws = PeerWorkspace.emulate(self.raster_settings, self.chunk, 1, device, S, layers)[0]
        return self._ws

    def pose_workspace(self) -> "PeerWorkspace":
        """The peer workspace composer.compose(rasterizer=self) sums its accumulator rows through (exchange="p2p"): the one this
        module's forward set up, so the composer's reduction takes no collective of its own."""
        if self._ws is None:
            raise _capi.SgrError("compose(rasterizer=...) with exchange='p2p' sums over the rasterizer's peer workspace: run the "
                                 "rasterizer's forward before the composer's backward")
        return self._ws

    def loss_workspace(self) -> "PeerWorkspace":
        """The peer workspace the band losses (band_losses.frame_losses / lidar_depth_loss with rasterizer=self) exchange their halo and
        partial sums through (exchange="p2p"): the one this module's forward set up, in its loss section."""
        if self._ws is None:
            raise _capi.SgrError("the band losses with rasterizer= and exchange='p2p' exchange over the rasterizer's peer workspace: run "
                                 "the rasterizer's forward before the losses")
        return self._ws

    def sky_workspace(self, R: int, device=None) -> "SkyWorkspace":
        """The sky section sky.sky_composite(rasterizer=self) exchanges the cube map's gradient through (exchange="p2p"): COLLECTIVE on
        first use and when R changes (allocate + rendezvous, keyed on (R, world)), so the sky composite's forward, which every rank
        runs, asks for it.  It is kept across repartition(); the exchange's barriers come from the current loss_workspace()."""
        sky = self._sky
        if sky is None or sky.R != int(R):
            if device is None:
                raise _capi.SgrError("the sky section is allocated in the sky composite's forward: pass its device")
            if self.world > 1:
                sky = SkyWorkspace(R, self.world, self.rank, device, self.group)
            else:
                sky = SkyWorkspace.emulate(R, 1, device)[0]
            self._sky = sky
        return sky

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

    def forward_layers(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None,
                       semantics=None, *, layers):
        """forward() plus render layers, as GaussianRasterizer.forward_layers returns them: ``layers`` is a sequence of RenderLayer whose
        ranges are in THIS rank's rows, and each layer's (color, depth, alpha) holds this rank's band of the layer rendered from the rows
        of every rank (zeros elsewhere; the ranks' images sum to the single-GPU layer of the rank-major concatenation of their rows).
        Every rank passes the same number of layers with the same bg, and every rank's loss must give the same layers a gradient (or
        none): an owner gathers the other ranks' layer rows only for the layers whose outputs got a gradient on its own rank.  Only the fused peer-memory step renders layers:
        exchange="p2p", fused=True, an InstanceCapacity that has learnt its capacity (a plain forward first), no feature channels and
        at most two layers."""
        mode = ("render layers under Gaussian sharding need the fused peer-memory step (elsewhere they are single-GPU: GaussianRasterizer): "
                "exchange='p2p', fused=True, an InstanceCapacity")
        exchange, fused, capacity = getattr(self, "exchange", None), getattr(self, "fused", False), getattr(self, "capacity", None)
        if exchange != "p2p" or not fused:
            raise _capi.SgrError(f"{mode} (this rasterizer has exchange={exchange!r}, fused={fused})")
        if capacity is None or capacity.capacity is None:
            raise _capi.SgrError(f"{mode} whose capacity is known: run a plain forward first")
        if semantics is not None:
            raise _capi.SgrError(f"{mode}, and no feature channels in the call")
        if len(layers) > _capi.MAX_SHARDED_LAYERS:
            raise _capi.SgrError(f"{mode}, and at most {_capi.MAX_SHARDED_LAYERS} layers (got {len(layers)})")
        layers = tuple(_check_layers(layers, int(means3D.shape[0])))
        shs, colors_precomp, scales, rotations, cov3D_precomp, _ = _reference_inputs(means3D, shs, colors_precomp, scales, rotations,
                                                                                     cov3D_precomp, None)
        if not means3D.is_cuda:
            raise _capi.SgrError("street_gaussians_b200 rasterizer needs CUDA tensors (there is no CPU fallback)")
        args = (means3D, means2D, shs, colors_precomp, None, opacities, scales, rotations, cov3D_precomp)
        differentiable = torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in args)
        out = _GaussianShardedLayers.apply(*args, self.raster_settings, self, differentiable, layers, *(l[3] for l in layers))
        return tuple(out[:5]) + (tuple(tuple(out[5 + 3 * k: 8 + 3 * k]) for k in range(len(layers))),)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None,
                semantics=None):
        shs, colors_precomp, scales, rotations, cov3D_precomp, semantics = _reference_inputs(means3D, shs, colors_precomp, scales, rotations,
                                                                                             cov3D_precomp, semantics)
        args = (means3D, means2D, shs, colors_precomp, semantics, opacities, scales, rotations, cov3D_precomp)
        differentiable = torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in args)
        return _GaussianShardedRasterize.apply(*args, self.raster_settings, self, differentiable)


# ---------------------------------------------------------------------------------------------------------------------
# Rebalancing Gaussian ownership after densification (DESIGN.md §8)
# ---------------------------------------------------------------------------------------------------------------------
class RebalanceMove(NamedTuple):
    """Rows [src_row_begin, src_row_end) of sub-model `model` on rank `src` become rows [dst_row_begin, ...) of that sub-model on
    rank `dst`.  In RebalancePlan.kept, src == dst: the rows a rank keeps, and where they land in its new tensors."""
    src: int
    dst: int
    model: int
    src_row_begin: int
    src_row_end: int
    dst_row_begin: int


class RebalancePlan(NamedTuple):
    moves: List[RebalanceMove]  # by model, then source rank, then destination rank
    kept: List[RebalanceMove]
    counts: List[List[int]]     # the new counts[world][n_models]


def rebalance_plan(counts: Sequence[Sequence[int]]) -> RebalancePlan:
    """Host-only plan of rebalance(): counts[r][m] rows of sub-model m on rank r (composition order), split as GaussianShardedRasterizer
    requires: the rank-major concatenation of the ranks' rows is the model-major global array.  Rank r ends up owning the global rows
    [B_r, B_{r+1}), B the even split (the first P_total % world ranks get one row more), and every row keeps its global position; a
    row moves only when its new owner is another rank, possibly past its neighbours."""
    counts = [[int(c) for c in row] for row in counts]
    world = len(counts)
    if world == 0:
        raise ValueError("counts: no ranks")
    nm = len(counts[0])
    if any(len(row) != nm for row in counts) or any(c < 0 for row in counts for c in row):
        raise ValueError(f"counts must be [world][n_models] non-negative integers, got {counts}")
    last = -1  # highest model a lower rank holds rows of: no later rank may hold rows of a model before it
    for r, row in enumerate(counts):
        held = [m for m, c in enumerate(row) if c]
        if held and held[0] < last:
            raise ValueError(f"rank {r} holds rows of model {held[0]} but a lower rank holds rows of model {last}: the ranks' rows are not "
                             "the rank-major split of the model-major global array")
        last = held[-1] if held else last
    base, extra = divmod(sum(map(sum, counts)), world)
    B = [r * base + min(r, extra) for r in range(world + 1)]
    new = [[0] * nm for _ in range(world)]
    moves, kept = [], []
    g0 = 0
    for m in range(nm):
        g1 = g0 + sum(row[m] for row in counts)
        nb = [max(B[d], g0) for d in range(world)]  # model m's new global range on rank d
        ne = [min(B[d + 1], g1) for d in range(world)]
        for d in range(world):
            new[d][m] = max(0, ne[d] - nb[d])
        a = g0
        for s in range(world):
            b = a + counts[s][m]
            for d in range(world):
                lo, hi = max(a, nb[d]), min(b, ne[d])
                if lo < hi:
                    (kept if d == s else moves).append(RebalanceMove(s, d, m, lo - a, hi - a, lo - nb[d]))
            a = b
        g0 = g1
    return RebalancePlan(moves, kept, new)


class ProcessGroupTransport:
    """rebalance()'s two exchanges over torch.distributed (NCCL or gloo): an all_gather of a small int64 table and the packed row
    buffers.  Tests substitute an object with the same four members that exchanges between emulated ranks."""

    def __init__(self, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0

    def all_gather(self, t: torch.Tensor) -> List[torch.Tensor]:
        """Every rank's `t` (a CPU tensor), as CPU tensors in rank order."""
        if self.world == 1:
            return [t]
        dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
        out = [torch.empty_like(t, device=dev) for _ in range(self.world)]
        dist.all_gather(out, t.to(dev), group=self.group)
        return list(torch.stack(out).cpu())

    def exchange(self, sends: dict, recvs: dict) -> None:
        """sends[dst] goes to rank dst and recvs[src] is filled from rank src, one batch_isend_irecv for all pairs."""
        peer = (lambda r: r) if self.group is None else (lambda r: dist.get_global_rank(self.group, r))
        ops = [dist.P2POp(dist.isend, b, peer(d), self.group) for d, b in sends.items()]
        ops += [dist.P2POp(dist.irecv, b, peer(s), self.group) for s, b in recvs.items()]
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()


def _rebalance_tables(L, ranges, buffers, dev):
    rt = (_capi.SgrRebalanceRange * max(1, len(ranges)))()
    for i, (seg, buf, src_row, dst_row, rows) in enumerate(ranges):
        rt[i].segment, rt[i].buffer, rt[i].src_row, rt[i].dst_row, rt[i].rows = seg, buf, src_row, dst_row, rows
    nb = len(buffers)
    bp = (C.c_void_p * max(1, nb))(*[b.data_ptr() for b in buffers])
    bf = (C.c_int64 * max(1, nb))(*[b.numel() for b in buffers])
    scratch = torch.empty((int(L.sgr_rebalance_scratch_bytes(len(ranges))),), dtype=torch.uint8, device=dev)
    return (rt, len(ranges), bp, bf, nb, ptr(scratch), scratch.numel()), scratch


def _row_table(models, optimizer, slots, dev, tr, what: str):
    """COLLECTIVE (one all_gather): this rank's sgr_rebalance_* segments of `models` (moment bits where Adam state exists) and the
    [world][n_models][11] table of every rank's counts, row widths and Adam steps (-1: no state), checked alike on every rank: the
    widths and steps must agree (ValueError otherwise, on every rank).  Returns (segments, [(params, moments)] per model, table)."""
    nm = len(models)
    segs = (_capi.SgrDensifySegment * nm)()
    infos = []
    meta = torch.full((nm, 4 + _capi.DENSIFY_TENSORS), -1, dtype=torch.int64)
    for k, m in enumerate(models):
        seg, params, moments, widths = _segment(m, k, optimizer, slots, dev)
        _stat_segment(seg, m, k, dev)
        meta[k, :4] = torch.tensor([seg.count, seg.dc_width, seg.rest_width, seg.semantic_width])
        for a, p in enumerate(params):
            if moments[a] is not None:
                opt = slots[id(p)][0]
                meta[k, 4 + a] = int(opt.state[p]["step"])
                if widths[a]:
                    seg.moments |= 1 << a
        segs[k] = seg
        infos.append((params, moments))
    table = torch.stack(tr.all_gather(meta)).tolist()  # [world][nm][11]
    for k in range(nm):
        for r in range(len(table)):
            if table[r][k][1:4] != table[0][k][1:4]:
                raise ValueError(f"model {k}: rows of {table[0][k][1:4]} (dc, rest, semantic floats) on rank 0, {table[r][k][1:4]} on rank {r}")
            for a in range(_capi.DENSIFY_TENSORS):
                if table[r][k][4 + a] != table[0][k][4 + a]:
                    st = lambda v: "no Adam state" if v < 0 else f"Adam step {v}"
                    raise ValueError(f"model {k}: {PARAM_NAMES[a]} has {st(table[0][k][4 + a])} on rank 0 and {st(table[r][k][4 + a])} on rank {r}; "
                                     f"{what} needs the same optimizer state on every rank")
    return segs, infos, table


def rebalance(models: Sequence, optimizer=None, group: Optional[dist.ProcessGroup] = None, rasterizer: Optional["GaussianShardedRasterizer"] = None,
              transport=None) -> int:
    """COLLECTIVE: even out the ranks' Gaussian counts after densify_and_prune, moving rows between ranks together with their Adam
    moments and densification statistics.  Returns the new local Gaussian count.

    models: this rank's sub-models in composition order (background, then actors; the attributes densify_and_prune reads: the seven
      parameters and max_radii2D, xyz_gradient_accum, denom), the same list on every rank; a sub-model may have 0 local rows.  The
      ranks' rows must form the split GaussianShardedRasterizer documents (rebalance_plan).  Afterwards rank r owns the global rows
      [B_r, B_{r+1}) of the even split and every row keeps its global position, so the Gaussian-sharded render is the same.
    optimizer: one optimizer or a list (as for densify_and_prune).  Parameters are replaced by new nn.Parameters in their groups, found
      by identity, and their state moves to the new key with the moments of the rows they now hold; step is unchanged and must be equal
      on every rank (ValueError otherwise, on every rank).
    rasterizer: its repartition() is called with the new counts' maximum (no further collective).
    transport: see ProcessGroupTransport; default ProcessGroupTransport(group).

    Communication: one all_gather of a [n_models, 11] int64 table (counts, row widths, Adam steps), the only host read, and, when some
    row moves, one batch_isend_irecv of one packed buffer per (source, destination) pair.  The rows are packed by one
    sgr_rebalance_pack launch and the new tensors written by one sgr_rebalance_splice launch; when no row moves (world 1, or ranks
    already balanced) nothing is launched."""
    tr = transport if transport is not None else ProcessGroupTransport(group)
    world, rank = int(tr.world), int(tr.rank)
    models = list(models)
    nm = len(models)
    if nm == 0:
        raise ValueError("rebalance needs the sub-models (background, then actors)")
    L = _capi.lib()
    dev = _attr(models[0], "_xyz").device
    slots = _param_slots(optimizer)
    segs, infos, table = _row_table(models, optimizer, slots, dev, tr, "rebalance")
    plan = rebalance_plan([[row[0] for row in table[r]] for r in range(world)])
    P_new = sum(plan.counts[rank])
    if rasterizer is not None:
        rasterizer.repartition(P_new, chunk=max(sum(c) for c in plan.counts))
    if not plan.moves:
        return P_new
    rf = [int(L.sgr_rebalance_row_floats(C.byref(segs[k]))) for k in range(nm)]
    # pack: one buffer per destination, its blocks in plan order (the receiver lists them in the same order)
    sends = [mv for mv in plan.moves if mv.src == rank]
    recvs = [mv for mv in plan.moves if mv.dst == rank]
    dsts = sorted({mv.dst for mv in sends})
    srcs = sorted({mv.src for mv in recvs})
    floats = lambda mvs, peer, side: sum((mv.src_row_end - mv.src_row_begin) * rf[mv.model] for mv in mvs if getattr(mv, side) == peer)
    send_bufs = [torch.empty((floats(sends, d, "dst"),), dtype=torch.float32, device=dev) for d in dsts]
    recv_bufs = [torch.empty((floats(recvs, s, "src"),), dtype=torch.float32, device=dev) for s in srcs]
    if sends:
        args, scratch = _rebalance_tables(L, [(mv.model, dsts.index(mv.dst), mv.src_row_begin, 0, mv.src_row_end - mv.src_row_begin)
                                              for mv in sends], send_bufs, dev)
        _capi.call("sgr_rebalance_pack", dev, segs, nm, *args)
    tr.exchange(dict(zip(dsts, send_bufs)), dict(zip(srcs, recv_bufs)))
    # splice: per model [received from lower ranks | kept | received from higher ranks]
    ranges = [(mv.model, srcs.index(mv.src), 0, mv.dst_row_begin, mv.src_row_end - mv.src_row_begin) for mv in recvs]
    ranges += [(mv.model, -1, mv.src_row_begin, mv.dst_row_begin, mv.src_row_end - mv.src_row_begin) for mv in plan.kept if mv.src == rank]
    ranges.sort(key=lambda t: (t[0], t[3]))
    outs = (_capi.SgrDensifyOutput * nm)()
    new = []
    for k, (params, moments) in enumerate(infos):
        n_new = plan.counts[rank][k]
        o = outs[k]
        o.count = n_new
        nps, nmom = [], []
        for a, p in enumerate(params):
            t = torch.empty((n_new,) + tuple(p.shape[1:]), dtype=torch.float32, device=dev)
            mv = None if moments[a] is None else (torch.empty_like(t), torch.empty_like(t))
            if n_new and t.numel():
                o.param[a] = t.data_ptr()
                if mv is not None:
                    o.exp_avg[a], o.exp_avg_sq[a] = mv[0].data_ptr(), mv[1].data_ptr()
            nps.append(t)
            nmom.append(mv)
        stats = (torch.empty(n_new, device=dev), torch.empty(n_new, 2, device=dev), torch.empty(n_new, 1, device=dev))
        if n_new:
            o.max_radii2D, o.xyz_gradient_accum, o.denom = (t.data_ptr() for t in stats)
        new.append((nps, nmom, stats))
    if ranges:
        args, scratch = _rebalance_tables(L, ranges, recv_bufs, dev)
        _capi.call("sgr_rebalance_splice", dev, segs, outs, nm, *args)
    for k, m in enumerate(models):
        _install(m, infos[k][0], *new[k], slots)
    return P_new


# ---------------------------------------------------------------------------------------------------------------------
# Checkpoints under Gaussian sharding (DESIGN.md §8): the files io.save_checkpoint / io.save_ply write on one GPU, and resuming from them
# at any world size
# ---------------------------------------------------------------------------------------------------------------------
def even_slices(totals: Sequence[int], world: int) -> List[List[tuple]]:
    """Rank r's rows [lo, hi) of every sub-model (totals[m] rows each, composition order) under the even split of the model-major global
    array that rebalance() leaves: rank r owns the global rows [B_r, B_{r+1}), the first P % world ranks one row more."""
    totals = [int(n) for n in totals]
    if world < 1 or any(n < 0 for n in totals):
        raise ValueError(f"even_slices needs world >= 1 and non-negative counts, got world={world}, {totals}")
    base, extra = divmod(sum(totals), world)
    B = [r * base + min(r, extra) for r in range(world + 1)]
    out = []
    for r in range(world):
        row, g0 = [], 0
        for n in totals:
            lo = min(max(B[r], g0), g0 + n)
            row.append((lo - g0, max(lo, min(B[r + 1], g0 + n)) - g0))
            g0 += n
        out.append(row)
    return out


def gather_pieces(counts: Sequence[Sequence[int]], row_bytes: Sequence[int], piece_bytes: int) -> List[tuple]:
    """The pieces gather_state sends: (source rank, [(model, first local row, rows), ...]) in rank-major, then model, then row order, every
    local row of every rank exactly once, each piece at most piece_bytes (row_bytes[m] bytes per row of model m; a model no rank holds rows
    of may have any width)."""
    need = max((int(row_bytes[k]) for row in counts for k, n in enumerate(row) if n), default=0)
    if piece_bytes < max(need, 1):
        raise ValueError(f"piece_bytes={piece_bytes} is smaller than one row ({need} bytes)")
    pieces = []
    for s, row in enumerate(counts):
        cur, used = [], 0
        for k, n in enumerate(row):
            at = 0
            while at < n:
                take = min((piece_bytes - used) // int(row_bytes[k]), n - at)
                if take == 0:
                    pieces.append((s, cur))
                    cur, used = [], 0
                    continue
                cur.append((k, at, take))
                used += take * int(row_bytes[k])
                at += take
        if cur:
            pieces.append((s, cur))
    return pieces


def _unpack_rows(flat: torch.Tensor, ranges, seg_info, host, at_rank):
    """Scatter a received piece (host fp32, the sgr_rebalance_pack block format) into the host arrays of every model at its global rows."""
    off = 0
    for k, first, rows in ranges:
        widths, moment_bits = seg_info[k]
        dst = host[k]
        g = at_rank[k] + first
        order = [dst[PARAM_NAMES[a]] for a in range(len(PARAM_NAMES)) if widths[a]]
        order += [dst["adam"][PARAM_NAMES[a]]["exp_avg"] for a in moment_bits]
        order += [dst["adam"][PARAM_NAMES[a]]["exp_avg_sq"] for a in moment_bits]
        order += [dst[s] for s in STAT_NAMES]
        for t in order:
            w = int(math.prod(t.shape[1:]))
            t.view(t.shape[0], w)[g:g + rows] = flat[off:off + rows * w].view(rows, w)
            off += rows * w


def gather_state(models: Sequence, optimizer=None, *, dst: int = 0, group=None, transport=None, piece_bytes: int = 1 << 30):
    """COLLECTIVE: every rank's rows of every sub-model, with their Adam moments and densification statistics, assembled on rank `dst` as
    the global tensors a single-GPU run of the same rows holds (rank-major order, as GaussianShardedRasterizer composes them).

    models: this rank's sub-models in composition order (the seven parameters and max_radii2D, xyz_gradient_accum, denom), the same list
      on every rank; a sub-model may have 0 local rows.  optimizer: one optimizer or a list; a parameter's moments are gathered where it has
      Adam state, and its step must be equal on every rank.  As in rebalance(), one all_gather of the per-model table comes first and a
      width or step mismatch raises ValueError on every rank before any row moves.
    Then the rows travel in pieces (gather_pieces) of at most piece_bytes: the owner packs one piece with sgr_rebalance_pack into a buffer
      it reuses, sends it to dst (transport.exchange), and dst copies it to the host and scatters it into the global host tensors.  Extra
      device memory is one piece buffer per rank (dst's own rows take the same path without the send); no live tensor is replaced.
    Returns on dst one dict per model: the seven parameters and three statistics by attribute name (CPU fp32), and "adam": {parameter name:
      {"step": int, "exp_avg", "exp_avg_sq"}} for the parameters with Adam state.  Other ranks return None."""
    tr = transport if transport is not None else ProcessGroupTransport(group)
    world, rank = int(tr.world), int(tr.rank)
    models = list(models)
    nm = len(models)
    if nm == 0:
        raise ValueError("gather_state needs the sub-models (background, then actors)")
    if not 0 <= int(dst) < world:
        raise ValueError(f"dst={dst} is not a rank of a group of {world}")
    if int(piece_bytes) <= 0:
        raise ValueError(f"piece_bytes must be positive, got {piece_bytes}")
    L = _capi.lib()
    dev = _attr(models[0], "_xyz").device
    slots = _param_slots(optimizer)
    segs, infos, table = _row_table(models, optimizer, slots, dev, tr, "gather_state")
    counts = [[row[0] for row in table[r]] for r in range(world)]
    rf = [int(L.sgr_rebalance_row_floats(C.byref(segs[k]))) for k in range(nm)]
    pieces = gather_pieces(counts, [4 * f for f in rf], int(piece_bytes))
    floats = lambda ranges: sum(rows * rf[k] for k, _, rows in ranges)
    cap = max((floats(r) for s, r in pieces if s == rank or rank == dst), default=0)
    buf = torch.empty((cap,), dtype=torch.float32, device=dev) if cap else None
    host = at_rank = seg_info = None
    if rank == dst:
        host, seg_info = [], []
        for k, (params, moments) in enumerate(infos):
            n = sum(counts[r][k] for r in range(world))
            h = {a: torch.empty((n,) + tuple(p.shape[1:]), dtype=torch.float32) for a, p in zip(PARAM_NAMES, params)}
            h.update(max_radii2D=torch.empty(n), xyz_gradient_accum=torch.empty(n, 2), denom=torch.empty(n, 1))
            h["adam"] = {PARAM_NAMES[a]: dict(step=table[0][k][4 + a], exp_avg=torch.empty_like(h[PARAM_NAMES[a]]),
                                              exp_avg_sq=torch.empty_like(h[PARAM_NAMES[a]]))
                         for a in range(len(PARAM_NAMES)) if table[0][k][4 + a] >= 0}
            host.append(h)
            w = [int(math.prod(p.shape[1:])) for p in params]
            seg_info.append((w, [a for a in range(len(PARAM_NAMES)) if (segs[k].moments >> a) & 1]))
        at_rank = [[sum(counts[q][k] for q in range(r)) for k in range(nm)] for r in range(world)]
    for s, ranges in pieces:
        n = floats(ranges)
        if rank == s:
            args, scratch = _rebalance_tables(L, [(k, 0, first, 0, rows) for k, first, rows in ranges], [buf[:n]], dev)
            _capi.call("sgr_rebalance_pack", dev, segs, nm, *args)
        if s != dst:
            tr.exchange({dst: buf[:n]} if rank == s else {}, {s: buf[:n]} if rank == dst else {})
        if rank == dst:
            _unpack_rows(buf[:n].cpu(), ranges, seg_info, host, at_rank[s])
    return host


# Host storage address -> the location torch.save records for it.  save_checkpoint assembles the global tensors on the host (so the device
# memory of dst stays bounded) but writes them as the single-GPU file holds them, on dst's CUDA device, so that a bare torch.load (the
# reference's train.py:42, scene.py:42) puts them there.  The tagger answers only while save_checkpoint is writing (_SAVE_AS non-empty).
_SAVE_AS = {}
_tagger = []


def _tag_host_storage(storage):
    if _SAVE_AS and storage.device.type == "cpu":
        return _SAVE_AS.get(storage.data_ptr())
    return None


@contextlib.contextmanager
def _saved_on(tensors, device):
    """torch.save inside the block records the host storages of `tensors` at `device` (torch.serialization.register_package)."""
    if not _tagger:
        torch.serialization.register_package(1, _tag_host_storage, lambda storage, location: None)
        _tagger.append(_tag_host_storage)
    for t in tensors:
        if t.device.type == "cpu" and t.numel():
            _SAVE_AS[t.untyped_storage().data_ptr()] = f"cuda:{device.index if device.index is not None else torch.cuda.current_device()}"
    try:
        yield
    finally:
        _SAVE_AS.clear()


def _checkpoint_entries(model, st, optimizer, is_final: bool, extra, dev, on_device: list):
    """One sub-model's entries of io.save_checkpoint from its gathered state: the parameters as nn.Parameters (the model's requires_grad),
    and unless is_final the training extras in GaussianModel.state_dict's order (gaussian_model.py:180-205), then the caller's `extra`.
    The gathered host tensors are appended to `on_device` (written at dev's location); an empty one is made on dev itself."""
    from .training import adam_state_dict

    def dev_tensor(t):
        if t.numel() == 0:
            return torch.empty(t.shape, dtype=t.dtype, device=dev)
        on_device.append(t)
        return t

    params = {a: nn.Parameter(dev_tensor(st[a]), requires_grad=_attr(model, a).requires_grad) for a in PARAM_NAMES}
    e = {}
    if not is_final:
        if _has(model, "spatial_lr_scale"):
            e["spatial_lr_scale"] = _attr(model, "spatial_lr_scale")
        e["denom"], e["max_radii2D"], e["xyz_gradient_accum"] = (dev_tensor(st[s]) for s in ("denom", "max_radii2D", "xyz_gradient_accum"))
        if _has(model, "active_sh_degree"):
            e["active_sh_degree"] = _attr(model, "active_sh_degree")
        if optimizer is not None:
            adam = {a: dict(step=v["step"], exp_avg=dev_tensor(v["exp_avg"]), exp_avg_sq=dev_tensor(v["exp_avg_sq"])) for a, v in st["adam"].items()}
            e["optimizer"] = adam_state_dict(model, optimizer, state=adam)
    e.update(extra or {})
    return params, e


def save_checkpoint(path: str, named_models, iteration: int, optimizer=None, *, is_final: bool = False, extras=None, dst: int = 0, group=None,
                    transport=None, piece_bytes: int = 1 << 30, **other) -> None:
    """COLLECTIVE: rank `dst` writes the .pth of train.py:218-223 that io.save_checkpoint writes on one GPU for the rank-major concatenation
    of the ranks' rows (gather_state).  named_models: {model_name: this rank's sub-model} in composition order, the same names on every
    rank.  Per model: the seven parameters and, unless is_final, spatial_lr_scale and active_sh_degree (where the model has them), denom,
    max_radii2D, xyz_gradient_accum and 'optimizer', the model's state in torch.optim.Adam.state_dict() format with the reference's group
    names (training.adam_state_dict, from the groups of this rank's `optimizer`).  extras: {model_name: {key: value}} added to a model's
    entries; **other (actor_pose, sky_cubemap, color_correction, pose_correction, ...: replicated state) is written by dst only.

    The file is the single-GPU one as the reference reads it with a bare torch.load: the parameters are nn.Parameters with the requires_grad
    of dst's model, and the parameters, moments and statistics are recorded at dst's CUDA device (the Adam steps on the CPU, as torch keeps
    them), although dst assembles them on the host and never holds the whole model on the device."""
    names = list(named_models)
    objs = [named_models[n] for n in names]
    state = gather_state(objs, None if is_final else optimizer, dst=dst, group=group, transport=transport, piece_bytes=piece_bytes)
    if state is None:
        return
    from . import io
    dev = _attr(objs[0], "_xyz").device
    models, ex, on_device = {}, {}, []
    for n, m, st in zip(names, objs, state):
        models[n], ex[n] = _checkpoint_entries(m, st, None if is_final else optimizer, is_final, (extras or {}).get(n), dev, on_device)
    with _saved_on(on_device, dev):
        io.save_checkpoint(path, models, iteration, ex, **other)


def save_ply(path: str, named_models, *, dst: int = 0, group=None, transport=None, piece_bytes: int = 1 << 30) -> None:
    """COLLECTIVE: rank `dst` writes the point_cloud.ply of Scene.save (street_gaussian_model.py:94-105), the bytes io.save_ply writes on one
    GPU for the rank-major concatenation of the ranks' rows.  named_models as for save_checkpoint; statistics are not needed."""
    names = list(named_models)
    objs = []
    for n in names:
        m = named_models[n]
        d = {a: _attr(m, a) for a in PARAM_NAMES}  # with zero statistics where the model has none: the row format carries them
        cnt, dev = int(d["_xyz"].shape[0]), d["_xyz"].device
        for s, shape in zip(STAT_NAMES, ((cnt,), (cnt, 2), (cnt, 1))):
            d[s] = _attr(m, s) if _has(m, s) else torch.zeros(shape, device=dev)
        objs.append(d)
    state = gather_state(objs, None, dst=dst, group=group, transport=transport, piece_bytes=piece_bytes)
    if state is None:
        return
    from . import io
    io.save_ply(path, {n: {a: st[a] for a in PARAM_NAMES} for n, st in zip(names, state)})


_CKPT_KEYS = ("xyz", "feature_dc", "feature_rest", "opacity", "scaling", "rotation", "semantic")  # gaussian_model.py:182-190, by PARAM_NAMES


def load_checkpoint(path: str, models, optimizer=None, *, group=None, transport=None, rasterizer: Optional["GaussianShardedRasterizer"] = None) -> int:
    """Resume from a .pth written by save_checkpoint, io.save_checkpoint or the reference's train.py, at any world size.  Returns the local
    Gaussian count.

    models: {model_name: this rank's sub-model} in composition order.  Rank r takes the global rows [B_r, B_{r+1}) of the even split of the
      model-major array (even_slices, the split rebalance() leaves; a sub-model may get 0 rows).  The file is opened with torch.load(mmap=True)
      and only this rank's slices are copied to the device of the model's _xyz, so no rank holds the whole model on the device.
    Parameters are replaced by new nn.Parameters (same requires_grad), in their groups of `optimizer` too (found by identity, as rebalance()
      does); where the file's 'optimizer' holds state for a parameter (matched by the reference's group names), its state becomes {step, the
      slices of exp_avg and exp_avg_sq}, otherwise any old state is dropped.  max_radii2D, xyz_gradient_accum and denom take their slices, or
      zeros when the file is final.  Group learning rates and every other entry of the file are left to the caller.
    rasterizer: its repartition() is called with the largest rank's count (no collective: every rank computes it from the file).
    transport / group: only for this rank's index and the world size (ProcessGroupTransport); nothing is exchanged."""
    tr = transport if transport is not None else ProcessGroupTransport(group)
    world, rank = int(tr.world), int(tr.rank)
    names = list(models)
    objs = [models[n] for n in names]
    if not objs:
        raise ValueError("load_checkpoint needs the sub-models (background, then actors)")
    sd = torch.load(path, map_location="cpu", mmap=True, weights_only=False)
    for n in names:
        if n not in sd or not isinstance(sd[n], dict) or "xyz" not in sd[n]:
            raise KeyError(f"{path} has no Gaussian model '{n}' (it holds {sorted(k for k, v in sd.items() if isinstance(v, dict) and 'xyz' in v)})")
    slices = even_slices([int(sd[n]["xyz"].shape[0]) for n in names], world)
    dev = _attr(objs[0], "_xyz").device
    slots = _param_slots(optimizer)
    for n, m, (lo, hi) in zip(names, objs, slices[rank]):
        e = sd[n]
        opt_state = {}
        if optimizer is not None and isinstance(e.get("optimizer"), dict):
            osd = e["optimizer"]
            for g in osd["param_groups"]:
                if g.get("name") in ADAM_GROUP_NAMES and len(g["params"]) == 1 and g["params"][0] in osd["state"]:
                    opt_state[PARAM_NAMES[ADAM_GROUP_NAMES.index(g["name"])]] = osd["state"][g["params"][0]]
        for a, key in zip(PARAM_NAMES, _CKPT_KEYS):
            old = _attr(m, a)
            t = e[key][lo:hi].to(device=dev, dtype=torch.float32).contiguous()
            p = nn.Parameter(t, requires_grad=old.requires_grad)
            if id(old) in slots:
                opt, grp, j = slots[id(old)]
                grp["params"][j] = p
                opt.state.pop(old, None)
                s = opt_state.get(a)
                if s is not None:
                    step = s["step"].clone() if isinstance(s["step"], torch.Tensor) else s["step"]
                    opt.state[p] = dict(step=step, **{mk: s[mk][lo:hi].to(device=dev, dtype=torch.float32).contiguous()
                                                      for mk in ("exp_avg", "exp_avg_sq")})
            _set(m, a, p)
        for s, shape in zip(STAT_NAMES, ((hi - lo,), (hi - lo, 2), (hi - lo, 1))):
            t = e[s][lo:hi].to(device=dev, dtype=torch.float32).reshape(shape).contiguous() if s in e else torch.zeros(shape, device=dev)
            _set(m, s, t)
    P_local = sum(hi - lo for lo, hi in slices[rank])
    if rasterizer is not None:
        rasterizer.repartition(P_local, chunk=max(sum(hi - lo for lo, hi in row) for row in slices))
    return P_local
