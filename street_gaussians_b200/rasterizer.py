"""Host side of the drop-in: the reference's Python surface over the C-ABI CUDA library.

Mirrors /root/reference/submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py (DGR below):
  * ``GaussianRasterizationSettings`` — same 12 fields in the same order (DGR :167-179);
  * ``GaussianRasterizer`` — ``forward`` / ``markVisible`` / ``visible_filter`` with the same signatures, defaults,
    argument checks (same two ``Exception`` messages, DGR :201-205) and the same 5-tuple result
    ``(color, radii, depth, alpha, semantic)`` (DGR :197-233, 186-195, 235-260);
  * ``rasterize_gaussians`` — the 10-positional-argument functional entry (DGR :21-44);
  * gradients for the same 8 inputs in the same order (DGR :152-163), including the 3-column ``means2D`` convention
    (x, y = NDC-scaled screen gradient, z = sum |gx|+|gy|).

PyTorch is plumbing here: it owns device memory (caching allocator), the current stream and autograd bookkeeping.
All arithmetic happens in libsgr.so (hand-written CUDA, sm_90a) through include/sgr.h.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional, Tuple

import torch
import torch.nn as nn

from . import _capi


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


class TileRowBand(NamedTuple):
    """Tile rows (16 px each) owned by this process: r in [begin, end) with (r - begin) % step == 0."""
    begin: int
    end: int
    step: int = 1


def _ptr(t: Optional[torch.Tensor]):
    if t is None or t.numel() == 0:
        return None
    return C.c_void_p(t.data_ptr())


def _dev_f32(t: torch.Tensor, device) -> torch.Tensor:
    """contiguous fp32 on `device` (the reference calls .contiguous() on every argument, DGR/rasterize_points.cu:92-118)."""
    if t.device != device or t.dtype != torch.float32:
        t = t.to(device=device, dtype=torch.float32)
    return t.contiguous()


def _none_if_empty(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    return None if t is None or t.numel() == 0 else t


def _make_frame(s: GaussianRasterizationSettings, P: int, M: int, S: int, device, band: Optional[TileRowBand]):
    keep = [_dev_f32(s.bg, device), _dev_f32(s.viewmatrix, device), _dev_f32(s.projmatrix, device), _dev_f32(s.campos, device)]
    fr = _capi.SgrFrame()
    fr.P, fr.D, fr.M, fr.S = int(P), int(s.sh_degree), int(M), int(S)
    fr.width, fr.height = int(s.image_width), int(s.image_height)
    fr.tan_fovx, fr.tan_fovy, fr.scale_modifier = float(s.tanfovx), float(s.tanfovy), float(s.scale_modifier)
    fr.prefiltered, fr.debug = int(bool(s.prefiltered)), int(bool(s.debug))
    if band is None:
        fr.row_begin = fr.row_end = fr.row_step = 0
    else:
        fr.row_begin, fr.row_end, fr.row_step = int(band.begin), int(band.end), int(band.step)
    fr.bg, fr.viewmatrix, fr.projmatrix, fr.campos = (k.data_ptr() for k in keep)
    return fr, keep


def _stream(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _dump(path: str, args) -> None:
    """CPU deep copy of the call's arguments, written with torch.save — the reference's debug post-mortem."""
    try:
        torch.save(tuple(a.detach().cpu().clone() if isinstance(a, torch.Tensor) else a for a in args), path)
    except Exception:
        pass


class _ForwardState:
    """Caller-owned forward->backward state (the reference keeps geomBuffer/binningBuffer/imgBuffer byte tensors)."""
    __slots__ = ("geom", "img", "binning", "num_instances")


def _reference_inputs(means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, semantics):
    """The reference's two argument checks (same messages, DGR :201-205) and its placeholders: an absent input becomes an empty
    tensor, absent semantics zeros(P, 0).  Returns (shs, colors_precomp, scales, rotations, cov3D_precomp, semantics)."""
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
            ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
    if semantics is None:
        semantics = torch.zeros(means3D.shape[0], 0, dtype=torch.float32, device=means3D.device)
    return (torch.Tensor([]) if shs is None else shs, torch.Tensor([]) if colors_precomp is None else colors_precomp,
            torch.Tensor([]) if scales is None else scales, torch.Tensor([]) if rotations is None else rotations,
            torch.Tensor([]) if cov3D_precomp is None else cov3D_precomp, semantics)


def _fp32_inputs(means3D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp):
    """The kernels' inputs as contiguous fp32 on means3D's device; an absent or empty optional input, and semantics without
    channels, is None."""
    if means3D.dim() != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # DGR/rasterize_points.cu:58-60
    if not means3D.is_cuda:
        raise _capi.SgrError("street_gaussians_b200 rasterizer needs CUDA tensors (there is no CPU fallback)")
    device = means3D.device
    S = int(semantics.shape[1]) if (semantics is not None and semantics.dim() == 2) else 0
    tensors = dict(means3D=_dev_f32(means3D, device), opacities=_dev_f32(opacities, device))
    for name, t in (("sh", _none_if_empty(sh)), ("colors_precomp", _none_if_empty(colors_precomp)), ("scales", _none_if_empty(scales)),
                    ("rotations", _none_if_empty(rotations)), ("cov3Ds_precomp", _none_if_empty(cov3Ds_precomp)),
                    ("semantics", semantics if S > 0 else None)):
        tensors[name] = _dev_f32(t, device) if t is not None else None
    return tensors


def _input_shapes(*inputs):
    """(shape, device, dtype) of each autograd input (None for None): what _fit_grads casts the gradients back to."""
    return tuple(None if t is None else (tuple(t.shape), t.device, t.dtype) for t in inputs)


def _fit_grads(shapes, grads):
    """Each gradient reshaped and cast to its input's shape, dtype and device; None for a None input, zeros for an input without a
    gradient (an empty placeholder)."""
    out = []
    for s, g in zip(shapes, grads):
        if s is None:
            out.append(None)
            continue
        shape, device, dtype = s
        out.append(torch.zeros(shape, device=device, dtype=dtype) if g is None else g.reshape(shape).to(device=device, dtype=dtype))
    return tuple(out)


def _image_grads(settings, device, grads, channels):
    """The upstream gradients of image outputs; an output autograd passed no gradient for contributes a zero [c, H, W] image."""
    H, W = int(settings.image_height), int(settings.image_width)
    return tuple(g if g is not None else torch.zeros((c, H, W), device=device, dtype=torch.float32) for g, c in zip(grads, channels))


def _geom_grad_buffers(tensors, P: int, device):
    """The 8 outputs of the per-Gaussian chain rule in sgr_backward_geom's order (torch.empty: the kernel writes every element)."""
    sh, colors, cov = tensors["sh"], tensors["colors_precomp"], tensors["cov3Ds_precomp"]
    M = int(sh.shape[1]) if sh is not None else 0
    e = lambda *shape: torch.empty(shape, device=device, dtype=torch.float32)
    return (e(P, 3), e(P, 3), e(P, M, 3) if sh is not None else None, e(P, 3) if colors is not None else None, e(P, 1),
            e(P, 3) if cov is None else None, e(P, 4) if cov is None else None, e(P, 6) if cov is not None else None)


def _copy_status(fr, geom, host_status: torch.Tensor, device):
    """sgr_forward_status_async: the status words of the forward just enqueued into pinned `host_status`, on the current stream."""
    rc = _capi.lib().sgr_forward_status_async(C.byref(fr), _ptr(geom), C.c_void_p(host_status.data_ptr()), _stream(device))
    _capi.check(rc, "sgr_forward_status_async")


class InstanceCapacity:
    """Opt-in, sync-free binning (include/sgr.h: sgr_forward_bounded).  The reference — and this library by default —
    blocks the host once per forward to read the instance count R back and size the sort buffers.  With a capacity
    object the buffers are sized from the largest R seen so far (x `headroom`), nothing is read back inside forward, and
    the true count of each frame arrives asynchronously in pinned memory; `check()` (called at the start of the next
    forward and from `GaussianRasterizer.synchronize_capacity()`) raises if a frame did not fit, after growing the capacity.
    The first frame(s) run in exact mode to learn R."""

    def __init__(self, headroom: float = 1.25, initial: Optional[int] = None):
        self.headroom, self.capacity = float(headroom), (int(initial) if initial else None)
        self.gaussian_capacity = None  # depth-order slots of the compacted Gaussian-sharded forward (sgr_sharded_forward)
        self.frozen = False            # freeze(): capacities fixed, no per-frame status copy / event (CUDA-graph capture of a step)
        self._pending = []  # (pinned int32[4], cuda event) in submission order
        self._pool = []     # pinned status words ready for reuse: no pin_memory() (a cudaHostAlloc) inside the steady-state step

    def observe(self, R: int):
        want = int(R * self.headroom) + 4096
        if self.capacity is None or want > self.capacity:
            self.capacity = want

    def freeze(self, frozen: bool = True):
        """Stop tracking: forwards neither copy their status words back nor record events, so a whole step (forward + backward) is a
        fixed sequence of stream operations that torch.cuda.graph can capture and replay.  Overflows are then only visible through
        an explicit sgr_forward_status; unfreeze to resume tracking."""
        if frozen:
            self.check(wait=True)
        self.frozen = bool(frozen)
        return self

    def observe_gaussians(self, n: int):
        want = int(n * self.headroom) + 1024
        if self.gaussian_capacity is None or want > self.gaussian_capacity:
            self.gaussian_capacity = want

    def status_word(self) -> torch.Tensor:
        """A pinned int32[8] for sgr_forward_status_async; recycled once its frame has been checked."""
        return self._pool.pop() if self._pool else torch.zeros(8, dtype=torch.int32).pin_memory()

    def track(self, host_status: torch.Tensor, event):
        self._pending.append((host_status, event))

    def record_status(self, fr, geom, device):
        """Track the bounded forward just enqueued on `device`'s current stream: its status words go into a pinned word
        asynchronously, and check() reads them once the event recorded behind the copy has completed."""
        host_status = self.status_word()
        _copy_status(fr, geom, host_status, device)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        self.track(host_status, ev)

    def check(self, wait: bool = False):
        """Examine the frames whose status has arrived (all of them with wait=True).  Raises on the FIRST overflowed frame
        after growing the capacity; the frames after it stay pending, so a later call still reports them.  An overflowed
        frame was rendered incomplete: call check(wait=True) (GaussianRasterizer.synchronize_capacity()) before the
        optimiser step when that matters, and re-render."""
        pending, self._pending = self._pending, []
        for i, (host_status, ev) in enumerate(pending):
            if wait:
                ev.synchronize()
            if not ev.query():
                self._pending.append((host_status, ev))
                continue
            R, overflow, n_sel, timed_out = int(host_status[0]), int(host_status[1]), int(host_status[3]), int(host_status[4])
            self._pool.append(host_status)
            if timed_out:
                self._pending.extend(pending[i + 1:])
                raise _capi.SgrError(f"the device barrier of epoch {timed_out} timed out (a peer rank never arrived within 2 s): that frame "
                                     "was rendered from incomplete peer data")
            old, old_g = self.capacity, self.gaussian_capacity
            self.observe(R)
            if n_sel:
                self.observe_gaussians(n_sel)
            if overflow:
                self._pending.extend(pending[i + 1:])
                what = (f"instance capacity {old} overflowed (frame needed {R}); capacity raised to {self.capacity}" if overflow & 1 else
                        f"Gaussian capacity {old_g} overflowed (band holds {n_sel}); capacity raised to {self.gaussian_capacity}")
                raise _capi.SgrError(what + " — re-render that frame")


def _forward_impl(means3D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp,
                  settings: GaussianRasterizationSettings, band: Optional[TileRowBand], capacity: Optional["InstanceCapacity"] = None):
    L = _capi.lib()
    tensors = _fp32_inputs(means3D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp)
    device = means3D.device
    P = means3D.shape[0]
    H, W = int(settings.image_height), int(settings.image_width)
    S = int(tensors["semantics"].shape[1]) if tensors["semantics"] is not None else 0
    M = int(tensors["sh"].shape[1]) if tensors["sh"] is not None else 0

    f32 = dict(device=device, dtype=torch.float32)
    whole = band is None
    alloc_img = torch.empty if whole else torch.zeros  # a partial band leaves foreign rows untouched -> hand back zeros there
    st = _ForwardState()
    st.num_instances = 0
    st.binning = None
    if P == 0:  # the reference short-circuits and returns zero-filled images (DGR/rasterize_points.cu:86)
        st.geom = st.img = None
        z = lambda c: torch.zeros((c, H, W), **f32)
        return z(3), torch.zeros((0,), device=device, dtype=torch.int32), z(1), z(1), z(S), st, None

    color = alloc_img((3, H, W), **f32)
    depth = alloc_img((1, H, W), **f32)
    alpha = alloc_img((1, H, W), **f32)
    semantic = alloc_img((S, H, W), **f32)
    radii = torch.empty((P,), device=device, dtype=torch.int32)

    fr, keep = _make_frame(settings, P, M, S, device, band)
    gb, ib = C.c_size_t(0), C.c_size_t(0)
    _capi.check(L.sgr_state_sizes(C.byref(fr), C.byref(gb), C.byref(ib)), "sgr_state_sizes")
    st.geom = torch.empty((gb.value,), device=device, dtype=torch.uint8)
    st.img = torch.empty((ib.value,), device=device, dtype=torch.uint8)

    if capacity is not None and not capacity.frozen:
        capacity.check()
    if capacity is not None and capacity.capacity is not None:
        # bounded mode: no host synchronisation anywhere in this call
        cap = int(capacity.capacity)
        nbytes = int(L.sgr_binning_bytes(cap))
        st.binning = torch.empty((nbytes,), device=device, dtype=torch.uint8)
        with torch.cuda.device(device):
            rc = L.sgr_forward_bounded(C.byref(fr), _ptr(tensors["means3D"]), _ptr(tensors["sh"]), _ptr(tensors["colors_precomp"]),
                                       _ptr(tensors["semantics"]), _ptr(tensors["opacities"]), _ptr(tensors["scales"]),
                                       _ptr(tensors["rotations"]), _ptr(tensors["cov3Ds_precomp"]), _ptr(color), _ptr(depth), _ptr(alpha),
                                       _ptr(semantic), _ptr(radii), _ptr(st.geom), gb.value, _ptr(st.img), ib.value, _ptr(st.binning), nbytes,
                                       cap, _stream(device))
            _capi.check(rc, "sgr_forward_bounded")
            if not capacity.frozen:
                capacity.record_status(fr, st.geom, device)
        st.num_instances = cap
        del keep
        return color, radii, depth, alpha, semantic, st, tensors

    def _alloc(_user, nbytes):
        st.binning = torch.empty((int(nbytes),), device=device, dtype=torch.uint8)
        return st.binning.data_ptr()

    cb = _capi.ALLOC_FN(_alloc)
    bin_ptr, n_inst = C.c_void_p(), C.c_int64(0)
    with torch.cuda.device(device):
        rc = L.sgr_forward(C.byref(fr), _ptr(tensors["means3D"]), _ptr(tensors["sh"]), _ptr(tensors["colors_precomp"]),
                           _ptr(tensors["semantics"]), _ptr(tensors["opacities"]), _ptr(tensors["scales"]),
                           _ptr(tensors["rotations"]), _ptr(tensors["cov3Ds_precomp"]), _ptr(color), _ptr(depth), _ptr(alpha),
                           _ptr(semantic), _ptr(radii), _ptr(st.geom), gb.value, _ptr(st.img), ib.value, cb, None,
                           C.byref(bin_ptr), C.byref(n_inst), _stream(device))
    _capi.check(rc, "sgr_forward")
    st.num_instances = int(n_inst.value)
    if capacity is not None:
        capacity.observe(st.num_instances)
    del keep
    return color, radii, depth, alpha, semantic, st, tensors


def _backward_blend_impl(settings, band, st: _ForwardState, tensors, alpha, grad_color, grad_depth, grad_alpha, grad_semantic,
                         grad2d_out: Optional[torch.Tensor] = None):
    """Stage 1: returns (grad2d[P,12], dL_dsemantics[P,S]) — the per-rank partial sums under tile-row sharding.
    grad2d_out: write the sums there instead of a fresh tensor (peer-mapped workspace of the Gaussian-sharded mode)."""
    L = _capi.lib()
    means3D = tensors["means3D"]
    device, P = means3D.device, means3D.shape[0]
    S = int(tensors["semantics"].shape[1]) if tensors["semantics"] is not None else 0
    M = int(tensors["sh"].shape[1]) if tensors["sh"] is not None else 0
    fr, keep = _make_frame(settings, P, M, S, device, band)
    grad2d = grad2d_out if grad2d_out is not None else torch.empty((P, 12), device=device, dtype=torch.float32)
    g_sem = torch.empty((P, S), device=device, dtype=torch.float32)
    gc, gd, ga = _dev_f32(grad_color, device), _dev_f32(grad_depth, device), _dev_f32(grad_alpha, device)
    gs = _dev_f32(grad_semantic, device) if S > 0 else None
    with torch.cuda.device(device):
        rc = L.sgr_backward_blend(C.byref(fr), st.num_instances, _ptr(tensors["semantics"]), _ptr(st.geom), _ptr(st.binning),
                                  _ptr(st.img), _ptr(alpha), _ptr(gc), _ptr(gd), _ptr(ga), _ptr(gs), _ptr(grad2d), _ptr(g_sem),
                                  _stream(device))
    _capi.check(rc, "sgr_backward_blend")
    del keep
    return grad2d, g_sem


def _backward_layer_blends(settings, st: _ForwardState, tensors, layers, layer_bgs, layer_states, layer_alphas, grad_layers, sink_wanted):
    """The layers' stage 1 (sgr_backward_blend_layer): returns (SgrLayerGrad table for _backward_geom_impl, gradient of each layer's
    means2D sink or None, tensors the table points into).  A layer with an empty range, or whose outputs got no upstream gradient,
    keeps a table row without grad2d and costs nothing."""
    L = _capi.lib()
    means3D = tensors["means3D"]
    dev, P = means3D.device, int(means3D.shape[0])
    S = int(tensors["semantics"].shape[1]) if tensors["semantics"] is not None else 0
    M = int(tensors["sh"].shape[1]) if tensors["sh"] is not None else 0
    fr, keep = _make_frame(settings, P, M, S, dev, None)
    table, sink_grads, keep_alive = [], [], []
    for k, (b, e, _, sink) in enumerate(layers):
        gc, gd, ga = grad_layers[3 * k: 3 * k + 3]
        lg = _capi.SgrLayerGrad(b, e, None, None)
        sg = None
        if (gc is not None or gd is not None or ga is not None) and e > b:
            gc, gd, ga = (_dev_f32(g, dev) for g in _image_grads(settings, dev, (gc, gd, ga), (3, 1, 1)))
            g2 = torch.empty((e - b, 12), device=dev, dtype=torch.float32)
            lay = _capi.SgrLayer(b, e, layer_bgs[k].data_ptr())
            with torch.cuda.device(dev):
                rc = L.sgr_backward_blend_layer(C.byref(fr), C.byref(lay), _ptr(st.geom), _ptr(layer_states[k]), _ptr(layer_alphas[k]),
                                                _ptr(gc), _ptr(gd), _ptr(ga), _ptr(g2), _stream(dev))
            _capi.check(rc, "sgr_backward_blend_layer")
            lg.grad2d = g2.data_ptr()
            keep_alive += [gc, gd, ga, g2]
            if sink is not None and sink_wanted[k]:
                sg = torch.empty((e - b, 3), device=dev, dtype=torch.float32)
                lg.dL_dmeans2D = sg.data_ptr()
        table.append(lg)
        sink_grads.append(None if sg is None else sg.to(dtype=sink.dtype, device=sink.device))
    del keep
    return table, sink_grads, keep_alive


def _backward_geom_impl(settings, band, st: _ForwardState, tensors, radii, grad2d, layers=None):
    """Stage 2: per-Gaussian chain rule.  Outputs are torch.empty — the kernel writes every element.  `layers`: the SgrLayerGrad
    table of _backward_layer_blends; the rows of its live layers are merged into grad2d (sgr_backward_geom_layered), while the
    main means2D gradient stays that of the main images."""
    L = _capi.lib()
    means3D = tensors["means3D"]
    device, P = means3D.device, means3D.shape[0]
    S = int(tensors["semantics"].shape[1]) if tensors["semantics"] is not None else 0
    sh, colors, scales, rots, cov = (tensors[k] for k in ("sh", "colors_precomp", "scales", "rotations", "cov3Ds_precomp"))
    M = int(sh.shape[1]) if sh is not None else 0
    fr, keep = _make_frame(settings, P, M, S, device, band)
    grads = _geom_grad_buffers(tensors, P, device)
    live = [lg for lg in layers or () if lg.grad2d]
    inputs = (C.byref(fr), _ptr(means3D), _ptr(sh), _ptr(colors), _ptr(scales), _ptr(rots), _ptr(cov), _ptr(radii), _ptr(st.geom),
              _ptr(grad2d))
    with torch.cuda.device(device):
        if not live:
            rc = L.sgr_backward_geom(*inputs, *map(_ptr, grads), _stream(device))
        else:
            lo, hi = min(lg.begin for lg in live), max(lg.end for lg in live)
            scratch = torch.empty((3 * (hi - lo),), device=device, dtype=torch.float32)
            table = (_capi.SgrLayerGrad * len(layers))(*layers)
            rc = L.sgr_backward_geom_layered(*inputs, table, len(layers), _ptr(scratch), *map(_ptr, grads), _stream(device))
    _capi.check(rc, "sgr_backward_geom_layered" if live else "sgr_backward_geom")
    del keep
    return grads


def _forward_or_dump(means3D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp, raster_settings, band, capacity):
    try:
        return _forward_impl(means3D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp, raster_settings, band,
                             capacity)
    except Exception:
        if raster_settings.debug:  # same post-mortem as the reference (DGR/diff_gaussian_rasterization/__init__.py:87-94)
            _dump("snapshot_fw.dump", (raster_settings.bg, means3D, colors_precomp, semantics, opacities, scales, rotations,
                                       raster_settings.scale_modifier, cov3Ds_precomp, raster_settings.viewmatrix,
                                       raster_settings.projmatrix, raster_settings.tanfovx, raster_settings.tanfovy,
                                       raster_settings.image_height, raster_settings.image_width, sh, raster_settings.sh_degree,
                                       raster_settings.campos, raster_settings.prefiltered, raster_settings.debug))
            print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
        raise


def _forward_layers(settings, st: _ForwardState, tensors, P: int, device, layers):
    """Renders every layer from the tile lists of the main forward in `st` (sgr_forward_layer).  Returns (bg tensor per layer, layer
    state per layer, [color, depth, alpha] of every layer in one flat list); an empty range needs no state."""
    L = _capi.lib()
    H, W = int(settings.image_height), int(settings.image_width)
    M = int(tensors["sh"].shape[1]) if tensors is not None and tensors["sh"] is not None else 0
    S = int(tensors["semantics"].shape[1]) if tensors is not None and tensors["semantics"] is not None else 0
    fr, keep = _make_frame(settings, P, M, S, device, None)
    f32 = dict(device=device, dtype=torch.float32)
    bgs, states, outs = [], [], []
    for b, e, bg, _ in layers:
        bg = _dev_f32(bg, device)
        c, d, a = torch.empty((3, H, W), **f32), torch.empty((1, H, W), **f32), torch.empty((1, H, W), **f32)
        lay = _capi.SgrLayer(b, e, bg.data_ptr())
        ls, nbytes = None, 0
        if e > b:
            nb = C.c_size_t(0)
            _capi.check(L.sgr_layer_state_sizes(C.byref(fr), st.num_instances, C.byref(nb)), "sgr_layer_state_sizes")
            ls, nbytes = torch.empty((nb.value,), device=device, dtype=torch.uint8), nb.value
        with torch.cuda.device(device):
            rc = L.sgr_forward_layer(C.byref(fr), C.byref(lay), st.num_instances, _ptr(st.geom), _ptr(st.binning), _ptr(st.img), _ptr(ls),
                                     nbytes, _ptr(c), _ptr(d), _ptr(a), _stream(device))
        _capi.check(rc, "sgr_forward_layer")
        bgs.append(bg)
        states.append(ls)
        outs += [c, d, a]
    del keep
    return bgs, states, outs


class _RasterizeGaussians(torch.autograd.Function):
    """Outputs (color, radii, depth, alpha, semantic), then (color, depth, alpha) per render layer (include/sgr.h, SgrLayer).
    `layers` holds _check_layers' tuples (whole image only; () for the plain call) and `sinks` their means2D tensors or None."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, band=None, grad_reduce=None, capacity=None, layers=(), *sinks):
        # with layers an output without upstream gradient arrives as None, so a layer without one costs nothing in backward
        ctx.set_materialize_grads(not layers)
        color, radii, depth, alpha, semantic, st, tensors = _forward_or_dump(means3D, sh, colors_precomp, semantics, opacities, scales,
                                                                             rotations, cov3Ds_precomp, raster_settings, band, capacity)
        bgs, states, layer_outs = (_forward_layers(raster_settings, st, tensors, int(means3D.shape[0]), means3D.device, layers)
                                   if layers else ((), (), []))
        ctx.raster_settings, ctx.band, ctx.state, ctx.grad_reduce = raster_settings, band, st, grad_reduce
        ctx.layers, ctx.layer_bgs, ctx.layer_states = layers, bgs, states
        ctx.shapes = _input_shapes(means3D, means2D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp)
        # The fp32-contiguous inputs go through save_for_backward like the reference's (DGR __init__.py:101), so autograd's
        # version counters catch an in-place update of a parameter between forward and backward instead of silently
        # differentiating the mutated values.
        ctx.tensor_keys = None if tensors is None else tuple(k for k, v in tensors.items() if v is not None)
        ctx.tensor_none = None if tensors is None else tuple(k for k, v in tensors.items() if v is None)
        ctx.save_for_backward(radii, alpha, *layer_outs[2::3], *([] if tensors is None else [tensors[k] for k in ctx.tensor_keys]))
        ctx.mark_non_differentiable(radii)
        return (color, radii, depth, alpha, semantic, *layer_outs)

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_depth, grad_alpha, grad_semantic, *grad_layers):
        n = len(ctx.layers)
        radii, alpha, *rest = ctx.saved_tensors
        layer_alphas, saved = rest[:n], rest[n:]
        st, settings, band, shapes = ctx.state, ctx.raster_settings, ctx.band, ctx.shapes
        nones = (None,) * 5  # raster_settings, band, grad_reduce, capacity, layers
        if ctx.tensor_keys is None:  # P == 0: every layer range is empty
            sink_grads = tuple(None if s is None else torch.zeros((0, 3), device=s.device, dtype=s.dtype) for _, _, _, s in ctx.layers)
            return _fit_grads(shapes, (None,) * 9) + nones + sink_grads
        tensors = dict(zip(ctx.tensor_keys, saved))
        tensors.update({k: None for k in ctx.tensor_none})
        S = int(tensors["semantics"].shape[1]) if tensors["semantics"] is not None else 0
        grad_color, grad_depth, grad_alpha, grad_semantic = _image_grads(settings, tensors["means3D"].device,
                                                                         (grad_color, grad_depth, grad_alpha, grad_semantic), (3, 1, 1, S))
        try:
            grad2d, g_sem = _backward_blend_impl(settings, band, st, tensors, alpha, grad_color, grad_depth, grad_alpha, grad_semantic)
            if ctx.grad_reduce is not None:  # multi-GPU: sum the per-band partial sums across ranks (one collective)
                grad2d, g_sem = ctx.grad_reduce(grad2d, g_sem)
            if n:
                table, sink_grads, keep_alive = _backward_layer_blends(settings, st, tensors, ctx.layers, ctx.layer_bgs, ctx.layer_states,
                                                                       layer_alphas, grad_layers, ctx.needs_input_grad[14:])
                grads = _backward_geom_impl(settings, band, st, tensors, radii, grad2d, table)
            else:
                sink_grads, grads = (), _backward_geom_impl(settings, band, st, tensors, radii, grad2d)
        except Exception:
            if settings.debug:  # DGR/diff_gaussian_rasterization/__init__.py:141-148
                _dump("snapshot_bw.dump", (settings.bg, tensors["means3D"], radii, tensors["colors_precomp"], tensors["scales"],
                                           tensors["rotations"], settings.scale_modifier, tensors["cov3Ds_precomp"], settings.viewmatrix,
                                           settings.projmatrix, settings.tanfovx, settings.tanfovy, grad_color, grad_depth, grad_alpha,
                                           grad_semantic, tensors["sh"], settings.sh_degree, settings.campos, alpha, tensors["semantics"],
                                           settings.debug))
                print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
            raise
        g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov = grads
        return _fit_grads(shapes, (g_means3D, g_means2D, g_sh, g_colors, g_sem if S > 0 else None, g_opac, g_scales, g_rots,
                                   g_cov)) + nones + tuple(sink_grads)


class RenderLayer(NamedTuple):
    """Rows [begin, end) of the call's Gaussians, rendered in the same call as the full frame over background `bg` (3 floats).
    The reference's objects-only render (render_object with parse_camera_again=False, train.py:114-122) is
    ``RenderLayer(n_bkgd, P, (1, 1, 1))`` on the composed tensors, its background-only render ``RenderLayer(0, n_bkgd, (1, 1, 1))``.
    The layer's (color, depth, alpha) equal a separate GaussianRasterizer call on the sliced tensors with this `bg` and no
    semantics; an empty range gives colour `bg` with zero depth and alpha.  `means2D` ([end - begin, 3], optional) receives the
    layer's own screen-space gradient, as the separate call's means2D would; the main call's means2D receives the main images' only."""
    begin: int
    end: int
    bg: object
    means2D: Optional[torch.Tensor] = None


def _check_layers(layers, P: int):
    """(begin, end, bg as a float32 tensor, means2D) per layer; raises ValueError before anything touches the GPU."""
    out = []
    for i, l in enumerate(layers):
        if not isinstance(l, RenderLayer):
            l = RenderLayer(*l)
        b, e = int(l.begin), int(l.end)
        if not 0 <= b <= e <= P:
            raise ValueError(f"layer {i}: range [{b}, {e}) is not inside [0, {P}]")
        bg = l.bg.detach() if isinstance(l.bg, torch.Tensor) else torch.as_tensor(l.bg, dtype=torch.float32)
        if bg.numel() != 3 or not (bg.is_floating_point() or bg.dtype in (torch.int32, torch.int64)):
            raise ValueError(f"layer {i}: bg must hold 3 floats, got shape {tuple(bg.shape)} of {bg.dtype}")
        if l.means2D is not None and tuple(l.means2D.shape) != (e - b, 3):
            raise ValueError(f"layer {i}: means2D must have shape ({e - b}, 3), got {tuple(l.means2D.shape)}")
        out.append((b, e, bg.reshape(3), l.means2D))
    return out


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, semantics, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings, None, None, None, ())


class GaussianRasterizer(nn.Module):
    """Same surface as the reference class (DGR :181-260).  ``band`` / ``grad_reduce`` (tile-row sharding across GPUs,
    street_gaussians_b200.sharded) and ``capacity`` (sync-free binning, InstanceCapacity) are the only additions:
    keyword-only, default off."""

    def __init__(self, raster_settings, *, band: Optional[TileRowBand] = None, grad_reduce=None,
                 capacity: Optional[InstanceCapacity] = None):
        super().__init__()
        self.raster_settings = raster_settings
        self.band = band
        self.grad_reduce = grad_reduce
        self.capacity = capacity  # opt-in sync-free binning; share ONE InstanceCapacity across the rasterizers of a training loop

    def synchronize_capacity(self):
        """Wait for the outstanding frame statuses of the sync-free mode and raise if any frame overflowed."""
        if self.capacity is not None:
            self.capacity.check(wait=True)

    def markVisible(self, positions):
        L = _capi.lib()
        s = self.raster_settings
        with torch.no_grad():
            if not positions.is_cuda:
                raise _capi.SgrError("markVisible needs a CUDA tensor")
            dev = positions.device
            pos = _dev_f32(positions, dev)
            P = pos.shape[0]
            visible = torch.zeros((P,), device=dev, dtype=torch.bool)
            if P:
                view, proj = _dev_f32(s.viewmatrix, dev), _dev_f32(s.projmatrix, dev)
                with torch.cuda.device(dev):
                    rc = L.sgr_mark_visible(P, _ptr(pos), _ptr(view), _ptr(proj), C.c_void_p(visible.data_ptr()), _stream(dev))
                _capi.check(rc, "sgr_mark_visible")
        return visible

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, semantics=None):
        return self._forward(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, semantics, None)

    def forward_layers(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                       cov3D_precomp=None, semantics=None, *, layers):
        """forward() plus render layers: ``layers`` is a sequence of RenderLayer, and the result gains a 6th element holding one
        (color[3,H,W], depth[1,H,W], alpha[1,H,W]) per layer, rendered from this call's tile lists (whole image on one GPU, default
        and InstanceCapacity modes).  The first five elements are what forward() returns.  (forward() itself keeps the
        reference's exact signature.)"""
        return self._forward(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, semantics, layers)

    def _forward(self, means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, semantics, layers):
        if layers is not None:
            if self.band is not None or self.grad_reduce is not None:
                raise _capi.SgrError("render layers need the whole image on one GPU (this rasterizer has a tile-row band / gradient reduction)")
            layers = tuple(_check_layers(layers, int(means3D.shape[0])))
        shs, colors_precomp, scales, rotations, cov3D_precomp, semantics = _reference_inputs(means3D, shs, colors_precomp, scales, rotations,
                                                                                             cov3D_precomp, semantics)
        if layers is None:
            return _RasterizeGaussians.apply(means3D, means2D, shs, colors_precomp, semantics, opacities, scales, rotations, cov3D_precomp,
                                             self.raster_settings, self.band, self.grad_reduce, self.capacity, ())
        if not means3D.is_cuda:
            raise _capi.SgrError("street_gaussians_b200 rasterizer needs CUDA tensors (there is no CPU fallback)")
        out = _RasterizeGaussians.apply(means3D, means2D, shs, colors_precomp, semantics, opacities, scales, rotations, cov3D_precomp,
                                        self.raster_settings, self.band, self.grad_reduce, self.capacity, layers, *(l[3] for l in layers))
        return tuple(out[:5]) + (tuple(tuple(out[5 + 3 * k: 8 + 3 * k]) for k in range(len(layers))),)

    def visible_filter(self, means3D, scales=None, rotations=None, cov3D_precomp=None) -> Tuple[torch.Tensor, torch.Tensor]:
        L = _capi.lib()
        s = self.raster_settings
        with torch.no_grad():
            if means3D.dim() != 2 or means3D.shape[1] != 3:
                raise RuntimeError("means3D must have dimensions (num_points, 3)")
            if not means3D.is_cuda:
                raise _capi.SgrError("visible_filter needs CUDA tensors")
            dev = means3D.device
            P = means3D.shape[0]
            radii = torch.zeros((P,), device=dev, dtype=torch.int32)
            means2D = torch.zeros((P, 2), device=dev, dtype=torch.float32)
            if P:
                m = _dev_f32(means3D, dev)
                sc, ro, cv = _none_if_empty(scales), _none_if_empty(rotations), _none_if_empty(cov3D_precomp)
                sc = _dev_f32(sc, dev) if sc is not None else None
                ro = _dev_f32(ro, dev) if ro is not None else None
                cv = _dev_f32(cv, dev) if cv is not None else None
                fr, keep = _make_frame(s, P, 0, 0, dev, None)
                with torch.cuda.device(dev):
                    rc = L.sgr_visible_filter(C.byref(fr), _ptr(m), _ptr(sc), _ptr(ro), _ptr(cv), _ptr(radii), _ptr(means2D), _stream(dev))
                _capi.check(rc, "sgr_visible_filter")
                del keep
        return radii, means2D


def distCUDA2(points: torch.Tensor) -> torch.Tensor:
    """simple_knn._C.distCUDA2 (KNN/spatial.cu:14-26): mean squared distance to the 3 nearest neighbours, [P] fp32."""
    L = _capi.lib()
    if not points.is_cuda:
        raise _capi.SgrError("distCUDA2 needs a CUDA tensor")
    dev = points.device
    pts = _dev_f32(points, dev)
    P = pts.shape[0]
    out = torch.zeros((P,), device=dev, dtype=torch.float32)
    if P:
        nbytes = L.sgr_knn_scratch_bytes(P)
        scratch = torch.empty((nbytes,), device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            rc = L.sgr_knn_mean_dist2(P, _ptr(pts), _ptr(out), _ptr(scratch), nbytes, _stream(dev))
        _capi.check(rc, "sgr_knn_mean_dist2")
    return out
