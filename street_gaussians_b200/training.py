"""Post-backward bookkeeping of a training iteration (SURVEY.md §8 row f3) over sgr_densify_stats / sgr_adam_step.

    add_densification_stats(models, radii, viewspace_point_grad)
        = StreetGaussianModel.set_max_radii2D + add_densification_stats (lib/models/street_gaussian_model.py:551-571) for all
        sub-models in one kernel.  `models`: objects / mappings exposing max_radii2D [n], xyz_gradient_accum [n,2], denom [n,1]
        (the attributes lib/models/gaussian_model.py:49-51 creates) in composition order (background, then the frame's actors).
    FusedAdam(param_groups, ...)
        torch.optim.Adam's interface (param_groups with per-group "lr" / "name", .step(), .zero_grad(), state_dict) for the way the
        reference uses it (gaussian_model.py:300-303: lr per group, eps=1e-15, no weight decay / amsgrad); ONE kernel updates every
        tensor of every group — pass the groups of all sub-models to a single FusedAdam to get a single launch per iteration.
    densify_and_prune(models, max_grad, min_opacity, prune_big_points, optimizer=None, *, grad_abs=False, seed=None, noise=None)
        = StreetGaussianModel.densify_and_prune (lib/models/street_gaussian_model.py:573-586) over GaussianModelBkgd /
        GaussianModelActor.densify_and_prune: clone, split and prune every sub-model in two kernels around ONE host read-back of the
        new sizes, resizing the parameters together with their Adam moments.  Works with one shared FusedAdam over all sub-models.
    reset_opacity(models, optimizer=None)
        = StreetGaussianModel.reset_opacity (:597-602 -> lib/models/gaussian_model.py:410-414), in place, one kernel.
    SparseAdam(param_groups, ...).step(models, radii)
        opt-in visibility-masked Adam (no reference counterpart; it deviates from the reference): FusedAdam's update on the rows
        with radii > 0 only, every other row's parameter and moments left untouched.
    CubeMapSparseAdam([cube_map], ...).step(blocks)
        opt-in block-masked Adam for the sky cube map (no reference counterpart; it deviates from the reference): FusedAdam's update
        on the 32 x 32-texel blocks sky.sky_composite(blocks=) marked, every other texel left untouched, and the map cleared.
CUDA tensors only; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Iterable, Sequence

import torch

from . import _capi
from ._capi import ptr


def _attr(model, name):
    return model[name] if isinstance(model, dict) else getattr(model, name)


def add_densification_stats(models: Sequence, radii: torch.Tensor, viewspace_point_grad: torch.Tensor) -> None:
    if not radii.is_cuda:
        raise _capi.SgrError("add_densification_stats needs CUDA tensors (there is no CPU fallback)")
    dev = radii.device
    n = len(models)
    segs = (_capi.SgrStatSegment * n)()
    start, keep = 0, []
    for k, m in enumerate(models):
        mr, ga, dn = _attr(m, "max_radii2D"), _attr(m, "xyz_gradient_accum"), _attr(m, "denom")
        for t, shape in ((mr, 1), (ga, 2), (dn, 1)):
            if t.dtype != torch.float32 or not t.is_contiguous() or t.device != dev:
                raise _capi.SgrError("densification statistics must be contiguous fp32 CUDA tensors (they are updated in place)")
        cnt = int(mr.shape[0])
        if ga.numel() != 2 * cnt or dn.numel() != cnt:
            raise ValueError(f"model {k}: xyz_gradient_accum must be [{cnt}, 2] and denom [{cnt}, 1]")
        s = segs[k]
        s.start, s.count = start, cnt
        s.max_radii2D, s.xyz_gradient_accum, s.denom = (t.data_ptr() if cnt else None for t in (mr, ga, dn))
        start += cnt
    if radii.numel() != start or viewspace_point_grad.shape != (start, 3):
        raise ValueError(f"radii must be [{start}] and the viewspace gradient [{start}, 3] for these models")
    r = radii if (radii.dtype == torch.int32 and radii.is_contiguous()) else radii.to(torch.int32).contiguous()
    g = _capi.f32(viewspace_point_grad)
    _capi.call("sgr_densify_stats", dev, segs, n, ptr(r), ptr(g))


def _advance_state(st, p):
    """torch.optim.Adam's per-parameter state {step, exp_avg, exp_avg_sq}, created at zero on first use, with step incremented."""
    if len(st) == 0:
        st["step"] = 0
        st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
    st["step"] = int(st["step"]) + 1
    return st


class FusedAdam(torch.optim.Optimizer):
    """torch.optim.Adam(params, lr, betas=(0.9, 0.999), eps) semantics, every parameter of every group updated by one kernel."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        buckets = {}  # (device, betas, eps) -> [(param, group)]
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                if not p.is_cuda:
                    raise _capi.SgrError("FusedAdam needs CUDA parameters (there is no CPU fallback)")
                if p.dtype != torch.float32 or not p.is_contiguous():
                    raise _capi.SgrError("FusedAdam updates contiguous fp32 parameters in place")
                buckets.setdefault((p.device, tuple(group["betas"]), float(group["eps"])), []).append((p, group))
        for (dev, betas, eps), items in buckets.items():
            tab = (_capi.SgrAdamTensor * len(items))()
            keep = []
            for k, (p, group) in enumerate(items):
                st = _advance_state(self.state[p], p)
                g = _capi.f32(p.grad)
                keep.append(g)
                t = tab[k]
                t.param, t.grad, t.exp_avg, t.exp_avg_sq = p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()
                t.numel, t.lr, t.step = p.numel(), float(group["lr"]), st["step"]
            _capi.call("sgr_adam_step", dev, tab, len(items), float(betas[0]), float(betas[1]), eps)
            del keep
        return loss


# ---- densification ----
PARAM_NAMES = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation", "_semantic")
STAT_NAMES = ("max_radii2D", "xyz_gradient_accum", "denom")
SCALAR_NAMES = ("points_total", "points_clone", "points_split", "points_below_min_opacity", "points_big_ws", "points_pruned")


def _has(model, name):
    return name in model if isinstance(model, dict) else hasattr(model, name)


def _set(model, name, value):
    if isinstance(model, dict):
        model[name] = value
    else:
        setattr(model, name, value)


def _per_model(v, n, what):
    if isinstance(v, (list, tuple)):
        if len(v) != n:
            raise ValueError(f"{what}: {len(v)} values for {n} models")
        return list(v)
    return [v] * n


def _f32(v) -> float:
    return float(torch.as_tensor(v, dtype=torch.float32).reshape(-1)[0])


def _times(t, f: float) -> float:
    """fp32 tensor x Python float, formed the way torch forms the reference's thresholds (percent_dense * extent, ...)."""
    return float((torch.as_tensor(t, dtype=torch.float32).detach().cpu().reshape(-1)[:1] * f)[0])


def _param_slots(optimizer):
    """id(param) -> (group, position): groups are matched by parameter identity, never by group['name'], so one optimizer over
    all sub-models (whose groups repeat the names "xyz", "f_dc", ...) works as well as one per sub-model."""
    slots = {}
    opts = [] if optimizer is None else list(optimizer) if isinstance(optimizer, (list, tuple)) else [optimizer]
    for opt in opts:
        for g in opt.param_groups:
            for j, p in enumerate(g["params"]):
                slots[id(p)] = (opt, g, j)
    return slots


def _moments(optimizer, slots, p):
    if id(p) not in slots:
        return None
    st = slots[id(p)][0].state.get(p, None)
    if not st or "exp_avg" not in st:
        return None
    return st["exp_avg"], st["exp_avg_sq"]


def _check_tensor(t, dev, what):
    if not t.is_cuda or t.device != dev:
        raise _capi.SgrError(f"{what} must be a CUDA tensor on {dev} (there is no CPU fallback)")
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise _capi.SgrError(f"{what} must be a contiguous fp32 tensor")


def _segment(model, k, optimizer, slots, dev):
    seg = _capi.SgrDensifySegment()
    params = [_attr(model, n) for n in PARAM_NAMES]
    n = int(params[0].shape[0])
    seg.count = n
    widths = [int(math.prod(p.shape[1:])) for p in params]
    seg.dc_width, seg.rest_width, seg.semantic_width = widths[1], widths[2], widths[6]
    moments = []
    for a, p in enumerate(params):
        _check_tensor(p, dev, f"model {k}: {PARAM_NAMES[a]}")
        if p.shape[0] != n:
            raise ValueError(f"model {k}: {PARAM_NAMES[a]} has {p.shape[0]} rows, _xyz {n}")
        mv = _moments(optimizer, slots, p)
        if mv is not None:
            for t in mv:
                _check_tensor(t, dev, f"model {k}: Adam state of {PARAM_NAMES[a]}")
                if t.shape != p.shape:
                    raise ValueError(f"model {k}: Adam state of {PARAM_NAMES[a]} has shape {tuple(t.shape)}, the parameter {tuple(p.shape)}")
        moments.append(mv)
        if n and widths[a]:
            seg.param[a] = p.data_ptr()
            if mv is not None:
                seg.exp_avg[a], seg.exp_avg_sq[a] = mv[0].data_ptr(), mv[1].data_ptr()
    return seg, params, moments, widths


def _stat_segment(seg, model, k, dev):
    """Check the model's densification statistics against seg.count rows and point the segment at them."""
    n = seg.count
    stats = [_attr(model, s) for s in STAT_NAMES]
    for t, w in zip(stats, (1, 2, 1)):
        _check_tensor(t, dev, f"model {k}: densification statistics")
        if t.numel() != w * n:
            raise ValueError(f"model {k}: max_radii2D must be [{n}], xyz_gradient_accum [{n}, 2] and denom [{n}, 1]")
    if n:
        seg.max_radii2D, seg.xyz_gradient_accum, seg.denom = (t.data_ptr() for t in stats)


def _install(model, params, new_params, new_moments, new_stats, slots):
    """Replace the model's parameters `params` by new nn.Parameters over `new_params` (same requires_grad), in their optimizer groups
    too (found by identity): each optimizer state moves to the new key with its step unchanged and the new moments (None: the state
    is kept as it is).  The statistics become `new_stats`."""
    for a, (old, t) in enumerate(zip(params, new_params)):
        p = torch.nn.Parameter(t, requires_grad=old.requires_grad)
        if id(old) in slots:
            opt, g, j = slots[id(old)]
            g["params"][j] = p
            st = opt.state.pop(old, None)
            if st is not None:
                if new_moments[a] is not None:
                    st["exp_avg"], st["exp_avg_sq"] = new_moments[a]
                opt.state[p] = st
        _set(model, PARAM_NAMES[a], p)
    for name, t in zip(STAT_NAMES, new_stats):
        _set(model, name, t)


ADAM_GROUP_NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic")  # gaussian_model.py:289-297, by PARAM_NAMES


def adam_state_dict(model, optimizer, *, state=None) -> dict:
    """One sub-model's optimizer state in the format torch.optim.Adam.state_dict() gives for the reference's per-model optimizer
    (GaussianModel.training_setup, gaussian_model.py:286-303): seven groups named xyz, f_dc, f_rest, opacity, scaling, rotation, semantic,
    parameter i in group i, each group with the lr, betas and eps of the group of `optimizer` (one optimizer or a list, e.g. a FusedAdam
    or SparseAdam over several sub-models) that holds the model's tensor, found by identity; state[i] = {step (fp32 CPU scalar tensor, as
    torch keeps it), exp_avg, exp_avg_sq} for the tensors with Adam state.  The moments are the optimizer's tensors, not copies.  state:
    {parameter name: {"step", "exp_avg", "exp_avg_sq"}} to use instead of the optimizer's (sharded.gather_state's "adam").  What
    GaussianModel.state_dict stores as 'optimizer', so a torch.optim.Adam built as the reference builds it load_state_dict()s it."""
    slots = _param_slots(optimizer)
    groups, packed = [], {}
    for i, (a, name) in enumerate(zip(PARAM_NAMES, ADAM_GROUP_NAMES)):
        p = _attr(model, a)
        if id(p) not in slots:
            raise ValueError(f"{a} is not held by the optimizer")
        opt, g, _ = slots[id(p)]
        groups.append(dict(params=[torch.zeros(0)], lr=g["lr"], betas=tuple(g["betas"]), eps=g["eps"], name=name))
        st = opt.state.get(p) if state is None else state.get(a)
        if st:
            packed[i] = dict(step=torch.tensor(float(int(st["step"])), dtype=torch.float32), exp_avg=st["exp_avg"], exp_avg_sq=st["exp_avg_sq"])
    sd = torch.optim.Adam(groups, lr=0.0, eps=1e-15).state_dict()
    sd["state"] = packed
    return sd


def _densify(models, max_grad, min_opacity, prune_big_points, optimizer=None, grad_abs=False, seed=None, noise=None, keep_masks=False):
    L = _capi.lib()
    models = list(models)
    nm = len(models)
    if nm == 0:
        return [], None
    dev = _attr(models[0], "_xyz").device
    slots = _param_slots(optimizer)
    max_grads, grad_abss = _per_model(max_grad, nm, "max_grad"), _per_model(grad_abs, nm, "grad_abs")
    segs = (_capi.SgrDensifySegment * nm)()
    infos = []
    for k, m in enumerate(models):
        seg, params, moments, widths = _segment(m, k, optimizer, slots, dev)
        _stat_segment(seg, m, k, dev)
        if _has(m, "scene_radius"):       # GaussianModelBkgd (gaussian_model_bkgd.py:21-23, 86-98)
            seg.kind, extent = _capi.DENSIFY_BACKGROUND, _attr(m, "scene_radius")
            c = torch.as_tensor(_attr(m, "sphere_center"), dtype=torch.float32).detach().cpu().reshape(-1)
            for a in range(3):
                seg.sphere_center[a] = float(c[a])
            seg.sphere_diameter = _f32(2 * torch.as_tensor(_attr(m, "sphere_radius"), dtype=torch.float32).detach().cpu().reshape(-1)[:1])
        elif _has(m, "extent"):           # GaussianModelActor (gaussian_model_actor.py:37-40, 218-247)
            seg.kind, extent = _capi.DENSIFY_ACTOR, _attr(m, "extent")
            lo = torch.as_tensor(_attr(m, "min_xyz"), dtype=torch.float32).detach().cpu().reshape(-1)
            hi = torch.as_tensor(_attr(m, "max_xyz"), dtype=torch.float32).detach().cpu().reshape(-1)
            for a in range(3):
                seg.min_xyz[a], seg.max_xyz[a] = float(lo[a]), float(hi[a])
        else:
            raise ValueError(f"model {k} has neither scene_radius (background) nor extent (actor)")
        seg.grad_col = 1 if grad_abss[k] else 0
        seg.prune_big = 1 if prune_big_points else 0
        seg.grad_threshold = _f32(max_grads[k])
        seg.dense_threshold = _times(extent, _attr(m, "percent_dense"))
        seg.big_threshold = _times(extent, _attr(m, "percent_big_ws"))
        seg.min_opacity = _f32(min_opacity)
        segs[k] = seg
        infos.append((params, moments, widths))
    P = sum(s.count for s in segs)
    if noise is not None:
        if tuple(noise.shape) != (P, _capi.DENSIFY_DRAWS):
            raise ValueError(f"noise must be [{P}, {_capi.DENSIFY_DRAWS}]")
        _check_tensor(noise, dev, "noise")
    if seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    nbytes = L.sgr_densify_scratch_bytes(nm, P)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    result = (C.c_int64 * (nm * _capi.DENSIFY_RESULT))()
    npp = ptr(noise) if noise is not None else None
    _capi.call("sgr_densify_plan", dev, segs, nm, C.c_uint64(seed), npp, scratch.data_ptr(), nbytes, result)
    outs = (_capi.SgrDensifyOutput * nm)()
    new = []
    for k, (params, moments, widths) in enumerate(infos):
        n_new = int(result[k * _capi.DENSIFY_RESULT])
        o = outs[k]
        o.count = n_new
        np_, nmom = [], []
        for a, p in enumerate(params):
            t = torch.empty((n_new,) + tuple(p.shape[1:]), dtype=torch.float32, device=dev)
            mv = None if moments[a] is None else (torch.empty_like(t), torch.empty_like(t))
            if n_new and widths[a]:
                o.param[a] = t.data_ptr()
                if mv is not None and segs[k].count:
                    o.exp_avg[a], o.exp_avg_sq[a] = mv[0].data_ptr(), mv[1].data_ptr()
            if mv is not None and segs[k].count == 0:
                mv = (torch.zeros_like(t), torch.zeros_like(t))
            np_.append(t)
            nmom.append(mv)
        stats = (torch.empty(n_new, device=dev), torch.empty(n_new, 2, device=dev), torch.empty(n_new, 1, device=dev))
        if n_new:
            o.max_radii2D, o.xyz_gradient_accum, o.denom = (t.data_ptr() for t in stats)
        new.append((np_, nmom, stats))
    _capi.call("sgr_densify_apply", dev, segs, outs, nm, C.c_uint64(seed), npp, scratch.data_ptr(), nbytes)
    scalars = []
    for k, m in enumerate(models):
        _install(m, infos[k][0], *new[k], slots)
        r = result[k * _capi.DENSIFY_RESULT:(k + 1) * _capi.DENSIFY_RESULT]
        d = dict(zip(SCALAR_NAMES, (int(v) for v in r[1:7])))
        if not prune_big_points:
            d.pop("points_big_ws")
        scalars.append(d)
    masks = None
    if keep_masks:  # the plan's per-parent 4-bit section masks (for tests): in the scratch, after the two tables and two start arrays
        al = lambda b: (b + 255) // 256 * 256
        off = al(C.sizeof(_capi.SgrDensifySegment) * nm) + al(C.sizeof(_capi.SgrDensifyOutput) * nm) + 2 * al(4 * (nm + 1))
        masks = scratch[off:off + P].clone()
    return scalars, masks


def densify_and_prune(models: Sequence, max_grad, min_opacity: float, prune_big_points: bool, optimizer=None, *, grad_abs=False,
                      seed=None, noise=None) -> list:
    """Clone, split and prune every sub-model (background and actors, in composition order) in one pass, as
    GaussianModelBkgd.densify_and_prune (lib/models/gaussian_model_bkgd.py:74-114) and GaussianModelActor.densify_and_prune
    (lib/models/gaussian_model_actor.py:204-261) do one model at a time.

    models: objects or mappings with the reference's attributes: the parameters _xyz, _features_dc, _features_rest, _opacity,
      _scaling, _rotation, _semantic; the statistics max_radii2D, xyz_gradient_accum, denom; percent_dense and percent_big_ws; and
      either scene_radius, sphere_center, sphere_radius (a background) or extent, min_xyz, max_xyz (an actor).
    max_grad, grad_abs: one value, or one per model.  The reference reads them from the config per kind
      (cfg.optim.densify_grad_threshold_bkgd / _obj and densify_grad_abs_bkgd / _obj); grad_abs selects column 1 of
      xyz_gradient_accum.  An actor with random_initialization or deformable uses the caller's max_grad with grad_abs=False.
    optimizer: one optimizer (e.g. a FusedAdam over all models) or a list of them (e.g. the reference's torch.optim.Adam per model).  Each parameter's group is found by identity, the
      parameter is replaced by a new nn.Parameter in that group, and its state (step unchanged) moves to the new key with the
      moments of surviving rows carried and zero moments for clones and children.
    seed: key of the Philox normal draws (None: drawn from torch's default generator).  noise: [P, 18] draws per parent instead
      (a test seam; see include/sgr.h).

    Returns one dict per model with points_total, points_clone, points_split, points_below_min_opacity, points_big_ws (with
    prune_big_points) and points_pruned.  The only host synchronisation is one read-back of the new sizes.  Unlike the reference it
    does not call torch.cuda.empty_cache(): the freed blocks stay in PyTorch's cache for the next iterations.  The number of
    Gaussians changes, so a CUDA graph that captured a training step must be captured again after this call."""
    return _densify(models, max_grad, min_opacity, prune_big_points, optimizer, grad_abs, seed, noise)[0]


def reset_opacity(models: Sequence, optimizer=None) -> None:
    """GaussianModel.reset_opacity (lib/models/gaussian_model.py:410-414) for every model in one kernel:
    _opacity = inverse_sigmoid(min(sigmoid(_opacity), 0.01)) and the opacity's Adam moments zeroed, in place (the parameter
    objects stay the same, so the optimizer needs no update)."""
    models = list(models)
    if not models:
        return
    slots = _param_slots(optimizer)
    segs = (_capi.SgrDensifySegment * len(models))()
    dev = _attr(models[0], "_opacity").device
    for k, m in enumerate(models):
        op = _attr(m, "_opacity")
        _check_tensor(op, dev, f"model {k}: _opacity")
        segs[k].count = int(op.numel())
        if op.numel():
            segs[k].param[3] = op.data_ptr()
            mv = _moments(optimizer, slots, op)
            if mv is not None:
                for t in mv:
                    _check_tensor(t, dev, f"model {k}: Adam state of _opacity")
                segs[k].exp_avg[3], segs[k].exp_avg_sq[3] = mv[0].data_ptr(), mv[1].data_ptr()
    _capi.call("sgr_reset_opacity", dev, segs, len(models))


# ---- visibility-masked Adam ----
class SparseAdam(torch.optim.Optimizer):
    """Visibility-masked ("sparse") Adam: an OPT-IN alternative to FusedAdam that updates only the rows of the Gaussians the frame
    rendered.  It changes training results against the reference (whose torch.optim.Adam also moves invisible rows on their decaying
    momentum), so FusedAdam stays the drop-in; use this one when the optimizer step's cost matters more than matching the reference.

    step(models, radii) — models: the frame's sub-models in composition order (background, then the frame's actors), the same list
    and radii [sum of rows] int32 (the rasterizer's output) that add_densification_stats gets.  Each model's per-Gaussian tensors are
    found by identity among _xyz, _features_dc, _features_rest, _opacity, _scaling, _rotation, _semantic.  For every such tensor this
    optimizer holds and that has a .grad:
      * row l of model k is visible iff radii[start_k + l] > 0 (the reference's visibility_filter);
      * visible rows get FusedAdam's update bit for bit, with the tensor's group lr / betas / eps and its step count;
      * invisible rows keep their parameter, exp_avg and exp_avg_sq, and their gradient is not read;
      * state["step"] goes up by one, as in FusedAdam: there are no per-row step counts.
    Rows that receive gradient from anything other than this frame's render (a regulariser, another camera's loss) are still
    skipped when their radii is 0.  Tensors held by this optimizer that belong to no model passed in this call (actors absent from
    the frame) keep their bits and their step count.  So do non-per-Gaussian parameters such as actor poses: put those in a
    FusedAdam.  The state stays {step, exp_avg, exp_avg_sq}, so densify_and_prune, reset_opacity, state_dict and load_state_dict
    work unchanged, and a state dict moves between FusedAdam and SparseAdam in either direction.  One kernel launch per (betas, eps)
    bucket; no host synchronisation.  CUDA tensors only."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))

    @torch.no_grad()
    def step(self, models: Sequence = None, radii: torch.Tensor = None, closure=None):
        if models is None or radii is None:
            raise TypeError("SparseAdam.step(models, radii) needs the frame's models and radii; it has no dense fallback "
                            "(use FusedAdam for a dense update)")
        loss = closure() if closure is not None else None
        models = list(models)
        params, rows = [], []
        for k, m in enumerate(models):
            ps = [_attr(m, n) for n in PARAM_NAMES]
            n = int(ps[0].shape[0])
            for a, p in enumerate(ps):
                if p.dim() == 0 or p.shape[0] != n:
                    raise ValueError(f"model {k}: {PARAM_NAMES[a]} has shape {tuple(p.shape)}, _xyz has {n} rows")
            params.append(ps)
            rows.append(n)
        if radii.dtype != torch.int32 or tuple(radii.shape) != (sum(rows),):
            raise ValueError(f"radii must be an int32 tensor of shape [{sum(rows)}] for these models, got {radii.dtype} {tuple(radii.shape)}")
        if not radii.is_cuda:
            raise _capi.SgrError("SparseAdam needs CUDA tensors (there is no CPU fallback)")
        dev = radii.device
        # What sgr_sparse_adam_step would reject is checked here, before any state changes, so that a bad group or tensor cannot
        # leave other tensors stepped.  Hyper-parameters once per group; the messages are only formatted on failure.
        hyper = {}  # id(group) -> (lr, (betas, eps))
        for g in self.param_groups:
            lr, betas = float(g["lr"]), tuple(float(b) for b in g["betas"])
            if not math.isfinite(lr):
                raise ValueError(f"a parameter group has a non-finite lr {lr}")
            if not all(0.0 <= b < 1.0 for b in betas):
                raise ValueError(f"a parameter group has betas {betas} outside [0, 1)")
            hyper[id(g)] = (lr, (betas, float(g["eps"])))
        group_of = {id(p): g for g in self.param_groups for p in g["params"]}
        f32 = torch.float32
        ok = lambda t: t.is_cuda and t.dtype == f32 and t.device == dev and t.is_contiguous()
        buckets = {}  # (betas, eps) -> [(model, tensor, param, lr, width)]; every tensor is on radii's device
        for k, ps in enumerate(params):
            for a, p in enumerate(ps):
                g = group_of.get(id(p))
                if g is None or p.grad is None:
                    continue
                if not ok(p):
                    _check_tensor(p, dev, f"model {k}: {PARAM_NAMES[a]}")
                st = self.state[p]
                if st:
                    m, v = st["exp_avg"], st["exp_avg_sq"]
                    if not (ok(m) and ok(v) and m.shape == p.shape and v.shape == p.shape):
                        for t in (m, v):
                            _check_tensor(t, dev, f"model {k}: Adam state of {PARAM_NAMES[a]}")
                        raise ValueError(f"model {k}: Adam state of {PARAM_NAMES[a]} has shapes {tuple(m.shape)} / {tuple(v.shape)}, "
                                         f"the parameter {tuple(p.shape)}")
                w = math.prod(p.shape[1:])
                if w > _capi.SPARSE_ADAM_MAX_WIDTH:
                    raise _capi.SgrError(f"model {k}: {PARAM_NAMES[a]} has {w} floats per row, more than {_capi.SPARSE_ADAM_MAX_WIDTH}")
                lr, key = hyper[id(g)]
                buckets.setdefault(key, []).append((k, a, p, lr, w))
        if not buckets:
            return loss
        r = radii.contiguous()
        for (betas, eps), items in buckets.items():
            # per model: param, grad, exp_avg, exp_avg_sq, width, lr, step of its 7 tensors, written into the ctypes record at once
            fields = [None] * len(models)
            keep = []
            for k, a, p, lr, w in items:
                st = _advance_state(self.state[p], p)
                if w == 0:
                    continue
                f = fields[k]
                if f is None:
                    f = fields[k] = [[None] * 7, [None] * 7, [None] * 7, [None] * 7, [0] * 7, [0.0] * 7, [0] * 7]
                f[4][a], f[5][a], f[6][a] = w, lr, st["step"]
                if p.numel():
                    g = _capi.f32(p.grad)
                    keep.append(g)
                    f[0][a], f[1][a], f[2][a], f[3][a] = p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()
            segs = (_capi.SgrSparseAdamSegment * len(models))()
            start = 0
            for k, n in enumerate(rows):
                s = segs[k]
                s.start, s.count = start, n
                start += n
                f = fields[k]
                if f is not None:
                    s.param[:], s.grad[:], s.exp_avg[:], s.exp_avg_sq[:], s.width[:], s.lr[:], s.step[:] = f
            _capi.call("sgr_sparse_adam_step", dev, segs, len(models), ptr(r), float(betas[0]), float(betas[1]), eps)
            del keep
        return loss


# ---- block-masked Adam of the sky cube map ----
class CubeMapSparseAdam(torch.optim.Optimizer):
    """Block-masked Adam for the sky cube map: an OPT-IN alternative to FusedAdam (the reference's torch.optim.Adam(eps=1e-15) of
    SkyCubeMap) that steps only the 32 x 32-texel blocks the frame's backward touched.  It changes training results against the
    reference, whose Adam keeps moving every texel on its decaying momentum, so FusedAdam stays the drop-in.

    It holds exactly one parameter, the contiguous fp32 CUDA cube map [6, R, R, 3].  step(blocks) — blocks: the uint8 map of
    sky.block_map(R, device) that sky.sky_composite(..., blocks=blocks) filled:
      * with a .grad, state["step"] goes up by one (as in FusedAdam: there are no per-block step counts), the moments are created at
        zero on first use, and ONE sgr_cube_sparse_adam_step call gives the marked blocks FusedAdam's update bit for bit, leaves every
        other texel's parameter and moments untouched (their gradient is not read), and clears `blocks` for the next frame;
      * without a .grad, nothing changes, the map included.
    The state is {step, exp_avg, exp_avg_sq}, so a state dict moves between FusedAdam and CubeMapSparseAdam in either direction, and
    param_groups[0]["lr"] can be scheduled.  No host synchronisation and, after the first step, no allocation; the grid depends on R
    only, so the step can be captured in a CUDA graph.  step() without a map raises TypeError: there is no dense fallback."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))
        ps = [p for g in self.param_groups for p in g["params"]]
        if len(ps) != 1:
            raise ValueError(f"CubeMapSparseAdam holds exactly one parameter (the cube map), got {len(ps)}")
        p = ps[0]
        if p.dim() != 4 or p.shape[0] != 6 or p.shape[1] != p.shape[2] or p.shape[3] != 3:
            raise ValueError(f"the cube map must be [6, R, R, 3], got {tuple(p.shape)}")
        if p.dtype != torch.float32 or not p.is_contiguous():
            raise ValueError(f"the cube map must be a contiguous fp32 tensor, got {p.dtype}")
        self._R = int(p.shape[1])
        self._nblocks = int(_capi.lib().sgr_sky_grad_blocks(self._R))
        if self._nblocks <= 0:
            raise ValueError(f"the cube map's R={self._R} is outside 0 < R <= 16384")
        self._rec = _capi.SgrAdamTensor()  # the entry's record, refilled in place every step
        self._rec.numel = p.numel()

    @torch.no_grad()
    def step(self, blocks: torch.Tensor = None, closure=None):
        if blocks is None:
            raise TypeError("CubeMapSparseAdam.step(blocks) needs the block map sky_composite(blocks=) filled; it has no dense fallback "
                            "(use FusedAdam for a dense update)")
        if blocks.dtype != torch.uint8 or blocks.numel() != self._nblocks or not blocks.is_contiguous():
            raise ValueError(f"blocks must be a contiguous uint8 map of sgr_sky_grad_blocks({self._R}) = {self._nblocks} bytes, got "
                             f"{blocks.dtype} {tuple(blocks.shape)}")
        loss = closure() if closure is not None else None
        group = self.param_groups[0]
        p = group["params"][0]
        if p.grad is None:
            return loss
        lr, (b1, b2), eps = float(group["lr"]), (float(b) for b in group["betas"]), float(group["eps"])
        if not math.isfinite(lr):
            raise ValueError(f"non-finite lr {lr}")
        if not (0.0 <= b1 < 1.0 and 0.0 <= b2 < 1.0):
            raise ValueError(f"betas ({b1}, {b2}) outside [0, 1)")
        dev = p.device
        if not p.is_cuda or blocks.device != dev:
            raise _capi.SgrError(f"CubeMapSparseAdam needs the cube map and blocks on one CUDA device (cube on {p.device}, blocks on "
                                 f"{blocks.device}; there is no CPU fallback)")
        if tuple(p.shape) != (6, self._R, self._R, 3) or p.dtype != torch.float32 or not p.is_contiguous():
            raise ValueError(f"the cube map changed to {p.dtype} {tuple(p.shape)}")
        st = self.state[p]
        if st:
            m, v = st["exp_avg"], st["exp_avg_sq"]
            for t in (m, v):
                if t.shape != p.shape or t.dtype != torch.float32 or t.device != dev or not t.is_contiguous():
                    raise ValueError(f"the cube map's Adam state is {t.dtype} {tuple(t.shape)} on {t.device}, the parameter "
                                     f"{p.dtype} {tuple(p.shape)} on {dev}")
        g = p.grad if (p.grad.dtype == torch.float32 and p.grad.is_contiguous()) else _capi.f32(p.grad)
        if g.shape != p.shape or g.device != dev:
            raise ValueError(f"the cube map's gradient is {tuple(g.shape)} on {g.device}, the parameter {tuple(p.shape)} on {dev}")
        st = _advance_state(st, p)
        r = self._rec
        r.param, r.grad, r.exp_avg, r.exp_avg_sq = p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()
        r.lr, r.step = lr, st["step"]
        _capi.call("sgr_cube_sparse_adam_step", dev, self._R, C.byref(r), blocks.data_ptr(), b1, b2, eps)
        return loss
