"""The renderer's feature channels (lib/models/street_gaussian_renderer.py:206-264: cfg.render.render_normal and cfg.data.use_semantic)
over the sgr_gaussian_normals_*, sgr_compose_semantics_* and sgr_finish_features_* entries (include/sgr.h).

    gaussian_normals(means3D, rotations, scales, camera_center)  -> normals [P, 3]
        GaussianModel.get_normals (gaussian_model.py:256-269) on the composed rows compose(...) returns: the column of
        quaternion_to_matrix(rotation) at argmin(scales), turned to face the camera.  Actor rows are their posed (and flipped) world
        rows and a pose-corrected background its corrected rows (DESIGN.md §2).  Differentiable in `rotations` only.
    compose_semantics(models, class_labels, mode)                 -> semantics [P, K]
        StreetGaussianModel.get_semantic (street_gaussian_model.py:417-431) over the [background, actor_0, ...] list compose takes.
    finish_features(rendered, normal_channels, semantic_mode)    -> (normals [3, H, W] or None, semantic [K, H, W] or None)
        the split, F.normalize and the probabilities' log of render_kernel (street_gaussian_renderer.py:245-264); with band= on the
        rows of a rank's TileRowBand only (sgr_band_finish_features_*).

The feature tensor the rasterizer takes is torch.cat([normals, semantics], -1) ([P, 3 + K]; training needs 3 + K <= 32).  CUDA tensors
only: there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import _capi
from ._capi import ptr
from .composer import _raw

MODES = {"logits": _capi.SEMANTIC_LOGITS, "probabilities": _capi.SEMANTIC_PROBABILITIES}


def _mode(mode: str) -> int:
    if mode not in MODES:
        raise ValueError(f"semantic mode must be 'logits' or 'probabilities', got {mode!r}")
    return MODES[mode]


def _cuda_f32(what: str, named: dict, device=None):
    for name, t in named.items():
        if t.dtype != torch.float32:
            raise ValueError(f"{name} must be float32, got {t.dtype}")
    for name, t in named.items():
        if not t.is_cuda:
            raise _capi.SgrError(f"street_gaussians_b200.{what} needs CUDA tensors ({name} is on {t.device}; there is no CPU fallback)")
        if device is not None and t.device != device:
            raise ValueError(f"{name} is on {t.device}, expected {device}")


class _GaussianNormals(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, rotations, scales, camera_center):
        P = int(means3D.shape[0])
        dev = means3D.device
        m, r, s, c = means3D.contiguous(), _capi.f32(rotations, align16=True), scales.contiguous(), camera_center.reshape(3).contiguous()
        normals = torch.empty((P, 3), device=dev, dtype=torch.float32)
        decision = torch.empty((P,), device=dev, dtype=torch.uint8)
        _capi.call("sgr_gaussian_normals_forward", dev, P, ptr(m), ptr(r), ptr(s), ptr(c), ptr(normals), ptr(decision))
        ctx.save_for_backward(r, decision)
        return normals

    @staticmethod
    def backward(ctx, g_normals):
        r, decision = ctx.saved_tensors
        if g_normals is None or not ctx.needs_input_grad[1]:
            return None, None, None, None
        dev = r.device
        g = g_normals.contiguous()
        g_rot = torch.empty_like(r)
        _capi.call("sgr_gaussian_normals_backward", dev, int(r.shape[0]), ptr(r), ptr(decision), ptr(g), ptr(g_rot))
        return None, g_rot, None, None


def gaussian_normals(means3D: torch.Tensor, rotations: torch.Tensor, scales: torch.Tensor, camera_center: torch.Tensor) -> torch.Tensor:
    """-> normals [P, 3]: column argmin(scales) (lowest index on ties) of quaternion_to_matrix(rotations), negated where it faces away
    from camera_center [3] (sum(-d n) < 0 or NaN, d the unit direction from the camera to the Gaussian).  means3D / scales [P, 3],
    rotations [P, 4], fp32 CUDA.  The gradient reaches `rotations` only; the column and the sign are the forward's."""
    P = int(means3D.shape[0]) if means3D.dim() == 2 else -1
    if means3D.dim() != 2 or means3D.shape[1] != 3:
        raise ValueError(f"means3D must be [P, 3], got {tuple(means3D.shape)}")
    if tuple(rotations.shape) != (P, 4) or tuple(scales.shape) != (P, 3):
        raise ValueError(f"rotations must be [{P}, 4] and scales [{P}, 3], got {tuple(rotations.shape)} and {tuple(scales.shape)}")
    if camera_center.numel() != 3:
        raise ValueError(f"camera_center must have 3 elements, got {tuple(camera_center.shape)}")
    _cuda_f32("gaussian_normals", dict(means3D=means3D, rotations=rotations, scales=scales, camera_center=camera_center), means3D.device)
    return _GaussianNormals.apply(means3D, rotations, scales, camera_center)


class _ComposeSemantics(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mode: int, labels: Tuple[int, ...], bg, *actors):
        dev = bg.device
        K = int(bg.shape[1])
        n_bg, n_act = int(bg.shape[0]), len(actors)
        bg_c = bg.contiguous()
        act_c = [a.contiguous() for a in actors]
        counts = (C.c_int32 * max(n_act, 1))(*[int(a.shape[0]) for a in act_c])
        lab = (C.c_int32 * max(n_act, 1))(*labels)
        ptrs = (C.c_void_p * max(n_act, 1))(*[a.data_ptr() if a.numel() else None for a in act_c])
        P = n_bg + sum(int(a.shape[0]) for a in act_c)
        out = torch.empty((P, K), device=dev, dtype=torch.float32)
        _capi.call("sgr_compose_semantics_forward", dev, K, mode, n_bg, ptr(bg_c), n_act, counts, lab, ptrs, ptr(out))
        ctx.args = (mode, K, n_bg, n_act, counts, lab, [tuple(a.shape) for a in act_c])
        ctx.save_for_backward(out)
        return out

    @staticmethod
    def backward(ctx, g_out):
        (out,) = ctx.saved_tensors
        mode, K, n_bg, n_act, counts, lab, shapes = ctx.args
        dev = out.device
        g = g_out.contiguous()
        need_bg = ctx.needs_input_grad[2]
        need_act = any(ctx.needs_input_grad[3:])
        g_bg = torch.empty((n_bg, K), device=dev, dtype=torch.float32) if need_bg else None
        g_act = [torch.empty(s, device=dev, dtype=torch.float32) for s in shapes] if need_act else None
        gptrs = (C.c_void_p * max(n_act, 1))(*[t.data_ptr() if t.numel() else None for t in g_act]) if need_act else None
        _capi.call("sgr_compose_semantics_backward", dev, K, mode, n_bg, n_act, counts, lab, ptr(out), ptr(g), ptr(g_bg), gptrs)
        return (None, None, g_bg) + (tuple(g_act) if need_act else (None,) * n_act)


def compose_semantics(models: Sequence, class_labels: Sequence[int] = (), mode: str = "logits") -> torch.Tensor:
    """-> semantics [P, K] in compose's row order: the background's _semantic [n_bg, K] ('logits') or its row softmax
    ('probabilities'), then per actor zeros with column class_labels[a] = its _semantic [n_a, 1] or the sigmoid of it.  Gradients reach
    every model's _semantic.  fp32 CUDA tensors."""
    m = _mode(mode)
    sems = [_raw(x, "semantic") for x in models]
    bg, actors = sems[0], sems[1:]
    labels = tuple(int(v) for v in class_labels)
    if bg.dim() != 2 or bg.shape[1] < 1:
        raise ValueError(f"the background's _semantic must be [n_bg, K] with K >= 1, got {tuple(bg.shape)}")
    K = int(bg.shape[1])
    if len(labels) != len(actors):
        raise ValueError(f"{len(actors)} actors but {len(labels)} class labels")
    for a, (s, lab) in enumerate(zip(actors, labels)):
        if s.dim() != 2 or s.shape[1] != 1:
            raise ValueError(f"actor {a}'s _semantic must be [n, 1], got {tuple(s.shape)}")
        if not 0 <= lab < K:
            raise ValueError(f"class label {lab} of actor {a} is outside [0, {K})")
    _cuda_f32("compose_semantics", {("background _semantic" if k == 0 else f"actor {k - 1} _semantic"): s for k, s in enumerate(sems)}, bg.device)
    return _ComposeSemantics.apply(m, labels, *sems)


class _FinishFeatures(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rendered, nc: int, mode: int, rows: Optional[Tuple[int, int, int]]):
        ctx.set_materialize_grads(False)
        S, H, W = (int(v) for v in rendered.shape)
        dev = rendered.device
        x = rendered.contiguous()
        new = torch.empty if rows is None else torch.zeros  # a band writes its rows only
        normals = new((nc, H, W), device=dev, dtype=torch.float32)
        semantic = new((S - nc, H, W), device=dev, dtype=torch.float32)
        if rows is None:
            _capi.call("sgr_finish_features_forward", dev, S, H, W, nc, mode, ptr(x), ptr(normals), ptr(semantic))
        else:
            _capi.call("sgr_band_finish_features_forward", dev, S, H, W, nc, mode, *rows, ptr(x), ptr(normals), ptr(semantic))
        ctx.save_for_backward(x)
        ctx.args = (S, H, W, nc, mode, rows)
        return normals, semantic

    @staticmethod
    def backward(ctx, g_normals, g_semantic):
        (x,) = ctx.saved_tensors
        S, H, W, nc, mode, rows = ctx.args
        dev = x.device
        gn = g_normals.contiguous() if g_normals is not None else None
        gs = g_semantic.contiguous() if g_semantic is not None else None
        if rows is None:
            g = torch.empty_like(x)
            _capi.call("sgr_finish_features_backward", dev, S, H, W, nc, mode, ptr(x), ptr(gn), ptr(gs), ptr(g))
        else:
            g = torch.zeros_like(x)
            _capi.call("sgr_band_finish_features_backward", dev, S, H, W, nc, mode, *rows, ptr(x), ptr(gn), ptr(gs), ptr(g))
        return g, None, None, None


def finish_features(rendered: torch.Tensor, normal_channels: int, semantic_mode: str = "logits", *, band=None
                    ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """rendered [S, H, W] (the rasterizer's feature image: normal_channels = 3 normal channels first, or 0, then the semantics)
    -> (normals [3, H, W] = per-pixel F.normalize, or None; semantic [S - normal_channels, H, W], or None): the semantic channels
    as they are ('logits') or log(x / (sum_c x + 1e-8) + 1e-8) ('probabilities').  Differentiable in `rendered`.

    band= (keyword-only, a TileRowBand of sharded.py): rendered holds the rendered rows of this rank's band, as a sharded rasterizer
    returns them.  The outputs and dL/drendered have the band's rows, zeros elsewhere, equal bit for bit to the whole-frame call's
    rows.  The operation is per pixel, so no collective is needed and the ranks' results summed are the whole frame's."""
    nc = int(normal_channels)
    if nc not in (0, 3):
        raise ValueError(f"normal_channels must be 0 or 3, got {normal_channels}")
    m = _mode(semantic_mode)
    if rendered.dim() != 3 or rendered.shape[0] < max(nc, 1) or rendered.shape[1] < 1 or rendered.shape[2] < 1:
        raise ValueError(f"rendered must be [S, H, W] with S >= max(normal_channels, 1), got {tuple(rendered.shape)}")
    rows = None
    if band is not None:  # a bad band fails before anything is launched
        from .band_losses import check_band
        rows = check_band(band, int(rendered.shape[1]))
    _cuda_f32("finish_features", dict(rendered=rendered))
    normals, semantic = _FinishFeatures.apply(rendered, nc, m, rows)
    return (normals if nc else None), (semantic if semantic.shape[0] else None)
