"""Host side of the scene-graph composer (SURVEY.md §8 row f1): the reference's StreetGaussianModel.get_xyz / get_rotation /
get_scaling / get_opacity / get_features (lib/models/street_gaussian_model.py:287-449) as ONE autograd.Function over
sgr_compose_forward / sgr_compose_backward (include/sgr.h).

    models : [background, actor_0, actor_1, ...] — each a mapping (or object) with the reference's raw parameters
             _xyz [n,3], _rotation [n,4], _scaling [n,3], _opacity [n,1], _features_dc [n,C,3], _features_rest [n,M-1,3]
             (lib/models/gaussian_model.py:41-47); the leading underscore is optional in mappings.
    poses  : [num_actors, 7] = (qw, qx, qy, qz, tx, ty, tz): the rows parse_camera expands into obj_rots / obj_trans (:258-273)
    idft   : [num_actors, C] IDFT(t, C) rows (lib/utils/sh_utils.py:120-130)
    flip   : optional bool [sum of actor counts] (the flip_mask of :275-284) with flip_quat [4] (the reference's flip_matrix)
    pose_correction : optional (rot [4], trans [3]), the caller's rows pose_correction_rots[id] / pose_correction_trans[id] of
             lib/models/camera_pose.py; the background is moved by them as correct_gaussian_xyz / correct_gaussian_rotation do
             (street_gaussian_model.py:311-312, 340-341).  None (the reference's 'test' mode) composes without a correction.

`compose(...)` returns (means3D, rotations, scales, opacities, shs) ready for GaussianRasterizer.forward; gradients flow to every
raw parameter, to `poses` and to the two correction rows.  PyTorch is plumbing (allocation, autograd bookkeeping); all arithmetic is in libsgr.so, and there
is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import _capi
from ._capi import ptr

RAW_KEYS = ("xyz", "rotation", "scaling", "opacity", "features_dc", "features_rest")


def _raw(model, key):
    if isinstance(model, dict):
        return model[key] if key in model else model["_" + key]
    return getattr(model, "_" + key)


class _Compose(torch.autograd.Function):
    @staticmethod
    def forward(ctx, poses, idft, flip, flip_quat, corr_rot, corr_trans, n_models, reduce, *raw):
        if not raw[0].is_cuda:
            raise _capi.SgrError("street_gaussians_b200 composer needs CUDA tensors (there is no CPU fallback)")
        dev = raw[0].device
        raw = tuple(_capi.f32(t) for t in raw)
        models = [raw[6 * k: 6 * k + 6] for k in range(n_models)]
        M = int(models[0][5].shape[1]) + 1
        nseg = n_models
        segs = (_capi.SgrSegment * nseg)()
        start = 0
        for k, m in enumerate(models):
            n, Cdim = int(m[0].shape[0]), int(m[4].shape[1])
            if Cdim > _capi.MAX_FOURIER:
                raise _capi.SgrError(f"fourier_dim {Cdim} exceeds SGR_MAX_FOURIER = {_capi.MAX_FOURIER}")
            s = segs[k]
            s.start, s.count, s.fourier_dim, s.posed = start, n, Cdim, int(k > 0)
            s.xyz, s.rotation, s.scaling, s.opacity, s.features_dc, s.features_rest = (t.data_ptr() if t.numel() else None for t in m)
            start += n
        P = start
        # per-segment pose / IDFT rows (row 0 = background, ignored by the kernels)
        pose_tab = torch.zeros((nseg, 8), device=dev, dtype=torch.float32)
        idft_tab = torch.zeros((nseg, _capi.MAX_FOURIER), device=dev, dtype=torch.float32)
        if nseg > 1:
            pose_tab[1:, :7] = poses.to(device=dev, dtype=torch.float32)
            idft_tab[1:, : idft.shape[1]] = idft.to(device=dev, dtype=torch.float32)
        flip_full = None
        if flip is not None and nseg > 1:
            flip_full = torch.zeros((P,), device=dev, dtype=torch.uint8)
            flip_full[int(models[0][0].shape[0]):] = flip.to(device=dev, dtype=torch.uint8)
            flip_quat = _capi.f32(flip_quat.reshape(4), dev)
        corr = None
        if corr_rot is not None:
            corr = torch.zeros((8,), device=dev, dtype=torch.float32)
            corr[:4] = corr_rot.reshape(4).to(device=dev, dtype=torch.float32)
            corr[4:7] = corr_trans.reshape(3).to(device=dev, dtype=torch.float32)
        e = lambda *shape: torch.empty(shape, device=dev, dtype=torch.float32)
        xyz, rot, scale, opac, sh = e(P, 3), e(P, 4), e(P, 3), e(P, 1), e(P, M, 3)
        fq = ptr(flip_quat) if flip_full is not None else None
        if corr is None:
            _capi.call("sgr_compose_forward", dev, segs, nseg, M, ptr(pose_tab), ptr(idft_tab), ptr(flip_full), fq, ptr(xyz), ptr(rot),
                       ptr(scale), ptr(opac), ptr(sh))
        else:
            _capi.call("sgr_compose_forward_corrected", dev, segs, nseg, M, ptr(pose_tab), ptr(idft_tab), ptr(flip_full), fq, ptr(corr),
                       ptr(xyz), ptr(rot), ptr(scale), ptr(opac), ptr(sh))
        ctx.segs, ctx.nseg, ctx.M, ctx.n_models = segs, nseg, M, n_models
        ctx.flip_full, ctx.flip_quat = flip_full, (flip_quat if flip_full is not None else None)
        ctx.pose_shape = None if poses is None else (tuple(poses.shape), poses.dtype, poses.device)
        ctx.corr_meta = None if corr is None else ((tuple(corr_rot.shape), corr_rot.dtype, corr_rot.device),
                                                   (tuple(corr_trans.shape), corr_trans.dtype, corr_trans.device))
        ctx.corr, ctx.reduce = corr, reduce
        ctx.save_for_backward(pose_tab, idft_tab, *raw)
        return xyz, rot, scale, opac, sh

    @staticmethod
    def backward(ctx, g_xyz, g_rot, g_scale, g_opac, g_sh):
        pose_tab, idft_tab, *raw = ctx.saved_tensors
        dev = pose_tab.device
        nseg, M = ctx.nseg, ctx.M
        P = sum(int(raw[6 * k].shape[0]) for k in range(nseg))
        z = lambda g, *shape: _capi.f32(g) if g is not None else torch.zeros(shape, device=dev, dtype=torch.float32)
        g_xyz, g_rot, g_scale, g_opac, g_sh = z(g_xyz, P, 3), z(g_rot, P, 4), z(g_scale, P, 3), z(g_opac, P, 1), z(g_sh, P, M, 3)
        grads = [torch.empty_like(t) for t in raw]
        gtab = (_capi.SgrSegmentGrads * nseg)()
        for k in range(nseg):
            g = gtab[k]
            g.xyz, g.rotation, g.scaling, g.opacity, g.features_dc, g.features_rest = (t.data_ptr() if t.numel() else None for t in grads[6 * k: 6 * k + 6])
        dposes = torch.empty((nseg, 8), device=dev, dtype=torch.float32)
        corr = ctx.corr
        dcorr = None if corr is None else torch.empty((8,), device=dev, dtype=torch.float32)
        if ctx.reduce is not None:
            _backward_rows_reduced(ctx.reduce, dev, ctx.segs, gtab, nseg, M, pose_tab, idft_tab, ctx.flip_full, ctx.flip_quat, corr,
                                   (g_xyz, g_rot, g_scale, g_opac, g_sh), dposes, dcorr)
        elif corr is None:
            scratch = torch.empty((nseg, 16), device=dev, dtype=torch.float32)
            _capi.call("sgr_compose_backward", dev, ctx.segs, gtab, nseg, M, ptr(pose_tab), ptr(idft_tab), ptr(ctx.flip_full), ptr(ctx.flip_quat),
                       ptr(g_xyz), ptr(g_rot), ptr(g_scale), ptr(g_opac), ptr(g_sh), ptr(dposes), ptr(scratch))
        else:
            scratch = torch.empty((nseg + 1, 16), device=dev, dtype=torch.float32)
            _capi.call("sgr_compose_backward_corrected", dev, ctx.segs, gtab, nseg, M, ptr(pose_tab), ptr(idft_tab), ptr(ctx.flip_full),
                       ptr(ctx.flip_quat), ptr(corr), ptr(g_xyz), ptr(g_rot), ptr(g_scale), ptr(g_opac), ptr(g_sh), ptr(dposes), ptr(dcorr),
                       ptr(scratch))
        g_poses = g_crot = g_ctrans = None
        if ctx.pose_shape is not None:
            shape, dtype, device = ctx.pose_shape
            g_poses = dposes[1:, :7].to(device=device, dtype=dtype).reshape(shape)
        if corr is not None:
            (rs, rd, rdev), (ts, td, tdev) = ctx.corr_meta
            g_crot, g_ctrans = dcorr[:4].to(device=rdev, dtype=rd).reshape(rs), dcorr[4:7].to(device=tdev, dtype=td).reshape(ts)
        return (g_poses, None, None, None, g_crot, g_ctrans, None, None) + tuple(grads)


def _backward_rows_reduced(reduce, dev, segs, gtab, nseg, M, pose_tab, idft_tab, flip_full, flip_quat, corr, upstream, dposes, dcorr):
    """The backward of one rank's rows under Gaussian sharding: its per-row gradients and accumulator rows, the rows summed over the
    ranks (COLLECTIVE), then dposes / dcorr finalized from the frame's sums, the same bytes on every rank."""
    L = _capi.lib()
    acc = torch.empty((int(L.sgr_compose_pose_rows(nseg, int(corr is not None))), 16), device=dev, dtype=torch.float32)
    _capi.call("sgr_compose_backward_rows", dev, segs, gtab, nseg, M, ptr(pose_tab), ptr(idft_tab), ptr(flip_full), ptr(flip_quat), ptr(corr),
               *(ptr(g) for g in upstream), ptr(acc), acc.numel() * 4)
    kind, arg = reduce
    if kind == "p2p":  # over the rasterizer's peer workspace: stage, barrier, sum in rank order, barrier per group of rows, then finalize
        ws = arg.pose_workspace()
        ws.next_epochs(2 * ((acc.shape[0] + _capi.POSE_ACC_ROWS - 1) // _capi.POSE_ACC_ROWS))
        _capi.call("sgr_compose_pose_reduce_peers", dev, C.byref(ws.peers), segs, nseg, ptr(pose_tab), ptr(corr), ptr(acc), acc.numel() * 4,
                   ptr(dposes), ptr(dcorr))
    else:
        from .band_losses import all_reduce_sum
        all_reduce_sum(acc, arg)
        _capi.call("sgr_compose_pose_finalize", dev, segs, nseg, ptr(pose_tab), ptr(corr), ptr(acc), acc.numel() * 4, ptr(dposes), ptr(dcorr))


def _reduction(group, rasterizer):
    """(kind, what) of the sum over the ranks, or None for the single-GPU call."""
    if rasterizer is None and group is None:
        return None
    if rasterizer is not None:
        if group is not None and group is not rasterizer.group:
            raise ValueError("compose: group= differs from the rasterizer's group")
        if rasterizer.exchange == "p2p":
            return ("p2p", rasterizer)
        group = rasterizer.group
    return ("nccl", group)


def compose(models: Sequence, poses: Optional[torch.Tensor] = None, idft: Optional[torch.Tensor] = None,
            flip: Optional[torch.Tensor] = None, flip_quat: Optional[torch.Tensor] = None, *,
            pose_correction: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, group=None, rasterizer=None):
    """-> (means3D[P,3], rotations[P,4], scales[P,3], opacities[P,1], shs[P,M,3]) of background + actors, differentiable.
    pose_correction = (rot [4], trans [3]) moves the background by the learned per-image correction; gradients return to both.

    group= / rasterizer= (Gaussian sharding, sharded.GaussianShardedRasterizer): `models` hold this rank's rows of every sub-model (any
    of them may have 0 rows, as sharded.rebalance can leave them) while poses, idft and pose_correction are the frame's, the same on every
    rank.  The composed rows are the single-GPU call's rows bit for bit.  COLLECTIVE in the backward: the per-segment pose and correction
    sums of every rank's rows are added before they become dL/dposes and dL/dcorrection, so those are the frame's gradients and the same
    bytes on every rank (up to the order of fp32 additions, they are the single-GPU call's), and replicated pose parameters step alike.
    rasterizer= with exchange="p2p" sums over its peer workspace, in ascending rank order, with device-side barriers and no NCCL call;
    otherwise (exchange="nccl", or group= alone) one all_reduce over the group.  None for both keeps the single-GPU call."""
    raw = [_raw(m, k) for m in models for k in RAW_KEYS]
    n_act = len(models) - 1
    if n_act > 0:
        if poses is None or tuple(poses.shape) != (n_act, 7):
            raise ValueError(f"poses must be [{n_act}, 7] (qw, qx, qy, qz, tx, ty, tz per actor)")
        if idft is None or idft.shape[0] != n_act:
            raise ValueError(f"idft must be [{n_act}, fourier_dim]")
    if flip is not None and flip_quat is None:
        raise ValueError("flip mask given without flip_quat (the reference's flip_matrix)")
    corr_rot = corr_trans = None
    if pose_correction is not None:
        corr_rot, corr_trans = pose_correction
        if corr_rot.numel() != 4 or corr_trans.numel() != 3:
            raise ValueError("pose_correction must be (rot [4] = qw, qx, qy, qz; trans [3])")
    return _Compose.apply(poses, idft, flip, flip_quat, corr_rot, corr_trans, len(models), _reduction(group, rasterizer), *raw)
