"""The tracked actor poses of the reference (lib/models/actor_pose.py, ActorPose, with model.nsg.opt_track) as
StreetGaussianModel.parse_camera composes them with the ego pose (street_gaussian_model.py:257-271), over sgr_actor_pose_forward /
sgr_actor_pose_backward (include/sgr.h).

    pose = ActorPose(obj_tracklets, tracklet_timestamps, camera_timestamps, obj_meta, fourier_dim=C)   # the reference's metadata
    poses, idft = pose(track_ids, timestamp=..., cam=..., is_val=..., ego_pose=..., frame=...)
    compose(models, poses, idft)

`poses` [n_act, 7] = (qw, qx, qy, qz, tx, ty, tz) per visible actor, differentiable in the parameters `opt_trans` [F, K, 3] and
`opt_rots` [F, K, 1] (the reference's names, so the `actor_pose['params']` of a reference checkpoint loads with load_state_dict);
`idft` [n_act, C] are the IDFT rows of gaussian_model_actor.py:71-77 at `frame`, or None without `frame`.  The track table lives on the
device from construction on; a call copies nothing and reads nothing back.  CUDA only: there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Mapping, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import _capi
from ._capi import ptr


def track_table(tracklets, tracklet_timestamps, camera_timestamps, obj_meta) -> dict:
    """Host arrays of the device track table.  A track's entries are np.argwhere(track_ids == track_id) of the [F, K] id plane in the
    reference's order (actor_pose.py:14, 29-30), each with its frame's tracklet timestamp in float64; cameras keep their training
    timestamps in the order given (actor_pose.py:96)."""
    tracklets = np.asarray(tracklets)
    ids = torch.from_numpy(tracklets).float()[..., 0].numpy()  # actor_pose.py:13-14 compares in float32
    ts = np.asarray(tracklet_timestamps, dtype=np.float64)
    track_ids, off, fc, ets, span, frames = [], [0], [], [], [], []
    for tid, meta in obj_meta.items():
        idx = np.argwhere(ids == tid).astype(np.int32).reshape(-1, 2)
        track_ids.append(tid)
        fc.append(idx)
        ets.append(ts[idx[:, 0]])
        off.append(off[-1] + len(idx))
        span.append((float(meta["start_timestamp"]), float(meta["end_timestamp"])))
        frames.append((int(meta["start_frame"]), int(meta["end_frame"])))
    cams = list((camera_timestamps or {}).keys())
    cam_off, cam_ts = [0], []
    for c in cams:
        t = np.asarray(camera_timestamps[c]["train_timestamps"], dtype=np.float64).reshape(-1)
        cam_ts.append(t)
        cam_off.append(cam_off[-1] + len(t))
    cat = lambda xs, dt, shape: np.concatenate(xs).astype(dt) if xs else np.zeros(shape, dt)
    return dict(track_ids=track_ids, cams=cams, counts=np.diff(off), track_off=np.asarray(off, np.int32),
                entry_fc=cat(fc, np.int32, (0, 2)).reshape(-1, 2), entry_ts=cat(ets, np.float64, (0,)),
                track_span=np.asarray(span, np.float64).reshape(-1, 2), track_frames=np.asarray(frames, np.int32).reshape(-1, 2),
                cam_off=np.asarray(cam_off, np.int32), cam_ts=cat(cam_ts, np.float64, (0,)))


class _PoseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, opt_trans, opt_rots, module, slots, timestamp, cam, is_val, ego, frame):
        n = len(slots)
        slots = slots if n else None
        dev = module.input_trans.device
        poses = torch.empty((n, 7), device=dev, dtype=torch.float32)
        idft = torch.empty((n, module.fourier_dim), device=dev, dtype=torch.float32) if frame is not None else None
        opt = opt_trans is not None
        _capi.call("sgr_actor_pose_forward", dev, *module._table_args(), n, slots, timestamp, cam, int(is_val), ptr(ego),
                   ptr(opt_trans) if opt else None, ptr(opt_rots) if opt else None, int(frame or 0), module.fourier_scale,
                   module.fourier_dim, ptr(poses), ptr(idft))
        ctx.module, ctx.args = module, (n, slots, timestamp, cam, is_val)
        if opt:
            ctx.save_for_backward(opt_trans, opt_rots, ego)
        if idft is not None:
            ctx.mark_non_differentiable(idft)
        return poses, idft

    @staticmethod
    def backward(ctx, g_poses, g_idft):
        L = _capi.lib()
        opt_trans, opt_rots, ego = ctx.saved_tensors
        n, slots, timestamp, cam, is_val = ctx.args
        dev = opt_trans.device
        g_trans, g_rots = torch.zeros_like(opt_trans), torch.zeros_like(opt_rots)
        if n and g_poses is not None:
            g = _capi.f32(g_poses)
            nbytes = int(L.sgr_actor_pose_scratch_bytes(n))
            scratch = torch.empty((nbytes,), device=dev, dtype=torch.uint8)
            _capi.call("sgr_actor_pose_backward", dev, *ctx.module._table_args(), n, slots, timestamp, cam, int(is_val), ptr(ego), ptr(opt_trans),
                       ptr(opt_rots), ptr(g), ptr(g_trans), ptr(g_rots), ptr(scratch), nbytes)
        return g_trans, g_rots, None, None, None, None, None, None, None


class ActorPose(nn.Module):
    """The reference's ActorPose (tracklets [F, K, 8] = track_id, x, y, z, qw, qx, qy, qz) with the pose composition of parse_camera.
    opt_track: learn opt_trans / opt_rots (model.nsg.opt_track, true in every shipped config).  fourier_dim / fourier_scale:
    model.gaussian.fourier_dim / fourier_scale, for the IDFT rows."""

    def __init__(self, tracklets, tracklet_timestamps, camera_timestamps, obj_meta: Mapping, *, opt_track: bool = True, fourier_dim: int = 1,
                 fourier_scale: float = 1.0, device="cuda"):
        super().__init__()
        device = torch.device(device)
        if device.type != "cuda":
            raise _capi.SgrError(f"street_gaussians_b200.ActorPose needs a CUDA device (got {device}; there is no CPU fallback)")
        if not 1 <= int(fourier_dim) <= _capi.MAX_FOURIER:
            raise ValueError(f"fourier_dim must be in [1, {_capi.MAX_FOURIER}], got {fourier_dim}")
        tracklets = np.asarray(tracklets, dtype=np.float32)
        if tracklets.ndim != 3 or tracklets.shape[2] != 8:
            raise ValueError(f"tracklets must be [num_frames, max_obj, 8], got {tracklets.shape}")
        tab = track_table(tracklets, tracklet_timestamps, camera_timestamps, obj_meta)
        self.opt_track, self.fourier_dim, self.fourier_scale = bool(opt_track), int(fourier_dim), float(fourier_scale)
        self.num_frames, self.max_obj = int(tracklets.shape[0]), int(tracklets.shape[1])
        self._slot = {tid: k for k, tid in enumerate(tab["track_ids"])}
        self._cam = {c: k for k, c in enumerate(tab["cams"])}
        self._counts = [int(c) for c in tab["counts"]]
        self._frames = [tuple(int(x) for x in f) for f in tab["track_frames"]]
        t = torch.from_numpy(tracklets).to(device)
        self.register_buffer("input_trans", t[..., 1:4].contiguous(), persistent=False)
        self.register_buffer("input_rots", t[..., 4:8].contiguous(), persistent=False)
        for k in ("track_off", "entry_fc", "entry_ts", "track_span", "track_frames", "cam_off", "cam_ts"):
            self.register_buffer("_" + k, torch.from_numpy(np.ascontiguousarray(tab[k])).to(device), persistent=False)
        if self.opt_track:
            self.opt_trans = nn.Parameter(torch.zeros_like(self.input_trans))
            self.opt_rots = nn.Parameter(torch.zeros_like(self.input_rots[..., :1]))

    def _table_args(self):
        return (len(self._counts), self.max_obj, ptr(self._track_off), ptr(self._entry_fc), ptr(self._entry_ts), ptr(self._track_span),
                ptr(self._track_frames), len(self._cam), ptr(self._cam_off), ptr(self._cam_ts), ptr(self.input_trans), ptr(self.input_rots))

    def forward(self, track_ids: Sequence, timestamp: float, cam=0, is_val: bool = False, ego_pose: Optional[torch.Tensor] = None,
                frame: Optional[int] = None):
        """-> (poses [n_act, 7], idft [n_act, fourier_dim] or None) for the visible actors `track_ids` (the reference's track ids, in
        the order compose takes them) on a camera with meta timestamp / cam / is_val and ego_pose [4, 4] (identity when None); idft at
        meta frame `frame`.  The validation path (is_val) applies with opt_track only, as in the reference."""
        dev = self.input_trans.device
        slots = []
        for tid in track_ids:
            if tid not in self._slot:
                raise KeyError(f"track id {tid} is not in obj_meta")
            s = self._slot[tid]
            if self._counts[s] < 2:  # actor_pose.py:87
                raise ValueError(f"track {tid} has {self._counts[s]} tracklet entries; interpolation needs at least 2")
            if frame is not None and self._frames[s][0] == self._frames[s][1]:
                raise ZeroDivisionError(f"track {tid} starts and ends on frame {self._frames[s][0]}: its IDFT time is undefined")
            slots.append(s)
        val = bool(is_val) and self.opt_track
        c = 0
        if val:
            if cam not in self._cam:
                raise KeyError(f"camera {cam} has no training timestamps in camera_timestamps")
            c = self._cam[cam]
        if ego_pose is None:
            ego_pose = torch.eye(4, device=dev)
        if tuple(ego_pose.shape) != (4, 4):
            raise ValueError(f"ego_pose must be [4, 4], got {tuple(ego_pose.shape)}")
        if ego_pose.device != dev:
            raise ValueError(f"ego_pose is on {ego_pose.device}, the track table on {dev}")
        ego = _capi.f32(ego_pose.detach())
        arr = (C.c_int32 * len(slots))(*slots)
        ot, orr = (self.opt_trans, self.opt_rots) if self.opt_track else (None, None)
        return _PoseFn.apply(ot, orr, self, arr, float(timestamp), c, val, ego, frame)
