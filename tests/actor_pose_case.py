"""The tracklets, parameters and cameras of the actor-pose fixture (tests/golden/callsite/actor_pose.npz).

Four tracks over F = 40 frames on non-uniform float64 timestamps near 1.6e9 s (steps of 12/128, 13/128 or 14/128 s, so every
difference is exact and ties can be built):
  track 0  frames 0-39 but 16-17 (more than 32 entries); column 0 on even frames, 1 on odd ones; its quaternion is negated on odd frames (the
           same rotation, so a slerp between neighbours without opt_track takes the shortest-arc flip)
  track 1  frames 10-11 only (exactly 2 entries), column 2; under camera 0 it has one training timestamp in its span (the fallback of
           actor_pose.py:127)
  track 2  frames 5-25 but 16-17 (starts and ends mid-sequence), column 1 on even frames, 0 on odd ones (it swaps columns with track 0)
  track 3  frames 12-19, column 3
Camera 0 trains on the even frames, camera 1 on every third.  Frames 15-17 are equally spaced, so a camera on frame 16 ties for
the second-nearest entry of track 3, and one midway between frames 16 and 17 ties for its nearest.  Parameter sets: `seeded` (opt_rots 3.6 on track 3's rows: the slerp ends have a negative dot product;
0.01 on track 1's rows: a dot product within 5e-5 of 1) and `zero` (the state training starts in).
Ego rotations: each camera's ego rotation selects one of matrix_to_quaternion's four branches."""
import math

import numpy as np
import torch

F, K = 40, 4
BASE = 1.6e9


def timestamps():
    g = np.random.default_rng(5)
    steps = g.choice([12, 13, 14], size=F - 1).astype(np.float64) / 128.0
    steps[15] = steps[16] = 13 / 128.0  # frames 15, 16, 17 equally spaced
    return BASE + np.concatenate([[0.0], np.cumsum(steps)])


_GAP = (16, 17)  # tracks 0 and 2 have no entry there, so the ties at frames 16-17 involve track 3 alone
TRACKS = {  # track id -> (frames, column of frame f)
    0: ([f for f in range(0, 40) if f not in _GAP], lambda f: f % 2),
    1: ([10, 11], lambda f: 2),
    2: ([f for f in range(5, 26) if f not in _GAP], lambda f: 1 - f % 2),
    3: (list(range(12, 20)), lambda f: 3),
}


def _yaw_quat(yaw, tilt):
    q = np.array([math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2)])
    t = np.array([math.cos(tilt / 2), math.sin(tilt / 2), 0.0, 0.0])
    w1, x1, y1, z1 = q
    w2, x2, y2, z2 = t
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                     w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def metadata():
    ts = timestamps()
    tr = np.zeros((F, K, 8), np.float32)
    tr[..., 0] = -1.0
    tr[..., 4] = 1.0
    obj_meta = {}
    for tid, (frames, col) in TRACKS.items():
        for f in frames:
            yaw = 0.4 * tid + 0.03 * f + 0.002 * f * f
            q = _yaw_quat(yaw, 0.02 * math.sin(f + tid))
            if tid == 0 and f % 2:
                q = -q
            tr[f, col(f)] = [tid, -6.0 + 4.0 * tid + 1.1 * f + 0.03 * f * f, 0.3 + 0.1 * tid, 14.0 + 3.0 * tid - 0.2 * f, *q]
        obj_meta[tid] = dict(track_id=tid, **{"class": "vehicle"}, class_label=0, deformable=False, start_frame=frames[0], end_frame=frames[-1],
                             start_timestamp=float(ts[frames[0]]), end_timestamp=float(ts[frames[-1]]), length=4.5, width=2.0, height=1.6)
    cams = {0: dict(train_timestamps=[float(ts[f]) for f in range(0, F, 2)], test_timestamps=[]),
            1: dict(train_timestamps=[float(ts[f]) for f in range(0, F, 3)], test_timestamps=[])}
    return dict(obj_tracklets=tr, tracklet_timestamps=ts, camera_timestamps=cams, obj_meta=obj_meta)


def params():
    g = np.random.default_rng(17)
    ot = (0.1 * g.standard_normal((F, K, 3))).astype(np.float32)
    orr = (0.3 * g.standard_normal((F, K, 1))).astype(np.float32)
    orr[12:20, 3] = 3.6   # track 3: the slerp's ends q1 (x) 3.6 and q1 (x) 3.6 (x) 3.6 have dot product cos(3.6) < 0
    orr[10:12, 2] = 0.01  # track 1: dot product cos(0.01)
    return dict(seeded=(ot, orr), zero=(np.zeros_like(ot), np.zeros_like(orr)))


def _rot(axis, angle):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(angle) * Kx + (1 - math.cos(angle)) * Kx @ Kx


EGO = {  # matrix_to_quaternion picks the branch of the largest of 1 + m00 + m11 + m22, 1 + m00 - m11 - m22, ...
    "b0": (_rot([0.1, 0.2, 1.0], 0.4), [12.0, -3.0, 0.4]),
    "b1": (_rot([1.0, 0.1, 0.05], 2.8), [-4.0, 8.0, 1.1]),
    "b2": (_rot([0.1, 1.0, -0.1], 2.9), [30.5, 2.0, -0.6]),
    "b3": (_rot([0.05, -0.1, 1.0], 2.7), [-7.25, -15.0, 0.2]),
}


def ego_pose(name):
    R, t = EGO[name]
    e = np.eye(4, dtype=np.float32)
    e[:3, :3], e[:3, 3] = R, t
    return e


_TS = timestamps()
CASES = [
    dict(name="train_mid", frame=13, t=_TS[13] + 3 / 128, cam=0, is_val=False, ego="b0", opt_track=True, params="seeded"),
    dict(name="tie", frame=16, t=_TS[16], cam=1, is_val=False, ego="b1", opt_track=True, params="seeded"),
    dict(name="midway", frame=16, t=_TS[16] + 6.5 / 128, cam=0, is_val=False, ego="b3", opt_track=True, params="seeded"),
    dict(name="val", frame=11, t=_TS[11], cam=0, is_val=True, ego="b2", opt_track=True, params="seeded"),
    dict(name="val_between", frame=22, t=_TS[22] + 2 / 128, cam=1, is_val=True, ego="b3", opt_track=True, params="seeded"),
    dict(name="edge", frame=5, t=_TS[5] - 2 / 128, cam=0, is_val=False, ego="b0", opt_track=True, params="seeded"),
    dict(name="zero", frame=13, t=_TS[13] + 3 / 128, cam=0, is_val=False, ego="b1", opt_track=True, params="zero"),
    dict(name="no_opt", frame=13, t=_TS[13] + 5 / 128, cam=0, is_val=False, ego="b2", opt_track=False, params=None),
]
BY_NAME = {c["name"]: c for c in CASES}


def visible(case):
    """StreetGaussianModel.parse_camera's actors (street_gaussian_model.py:243-247): start_frame <= frame <= end_frame, in track order."""
    return [tid for tid, (frames, _) in TRACKS.items() if frames[0] <= case["frame"] <= frames[-1]]


def functional(case, n):
    """Weights w [n, 7] of the seeded linear functional sum(w * poses) whose gradient the fixture stores."""
    return np.random.default_rng(100 + CASES.index(case)).standard_normal((n, 7)).astype(np.float32)


def camera(ns, case, width=64, height=48):
    """A reference Camera (lib/utils/camera_utils.py) carrying the case's meta."""
    meta = dict(frame=case["frame"], frame_idx=case["frame"], is_val=case["is_val"], timestamp=float(case["t"]), cam=case["cam"],
                ego_pose=ego_pose(case["ego"]))
    return ns.camera_utils.Camera(id=0, R=np.eye(3), T=np.zeros(3), FoVx=1.0, FoVy=0.8, K=None, image=torch.zeros(3, height, width),
                                  image_name="synthetic", metadata=meta)
