"""Torch restatement of the reference's tracked actor poses (lib/models/actor_pose.py with the composition of
street_gaussian_model.py:257-265), used by tests/test_actor_pose_cpu.py and tests/test_actor_pose_gpu.py.

poses(...) runs the reference's torch lines one actor at a time, on whatever device its tensors are on:
  * dtype float32: the reference's fp32 ops in its order (timestamp differences in float64 rounded once to fp32, the slerp step
    through torch.tensor([r]).float(), the textbook slerp tests/refharness.py stands in for roma).  finite=False keeps the
    reference's where-based slerp, whose gradient is NaN where the slerp's ends coincide exactly; finite=True takes the small-angle
    branch's finite gradient there, as the kernels do.
  * dtype float64: the same lines in float64 with the timestamp factors unrounded and the finite small-angle gradient: the exact
    value the fp32 lines approximate, with per-element bounds from bounds().
tie="first" is the project's rule for equal distances (the earlier entry of the track); tie="last" is the other choice, for tests
that show which outputs depend on it.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as Fn

U32 = 2.0 ** -24  # unit roundoff of fp32


def nearest_two(values, t, tie="first"):
    d = np.abs(np.asarray(values, np.float64) - t)
    idx = np.arange(len(d))
    order = np.lexsort((idx if tie == "first" else -idx, d))
    return int(order[0]), int(order[1])


class Table:
    """argwhere entries per track (actor_pose.py:29-30) and the metadata the lookups need."""

    def __init__(self, tracklets, timestamps, camera_timestamps, obj_meta):
        ids = torch.from_numpy(np.asarray(tracklets, np.float32))[..., 0]
        self.ts = np.asarray(timestamps, np.float64)
        self.idx = {tid: torch.argwhere(ids == tid).numpy() for tid in obj_meta}
        self.meta = obj_meta
        self.cams = {c: np.asarray(v["train_timestamps"], np.float64) for c, v in camera_timestamps.items()}


def mul_theta(a, theta):  # general_utils.py:252-259
    aw, ax, ay, az = torch.unbind(a, -1)
    bw, bz = torch.cos(theta), torch.sin(theta)
    return torch.stack((aw * bw - az * bz, ax * bw + ay * bz, ay * bw - ax * bz, az * bw + aw * bz), -1)


def quat_mul(a, b):  # general_utils.py:232-238
    aw, ax, ay, az = torch.unbind(a, -1)
    bw, bx, by, bz = torch.unbind(b, -1)
    return torch.stack((aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                        aw * bz + ax * by - ay * bx + az * bw), -1)


def matrix_to_quaternion(m):  # general_utils.py:159-218, one [3, 3] matrix
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = torch.unbind(m.reshape(9), -1)
    x = torch.stack([1.0 + m00 + m11 + m22, 1.0 + m00 - m11 - m22, 1.0 - m00 + m11 - m22, 1.0 - m00 - m11 + m22])
    qa = torch.where(x > 0, torch.sqrt(torch.where(x > 0, x, torch.ones_like(x))), torch.zeros_like(x))
    rows = torch.stack([torch.stack([qa[0] ** 2, m21 - m12, m02 - m20, m10 - m01]), torch.stack([m21 - m12, qa[1] ** 2, m10 + m01, m02 + m20]),
                        torch.stack([m02 - m20, m10 + m01, qa[2] ** 2, m12 + m21]), torch.stack([m10 - m01, m20 + m02, m21 + m12, qa[3] ** 2])])
    k = int(torch.argmax(qa))
    return rows[k] / (2.0 * qa[k].clamp_min(0.1))


def slerp(q0, q1, step, finite, info=None):
    """quaternion_slerp (general_utils.py:277-303) over the harness's unitquat_slerp."""
    dt = q0.dtype
    q0 = Fn.normalize(q0.unsqueeze(0))[..., [1, 2, 3, 0]]
    q1 = Fn.normalize(q1.unsqueeze(0))[..., [1, 2, 3, 0]]
    t = torch.tensor([step], dtype=torch.float64, device=q0.device).to(dt).view(-1, 1, 1)
    d = (q0 * q1).sum(-1, keepdim=True)
    q1 = torch.where(d < 0, -q1, q1)
    d = d.abs().clamp(-1.0, 1.0)
    small = bool((torch.sin(torch.acos(d.detach())).abs() < 1e-6).all())
    if finite and small:
        w0, w1 = 1.0 - t, t
        theta = torch.zeros_like(d)
    else:
        theta = torch.acos(d)
        s = torch.sin(theta)
        sm = s.abs() < 1e-6
        w0 = torch.where(sm, 1.0 - t, torch.sin((1.0 - t) * theta) / torch.where(sm, torch.ones_like(s), s))
        w1 = torch.where(sm, t, torch.sin(t * theta) / torch.where(sm, torch.ones_like(s), s))
    if info is not None:
        info.append(float(torch.sin(theta.detach()).abs().min()))
    return (w0 * q0 + w1 * q1)[..., [3, 0, 1, 2]].reshape(4)


def _scal(x, dtype):
    """A float64 timestamp expression as the reference hands it to torch: rounded once to fp32 in the fp32 lines, kept in float64."""
    return float(np.float32(x)) if dtype == torch.float32 else float(x)


def _sub(T, tid, tq, in_t, in_r, ot, orr, opt, dtype, tie, finite, info):
    idx = T.idx[tid]
    i1, i2 = nearest_two(T.ts[idx[:, 0]], tq, tie)
    (f1, c1), (f2, c2) = idx[i1], idx[i2]
    t1, t2 = T.ts[f1], T.ts[f2]
    if opt:
        tr1, tr2 = in_t[f1, c1] + ot[f1, c1], in_t[f2, c2] + ot[f2, c2]
        r1 = mul_theta(in_r[f1, c1], orr[f1, c1, 0])
        r2 = mul_theta(r1, orr[f1, c2, 0])  # actor_pose.py:148-150: theta of (frame_ind1, column_ind2), rots1 twice
    else:
        tr1, tr2 = in_t[f1, c1], in_t[f2, c2]
        r1, r2 = in_r[f1, c1], in_r[f2, c2]
    trans = (tr1 * _scal(t2 - tq, dtype) + tr2 * _scal(tq - t1, dtype)) / _scal(t2 - t1, dtype)
    if info is not None:  # the size of the terms the interpolation adds: max |tr| (|a| + |b|) / |c|
        info.append(("terms", float(torch.stack([tr1, tr2]).detach().abs().max()) * (abs(t2 - tq) + abs(tq - t1)) / abs(t2 - t1)))
    rot = slerp(r1, r2, (tq - t1) / (t2 - t1), finite, info)
    if info is not None:
        info.append(("rows", (int(f1), int(c1)), (int(f2), int(c2)), (int(f1), int(c2))))
    return trans, rot


def actor(T, tid, t, cam, is_val, in_t, in_r, ot, orr, opt, dtype, tie="first", finite=True, info=None):
    """(rot [4], trans [3]) of get_tracking_rotation / get_tracking_translation (actor_pose.py:124-173) before the ego pose."""
    if opt and is_val:
        m = T.meta[tid]
        ct = T.cams[cam]
        inside = ct[(ct >= m["start_timestamp"]) & (ct <= m["end_timestamp"])]
        if len(inside) >= 2:
            j1, j2 = nearest_two(inside, t, tie)
            c1, c2 = inside[j1], inside[j2]
            ta, ra = _sub(T, tid, c1, in_t, in_r, ot, orr, opt, dtype, tie, finite, info)
            tb, rb = _sub(T, tid, c2, in_t, in_r, ot, orr, opt, dtype, tie, finite, info)
            trans = (ta * _scal(c2 - t, dtype) + tb * _scal(t - c1, dtype)) / _scal(c2 - c1, dtype)
            if info is not None:
                info.append(("outer", (abs(c2 - t) + abs(t - c1)) / abs(c2 - c1)))
            return slerp(ra, rb, (t - c1) / (c2 - c1), finite, info), trans
    tr, ro = _sub(T, tid, t, in_t, in_r, ot, orr, opt, dtype, tie, finite, info)
    return ro, tr


def poses(T, track_ids, t, cam, is_val, ego, input_trans, input_rots, opt_trans=None, opt_rots=None, dtype=torch.float32, tie="first", finite=True,
          info=None):
    """[n_act, 7] = (ego_q (x) rot, R_ego trans + t_ego) per actor (street_gaussian_model.py:260-265).  opt_trans [F, K, 3] /
    opt_rots [F, K, 1] are used as given (leaf tensors for autograd); None without opt_track."""
    opt = opt_trans is not None
    e = ego.to(dtype)
    eq = matrix_to_quaternion(e[:3, :3])
    out = []
    for tid in track_ids:
        rot, trans = actor(T, tid, t, cam, is_val, input_trans.to(dtype), input_rots.to(dtype), opt_trans, opt_rots, opt, dtype, tie, finite, info)
        out.append(torch.cat([quat_mul(eq, rot), e[:3, :3] @ trans + e[:3, 3]]))
    if not out:
        return torch.zeros((0, 7), dtype=dtype, device=ego.device)
    return torch.stack(out)


def idft_rows(T, track_ids, frame, C, scale):
    """IDFT(fourier_scale (frame - start) / (end - start), C)[0] per actor (sh_utils.py:120-130, gaussian_model_actor.py:71-77)."""
    rows = []
    for tid in track_ids:
        m = T.meta[tid]
        t = torch.tensor(scale * ((frame - m["start_frame"]) / (m["end_frame"] - m["start_frame"]))).view(-1, 1).float()
        r = torch.zeros(C)
        k = torch.arange(C)
        r[k[::2]] = torch.cos(torch.pi * t * k[::2])[0]
        r[k[1::2]] = torch.sin(torch.pi * t * (k[1::2] + 1))[0]
        rows.append(r)
    return torch.stack(rows) if rows else torch.zeros((0, C))


def bounds(T, track_ids, t, cam, is_val, ego, input_trans, input_rots, opt_trans, opt_rots, w):
    """The float64 value of the poses and of the gradients of sum(w * poses), with per-element bounds on what fp32 arithmetic gives.

    Values.  Every fp32 operation rounds with relative error <= u = 2^-24.  A translation element is a chain of at most 9 roundings
    (one offset add, three timestamp factors, two products, a sum, the scaling, then three products and three sums of the ego
    mat-vec; twice that many on the validation path), each acting on a term no larger than
        S_t = max_i sum_j |R_ij| max(|tr1|, |tr2|) (|a| + |b|) / |c| + |t_ego|,
    so |fp32 - exact| <= 2 * 18 u S_t with a factor 2 for the second-order terms (on the validation path S_t takes the outer
    interpolation's factor (|a'| + |b'|) / |c'| as well: its two terms can cancel).  A rotation element is a unit quaternion carried
    through two yaw products, two normalisations, the slerp (cos / sin / acos to 2 ulp) and the ego product, at most 40 roundings
    of quantities <= 1 in magnitude on the validation path, plus the slerp's angle: acos amplifies the error of the dot product
    d (<= 8 u) by 1 / sin(theta), and the weights move by at most |t (1 - t)| theta times that, which is <= 8 u as well; we take
    |fp32 - exact| <= 2 * 64 u.
    Gradients.  The gradient of one row sums <= 8 contributions per actor, each a product chain of the same depth through the
    transposed Jacobians; the slerp's angle term carries 1 / sin(theta) (the conditioning of acos), so a gradient element gets
        |fp32 - exact| <= 2 * 128 u (1 + 1 / s_min) G
    with G the largest |contribution| magnitude of the case (the largest |gradient element|, a lower bound of it, times the number of
    actors) and s_min the smallest sin(theta) of the case's slerps outside the small-angle branch."""
    F64 = torch.float64
    info = []
    ot = opt_trans.detach().to(F64).clone().requires_grad_(True) if opt_trans is not None else None
    orr = opt_rots.detach().to(F64).clone().requires_grad_(True) if opt_rots is not None else None
    p = poses(T, track_ids, t, cam, is_val, ego, input_trans, input_rots, ot, orr, dtype=F64, info=info)
    e = ego.to(F64)
    b = torch.zeros_like(p)
    b[:, :4] = 2 * 64 * U32
    for a, tid in enumerate(track_ids):  # S_t per actor: the largest interpolation term, times the outer factor on the validation path
        ia = []
        poses(T, [tid], t, cam, is_val, ego, input_trans, input_rots, opt_trans, opt_rots, dtype=F64, info=ia)
        terms = max(x[1] for x in ia if isinstance(x, tuple) and x[0] == "terms")
        outer = max([x[1] for x in ia if isinstance(x, tuple) and x[0] == "outer"] or [1.0])
        S = float(e[:3, :3].abs().sum(1).max()) * terms * outer + e[:3, 3].abs()
        b[a, 4:] = 2 * 18 * U32 * S
    out = dict(poses=p.detach(), b_poses=b)
    if ot is not None and len(track_ids):
        (p * w.to(F64)).sum().backward()
        s_min = min([x for x in info if isinstance(x, float) and x > 1e-6] or [1.0])
        for name, g in (("dtrans", ot.grad), ("drots", orr.grad)):
            G = float(g.abs().max()) * len(track_ids) + 1e-30
            out[name] = g.detach()
            out["b_" + name] = torch.full_like(g, 2 * 128 * U32 * (1 + 1 / s_min) * G)
    return out
