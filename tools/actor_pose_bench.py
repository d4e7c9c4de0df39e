"""Times the tracked actor poses, forward + backward, with 8 and with 40 visible actors on a training camera.  Arms, alternating call
by call in one process, median and p10-p90 of STEPS after WARMUP, each call ending in a device synchronise:
  fused           street_gaussians_b200.ActorPose: one kernel forward, two backward, no host synchronisation
  reference_lines the reference's torch lines as they run (lib/models/actor_pose.py, parse_camera's composition): the track's
                  argwhere rows on the device brought to the host with .cpu() and ranked by np.argsort, the tracklet timestamps
                  indexed with .cpu() indices, rotation and translation looked up separately, one small torch op at a time, and
                  matrix_to_quaternion of the ego pose redone per actor; the slerp is the textbook one the tests stand in for roma
Reported per arm: host wall time per call and CUDA-event time per call; then the device time per call of each kernel of the fused
arm from a separately profiled run, and the host time of the fused call's pieces (forward, backward, and inside the forward the table
arguments and the bare ctypes call); then the composed training step at config C (poses -> compose -> rasterize -> photometric_loss
-> backward -> FusedAdam over the Gaussians and the pose offsets) with each arm training its own copy of the Gaussians from the same
non-zero offsets, alternating; after the timed loop every step's loss and poses are checked to be finite.  Prints one JSON line with
the GPU name and its enforced power limit.
python tools/actor_pose_bench.py"""
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import actor_pose_oracle as AO  # noqa: E402
from loss_bench import power_limit_w  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import losses, synthetic  # noqa: E402
from street_gaussians_b200.training import FusedAdam  # noqa: E402

DEV = "cuda"
STEPS, WARMUP = int(os.environ.get("STEPS", 80)), int(os.environ.get("WARMUP", 10))
KERNELS = ("actor_pose_fwd_kernel", "actor_pose_bwd_kernel", "actor_pose_accum_kernel")


class ReferenceLines(torch.nn.Module):
    """The reference's per-actor lookups as it runs them, host round trips included."""

    def __init__(self, tracklets, timestamps, obj_meta):
        super().__init__()
        t = torch.from_numpy(tracklets).float().to(DEV)
        self.track_ids, self.input_trans, self.input_rots = t[..., 0], t[..., 1:4], t[..., 4:8]
        self.timestamps = timestamps
        self.opt_trans = torch.nn.Parameter(torch.zeros_like(self.input_trans))
        self.opt_rots = torch.nn.Parameter(torch.zeros_like(self.input_rots[..., :1]))
        self.track_idx = {tid: torch.argwhere(self.track_ids == tid) for tid in obj_meta}

    def _closest(self, tid, t):
        idx = self.track_idx[tid]
        frames = idx[:, 0].cpu()                                            # device -> host
        d = np.abs(np.array(self.timestamps[frames]) - t)
        i1, i2 = np.argsort(d)[:2]
        return idx[i1], idx[i2]

    def translation(self, tid, t):
        a, b = self._closest(tid, t)
        t1, t2 = self.timestamps[a[0].cpu()], self.timestamps[b[0].cpu()]  # two more round trips
        tr1 = self.input_trans[a[0], a[1]] + self.opt_trans[a[0], a[1]]
        tr2 = self.input_trans[b[0], b[1]] + self.opt_trans[b[0], b[1]]
        return (tr1 * (t2 - t) + tr2 * (t - t1)) / (t2 - t1)

    def rotation(self, tid, t):
        a, b = self._closest(tid, t)
        t1, t2 = self.timestamps[a[0].cpu()], self.timestamps[b[0].cpu()]
        r1 = AO.mul_theta(self.input_rots[a[0], a[1]], self.opt_rots[a[0], a[1]][0])
        r2 = AO.mul_theta(r1, self.opt_rots[a[0], b[1]][0])
        return AO.slerp(r1, r2, (t - t1) / (t2 - t1), finite=False)

    def forward(self, track_ids, t, ego):
        out = []
        for tid in track_ids:
            rot, trans = self.rotation(tid, t), self.translation(tid, t)
            eq = AO.matrix_to_quaternion(ego[:3, :3])                       # per actor, as parse_camera does
            out.append(torch.cat([AO.quat_mul(eq, rot), ego[:3, :3] @ trans + ego[:3, 3]]))
        return torch.stack(out)


def table(n, F=198, K=None, seed=0):
    """n tracks over F frames (Waymo's ~20 s at 10 Hz), each present on 40-120 consecutive frames on changing columns."""
    g = np.random.default_rng(seed)
    K = K or n
    ts = 1.6e9 + np.concatenate([[0.0], np.cumsum(g.uniform(0.095, 0.105, F - 1))])
    tr = np.zeros((F, K, 8), np.float32)
    tr[..., 0] = -1
    meta = {}
    for k in range(n):
        s = int(g.integers(0, F // 2))
        e = min(F - 1, s + int(g.integers(40, 120)))
        for f in range(s, e + 1):
            q = g.standard_normal(4)
            tr[f, (k + f) % K] = [k, *(g.standard_normal(3) * 20), *(q / np.linalg.norm(q))]
        meta[k] = dict(start_frame=s, end_frame=e, start_timestamp=float(ts[s]), end_timestamp=float(ts[e]))
    return tr, ts, meta


def timed(calls, iters=STEPS, warmup=WARMUP):
    host = [[] for _ in calls]
    dev = [[] for _ in calls]
    for it in range(warmup + iters):
        for k, fn in enumerate(calls):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            if it >= warmup:
                host[k].append((t1 - t0) * 1e3)
                dev[k].append(a.elapsed_time(b))
    st = lambda x: dict(median_ms=float(np.median(x)), p10_ms=float(np.percentile(x, 10)), p90_ms=float(np.percentile(x, 90)))
    return [dict(host=st(h), events=st(d)) for h, d in zip(host, dev)]


def kernel_us(fn, calls=10):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        name = ev.key.split("(")[0].split("::")[-1].split("<")[0]
        if name in out:
            out[name] += ev.device_time_total / calls
    return out


def host_split(fused, ids, t, ego, w, iters=200):
    """Median host time (no synchronise) of the pieces of one fused forward + backward: the whole forward call, the whole backward
    call, and inside the forward the conversion of the table arguments and the bare ctypes call of sgr_actor_pose_forward."""
    from street_gaussians_b200 import _capi
    from street_gaussians_b200._capi import ptr, stream
    L = _capi.lib()
    slots = (ctypes.c_int32 * len(ids))(*[fused._slot[i] for i in ids])
    poses = torch.empty((len(ids), 7), device=DEV)
    parts = {k: [] for k in ("forward_call", "backward_call", "table_args", "ctypes_forward")}
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        p, _ = fused(ids, timestamp=t, cam=0, is_val=False, ego_pose=ego)
        t1 = time.perf_counter()
        (p * w).sum().backward()
        t2 = time.perf_counter()
        args = fused._table_args()
        t3 = time.perf_counter()
        rc = L.sgr_actor_pose_forward(*args, len(ids), slots, t, 0, 0, ptr(ego), ptr(fused.opt_trans), ptr(fused.opt_rots), 0, 1.0, 1,
                                      ptr(poses), None, stream(ego.device))
        t4 = time.perf_counter()
        assert rc == 0
        for k, d in zip(parts, (t1 - t0, t2 - t1, t3 - t2, t4 - t3)):
            parts[k].append(d * 1e3)
    torch.cuda.synchronize()
    return {k: float(np.median(v)) for k, v in parts.items()}


def arms(n, seed=0):
    tr, ts, meta = table(n, seed=seed)
    fused = sgb.ActorPose(tr, ts, {0: dict(train_timestamps=list(ts))}, meta, fourier_dim=1)
    ref = ReferenceLines(tr, ts, meta)
    g = np.random.default_rng(seed + 1)
    ot = torch.from_numpy((0.05 * g.standard_normal(tuple(fused.opt_trans.shape))).astype(np.float32))
    orr = torch.from_numpy((0.1 * g.standard_normal(tuple(fused.opt_rots.shape))).astype(np.float32))
    with torch.no_grad():
        for m in (fused, ref):
            m.opt_trans.copy_(ot)
            m.opt_rots.copy_(orr)
    ids = list(meta)
    t = float(ts[60] + 0.03)
    ego = torch.eye(4, device=DEV)
    ego[:3, 3] = torch.tensor([3.0, -1.0, 0.5])
    w = torch.randn(n, 7, device=DEV)
    return fused, ref, ids, t, ego, w


def main():
    assert torch.cuda.is_available(), "tools/actor_pose_bench.py needs a CUDA device"
    out = dict(gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w(), steps=STEPS, warmup=WARMUP, calls={})
    for n in (8, 40):
        fused, ref, ids, t, ego, w = arms(n)

        def f_call():
            poses, _ = fused(ids, timestamp=t, cam=0, is_val=False, ego_pose=ego)
            (poses * w).sum().backward()

        def r_call():
            (ref(ids, t, ego) * w).sum().backward()

        p_f = fused(ids, timestamp=t, cam=0, is_val=False, ego_pose=ego)[0]
        p_r = ref(ids, t, ego)
        assert bool(torch.isfinite(p_f).all() and torch.isfinite(p_r).all())
        fa, ra = timed([f_call, r_call])
        out["calls"][f"{n}_actors"] = dict(fused=fa, reference_lines=ra, kernel_us=kernel_us(f_call), host_split_ms=host_split(fused, ids, t, ego, w),
                                           max_abs_pose_diff=float((p_f.detach() - p_r.detach()).abs().max()))
    # the composed training step at config C
    sc = synthetic.make_config("C", seed=0, with_raw=True)
    raw, cam = sc["raw"], sc["cam"]
    H, W = cam["image_height"], cam["image_width"]
    n = raw["poses"].shape[0]
    F = 8
    ts = 1.6e9 + np.arange(F) * 0.1
    tr = np.zeros((F, n, 8), np.float32)
    for k in range(n):
        for f in range(F):
            # in front of the background field, which starts 2 m out and would hide the vehicles (and zero their gradient)
            tr[f, k] = [k, -1.0 + 0.3 * k + 0.05 * (f - 4), 0.1, 1.6 + 0.05 * k, *raw["poses"][k, :4].numpy()]
    meta = {k: dict(start_frame=0, end_frame=F - 1, start_timestamp=float(ts[0]), end_timestamp=float(ts[-1])) for k in range(n)}
    fused = sgb.ActorPose(tr, ts, {0: dict(train_timestamps=list(ts))}, meta, fourier_dim=1)
    ref = ReferenceLines(tr, ts, meta)
    g = np.random.default_rng(7)
    # non-zero offsets in both arms: at zero offsets the slerp's two ends coincide and the reference's where-based slerp returns a NaN
    # gradient, which Adam would write into opt_rots
    ot = torch.from_numpy((0.02 * g.standard_normal(tuple(fused.opt_trans.shape))).astype(np.float32))
    orr = torch.from_numpy((0.05 * g.standard_normal(tuple(fused.opt_rots.shape))).astype(np.float32))
    with torch.no_grad():
        for m in (fused, ref):
            m.opt_trans.copy_(ot)
            m.opt_rots.copy_(orr)
    ids, t, ego = list(range(n)), float(ts[4] + 0.03), torch.eye(4, device=DEV)
    idft = torch.ones(n, 1, device=DEV)
    st = sgb.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=DEV),
                                           scale_modifier=1.0, viewmatrix=cam["viewmatrix"].to(DEV), projmatrix=cam["projmatrix"].to(DEV),
                                           sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    rast = sgb.GaussianRasterizer(st)
    gt = torch.rand(3, H, W, device=DEV)
    arm = {}
    for name, m in (("fused", fused), ("reference_lines", ref)):  # each arm trains its own copy of the Gaussians
        models = [{k: v.to(DEV).clone().requires_grad_(True) for k, v in mm.items()} for mm in raw["models"]]
        gauss = [v for mm in models for v in mm.values()]
        arm[name] = dict(pose=m, models=models, losses=[], poses=[],
                         opt=FusedAdam([{"params": gauss, "lr": 1e-5}, {"params": [m.opt_trans, m.opt_rots], "lr": 1e-6}], eps=1e-15))

    def step(which):
        a = arm[which]

        def go():
            a["opt"].zero_grad(set_to_none=True)
            poses = fused(ids, timestamp=t, cam=0, is_val=False, ego_pose=ego)[0] if which == "fused" else ref(ids, t, ego)
            xyz, rot, scale, opac, sh = sgb.compose(a["models"], poses, idft)
            m2d = torch.zeros_like(xyz, requires_grad=True)
            img = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot)[0]
            loss = losses.photometric_loss(img, gt, None, 1.0, 0.2)
            loss.backward()
            a["opt"].step()
            a["losses"].append(loss.detach())   # checked after the timed loop: no synchronisation inside it
            a["poses"].append(poses.detach())
        return go

    fs, rs = timed([step("fused"), step("reference_lines")], iters=max(STEPS, 60), warmup=WARMUP)
    for name, a in arm.items():  # every timed step ran on finite poses and a finite loss, with gradient reaching the offsets
        assert bool(torch.isfinite(torch.stack(a["losses"])).all()), f"{name}: non-finite loss"
        assert bool(torch.isfinite(torch.stack(a["poses"])).all()), f"{name}: non-finite poses"
        assert bool(torch.isfinite(a["pose"].opt_rots).all() and torch.isfinite(a["pose"].opt_trans).all()), f"{name}: non-finite offsets"
        assert bool((a["pose"].opt_rots.grad != 0).any()), f"{name}: no gradient reached opt_rots"
    diff = float((arm["fused"]["poses"][-1] - arm["reference_lines"]["poses"][-1]).abs().max())
    out["composed_step_config_C"] = dict(actors=n, fused=fs, reference_lines=rs, last_step_max_abs_pose_diff=diff,
                                         last_loss=dict(fused=float(arm["fused"]["losses"][-1]), reference_lines=float(arm["reference_lines"]["losses"][-1])))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
