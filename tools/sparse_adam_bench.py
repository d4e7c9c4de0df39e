"""Times the optimizer step at config C (1.5 M background + 8 x 50 k actor Gaussians, SH degree 3, M = 16, 59 floats per row): the
dense training.FusedAdam against the visibility-masked training.SparseAdam, over all nine sub-models.

Visibility comes from real renders of config C's raw scene with the camera yawed by 0, 45, 90 and 180 degrees about the vertical
axis (the scene lies in front of the unyawed camera), plus fixed random masks with 10 %, 30 % and 100 % of the rows visible.  For
each mask: CUDA events around the whole step() call (host work included), median of 60 calls after 10 warm-up calls, the two
optimizers alternating call by call in one process; then each kernel's own device time from torch.profiler over 5 more calls.  The
bytes are the algorithmic traffic: 28 B per element for the dense step (read param, grad, exp_avg, exp_avg_sq; write param, exp_avg,
exp_avg_sq) and 4 B per row of radii + 28 B per element of a visible row for the masked one.

Then one whole training iteration with each optimizer, at yaw 0 and at the yaw that culls the most: compose -> rasterize ->
photometric_loss -> backward -> add_densification_stats -> optimizer step, median of 30 iterations after 5 warm-up iterations,
alternating.  Prints one JSON line with the GPU name and its enforced power limit.
python tools/sparse_adam_bench.py"""
import json
import math
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from loss_bench import power_limit_w  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import losses, synthetic, training  # noqa: E402

DEV = "cuda"
YAWS = (0, 45, 90, 180)
FRACTIONS = (0.1, 0.3, 1.0)
STEP_ITERS, STEP_WARMUP = 60, 10
ITER_ITERS, ITER_WARMUP = 30, 5
# Every step runs with lr = 0: Adam still reads and writes every byte it would (its cost does not depend on the values), but the
# parameters stay exactly those of config C.  With a real lr, the hundreds of timed steps would move every row by ~lr per step and
# the training iterations would render a distorted scene (saturated opacities, rescaled splats) instead of config C.
LR = 0.0


def scene_models():
    cfg = dict(synthetic.CONFIGS["C"])
    cfg.pop("kind")
    sc = synthetic.make_scene(seed=0, with_raw=True, **cfg)
    objs = []
    for r in sc["raw"]["models"]:
        n = r["xyz"].shape[0]
        o = types.SimpleNamespace(**{"_" + a: torch.nn.Parameter(v.to(DEV)) for a, v in r.items()})
        o._semantic = torch.nn.Parameter(torch.zeros(n, 0, device=DEV))
        o.max_radii2D, o.xyz_gradient_accum, o.denom = torch.zeros(n, device=DEV), torch.zeros(n, 2, device=DEV), torch.zeros(n, 1, device=DEV)
        objs.append(o)
    return sc, objs


def camera(sc, yaw_deg):
    c, s = math.cos(math.radians(yaw_deg)), math.sin(math.radians(yaw_deg))
    w2c = torch.eye(4)
    w2c[:3, :3] = torch.tensor([[c, 0.0, -s], [0.0, 1.0, 0.0], [s, 0.0, c]])
    cam = synthetic.make_camera(sc["cam"]["image_width"], sc["cam"]["image_height"], 50.0, w2c, 3)
    return sgb.GaussianRasterizer(sgb.GaussianRasterizationSettings(
        image_height=cam["image_height"], image_width=cam["image_width"], tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"],
        bg=cam["bg"].to(DEV), scale_modifier=cam["scale_modifier"], viewmatrix=cam["viewmatrix"].to(DEV),
        projmatrix=cam["projmatrix"].to(DEV), sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV), prefiltered=False, debug=False))


def optimizers(objs):
    groups = lambda: [{"params": [getattr(o, n)], "lr": LR, "name": n} for o in objs for n in training.PARAM_NAMES]
    return training.FusedAdam(groups(), eps=1e-15), training.SparseAdam(groups(), eps=1e-15)


def events_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def alternate(calls, iters, warmup):
    """Median ms of each call, the calls alternating one after the other."""
    ts = [[] for _ in calls]
    for it in range(warmup + iters):
        for k, fn in enumerate(calls):
            t = events_ms(fn)
            if it >= warmup:
                ts[k].append(t)
    return [float(np.median(t)) for t in ts]


def kernel_us(fn, name, calls=5):
    """Mean device time of the kernel `name` per call, from torch.profiler (the event times above include the host's work in step())."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    total = sum(ev.device_time_total for ev in prof.key_averages() if ev.key.split("(")[0].split("::")[-1] == name)
    return total / calls


def main():
    assert torch.cuda.is_available(), "tools/sparse_adam_bench.py needs a CUDA device"
    dev = torch.cuda.current_device()
    sc, objs = scene_models()
    pristine = [getattr(o, n).detach().clone() for o in objs for n in training.PARAM_NAMES]
    poses, idft = sc["raw"]["poses"].to(DEV), sc["raw"]["idft"].to(DEV)
    counts = [o._xyz.shape[0] for o in objs]
    P = sum(counts)
    widths = [sum(int(math.prod(getattr(o, n).shape[1:])) for n in training.PARAM_NAMES) for o in objs]
    assert widths[0] == 59
    gt = torch.rand(3, sc["cam"]["image_height"], sc["cam"]["image_width"], generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)

    def render(rast):
        xyz, rot, scale, opac, sh = sgb.compose(objs, poses, idft)
        m2d = torch.zeros_like(xyz, requires_grad=True)
        col, radii, _, _, _ = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot)
        return col, radii, m2d

    masks = {}
    with torch.no_grad():
        for yaw in YAWS:
            masks[f"yaw{yaw}"] = render(camera(sc, yaw))[1].clone()
    g = torch.Generator(device=DEV).manual_seed(2)
    for f in FRACTIONS:
        masks[f"random{int(round(f * 100))}"] = (torch.rand(P, generator=g, device=DEV) < f).to(torch.int32)

    fused, sparse = optimizers(objs)
    for o in objs:   # gradients of a realistic magnitude
        for n in training.PARAM_NAMES:
            p = getattr(o, n)
            p.grad = torch.randn(p.shape, generator=g, device=DEV) * 1e-4
    dense_bytes = 28 * sum(c * w for c, w in zip(counts, widths))
    steps = {}
    for name, radii in masks.items():
        vis = radii > 0
        vis_rows = [int(vis[s:s + c].sum()) for s, c in zip(np.cumsum([0] + counts[:-1]).tolist(), counts)]
        sparse_bytes = 4 * P + 28 * sum(v * w for v, w in zip(vis_rows, widths))
        fused_ms, sparse_ms = alternate([fused.step, lambda: sparse.step(objs, radii)], STEP_ITERS, STEP_WARMUP)
        fused_k = kernel_us(fused.step, "adam_kernel")
        sparse_k = kernel_us(lambda: sparse.step(objs, radii), "sparse_adam_kernel")
        steps[name] = dict(visible_fraction=sum(vis_rows) / P, fused_ms=fused_ms, sparse_ms=sparse_ms, sparse_over_fused=sparse_ms / fused_ms,
                           fused_kernel_us=fused_k, sparse_kernel_us=sparse_k, fused_bytes=dense_bytes, sparse_bytes=sparse_bytes,
                           fused_kernel_tbps=dense_bytes / max(fused_k, 1e-3) / 1e6, sparse_kernel_tbps=sparse_bytes / max(sparse_k, 1e-3) / 1e6)

    # one whole training iteration with each optimizer
    culled = min(YAWS, key=lambda y: steps[f"yaw{y}"]["visible_fraction"])
    iteration = {}
    for yaw in sorted({0, culled}):
        rast = camera(sc, yaw)

        def it(opt, masked):
            col, radii, m2d = render(rast)
            loss = losses.photometric_loss(col, gt, None, 1.0, 0.2)
            opt.zero_grad()
            loss.backward()
            training.add_densification_stats(objs, radii, m2d.grad)
            if masked:
                opt.step(objs, radii)
            else:
                opt.step()

        fused_ms, sparse_ms = alternate([lambda: it(fused, False), lambda: it(sparse, True)], ITER_ITERS, ITER_WARMUP)
        iteration[f"yaw{yaw}"] = dict(visible_fraction=steps[f"yaw{yaw}"]["visible_fraction"], fused_ms=fused_ms, sparse_ms=sparse_ms)
    # every step and every iteration above ran on config C's scene as generated
    assert all(torch.equal(getattr(o, n).detach(), t) for (o, n), t in zip([(o, n) for o in objs for n in training.PARAM_NAMES], pristine))
    out = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), P=P, counts=counts, floats_per_row=widths[0],
               step_iters=STEP_ITERS, iteration_iters=ITER_ITERS, optimizer_step=steps, training_iteration=iteration)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
