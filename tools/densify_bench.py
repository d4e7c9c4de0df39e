"""Times densification at config C (1.5 M background + 8 x 50 k actor Gaussians, SH degree 3, M = 16): the fused
training.densify_and_prune (plan kernel, scan, one read-back, apply kernel) against the reference's torch lines restated in
oracle/densify_oracle.py, run per sub-model on the same GPU.  Seeded statistics give a few percent each of clone, split and prune.
Densification is destructive, so every call starts from a fresh copy of the pristine scene, made outside the timed window.
CUDA events, median of 20 calls after 3 warm-up calls.  The apply kernel's own time comes from torch.profiler, and its bandwidth is
the bytes it must move (computed from the shapes and the counts) over that time.  Prints one JSON line with the GPU name and its
enforced power limit.
python tools/densify_bench.py"""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from loss_bench import power_limit_w  # noqa: E402
from oracle import densify_oracle as DO  # noqa: E402
from street_gaussians_b200 import synthetic, training  # noqa: E402

NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic")
ATTR = dict(xyz="_xyz", f_dc="_features_dc", f_rest="_features_rest", opacity="_opacity", scaling="_scaling", rotation="_rotation",
            semantic="_semantic")
ITERS, WARMUP = 20, 3


def pristine(seed=0):
    sc = synthetic.make_scene(P=1_500_000, width=1920, height=1280, sh_degree=3, seed=seed, n_vehicles=8, per_vehicle=50_000,
                              with_raw=True, scale_med=0.02)
    g = torch.Generator().manual_seed(seed + 1)
    models = []
    for k, r in enumerate(sc["raw"]["models"]):
        n = r["xyz"].shape[0]
        t = dict(xyz=r["xyz"], f_dc=r["features_dc"], f_rest=r["features_rest"], opacity=r["opacity"], scaling=r["scaling"],
                 rotation=r["rotation"], semantic=torch.zeros(n, 0))
        denom = torch.randint(1, 6, (n, 1), generator=g).float()
        # ~4 % of the parents above the gradient threshold; the scales decide clone or split
        hot = (torch.rand(n, 1, generator=g) < 0.04).float()
        t["xyz_gradient_accum"] = denom * (hot * 2.0 + torch.rand(n, 2, generator=g) * 0.9) * (6e-4 if k == 0 else 2e-4)
        t["denom"], t["max_radii2D"] = denom, torch.rand(n, generator=g) * 20
        t["exp_avg"] = {a: torch.randn(t[a].shape, generator=g) * 1e-3 for a in NAMES}
        t["exp_avg_sq"] = {a: torch.rand(t[a].shape, generator=g) * 1e-6 for a in NAMES}
        meta = dict(kind="background" if k == 0 else "actor", t={a: (v.cuda() if torch.is_tensor(v) else {b: x.cuda() for b, x in v.items()})
                                                                 for a, v in t.items()},
                    grad_col=1 if k == 0 else 0, grad_threshold=6e-4 if k == 0 else 2e-4, percent_dense=0.01, percent_big_ws=0.1)
        if k == 0:
            meta.update(extent=torch.tensor([float(sc["raw"]["models"][0]["xyz"].norm(dim=1).quantile(0.9))]).cuda(),
                        sphere_center=torch.zeros(3).cuda(), sphere_radius=torch.tensor([30.0]).cuda())
        else:
            meta.update(extent=torch.tensor([3.375]).cuda(), min_xyz=torch.tensor([-2.3, -0.85, -1.05]).cuda(),
                        max_xyz=torch.tensor([2.3, 0.85, 1.05]).cuda())
        models.append(meta)
    return models


def fresh(models):
    """Product-side models and one FusedAdam over all of them, from a copy of the pristine tensors."""
    objs, groups = [], []
    for m in models:
        o = types.SimpleNamespace()
        for a in NAMES:
            setattr(o, ATTR[a], torch.nn.Parameter(m["t"][a].clone()))
        for s in ("xyz_gradient_accum", "denom", "max_radii2D"):
            setattr(o, s, m["t"][s].clone())
        o.percent_dense, o.percent_big_ws = m["percent_dense"], m["percent_big_ws"]
        if m["kind"] == "background":
            o.scene_radius, o.sphere_center, o.sphere_radius = m["extent"], m["sphere_center"], m["sphere_radius"]
        else:
            o.extent, o.min_xyz, o.max_xyz = m["extent"], m["min_xyz"], m["max_xyz"]
        objs.append(o)
        groups += [{"params": [getattr(o, ATTR[a])], "lr": 0.0, "name": a} for a in NAMES]
    opt = training.FusedAdam(groups, lr=0.0, eps=1e-15)
    for o, m in zip(objs, models):
        for a in NAMES:
            opt.state[getattr(o, ATTR[a])] = {"step": 100, "exp_avg": m["t"]["exp_avg"][a].clone(), "exp_avg_sq": m["t"]["exp_avg_sq"][a].clone()}
    return objs, opt


def fresh_oracle(models):
    out = []
    for m in models:
        t = {a: (v.clone() if torch.is_tensor(v) else {b: x.clone() for b, x in v.items()}) for a, v in m["t"].items()}
        out.append(t)
    return out


def oracle_kwargs(m):
    kw = dict(grad_threshold=m["grad_threshold"], grad_col=m["grad_col"], extent=m["extent"], percent_dense=m["percent_dense"],
              percent_big_ws=m["percent_big_ws"], min_opacity=0.005, prune_big_points=True)
    if m["kind"] == "background":
        kw.update(sphere_center=m["sphere_center"], sphere_radius=m["sphere_radius"])
    else:
        kw.update(min_xyz=m["min_xyz"], max_xyz=m["max_xyz"])
    return kw


def timed(setup, call):
    ts = []
    for it in range(WARMUP + ITERS):
        state = setup()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        res = call(state)
        b.record()
        torch.cuda.synchronize()
        if it >= WARMUP:
            ts.append(a.elapsed_time(b))
        del state
    return float(np.median(ts)), res


def main():
    assert torch.cuda.is_available(), "tools/densify_bench.py needs a CUDA device"
    dev = torch.cuda.current_device()
    models = pristine()
    draws = [torch.randn(m["t"]["xyz"].shape[0], 18, device="cuda") for m in models]
    P = sum(m["t"]["xyz"].shape[0] for m in models)
    fused_ms, scal = timed(lambda: fresh(models), lambda s: training.densify_and_prune(
        s[0], [m["grad_threshold"] for m in models], 0.005, True, s[1], grad_abs=[m["grad_col"] == 1 for m in models], seed=1))
    ref_ms, _ = timed(lambda: fresh_oracle(models), lambda ts: [DO.densify_model(t, m["kind"], d, **oracle_kwargs(m))
                                                                 for t, m, d in zip(ts, models, draws)])
    # the apply kernel alone, from the profiler
    kernel_us = {}
    for _ in range(3):
        objs, opt = fresh(models)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            training.densify_and_prune(objs, [m["grad_threshold"] for m in models], 0.005, True, opt,
                                       grad_abs=[m["grad_col"] == 1 for m in models], seed=1)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            for key in ("densify_apply_kernel", "densify_plan_kernel"):
                if key in ev.key:
                    kernel_us.setdefault(key, []).append(ev.device_time_total / max(ev.count, 1))
        del objs, opt
    apply_us = float(np.median(kernel_us["densify_apply_kernel"]))
    plan_us = float(np.median(kernel_us["densify_plan_kernel"]))
    # bytes the apply kernel must move: every output row read from its parent and written (params + both moments where carried),
    # the carried moments of kept originals read, and the three statistics written
    nbytes = 0
    for m, s in zip(models, scal):
        w = sum(int(np.prod(m["t"][a].shape[1:])) for a in NAMES)
        n_new = (s["points_total"] + s["points_clone"] + s["points_split"]) - s["points_pruned"]
        kept_orig = s["points_total"] - s["points_split"]  # upper bound of section 0
        nbytes += 4 * w * (n_new + 3 * n_new + 2 * kept_orig) + 16 * n_new
    out = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), P=P, M=16, iters=ITERS,
               fused_ms=fused_ms, reference_lines_ms=ref_ms, speedup=ref_ms / fused_ms, plan_kernel_us=plan_us, apply_kernel_us=apply_us,
               apply_bytes=nbytes, apply_gbps=nbytes / (apply_us * 1e-6) / 1e9,
               scalars={k: sum(s.get(k, 0) for s in scal) for k in training.SCALAR_NAMES})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
