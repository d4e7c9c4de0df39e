"""Times the objects-only render at config C (1.5 M background + 8 x 50 k actor Gaussians, 1920x1280, SH degree 3, through compose):
the reference's shape (a second GaussianRasterizer call on the actor rows) against one call with a render layer
(GaussianRasterizer.forward_layers).

  training shape (train.py:94-122), compose -> rasterize -> photometric_loss + sky_loss + obj_acc_loss -> backward:
    two_calls   the main call plus a separate call on the actor slice [n_bkgd, P) over a white background
    layered     one call with RenderLayer(n_bkgd, P, white)
  render_all shape (street_gaussian_renderer.py:13-40), no gradient, white background:
    three_calls full, background-only and objects-only calls
    layered     one call with the background and the objects layers

Both modes: the default one (one blocking instance-count read-back per call) and the bounded one (InstanceCapacity).  The two arms of
each comparison alternate call by call in one process; CUDA events around each step, median of STEPS after WARMUP.  The outputs of the
two arms are compared first (images bit-equal).  Then, in a separate profiled run of the layered training step, the device time of
each kernel per step from torch.profiler.  Prints one JSON line with the GPU name and its enforced power limit.
python tools/layer_bench.py"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from loss_bench import power_limit_w  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import losses, synthetic  # noqa: E402
from street_gaussians_b200 import rasterizer as R  # noqa: E402

DEV = "cuda"
STEPS, WARMUP = 60, 10
KERNELS = ("layer_count_kernel", "layer_scan_kernel", "layer_compact_kernel", "layer_stash_kernel", "layer_merge_kernel", "blend_fwd_kernel",
           "blend_bwd2_kernel", "preprocess_fwd_kernel", "preprocess_bwd_tma_kernel", "emit_pairs_kernel", "tile_ranges_kernel")


def events_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def alternate(calls, iters=STEPS, warmup=WARMUP):
    ts = [[] for _ in calls]
    for it in range(warmup + iters):
        for k, fn in enumerate(calls):
            t = events_ms(fn)
            if it >= warmup:
                ts[k].append(t)
    return [dict(median_ms=float(np.median(t)), p10_ms=float(np.percentile(t, 10)), p90_ms=float(np.percentile(t, 90))) for t in ts]


def kernel_us(fn, calls=5):
    """Device time per call of each kernel in KERNELS (summed over its instantiations and launches), from torch.profiler."""
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
    out["all_kernels"] = sum(ev.device_time_total for ev in prof.key_averages()) / calls
    return out


def main():
    assert torch.cuda.is_available(), "tools/layer_bench.py needs a CUDA device"
    dev = torch.cuda.current_device()
    cfg = dict(synthetic.CONFIGS["C"])
    cfg.pop("kind")
    sc = synthetic.make_scene(seed=0, with_raw=True, **cfg)
    raw = sc["raw"]
    models = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in raw["models"]]
    poses, idft = raw["poses"].to(DEV).requires_grad_(True), raw["idft"].to(DEV)
    nb = models[0]["xyz"].shape[0]
    cam = sc["cam"]
    H, W = cam["image_height"], cam["image_width"]
    white = torch.ones(3, device=DEV)
    st = sgb.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=white,
                                           scale_modifier=cam["scale_modifier"], viewmatrix=cam["viewmatrix"].to(DEV),
                                           projmatrix=cam["projmatrix"].to(DEV), sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV),
                                           prefiltered=False, debug=False)
    g = torch.Generator(device=DEV).manual_seed(1)
    gt = torch.rand(3, H, W, generator=g, device=DEV)
    sky = torch.rand(1, H, W, generator=g, device=DEV) > 0.8
    obj_bound = torch.rand(1, H, W, generator=g, device=DEV) > 0.9
    leaves = [v for m in models for v in m.values()] + [poses]

    with torch.no_grad():
        xyz, rot, scale, opac, sh = sgb.compose(models, poses, idft)
        P = xyz.shape[0]
        inst = lambda sl: R._forward_impl(xyz[sl], sh[sl], None, None, opac[sl], scale[sl], rot[sl], None, st, None)[5].num_instances
        counts = dict(P=P, n_bkgd=nb, main_instances=inst(slice(0, P)), objects_instances=inst(slice(nb, P)),
                      background_instances=inst(slice(0, nb)))

    def make(mode):
        cap = None
        if mode == "bounded":
            cap = sgb.InstanceCapacity()
            with torch.no_grad():
                x, r_, s_, o_, h_ = sgb.compose(models, poses, idft)
                sgb.GaussianRasterizer(st, capacity=cap)(means3D=x, means2D=None, opacities=o_, shs=h_, scales=s_, rotations=r_)
        rast = sgb.GaussianRasterizer(st, capacity=cap)

        def train(layered):
            for v in leaves:
                v.grad = None
            x, r_, s_, o_, h_ = sgb.compose(models, poses, idft)
            m2d = torch.zeros_like(x, requires_grad=True)
            kw = dict(means3D=x, opacities=o_, shs=h_, scales=s_, rotations=r_)
            if layered:
                color, radii, depth, acc, _, ((_, _, oacc),) = rast.forward_layers(means2D=m2d, layers=[sgb.RenderLayer(nb, P, white)], **kw)
            else:
                color, radii, depth, acc, _ = rast(means2D=m2d, **kw)
                s2d = torch.zeros((P - nb, 3), device=DEV, requires_grad=True)
                _, _, _, oacc, _ = rast(means2D=s2d, **{k: v[nb:] for k, v in kw.items()})
            loss = losses.photometric_loss(color, gt, None, 1.0, 0.2) + losses.sky_loss(acc, sky, 0.05) + losses.obj_acc_loss(oacc, obj_bound, 0.1)
            loss.backward()
            return color.detach(), oacc.detach(), m2d.grad

        def render_all(layered):
            with torch.no_grad():
                x, r_, s_, o_, h_ = sgb.compose(models, poses, idft)
                kw = dict(means3D=x, opacities=o_, shs=h_, scales=s_, rotations=r_)
                if layered:
                    out = rast.forward_layers(means2D=None, layers=[sgb.RenderLayer(0, nb, white), sgb.RenderLayer(nb, P, white)], **kw)
                    return out[0], out[5][0][0], out[5][1][0]
                full = rast(means2D=None, **kw)[0]
                bkgd = rast(means2D=None, **{k: v[:nb] for k, v in kw.items()})[0]
                obj = rast(means2D=None, **{k: v[nb:] for k, v in kw.items()})[0]
                return full, bkgd, obj
        return rast, train, render_all

    results, same = {}, {}
    for mode in ("default", "bounded"):
        rast, train, render_all = make(mode)
        a, b = train(False), train(True)
        same[f"{mode}_train_images_equal"] = bool(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]))
        same[f"{mode}_train_means2D_rel_err"] = float((a[2] - b[2]).abs().max() / (b[2].abs().max() + 1e-30))
        a, b = render_all(False), render_all(True)
        same[f"{mode}_render_all_images_equal"] = bool(all(torch.equal(x, y) for x, y in zip(a, b)))
        two, one = alternate([lambda: train(False), lambda: train(True)])
        three, lay = alternate([lambda: render_all(False), lambda: render_all(True)])
        results[mode] = dict(train_two_calls=two, train_layered=one, train_speedup=two["median_ms"] / one["median_ms"],
                             render_all_three_calls=three, render_all_layered=lay, render_all_speedup=three["median_ms"] / lay["median_ms"])
        rast.synchronize_capacity()
    _, train, _ = make("default")
    kernels = dict(train_layered=kernel_us(lambda: train(True)), train_two_calls=kernel_us(lambda: train(False)))
    out = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(), width=W, height=H, steps=STEPS, warmup=WARMUP,
               **counts, outputs=same, times=results, kernel_us_per_step=kernels)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
