"""Feature channels in multi-GPU training, timed on ONE GPU.

    python tools/sharded_feature_bench.py [--steps 20 --K 19 --iters 50 --repeats 7] [--out FILE]

Leg 1, the Gaussian-sharded step at world 1 on config C (1.9 M Gaussians, 1920x1280, SH 3) with S = 3 (normals) and S = 3 + 19 feature
channels: GaussianShardedRasterizer(exchange="p2p") forward + backward, fused (sgr_sharded_forward_features / _backward_features, one
C call each way) against staged (project, peer scatter, forward_records, backward_blend, peer gather, backward_geom: the path a frame
with feature channels took before the fused step carried them).  CUDA events per step, the arms alternating step by step, median and
p10-p90 of --steps steps after 3 warm-up frames (the fused arm needs two to learn its capacities).  At world 1 there is no peer and no
NCCL traffic: the numbers compare the launch structure and the host work of the two paths, not a multi-GPU exchange.

Leg 2, finish_features on a tile-row band against the whole frame, ranks EMULATED: at config C's frame size with 3 normal channels and
K semantic classes, every rank's band forward + backward (sgr_band_finish_features_*) for world 1, 2, 4 and 8 (both layouts) runs alone,
one rank after another, timed with CUDA events; the slowest rank is given beside the whole-frame call.  Each time is the median of
`repeats` windows of `iters` calls, the arms alternating window by window, host cost of the ctypes calls included.  These say what one
rank's share of the work costs on one H100, not what several H100s reach together (the op is per pixel: no collective to time).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from street_gaussians_b200 import _capi  # noqa: E402
from street_gaussians_b200._capi import ptr  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import synthetic  # noqa: E402
from street_gaussians_b200.sharded import GaussianShardedRasterizer, contiguous_band, cyclic_band  # noqa: E402


def window(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def step_leg(dev, S, steps):
    """Fused and staged sharded steps at world 1, S feature channels: {arm: (median ms, p10, p90)}."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    import util
    scene = synthetic.make_config("C", seed=0, semantics=S)
    st = util.settings_from(sgb, scene["cam"], dev)
    keys = ("means3D", "shs", "opacities", "scales", "rotations", "semantics")
    leaves = {k: scene[k].to(dev).contiguous().requires_grad_(True) for k in keys}
    ups = [scene[k].to(dev) for k in ("grad_color", "grad_depth", "grad_alpha")] + [scene["grad_semantic"].to(dev)]
    arms = {name: GaussianShardedRasterizer(st, capacity=sgb.InstanceCapacity(), exchange="p2p", fused=fused)
            for name, fused in (("fused", True), ("staged", False))}

    def step(mod):
        color, _, depth, alpha, semantic = mod(means3D=leaves["means3D"], means2D=None, opacities=leaves["opacities"], shs=leaves["shs"],
                                               scales=leaves["scales"], rotations=leaves["rotations"], semantics=leaves["semantics"])
        torch.autograd.backward([color, depth, alpha, semantic], ups)
        for t in leaves.values():
            t.grad = None
        return bool(getattr(color.grad_fn, "fused", False))

    for name, mod in arms.items():
        for _ in range(3):
            took = step(mod)
            mod.synchronize_capacity()
        assert took == (name == "fused"), (name, took)
    times = {k: [] for k in arms}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(steps):
        for name, mod in arms.items():
            torch.cuda.synchronize()
            a.record()
            step(mod)
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b))
    out = {}
    for k, v in times.items():
        q = statistics.quantiles(v, n=10)
        out[k] = dict(median_ms=round(statistics.median(v), 3), p10_ms=round(q[0], 3), p90_ms=round(q[-1], 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--H", type=int, default=1280)
    ap.add_argument("--W", type=int, default=1920)
    ap.add_argument("--K", type=int, default=19)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sharded_feature_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    steps = {f"S={S}": step_leg(dev, S, args.steps) for S in (3, 3 + args.K)}
    torch.cuda.empty_cache()
    H, W, nc, K = args.H, args.W, 3, args.K
    S = nc + K
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand(S, H, W, device=dev, generator=g)
    x[:nc] = 2 * x[:nc] - 1
    gn, gs = torch.randn(nc, H, W, device=dev, generator=g), torch.randn(K, H, W, device=dev, generator=g)
    n, s, gx = torch.empty(nc, H, W, device=dev), torch.empty(K, H, W, device=dev), torch.empty(S, H, W, device=dev)

    def whole(mode):
        def fn():
            _capi.call("sgr_finish_features_forward", dev, S, H, W, nc, mode, ptr(x), ptr(n), ptr(s))
            _capi.call("sgr_finish_features_backward", dev, S, H, W, nc, mode, ptr(x), ptr(gn), ptr(gs), ptr(gx))
        return fn

    def band(mode, b, e, st):
        def fn():
            _capi.call("sgr_band_finish_features_forward", dev, S, H, W, nc, mode, b, e, st, ptr(x), ptr(n), ptr(s))
            _capi.call("sgr_band_finish_features_backward", dev, S, H, W, nc, mode, b, e, st, ptr(x), ptr(gn), ptr(gs), ptr(gx))
        return fn

    results = []
    for mode_name, mode in (("logits", _capi.SEMANTIC_LOGITS), ("probabilities", _capi.SEMANTIC_PROBABILITIES)):
        for layout in ("cyclic", "contiguous"):
            mk = cyclic_band if layout == "cyclic" else contiguous_band
            for world in (1, 2, 4, 8):
                arms = {"whole": whole(mode)}
                arms.update({f"rank{r}": band(mode, *mk(H, r, world)) for r in range(world)})
                for fn in arms.values():  # warm-up
                    for _ in range(3):
                        fn()
                times = {k: [] for k in arms}
                for _ in range(args.repeats):
                    for k, fn in arms.items():
                        times[k].append(window(fn, args.iters))
                med = {k: statistics.median(v) for k, v in times.items()}
                slow = max((k for k in arms if k != "whole"), key=lambda k: med[k])
                results.append(dict(mode=mode_name, layout=layout, world=world, whole_frame_ms=round(med["whole"], 4),
                                    slowest_rank_ms=round(med[slow], 4), slowest_rank=slow,
                                    slowest_rank_p10_p90=[round(v, 4) for v in statistics.quantiles(times[slow], n=10)[::8]]))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    doc = dict(gpu=gpu, sharded_step_world1_config_C=steps,
               finish_features_band=dict(H=H, W=W, S=S, ranks="emulated on one GPU, one after another", results=results))
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
