"""Per-kernel device time of the single-GPU config-C step (bench.py's timed workload: 1.9 M Gaussians, 1920x1280, SH 3, forward +
backward, bounded binning mode) from torch.profiler, grouped into the stages of the rasterizer:
    python tools/binning_profile.py [--out DIR] [--steps N] [--lib path/to/libsgr.so]
preprocess (preprocess_fwd_kernel), binning (every kernel between the projection and blend_fwd, each listed: depth sort, scan,
emission, tile bucketing), blend_fwd, blend_bwd2 and preprocess_bwd; the card's name and power limit are read in the same run.
Writes DIR/binning_profile.pt.trace.json (chrome trace) and DIR/binning_profile.txt.  --lib profiles another build of
libsgr.so (e.g. the parent commit's) with this tree's Python."""
import argparse
import collections
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name()


def stage_of(name, in_binning):
    for key, stage in (("preprocess_fwd", "preprocess"), ("blend_fwd", "blend_fwd"), ("blend_bwd2", "blend_bwd2"),
                       ("preprocess_bwd", "preprocess_bwd")):
        if key in name:
            return stage
    return "binning" if in_binning else "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "binning_profile_out"))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--lib", default=None, help="libsgr.so to load instead of the in-tree build")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("binning_profile.py needs a CUDA device")
    from street_gaussians_b200 import _capi
    if args.lib:
        _capi.LIB_PATH = os.path.abspath(args.lib)
    import bench
    import street_gaussians_b200 as sgb
    from street_gaussians_b200 import synthetic

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scene = synthetic.make_config("C", seed=0)
    cam = scene["cam"]
    P = scene["means3D"].shape[0]
    rast = sgb.GaussianRasterizer(bench.make_settings(sgb, cam, dev), capacity=sgb.InstanceCapacity())
    params = {k: scene[k].to(dev).requires_grad_(True) for k in bench.PARAM_KEYS}
    m2d = torch.zeros((P, 3), device=dev, requires_grad=True)
    gc, gd, ga = (scene[k].to(dev) for k in ("grad_color", "grad_depth", "grad_alpha"))

    def step():
        for v in params.values():
            v.grad = None
        m2d.grad = None
        c, r, d, a, s = rast(means3D=params["means3D"], means2D=m2d, opacities=params["opacities"], shs=params["shs"],
                             scales=params["scales"], rotations=params["rotations"])
        torch.autograd.backward([c, d, a], [gc, gd, ga])

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(args.out, "binning_profile.pt.trace.json"))

    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    evs.sort(key=lambda e: e.time_range.start)
    starts = [i for i, e in enumerate(evs) if "preprocess_fwd_kernel" in e.name]
    if len(starts) < 2:
        raise SystemExit("fewer than two steps in the trace")
    nstep = len(starts) - 1
    per_kernel = collections.OrderedDict()  # (stage, name) -> total us over the nstep whole steps
    stage_us = collections.OrderedDict((s, 0.0) for s in ("preprocess", "binning", "blend_fwd", "blend_bwd2", "preprocess_bwd", "other"))
    wall = 0.0
    for k in range(nstep):
        seg = evs[starts[k]:starts[k + 1]]
        wall += evs[starts[k + 1]].time_range.start - seg[0].time_range.start
        in_binning = False
        for e in seg:
            if "preprocess_fwd" in e.name:
                in_binning = True
            elif "blend_fwd" in e.name:
                in_binning = False
            st = stage_of(e.name, in_binning and "preprocess_fwd" not in e.name)
            d = e.time_range.end - e.time_range.start
            key = (st, e.name)
            per_kernel[key] = per_kernel.get(key, 0.0) + d
            stage_us[st] += d
    lines = [f"# card: {card()}", f"# config C: P={P}, {cam['image_width']}x{cam['image_height']}, bounded mode, {nstep} profiled steps",
             f"# step (projection start to next projection start): {wall / nstep:.1f} us; sum of device time {sum(stage_us.values()) / nstep:.1f} us",
             "# stage / kernel: us per step"]
    for st, tot in stage_us.items():
        lines.append(f"{st:15s} {tot / nstep:9.1f}")
        if st in ("binning", "other"):
            for (s2, name), us in per_kernel.items():
                if s2 == st:
                    lines.append(f"    {us / nstep:9.1f}  {name[:120]}")
    text = "\n".join(lines) + "\n"
    with open(os.path.join(args.out, "binning_profile.txt"), "w") as f:
        f.write(text)
    print(text)


if __name__ == "__main__":
    main()
