"""A/B of two libsgr.so builds on config C (1.5 M background + 8 x 50 k actor Gaussians, 1920x1280, SH degree 3, fwd+bwd), alternating in
one process: typically the build before and the build after the forward started storing the SH colour's direction Jacobian, so that
the preprocess backward reads 48 B per visible Gaussian instead of the 192-B coefficient row and a sector of the blend record.

Both libraries are loaded side by side (ctypes loads each with its own symbol scope); the package's calls go to whichever one is
current.  For each build, per round and alternating:
  * the bench-style training step (GaussianRasterizer with InstanceCapacity, forward + backward with bench.py's upstream gradients),
    CUDA events around STEPS eager steps after a warm-up;
  * in a separate profiled run, the device time per step of preprocess_fwd_kernel and preprocess_bwd_tma_kernel from torch.profiler,
    with the algorithmic bytes of each kernel computed from P, V (visible Gaussians) and M, and the rate they imply.
The two builds' outputs of one step are compared first (images and radii bit-equal, largest gradient differences).
Prints one JSON line with the GPU name and its enforced power limit.

python tools/sh_jacobian_ab.py --parent PATH/libsgr.so [--new PATH/libsgr.so] [--rounds 3] [--steps 50]"""
import argparse
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
from street_gaussians_b200 import _capi, synthetic  # noqa: E402

DEV = "cuda"
KEYS = ("means3D", "shs", "opacities", "scales", "rotations")
KERNELS = ("preprocess_fwd_kernel", "preprocess_bwd_tma_kernel")


def load(path):
    _capi.LIB_PATH, _capi._lib = path, None
    return _capi.lib()


def kernel_bytes(P, V, M, jacobian):
    """Algorithmic DRAM bytes per step of the two preprocess kernels (fp32, SH rows of 12 M bytes).
    forward : reads position, opacity, scale, rotation of every Gaussian and the SH row of the visible ones; writes radius, tile count,
              depth key and index of every Gaussian, the 48-B record of the visible ones (+ the 48-B Jacobian with `jacobian`).
    backward: reads radius, position, scale, rotation and the 48-B grad2d row of every Gaussian, and either the SH row of every
              Gaussian plus one 32-B sector of its record (before) or the 48-B Jacobian of the visible ones (after); writes the
              gradients of position, screen position, opacity, scale, rotation and the SH row of every Gaussian."""
    row = 12 * M
    fwd = P * (12 + 4 + 12 + 16) + V * row + P * 16 + V * 48 + (V * 48 if jacobian else 0)
    bwd_in = P * (4 + 12 + 12 + 16 + 48) + (V * 48 if jacobian else P * (row + 32))
    bwd_out = P * (12 + 12 + 4 + 12 + 16 + row)
    return fwd, bwd_in + bwd_out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True, help="libsgr.so of the build to compare against")
    ap.add_argument("--new", default=_capi.LIB_PATH)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--profile-steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    libs = {"parent": load(os.path.abspath(args.parent)), "new": load(os.path.abspath(args.new))}

    scene = synthetic.make_config("C", seed=0, with_raw=True)
    cam = scene["cam"]
    params = {k: scene[k].to(DEV).requires_grad_(True) for k in KEYS}
    P, M = int(params["means3D"].shape[0]), int(params["shs"].shape[1])
    means2D = torch.zeros((P, 3), device=DEV, requires_grad=True)
    up = [scene[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
    settings = sgb.GaussianRasterizationSettings(
        image_height=cam["image_height"], image_width=cam["image_width"], tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"],
        bg=cam["bg"].to(DEV), scale_modifier=cam["scale_modifier"], viewmatrix=cam["viewmatrix"].to(DEV),
        projmatrix=cam["projmatrix"].to(DEV), sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    rast = {k: sgb.GaussianRasterizer(settings, capacity=sgb.InstanceCapacity()) for k in libs}

    def step(name):
        _capi._lib = libs[name]
        for v in list(params.values()) + [means2D]:
            v.grad = None
        color, radii, depth, alpha, _ = rast[name](means3D=params["means3D"], means2D=means2D, opacities=params["opacities"],
                                                   shs=params["shs"], scales=params["scales"], rotations=params["rotations"])
        torch.autograd.backward([color, depth, alpha], up)
        return color, radii, depth, alpha

    # ---- outputs of one step, both builds ----
    outs = {}
    for name in libs:
        for _ in range(3):  # (the first call learns the instance capacity)
            step(name)
        c, r, d, a = step(name)
        outs[name] = dict(color=c.clone(), radii=r.clone(), depth=d.clone(), alpha=a.clone(),
                          **{"grad_" + k: params[k].grad.clone() for k in KEYS})
    torch.cuda.synchronize()
    V = int((outs["new"]["radii"] > 0).sum())
    compare = {}
    for k, v in outs["new"].items():
        w = outs["parent"][k]
        if k in ("color", "depth", "alpha", "radii"):
            compare[k + "_bit_equal"] = bool(torch.equal(v, w))
        else:
            diff = (v.double() - w.double()).abs()
            compare[k] = dict(max_abs=float(diff.max()), max_abs_value=float(w.abs().max()), n_differ=int((v != w).sum()))

    # ---- step times, alternating ----
    step_ms = {k: [] for k in libs}
    for _ in range(args.rounds):
        for name in libs:
            for _ in range(3):
                step(name)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(name)
            e1.record()
            torch.cuda.synchronize()
            step_ms[name].append(e0.elapsed_time(e1) / args.steps)

    # ---- kernel times (profiled separately), alternating ----
    kern_us = {k: {n: [] for n in KERNELS} for k in libs}
    for _ in range(args.rounds):
        for name in libs:
            step(name)
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.profile_steps):
                    step(name)
                torch.cuda.synchronize()
            for n in KERNELS:
                kern_us[name][n].append(sum(ev.device_time_total for ev in prof.key_averages() if n in ev.key) / args.profile_steps)

    result = dict(tool="sh_jacobian_ab", gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w(), P=P, V=V, M=M,
                  rounds=args.rounds, steps=args.steps, outputs=compare, builds={})
    for name in libs:
        fwd_b, bwd_b = kernel_bytes(P, V, M, jacobian=name == "new")
        kt = {n: float(np.median(v)) for n, v in kern_us[name].items()}
        result["builds"][name] = dict(
            step_ms=[round(x, 4) for x in step_ms[name]], step_ms_median=float(np.median(step_ms[name])),
            kernels={n: dict(us=round(kt[n], 2), bytes=b, gb_per_s=round(b / (kt[n] * 1e-6) / 1e9, 1) if kt[n] > 0 else None)
                     for n, b in zip(KERNELS, (fwd_b, bwd_b))})
    print(json.dumps(result))
    return 0


if __name__ == "__main__":
    sys.exit(main())
