"""A/B of two libsgr.so builds on config C (1.5 M background + 8 x 50 k actor Gaussians, 1920x1280, SH degree 3, fwd+bwd), alternating in
one process: typically the build before and the build after the forward started binning the far Gaussians only into the tiles the
near ones left unsaturated (the saturation split, include/sgr.h sgr_set_near_budget).

Both libraries are loaded side by side (ctypes loads each with its own symbol scope); the package's calls go to whichever one is
current.  For each build, per round and alternating:
  * the bench-style training step (GaussianRasterizer with InstanceCapacity, forward + backward with bench.py's upstream gradients),
    CUDA events around STEPS eager steps after a warm-up;
  * in a separate profiled run, the device time per step of every kernel from torch.profiler.
The two builds' outputs of one step are compared first (images and radii bit-equal, largest gradient differences), and the
instances each build emits (status word 3) are read from an exact-mode forward.  --sweep also times the new build at the budgets
R / d for each d given (the rule of the library is R / 8).  --sweep-parts builds one more library per value n, with the bucketing's
partition target (csrc/binning.cu kBucketTargetParts) set to n, and times and profiles each next to parent and new.
Prints one JSON line with the GPU name and its enforced power limit.

python tools/saturation_split_ab.py --parent PATH/libsgr.so [--new PATH/libsgr.so] [--rounds 3] [--steps 50] [--sweep 16 8 4 2]
                                    [--sweep-parts 132 264 396 528]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from loss_bench import power_limit_w  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import _capi, synthetic  # noqa: E402
from street_gaussians_b200 import rasterizer as R  # noqa: E402

DEV = "cuda"
KEYS = ("means3D", "shs", "opacities", "scales", "rotations")


def load(path, symbols):
    _capi.LIB_PATH, _capi._lib, saved = path, None, _capi.SYMBOLS
    _capi.SYMBOLS = symbols
    try:
        return _capi.lib()
    finally:
        _capi.SYMBOLS = saved


def build_target_parts(values, out_dir):
    """One libsgr.so per partition target: binning.cu recompiled with SGR_BUCKET_TARGET_PARTS=n, linked with the objects build()
    left in the package's _obj/."""
    from street_gaussians_b200 import build as B
    nvcc = B._nvcc()
    others = [os.path.join(B.OBJ, s + ".o") for s in B.SOURCES if s != "binning.cu"]
    missing = [o for o in others if not os.path.exists(o)]
    if values and missing:
        raise SystemExit(f"--sweep-parts links the objects of the package build; missing: {missing}")

    def one(n):
        obj, lib = os.path.join(out_dir, f"binning_{n}.o"), os.path.join(out_dir, f"libsgr_parts{n}.so")
        subprocess.run([nvcc, "-c", os.path.join(B.CSRC, "binning.cu"), "-o", obj, f"-DSGR_BUCKET_TARGET_PARTS={n}"] + B.NVCC_FLAGS,
                       check=True)
        subprocess.run([nvcc, "-shared", "-o", lib, obj] + others + ["-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC"],
                       check=True)
        return lib

    with ThreadPoolExecutor(max_workers=max(1, len(values))) as ex:
        return dict(zip(values, ex.map(one, values)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True, help="libsgr.so of the build to compare against")
    ap.add_argument("--new", default=_capi.LIB_PATH)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--profile-steps", type=int, default=10)
    ap.add_argument("--sweep", type=int, nargs="*", default=[], help="divisors d: also time the new build at budget R / d")
    ap.add_argument("--sweep-parts", type=int, nargs="*", default=[],
                    help="partition targets n: also time and profile the new sources built with SGR_BUCKET_TARGET_PARTS=n")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    old_symbols = [s for s in _capi.SYMBOLS if s != "sgr_set_near_budget"]
    libs = {"parent": load(os.path.abspath(args.parent), old_symbols), "new": load(os.path.abspath(args.new), _capi.SYMBOLS)}
    tmp = tempfile.TemporaryDirectory(prefix="sgr_parts_")
    for n, path in build_target_parts(args.sweep_parts, tmp.name).items():
        libs[f"parts={n}"] = load(path, _capi.SYMBOLS)

    scene = synthetic.make_config("C", seed=0)
    cam = scene["cam"]
    params = {k: scene[k].to(DEV).requires_grad_(True) for k in KEYS}
    P = int(params["means3D"].shape[0])
    means2D = torch.zeros((P, 3), device=DEV, requires_grad=True)
    up = [scene[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
    settings = sgb.GaussianRasterizationSettings(
        image_height=cam["image_height"], image_width=cam["image_width"], tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"],
        bg=cam["bg"].to(DEV), scale_modifier=cam["scale_modifier"], viewmatrix=cam["viewmatrix"].to(DEV),
        projmatrix=cam["projmatrix"].to(DEV), sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    variants = {name: (name, None) for name in libs}
    rast = {k: sgb.GaussianRasterizer(settings, capacity=sgb.InstanceCapacity()) for k in variants}

    def emitted(name):
        """(R, E): instances of the frame and instances the binning emitted, from an exact-mode forward."""
        _capi._lib = libs[name]
        with torch.no_grad():
            out = R._forward_impl(params["means3D"], params["shs"], None, None, params["opacities"], params["scales"], params["rotations"],
                                  None, settings, None)
        torch.cuda.synchronize()
        st = R.state_views(settings, out[5], P)["status"].tolist()
        return st[_capi.STATUS_INSTANCES], st[_capi.STATUS_EMITTED]

    R_total, E_parent = emitted("parent")
    for d in args.sweep:
        variants[f"new_R/{d}"] = ("new", R_total // d)
        rast[f"new_R/{d}"] = sgb.GaussianRasterizer(settings, capacity=sgb.InstanceCapacity())

    def step(name):
        lib_name, budget = variants[name]
        _capi._lib = libs[lib_name]
        for v in list(params.values()) + [means2D]:
            v.grad = None
        if budget is None:
            color, radii, depth, alpha, _ = rast[name](means3D=params["means3D"], means2D=means2D, opacities=params["opacities"],
                                                       shs=params["shs"], scales=params["scales"], rotations=params["rotations"])
        else:
            with _capi.near_budget(budget):
                color, radii, depth, alpha, _ = rast[name](means3D=params["means3D"], means2D=means2D, opacities=params["opacities"],
                                                           shs=params["shs"], scales=params["scales"], rotations=params["rotations"])
        torch.autograd.backward([color, depth, alpha], up)
        return color, radii, depth, alpha

    # ---- outputs of one step, every variant against the parent ----
    outs = {}
    for name in variants:
        for _ in range(3):  # (the first call learns the instance capacity)
            step(name)
        c, r, d, a = step(name)
        outs[name] = dict(color=c.clone(), radii=r.clone(), depth=d.clone(), alpha=a.clone(),
                          **{"grad_" + k: params[k].grad.clone() for k in KEYS})
    torch.cuda.synchronize()
    compare = {}
    for name in variants:
        if name == "parent":
            continue
        cmp = {}
        for k, v in outs[name].items():
            w = outs["parent"][k]
            if k in ("color", "depth", "alpha", "radii"):
                cmp[k + "_bit_equal"] = bool(torch.equal(v, w))
            else:
                diff = (v.double() - w.double()).abs()
                cmp[k] = dict(max_abs=float(diff.max()), max_abs_value=float(w.abs().max()), n_differ=int((v != w).sum()))
        compare[name] = cmp

    # ---- step times, alternating ----
    step_ms = {k: [] for k in variants}
    for _ in range(args.rounds):
        for name in variants:
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

    # ---- kernel times (profiled separately), alternating: each library at its own budget rule ----
    kern_us = {k: {} for k in libs}
    for _ in range(args.rounds):
        for name in kern_us:
            step(name)
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.profile_steps):
                    step(name)
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                if ev.device_time_total > 0:
                    kern_us[name].setdefault(ev.key[:90], []).append(ev.device_time_total / args.profile_steps)
    table = {}
    for name in kern_us:
        for k, v in kern_us[name].items():
            table.setdefault(k, {n: 0.0 for n in kern_us})[name] = round(float(np.median(v)), 1)
    table = dict(sorted(table.items(), key=lambda kv: -max(kv[1].values())))

    _, E_new = emitted("new")
    result = dict(tool="saturation_split_ab", gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w(), P=P,
                  instances=R_total, emitted=dict(parent=E_parent, new=E_new), rounds=args.rounds, steps=args.steps,
                  outputs=compare, step_ms={k: dict(runs=[round(x, 4) for x in v], median=round(float(np.median(v)), 4))
                                            for k, v in step_ms.items()},
                  kernels_us_per_step=table)
    print(json.dumps(result))
    return 0


if __name__ == "__main__":
    sys.exit(main())
