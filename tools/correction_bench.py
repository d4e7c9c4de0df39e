"""Times the background pose correction and the colour correction at config C (1.5 M background + 8 x 50 k actor Gaussians, M = 16,
1920x1280).  Arms, alternating call by call in one process, CUDA events around each call, median and p10-p90 of STEPS after WARMUP:
  compose            compose forward + backward without a correction
  compose_corrected  the same with pose_correction = (rot, trans)
  reference_torch    the reference's torch lines with the pose correction (compose_oracle + correct_gaussian_xyz / _rotation), which is
                     what a user who turns the correction on runs today
  color_correct      color_correct forward + backward on a 3x1280x1920 image
  color_einsum       the reference's einsum lines, forward + backward
Then, in a separate profiled run, the device time per call of each kernel (torch.profiler).  Prints one JSON line with the GPU name
and its enforced power limit.
python tools/correction_bench.py"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from layer_bench import alternate  # noqa: E402
from loss_bench import power_limit_w  # noqa: E402
import correction_oracle as CR  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import synthetic  # noqa: E402

DEV = "cuda"
KERNELS = ("compose_fwd_kernel", "compose_bwd_kernel", "compose_pose_finalize_kernel", "color_correct_fwd_kernel", "color_correct_bwd_kernel",
           "color_correct_finish_kernel")


def kernel_us(fn, calls=10):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key.split("(")[0].split("::")[-1].split("<")[0]
        if name in KERNELS:
            out[name] = out.get(name, 0.0) + ev.device_time_total / calls
    return out


def main():
    assert torch.cuda.is_available(), "tools/correction_bench.py needs a CUDA device"
    cfg = dict(synthetic.CONFIGS["C"])
    cfg.pop("kind")
    sc = synthetic.make_scene(seed=0, with_raw=True, **cfg)
    raw = sc["raw"]
    models = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in raw["models"]]
    poses, idft = raw["poses"].to(DEV).requires_grad_(True), raw["idft"].to(DEV)
    rot = torch.tensor([0.999, 0.01, -0.02, 0.015], device=DEV, requires_grad=True)
    trans = torch.tensor([0.05, -0.02, 0.03], device=DEV, requires_grad=True)
    P = sum(int(m["xyz"].shape[0]) for m in models)
    M = int(models[0]["features_rest"].shape[1]) + 1
    g = torch.Generator(device=DEV).manual_seed(1)
    up = [torch.randn(s, generator=g, device=DEV) for s in ((P, 3), (P, 4), (P, 3), (P, 1), (P, M, 3))]
    H, W = 1280, 1920
    img = torch.rand(3, H, W, generator=g, device=DEV, requires_grad=True)
    gimg = torch.randn(3, H, W, generator=g, device=DEV)
    aff = (torch.eye(4, device=DEV)[:3] + 0.05 * torch.randn(3, 4, generator=g, device=DEV)).requires_grad_(True)
    leaves = [v for m in models for v in m.values()] + [poses, rot, trans, img, aff]

    def clear():
        for x in leaves:
            x.grad = None

    def compose(corr):
        def run():
            clear()
            out = sgb.compose(models, poses, idft, pose_correction=(rot, trans) if corr else None)
            torch.autograd.backward(list(out), up)
        return run

    def reference():
        clear()
        o = CR.compose(models, poses, idft, None, None, (rot, trans))
        torch.autograd.backward([o[k] for k in CR.NAMES], up)

    def color(fn):
        def run():
            clear()
            fn(img, aff).backward(gimg)
        return run

    # outputs agree before anything is timed
    with torch.no_grad():
        a = sgb.compose(models, poses, idft, pose_correction=(rot, trans))
        b = CR.compose(models, poses, idft, None, None, (rot, trans))
        comp_err = max(float((x - b[k]).abs().max()) for x, k in zip(a, CR.NAMES))
        cc_err = float((sgb.color_correct(img, aff) - CR.color(img, aff)).abs().max())
    del a, b
    arms = dict(compose=compose(False), compose_corrected=compose(True), reference_torch=reference, color_correct=color(sgb.color_correct),
                color_einsum=color(CR.color))
    times = alternate(list(arms.values()))
    res = dict(gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w(), P=P, M=M, image=[3, H, W], max_abs_diff_compose=comp_err,
               max_abs_diff_color=cc_err, ms={k: t for k, t in zip(arms, times)})
    res["kernel_us"] = {k: kernel_us(arms[k]) for k in ("compose", "compose_corrected", "color_correct")}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
