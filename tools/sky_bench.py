"""Times the sky cube map composite at 1920x1280 with R = 1024 (the reference's default model.sky.resolution), Waymo-like K, a camera
that sees three cube faces, a sky mask over half the frame (training shape, jittered).  Arms, alternating call by call in one process,
CUDA events around each call, median and p10-p90 of STEPS after WARMUP, forward + backward each:
  sky_composite      street_gaussians_b200.sky_composite
  torch_restatement  the reference's torch lines with the restated cube lookup in fp32 torch (tests/sky_oracle.composite).  It is not
                     nvdiffrast, which is not available to time here; no comparison with nvdiffrast is made.
Then a separately profiled run with the device time per call of each sky kernel (torch.profiler), and the composed training step
(compose -> rasterize -> sky -> color_correct -> photometric + sky loss -> backward) at config B's scene (500 k Gaussians, SH degree 3)
with and without the sky, alternating.  Prints one JSON line with the GPU name and its enforced power limit.
python tools/sky_bench.py"""
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
import sky_oracle as SO  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import losses, synthetic  # noqa: E402

DEV = "cuda"
H, W, RES = 1280, 1920, 1024
KERNELS = ("sky_composite_fwd_kernel", "sky_composite_bwd_kernel")


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


def look_at(target):
    z = torch.tensor(target)
    z = z / z.norm()
    x = torch.linalg.cross(torch.tensor([0.0, 1.0, 0.0]), z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    w2c = torch.eye(4)
    w2c[:3, :3] = torch.stack([x, y, z], 1).T
    return w2c.to(DEV)


def main():
    assert torch.cuda.is_available(), "tools/sky_bench.py needs a CUDA device"
    g = torch.Generator(device=DEV).manual_seed(0)
    K = torch.tensor([[2055.6, 0.0, 939.7], [0.0, 2051.3, 641.1], [0.0, 0.0, 1.0]], device=DEV)
    w2c = look_at([1.0, -1.0, 1.0])
    cube = (0.999 * torch.ones(6, RES, RES, 3, device=DEV)).requires_grad_(True)
    rgb = torch.rand(3, H, W, generator=g, device=DEV, requires_grad=True)
    acc = torch.rand(1, H, W, generator=g, device=DEV, requires_grad=True)
    mask = torch.rand(1, H, W, generator=g, device=DEV) < 0.5
    up = torch.randn(3, H, W, generator=g, device=DEV)
    leaves = (cube, rgb, acc)

    def arm(fn):
        def run():
            for x in leaves:
                x.grad = None
            fn().backward(up)
        return run

    def ours():
        return sgb.sky_composite(rgb, acc, cube, K, w2c, sky_mask=mask, perturb=True)

    def torch_restatement():
        jx = torch.rand(H, W, device=DEV)
        jy = torch.rand(H, W, device=DEV)
        return SO.composite(rgb, acc, cube, K, w2c, mask, jx, jy, 1.0)

    with torch.no_grad():  # the arms agree before anything is timed
        torch.manual_seed(1)
        a = ours()
        torch.manual_seed(1)
        b = torch_restatement()
        diff = float((a - b).abs().max())
    del a, b
    arms = dict(sky_composite=arm(ours), torch_restatement=arm(torch_restatement))
    times = alternate(list(arms.values()))
    res = dict(gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w(), image=[3, H, W], resolution=RES, max_abs_diff=diff,
               ms={k: t for k, t in zip(arms, times)}, kernel_us=kernel_us(arms["sky_composite"]))

    # the composed training step with and without the sky
    cfg = dict(synthetic.CONFIGS["B"])
    cfg.pop("kind")
    sc = synthetic.make_scene(seed=0, with_raw=True, **cfg)
    raw, cam = sc["raw"], sc["cam"]
    st = sgb.GaussianRasterizationSettings(image_height=cam["image_height"], image_width=cam["image_width"], tanfovx=cam["tanfovx"],
                                           tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=DEV), scale_modifier=1.0,
                                           viewmatrix=cam["viewmatrix"].to(DEV), projmatrix=cam["projmatrix"].to(DEV), sh_degree=cam["sh_degree"],
                                           campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    Hs, Ws = cam["image_height"], cam["image_width"]
    Ks = torch.tensor([[Ws / (2 * cam["tanfovx"]), 0, Ws / 2], [0, Hs / (2 * cam["tanfovy"]), Hs / 2], [0, 0, 1.0]], device=DEV)
    w2cs = cam["viewmatrix"].to(DEV).T.contiguous()
    models = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in raw["models"]]
    poses, idft = raw["poses"].to(DEV), raw["idft"].to(DEV)
    gt = torch.rand(3, Hs, Ws, generator=g, device=DEV)
    smask = torch.rand(1, Hs, Ws, generator=g, device=DEV) < 0.3
    lmask = smask.clone()
    lmask[:, :50] = True
    affine = (torch.eye(4, device=DEV)[:3] + 0.05 * torch.randn(3, 4, generator=g, device=DEV)).requires_grad_(True)
    rast = sgb.GaussianRasterizer(st)
    params = [v for m in models for v in m.values()] + [cube, affine]

    def step(with_sky):
        def run():
            for p in params:
                p.grad = None
            xyz, rot, scale, opac, sh = sgb.compose(models, poses, idft)
            m2d = torch.zeros_like(xyz, requires_grad=True)
            out = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot)
            col, a_ = out[0], out[3]
            if with_sky:
                col = sgb.sky_composite(col, a_, cube, Ks, w2cs, sky_mask=smask, perturb=True)
            col = sgb.color_correct(col, affine)
            loss = losses.photometric_loss(col, gt, None, 1.0, 0.2) + losses.sky_loss(a_, lmask, 1.0)
            loss.backward()
        return run

    st_times = alternate([step(True), step(False)], iters=30, warmup=5)
    res["step_ms"] = dict(with_sky=st_times[0], without_sky=st_times[1], P=sum(int(m["xyz"].shape[0]) for m in models), image=[3, Hs, Ws])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
