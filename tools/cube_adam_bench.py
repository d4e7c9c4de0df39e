"""Times the sky cube map's optimizer step at R = 1024 (the reference's default model.sky.resolution, [6, 1024, 1024, 3] = 18.9 M
floats): the dense training.FusedAdam against the block-masked training.CubeMapSparseAdam.

Block maps come from real sky composites of a 1920x1280 frame (Waymo-like K, a sky mask over half the frame, jittered), backward with
sky_composite(blocks=), with the camera yawed by 0, 90, 180 and 270 degrees about the vertical axis, plus the all-marked map.  For each
map: CUDA events around each step() call (host work included), the two optimizers alternating call by call, median and p10-p90 of
STEPS calls after WARMUP; the map is refilled before each masked call, outside the timed window.  lr = 0, so every call moves the same
bytes and the cube stays put; after the timed calls the two optimizers' exp_avg and exp_avg_sq must be equal bit for bit on the marked
blocks (same gradient, same step count).  Then each kernel's device time from torch.profiler in a separate run.  Bytes are the
algorithmic traffic: 28 B per float for the dense step, 1 B per block + 28 B per float of a marked block for the masked one.

Then the composed training step at config B's scene (500 k Gaussians, SH degree 3, 1920x1280: compose -> rasterize -> sky(blocks=) ->
color_correct -> photometric + sky loss -> backward -> the cube's optimizer step) with each optimizer for the cube, alternating.  Prints
one JSON line with the GPU name and its enforced power limit.
python tools/cube_adam_bench.py"""
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from layer_bench import alternate  # noqa: E402
from loss_bench import power_limit_w  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import losses, sky, synthetic  # noqa: E402
from street_gaussians_b200.training import CubeMapSparseAdam, FusedAdam  # noqa: E402

DEV = "cuda"
H, W, RES = 1280, 1920, 1024
YAWS = (0, 90, 180, 270)
STEPS, WARMUP = 100, 10
KERNELS = ("adam_kernel", "cube_sparse_adam_kernel")


def look_at(yaw_deg):
    """w2c of a camera at the origin looking along (1, -1, 1) turned by yaw_deg about the world's y axis: it sees three cube faces."""
    a = math.radians(yaw_deg)
    d = torch.tensor([math.cos(a) + math.sin(a), -1.0, -math.sin(a) + math.cos(a)])
    z = d / d.norm()
    x = torch.linalg.cross(torch.tensor([0.0, 1.0, 0.0]), z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    w2c = torch.eye(4)
    w2c[:3, :3] = torch.stack([x, y, z], 1).T
    return w2c.to(DEV)


def frame_map(yaw, K, rgb, acc, mask, up):
    cube = torch.full((6, RES, RES, 3), 0.5, device=DEV, requires_grad=True)
    blocks = sky.block_map(RES, DEV)
    sgb.sky_composite(rgb, acc, cube, K, look_at(yaw), sky_mask=mask, perturb=True, blocks=blocks).backward(up)
    return blocks


def events_ms(fn, before=None):
    if before is not None:
        before()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def stats(t):
    return dict(median_ms=float(np.median(t)), p10_ms=float(np.percentile(t, 10)), p90_ms=float(np.percentile(t, 90)))


def kernel_us(fn, before, calls=10):
    out = {k: 0.0 for k in KERNELS}
    before()
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            before()
            fn()
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        name = ev.key.split("(")[0].split("::")[-1].split("<")[0]
        if name in out:
            out[name] += ev.device_time_total / calls
    return out


def main():
    assert torch.cuda.is_available(), "tools/cube_adam_bench.py needs a CUDA device"
    g = torch.Generator(device=DEV).manual_seed(0)
    K = torch.tensor([[2055.6, 0.0, 939.7], [0.0, 2051.3, 641.1], [0.0, 0.0, 1.0]], device=DEV)
    rgb = torch.rand(3, H, W, generator=g, device=DEV)
    acc = torch.rand(1, H, W, generator=g, device=DEV)
    mask = torch.rand(1, H, W, generator=g, device=DEV) < 0.5
    up = torch.randn(3, H, W, generator=g, device=DEV)
    maps = {f"yaw_{y}": frame_map(y, K, rgb, acc, mask, up) for y in YAWS}
    maps["all_marked"] = torch.ones_like(maps["yaw_0"])
    nb = -(-RES // 32)
    tb = torch.arange(6 * nb * nb, device=DEV).view(6, nb, 1, nb, 1).expand(6, nb, 32, nb, 32).reshape(6, nb * 32, nb * 32)[:, :RES, :RES]
    floats = 18 * RES * RES
    res = dict(gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w(), resolution=RES, image=[3, H, W], maps={})
    for name, saved in maps.items():
        pd = torch.nn.Parameter(0.2 * torch.randn(6, RES, RES, 3, generator=g, device=DEV))
        ps = torch.nn.Parameter(pd.detach().clone())
        pd.grad = torch.randn(6, RES, RES, 3, generator=g, device=DEV)
        ps.grad = pd.grad.clone()
        dense, masked = FusedAdam([pd], lr=0.0, eps=1e-15), CubeMapSparseAdam([ps], lr=0.0, eps=1e-15)
        blocks = saved.clone()
        refill = lambda: blocks.copy_(saved)  # noqa: E731
        td, ts = [], []
        for it in range(WARMUP + STEPS):
            a = events_ms(dense.step)
            b = events_ms(lambda: masked.step(blocks), refill)
            if it >= WARMUP:
                td.append(a)
                ts.append(b)
        torch.cuda.synchronize()
        marked = saved.bool()[tb].unsqueeze(-1).expand(6, RES, RES, 3)
        same = all(torch.equal(dense.state[pd][k].view(torch.int32)[marked], masked.state[ps][k].view(torch.int32)[marked])
                   for k in ("exp_avg", "exp_avg_sq"))
        n_marked = int(saved.bool().sum())
        marked_floats = int(marked.sum())
        kd = kernel_us(dense.step, lambda: None)
        ks = kernel_us(lambda: masked.step(blocks), refill)
        dense_bytes, masked_bytes = 28 * floats, saved.numel() + 28 * marked_floats
        res["maps"][name] = dict(
            blocks_marked=n_marked, blocks=saved.numel(), fraction=n_marked / saved.numel(), moments_equal_on_marked=same,
            fused_adam=dict(step=stats(td), kernel_us=kd["adam_kernel"], bytes=dense_bytes,
                            tb_per_s=dense_bytes / (kd["adam_kernel"] * 1e-6) / 1e12 if kd["adam_kernel"] else None),
            cube_sparse_adam=dict(step=stats(ts), kernel_us=ks["cube_sparse_adam_kernel"], bytes=masked_bytes,
                                  tb_per_s=masked_bytes / (ks["cube_sparse_adam_kernel"] * 1e-6) / 1e12 if ks["cube_sparse_adam_kernel"] else None))
        del pd, ps, dense, masked

    # config B's composed training step with the sky, the cube stepped by each optimizer
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
    cubes = {k: torch.nn.Parameter(0.999 * torch.ones(6, RES, RES, 3, device=DEV)) for k in ("fused_adam", "cube_sparse_adam")}
    opts = dict(fused_adam=FusedAdam([cubes["fused_adam"]], lr=0.0, eps=1e-15),
                cube_sparse_adam=CubeMapSparseAdam([cubes["cube_sparse_adam"]], lr=0.0, eps=1e-15))
    blocks = sky.block_map(RES, DEV)
    params = [v for m in models for v in m.values()] + [affine]

    def step(kind):
        cube, opt = cubes[kind], opts[kind]

        def run():
            for p in params + [cube]:
                p.grad = None
            xyz, rot, scale, opac, sh = sgb.compose(models, poses, idft)
            m2d = torch.zeros_like(xyz, requires_grad=True)
            out = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot)
            col, a_ = out[0], out[3]
            col = sgb.sky_composite(col, a_, cube, Ks, w2cs, sky_mask=smask, perturb=True,
                                    blocks=blocks if kind == "cube_sparse_adam" else None)
            col = sgb.color_correct(col, affine)
            loss = losses.photometric_loss(col, gt, None, 1.0, 0.2) + losses.sky_loss(a_, lmask, 1.0)
            loss.backward()
            if kind == "cube_sparse_adam":
                opt.step(blocks)
            else:
                opt.step()
        return run

    t = alternate([step("fused_adam"), step("cube_sparse_adam")], iters=30, warmup=5)
    res["config_b_step_ms"] = dict(fused_adam=t[0], cube_sparse_adam=t[1], P=sum(int(m["xyz"].shape[0]) for m in models), image=[3, Hs, Ws])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
