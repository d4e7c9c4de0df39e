"""Per-rank kernel time of the losses on a tile-row band (band_losses.py) against the whole-frame calls, on ONE GPU.

    python tools/band_loss_bench.py [--H 1280 --W 1920 --iters 50]

For emulated world sizes 1, 2, 4 and 8 (both layouts) every rank's stages run alone on its banded inputs and are timed with CUDA
events; the table gives the slowest rank (the step waits for it) beside the whole-frame photometric, sky and LiDAR calls.  The halo's
bytes per rank are computed from the shapes (fp32, both directions).  The collectives between the stages (one halo exchange, one
all-reduce of 5 doubles, four all-reduces of the LiDAR select of 8 KB each and one of 8 (1 + H/16) bytes) are NOT timed here: that
needs several GPUs under torchrun, and no number is estimated for them.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from street_gaussians_b200 import _capi, band_losses  # noqa: E402
from street_gaussians_b200._capi import ptr  # noqa: E402
from street_gaussians_b200.sharded import contiguous_band, cyclic_band  # noqa: E402


def timed(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=1280)
    ap.add_argument("--W", type=int, default=1920)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("band_loss_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    H, W = args.H, args.W
    g = torch.Generator(device=dev).manual_seed(0)
    img, gt = torch.rand(3, H, W, device=dev, generator=g), torch.rand(3, H, W, device=dev, generator=g)
    mask = (torch.rand(H * W, device=dev, generator=g) > 0.1).to(torch.uint8)
    acc = torch.rand(1, H, W, device=dev, generator=g)
    sky = (torch.rand(H * W, device=dev, generator=g) > 0.5).to(torch.uint8)
    lidar = torch.rand(1, H, W, device=dev, generator=g) * 50
    lidar[torch.rand(1, H, W, device=dev, generator=g) < 0.9] = 0.0
    depth = lidar + torch.randn(1, H, W, device=dev, generator=g)
    L = _capi.lib()

    nb = int(L.sgr_image_loss_scratch_bytes(3, H, W))
    scr = torch.empty(nb, device=dev, dtype=torch.uint8)
    grad, sc = torch.empty_like(img), torch.empty(4, device=dev)
    ga, sc2, s64 = torch.empty_like(acc), torch.empty(2, device=dev), torch.empty(64, device=dev, dtype=torch.uint8)
    nl = int(L.sgr_lidar_depth_loss_scratch_bytes(H * W))
    scl = torch.empty(nl, device=dev, dtype=torch.uint8)
    gd, gl, sc4 = torch.empty_like(depth), torch.empty_like(acc), torch.empty(4, device=dev)
    whole = dict(
        photometric=timed(lambda: _capi.call("sgr_image_loss", dev, 3, H, W, ptr(img), ptr(gt), ptr(mask), 0.8, -0.2, ptr(grad), ptr(sc),
                                             ptr(scr), nb), args.iters),
        sky=timed(lambda: _capi.call("sgr_sky_loss", dev, H * W, ptr(acc), ptr(sky), 1.0, ptr(ga), ptr(sc2), ptr(s64)), args.iters),
        lidar=timed(lambda: _capi.call("sgr_lidar_depth_loss", dev, H * W, ptr(depth), ptr(acc), ptr(lidar), ptr(mask), 0.95, 1.0, ptr(gd),
                                       ptr(gl), ptr(sc4), ptr(scl), nl), args.iters))

    rows_out = []
    for layout in ("cyclic", "contiguous"):
        for world in (1, 2, 4, 8):
            mk = cyclic_band if layout == "cyclic" else contiguous_band
            worst = dict(photometric=0.0, sky=0.0, lidar=0.0)
            halo_bytes = 0
            for r in range(world):
                band = mk(H, r, world)
                partials, scratch = band_losses.image_loss_stats(img, gt, mask, band)
                photo = lambda: (band_losses.image_loss_stats(img, gt, mask, band, partials),
                                 band_losses.image_loss_grad(img, gt, mask, band, 0.8, -0.2, partials, scratch))
                part = torch.empty(1, device=dev, dtype=torch.float64)
                skyf = lambda: band_losses.acc_loss_band("sgr_band_sky_loss", acc, sky, 1.0, band, True, part)

                def lid():
                    st, s = band_losses.lidar_keys(depth, acc, lidar, mask, band)
                    for lv in (1, 2):
                        band_losses.lidar_select(lv, 0.95, H, W, band, st, s)
                    sums = band_losses.lidar_select(3, 0.95, H, W, band, st, s)
                    band_losses.lidar_grad(depth, acc, lidar, 1.0, band, st, sums, s)

                for k, fn in (("photometric", photo), ("sky", skyf), ("lidar", lid)):
                    worst[k] = max(worst[k], timed(fn, args.iters))
                halo_bytes = max(halo_bytes, 4 * 3 * W * sum(band_losses.halo_rows(H, band, s) for s in range(4)))
            rows_out.append(dict(layout=layout, world=world, halo_bytes_per_rank=halo_bytes, **{f"{k}_ms_slowest_rank": v for k, v in worst.items()}))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu, H=H, W=W, whole_frame_ms=whole, bands=rows_out, collectives="not measured (needs several GPUs)"), indent=1))


if __name__ == "__main__":
    main()
