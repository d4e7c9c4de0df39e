"""Per-rank kernel time of the sky composite and the colour correction on a tile-row band against the whole-frame calls, on ONE GPU.

    python tools/band_image_bench.py [--H 1280 --W 1920 --R 1024 --iters 50]

For emulated world sizes 1, 2, 4 and 8 (both layouts) every rank's band calls run alone on its banded inputs and are timed with CUDA
events, each stage forward + backward (the sky with the SGR_SKY_MASK_GIVEN rule and the cube gradient, the colour correction with its
12 partial sums and the finishing call); the table gives the slowest rank (the step waits for it) beside the whole-frame calls.  Each time
includes the host cost of the ctypes calls.  The collectives between a rank's backward and the optimiser are NOT timed here: the
all-reduce of the dense 6 R^2 3 fp32 cube gradient (75 MB at R = 1024) and of the 12 doubles of the affine.  That needs several GPUs
under torchrun, and no number is estimated for them.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from street_gaussians_b200 import _capi  # noqa: E402
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
    ap.add_argument("--R", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("band_image_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    H, W, R = args.H, args.W, args.R
    g = torch.Generator(device=dev).manual_seed(0)
    rgb, up = torch.rand(3, H, W, device=dev, generator=g), torch.randn(3, H, W, device=dev, generator=g)
    acc = torch.rand(1, H, W, device=dev, generator=g)
    acc = torch.where(torch.rand(1, H, W, device=dev, generator=g) < 0.4, torch.zeros_like(acc), acc)
    mask = (torch.rand(H, W, device=dev, generator=g) < 0.3).to(torch.uint8)
    cube = torch.rand(6, R, R, 3, device=dev, generator=g)
    K = torch.tensor([[1.07 * W, 0.0, W / 2], [0.0, 1.07 * W, H / 2], [0.0, 0.0, 1.0]], device=dev)
    w2c = torch.eye(4, device=dev)
    A = torch.eye(4, device=dev)[:3] + 0.05 * torch.randn(3, 4, device=dev, generator=g)
    out, gimg, gacc, gcube = torch.empty_like(rgb), torch.empty_like(rgb), torch.empty_like(acc), torch.zeros_like(cube)
    gA, sums = torch.empty(3, 4, device=dev), torch.empty(12, device=dev, dtype=torch.float64)
    L = _capi.lib()
    nb = int(L.sgr_color_correct_scratch_bytes(H, W))
    scr = torch.empty(nb, device=dev, dtype=torch.uint8)
    nbb = int(L.sgr_band_color_correct_scratch_bytes(H, W))
    scrb = torch.empty(nbb, device=dev, dtype=torch.uint8)
    mode = _capi.SKY_MASK_GIVEN

    def sky_whole():
        _capi.call("sgr_sky_composite_forward", dev, H, W, R, mode, 1.0, ptr(rgb), ptr(acc), ptr(mask), ptr(cube), ptr(K), ptr(w2c), None, None,
                   ptr(out))
        _capi.call("sgr_sky_composite_backward", dev, H, W, R, mode, 1.0, ptr(acc), ptr(mask), ptr(cube), ptr(K), ptr(w2c), None, None, ptr(up),
                   ptr(gacc), ptr(gcube))

    def cc_whole():
        _capi.call("sgr_color_correct_forward", dev, H, W, ptr(rgb), ptr(A), ptr(out))
        _capi.call("sgr_color_correct_backward", dev, H, W, ptr(rgb), ptr(A), ptr(up), ptr(gimg), ptr(gA), ptr(scr), nb)

    whole = dict(sky=timed(sky_whole, args.iters), color_correct=timed(cc_whole, args.iters))

    rows_out = []
    for layout in ("cyclic", "contiguous"):
        for world in (1, 2, 4, 8):
            mk = cyclic_band if layout == "cyclic" else contiguous_band
            worst = dict(sky=0.0, color_correct=0.0)
            for r in range(world):
                b, e, s = mk(H, r, world)

                def sky_band():
                    _capi.call("sgr_band_sky_composite_forward", dev, H, W, b, e, s, R, mode, 1.0, ptr(rgb), ptr(acc), ptr(mask), ptr(cube), ptr(K),
                               ptr(w2c), None, None, ptr(out))
                    _capi.call("sgr_band_sky_composite_backward", dev, H, W, b, e, s, R, mode, 1.0, ptr(acc), ptr(mask), ptr(cube), ptr(K), ptr(w2c),
                               None, None, ptr(up), ptr(gacc), ptr(gcube))

                def cc_band():
                    _capi.call("sgr_band_color_correct_forward", dev, H, W, b, e, s, ptr(rgb), ptr(A), ptr(out))
                    _capi.call("sgr_band_color_correct_backward", dev, H, W, b, e, s, ptr(rgb), ptr(A), ptr(up), ptr(gimg), ptr(sums), ptr(scrb), nbb)
                    _capi.call("sgr_band_color_correct_affine_grad", dev, ptr(sums), ptr(gA))

                worst["sky"] = max(worst["sky"], timed(sky_band, args.iters))
                worst["color_correct"] = max(worst["color_correct"], timed(cc_band, args.iters))
            rows_out.append(dict(layout=layout, world=world, **{f"{k}_ms_slowest_rank": v for k, v in worst.items()}))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu, H=H, W=W, R=R, whole_frame_ms=whole, bands=rows_out,
                          collectives="not measured (needs several GPUs): cube gradient all-reduce of 6 R^2 3 fp32, affine sums of 12 doubles"),
                     indent=1))


if __name__ == "__main__":
    main()
