"""Time of scoring 50 views on ONE GPU: ViewMetrics against the reference's scoring lines restated as torch ops, and band scoring.

    python tools/eval_bench.py [--views 50 --reps 11]

Sizes: 1600 x 1066 (the reference's training-width cap, camera_utils.py:140) and 1920 x 1280.  Each row is the host time of one whole
scoring pass over the views, ending in the host read of its numbers: [median, min, max] over --reps passes after a warm-up pass.  These
passes are bound by the host work of the Python calls, so they vary with the host's load; they are not kernel times.  The kernel time of
the views' scoring is given separately: `device_ms_*` replays the accumulate calls of all views from one CUDA graph, timed with CUDA
events (median of 20 replays), which leaves the host out:
  view_metrics_train   ViewMetrics() add per view + result(): clamp, masked L1 / PSNR / SSIM, one read;
  torch_train_report   train.py:283-296 as torch ops: clamp, l1_loss and psnr with their boolean-index masking, summed per view;
  view_metrics_png     ViewMetrics(quantize8=True, ssim_masked=False): the save_image PNG round trip, unmasked SSIM and PSNR;
  torch_metrics_py     metrics.py:76-81 as torch ops on the 8-bit images (save_image's rounding, read back / 255): ssim (grouped
                       F.conv2d, 11x11 window) and psnr per view,
                       read as torch.tensor(list) like the reference;
  band_w{2,4,8}_slowest  the rank with the slowest median of an emulated cyclic world: per view the halo pack / unpack of its own sides and the band
                       accumulate, then the finish and one read.  The halo transfer and the all-reduce are NOT timed (they need several
                       GPUs under torchrun).
Prints one JSON line with the GPU's name and power limit beside the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from street_gaussians_b200 import _capi, band_losses, metrics  # noqa: E402
from street_gaussians_b200.sharded import cyclic_band  # noqa: E402

DEV = torch.device("cuda", 0)


def host_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()  # every pass ends in a host read
        ts.append((time.perf_counter() - t0) * 1e3)
    return [round(statistics.median(ts), 3), round(min(ts), 3), round(max(ts), 3)]


def device_time(imgs, gts, masks, flags, replays=20):
    """ms of the accumulate calls of all views replayed from one CUDA graph (CUDA events, median of `replays`)."""
    V = len(imgs)
    sums = torch.zeros(V, _capi.EVAL_SUMS, device=DEV, dtype=torch.float64)
    ms = [None if m is None else m.reshape(1, -1).to(torch.uint8) for m in masks]

    def body():
        for i in range(V):
            metrics.accumulate(imgs[i][None], gts[i][None], ms[i], sums[i:i + 1], flags)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        body()  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        body()
    times = []
    for _ in range(replays):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return round(statistics.median(times), 4)


# ---- the reference's lines, restated as torch ops ----
def _l1_loss(x, y, mask):
    x, y = x.permute(1, 2, 0), y.permute(1, 2, 0)
    m = mask.squeeze(0)
    return torch.abs(x[m] - y[m]).mean()


def _psnr(x, y, mask=None):
    x, y = x.permute(1, 2, 0), y.permute(1, 2, 0)
    if mask is not None:
        m = mask.squeeze(0)
        x, y = x[m], y[m]
    mse = torch.mean((x - y) ** 2)
    return 20 * torch.log10(1.0 / torch.sqrt(mse))


def _window(C):
    g = torch.tensor([float(torch.exp(torch.tensor(-(k - 5) ** 2 / 4.5))) for k in range(11)])
    g = g / g.sum()
    w = (g[:, None] @ g[None, :]).float()
    return w.expand(C, 1, 11, 11).contiguous().to(DEV)


def _ssim(x, y, win):
    C = x.shape[-3]
    mu1, mu2 = F.conv2d(x, win, padding=5, groups=C), F.conv2d(y, win, padding=5, groups=C)
    s11 = F.conv2d(x * x, win, padding=5, groups=C) - mu1 ** 2
    s22 = F.conv2d(y * y, win, padding=5, groups=C) - mu2 ** 2
    s12 = F.conv2d(x * y, win, padding=5, groups=C) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 ** 2 + mu2 ** 2 + C1) * (s11 + s22 + C2))).mean()


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=50)
    ap.add_argument("--reps", type=int, default=11)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench needs a CUDA device")
    V = args.views
    res = {"gpu": gpu_info(), "views": V}
    win = _window(3)
    for (W, H) in ((1600, 1066), (1920, 1280)):
        g = torch.Generator(device=DEV).manual_seed(0)
        imgs = [torch.rand(3, H, W, device=DEV, generator=g) * 1.1 - 0.05 for _ in range(V)]
        gts = [torch.rand(3, H, W, device=DEV, generator=g) for _ in range(V)]
        masks = [torch.rand(1, H, W, device=DEV, generator=g) > 0.1 for _ in range(V)]
        pngs = [torch.clamp(x, 0, 1).mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).float().div(255) for x in imgs]
        png_gts = [x.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).float().div(255) for x in gts]

        def vm_train():
            vm = metrics.ViewMetrics()
            for x, y, m in zip(imgs, gts, masks):
                vm.add(x, y, m)
            return vm.result()["mean"]["psnr"]

        def torch_train():
            l1_test, psnr_test = 0.0, 0.0
            for x, y, m in zip(imgs, gts, masks):
                image, gt = torch.clamp(x, 0.0, 1.0), torch.clamp(y, 0.0, 1.0)
                l1_test += _l1_loss(image, gt, m).mean().double()
                psnr_test += _psnr(image, gt, m).mean().double()
            return float(psnr_test / V), float(l1_test / V)

        def vm_png():
            vm = metrics.ViewMetrics(quantize8=True, ssim_masked=False)
            for x, y in zip(imgs, gts):
                vm.add(x, y)
            return vm.result()["mean"]["ssim"]

        def torch_png():
            ssims, psnrs = [], []
            for x, y in zip(pngs, png_gts):
                ssims.append(_ssim(x, y, win))
                psnrs.append(_psnr(x, y))
            return torch.tensor(ssims).mean().item(), torch.tensor(psnrs).mean().item()

        key = f"{W}x{H}"
        res[key] = {"view_metrics_train_ms": host_time(vm_train, args.reps), "torch_train_report_ms": host_time(torch_train, args.reps),
                    "view_metrics_png_ms": host_time(vm_png, args.reps), "torch_metrics_py_ms": host_time(torch_png, args.reps)}
        res[key]["device_ms_train"] = device_time(imgs, gts, masks, metrics._flags(True, False, True))
        res[key]["device_ms_png"] = device_time(imgs, gts, [None] * V, metrics._flags(True, True, False))
        # the two paths agree on the numbers they both compute
        res[key]["mean_psnr_view_metrics_vs_torch"] = [vm_train(), torch_train()[0]]
        res[key]["mean_ssim_png_view_metrics_vs_torch"] = [vm_png(), torch_png()[0]]
        for world in (2, 4, 8):
            per_rank = []
            for r in range(world):
                band = cyclic_band(H, r, world)
                rows = torch.zeros(H, dtype=torch.bool, device=DEV)
                for t in range(band.begin, band.end, band.step):
                    rows[16 * t:16 * t + 16] = True
                local = [torch.where(rows.view(1, -1, 1), x, torch.zeros_like(x)) for x in imgs]
                recv = {s: torch.zeros(3, band_losses.halo_rows(H, band, s), W, device=DEV) for s in (band_losses.RECV_UP, band_losses.RECV_DOWN)}
                flags = metrics._flags(True, False, True)

                def rank_pass():
                    sums = torch.zeros(V, _capi.EVAL_SUMS, device=DEV, dtype=torch.float64)
                    for i, (x, y, m) in enumerate(zip(local, gts, masks)):
                        img = x.clone()
                        for s in (band_losses.SEND_DOWN, band_losses.SEND_UP):
                            band_losses.halo_pack(img, band, s)
                        for s, buf in recv.items():
                            if buf.numel():
                                band_losses.halo_unpack(img, band, s, buf)
                        metrics.accumulate(img[None], y[None], m.reshape(1, -1).to(torch.uint8), sums[i:i + 1], flags, band)
                    return metrics.finish(sums).cpu()

                per_rank.append(host_time(rank_pass, args.reps))
            res[key][f"band_w{world}_slowest_ms"] = max(per_rank)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
