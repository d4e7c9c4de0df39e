"""Kernel time of the band losses over peer memory (band_losses.frame_losses + lidar_depth_loss with rasterizer= of a p2p rasterizer),
with the ranks EMULATED on ONE GPU, beside the whole-frame calls.

    python tools/band_loss_p2p_bench.py [--H 1280 --W 1920 --steps 10]

For world 1, 2, 4 and 8 (cyclic bands) the ranks run as threads on streams of one GPU over PeerWorkspace.emulate (as
tests/test_band_losses_p2p_gpu.py does); one step is the photometric, sky and object-accumulation losses (one halo exchange, one sum of
five doubles) and the LiDAR loss (four sums) of every rank.  torch.profiler's kernel records give, per rank and step: the time of the new
exchange kernels (halo copies, the sums' stage and add kernels), the barrier kernels (which, emulated, mostly wait for the other ranks'
work on the same GPU), and every kernel of the step.  The whole-frame calls (sgr_image_loss, sgr_sky_loss, sgr_obj_acc_loss,
sgr_lidar_depth_loss) are profiled the same way.  These are emulated, single-GPU numbers, not a multi-GPU time: NVLink traffic and
the barriers' cost across GPUs are not measured.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import types
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
from street_gaussians_b200 import band_losses, losses  # noqa: E402
from street_gaussians_b200 import sharded as SH  # noqa: E402
from street_gaussians_b200.rasterizer import GaussianRasterizationSettings  # noqa: E402
from rank_threads import run_ranks  # noqa: E402

GROUPS = (("halo", ("halo_copy_kernel",)), ("sum", ("loss_stage_kernel", "loss_sum_kernel")), ("barrier", ("peer_barrier_kernel",)))


def kernel_ms(fn):
    """Run fn under torch.profiler; {kernel name: total device ms} from the trace's kernel records."""
    with tempfile.TemporaryDirectory() as d:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    out = defaultdict(float)
    for e in trace.get("traceEvents", []):
        if e.get("cat") == "kernel":
            out[e["name"]] += e.get("dur", 0.0) / 1000.0
    return out


def grouped(ms):
    res = {g: sum(v for k, v in ms.items() if any(n in k for n in names)) for g, names in GROUPS}
    res["all_kernels"] = sum(ms.values())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=1280)
    ap.add_argument("--W", type=int, default=1920)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("band_loss_p2p_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    H, W, K = args.H, args.W, args.steps
    g = torch.Generator(device=dev).manual_seed(0)
    img, gt = torch.rand(3, H, W, device=dev, generator=g), torch.rand(3, H, W, device=dev, generator=g)
    mask = torch.rand(1, H, W, device=dev, generator=g) > 0.1
    acc = torch.rand(1, H, W, device=dev, generator=g)
    sky = torch.rand(1, H, W, device=dev, generator=g) > 0.5
    obj = torch.rand(1, H, W, device=dev, generator=g) > 0.7
    lidar = torch.rand(1, H, W, device=dev, generator=g) * 50
    lidar[torch.rand(1, H, W, device=dev, generator=g) < 0.9] = 0.0
    depth = lidar + torch.randn(1, H, W, device=dev, generator=g)
    z = torch.zeros(3, device=dev)
    st = GaussianRasterizationSettings(H, W, 0.5, 0.5, z, 1.0, torch.eye(4, device=dev), torch.eye(4, device=dev), 0, z, False, False)

    def whole():
        for _ in range(K):
            losses.photometric_loss(img, gt, mask), losses.sky_loss(acc, sky), losses.obj_acc_loss(acc, obj)
            losses.lidar_depth_loss(depth, acc, lidar, mask)

    whole()
    # every exchange kernel loaded before emulated ranks spin (see tests/test_band_losses_p2p_gpu._warm_up): the halo copies directly,
    # then the sums and the barrier of two ranks enqueued one after the other from this thread
    b = SH.cyclic_band(H, 0, 2)
    for side in (band_losses.SEND_UP, band_losses.SEND_DOWN):
        band_losses.halo_pack(img, b, side)
    for side in (band_losses.RECV_UP, band_losses.RECV_DOWN):
        band_losses.halo_unpack(img.clone(), b, side, torch.zeros(3, band_losses.halo_rows(H, b, side), W, device=dev))
    pair = SH.PeerWorkspace.emulate(st, 8, 2, dev)
    pst = [torch.cuda.Stream(device=dev) for _ in range(2)]
    tw = [(torch.zeros(5, device=dev, dtype=torch.float64), torch.zeros(5, device=dev, dtype=torch.int32)) for _ in range(2)]
    torch.cuda.synchronize()
    for r in range(2):
        with torch.cuda.stream(pst[r]):
            for t in tw[r]:
                band_losses.peer_sum(pair[r], t)
    torch.cuda.synchronize()
    res = dict(whole_frame=grouped(kernel_ms(whole)))
    res["whole_frame"] = {k: v / K for k, v in res["whole_frame"].items()}
    rows = []
    for world in (1, 2, 4, 8):
        wss = SH.PeerWorkspace.emulate(st, 8, world, dev)
        bands = [SH.cyclic_band(H, r, world) if world > 1 else None for r in range(world)]
        ris = [types.SimpleNamespace(exchange="p2p", group=None, band=bands[r], loss_workspace=(lambda w=wss[r]: w)) for r in range(world)]
        own = [SH.band_of_rows(H, r, world).to(dev).view(1, H, 1) for r in range(world)]
        ins = [[torch.where(own[r], t, torch.zeros_like(t)) for t in (img, acc, depth)] for r in range(world)]
        streams = [torch.cuda.Stream(device=dev) for _ in range(world)]

        def steps(n):
            def rank(r, _tr):
                x, a, d = ins[r]
                with torch.cuda.stream(streams[r]):
                    for _ in range(n):
                        band_losses.frame_losses(x, gt, mask, acc=a, sky_mask=sky, acc_obj=a, obj_bound=obj, rasterizer=ris[r])
                        band_losses.lidar_depth_loss(d, a, lidar, mask, rasterizer=ris[r])
            torch.cuda.synchronize()
            run_ranks(world, rank)
            torch.cuda.synchronize()

        steps(2)  # warm: every kernel loaded, the allocator's blocks in place
        ms = grouped(kernel_ms(lambda: steps(K)))
        rows.append(dict(world=world, **{f"{k}_ms_per_rank_step": v / (K * world) for k, v in ms.items()}))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu, tool="torch.profiler kernel records", H=H, W=W, steps=K, whole_frame_ms_per_step=res["whole_frame"],
                          p2p_emulated=rows, note="emulated on one GPU, not a multi-GPU time; barrier time is mostly waiting for the "
                          "other emulated ranks"), indent=1))


if __name__ == "__main__":
    main()
