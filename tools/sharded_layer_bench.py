"""Render layers in the fused Gaussian-sharded step, timed on ONE GPU with the ranks EMULATED.

    python tools/sharded_layer_bench.py [--steps 10] [--out FILE]

Config C (1.5 M background rows and 8 actors of 50 k rows, 1920x1280, SH 3) split rank-major over world = 1, 2, 4 and 8 emulated ranks,
each on its own stream of one GPU with its own peer workspace.  A step is every rank's fused forward + backward (sgr_sharded_forward /
_backward) without a layer, or with the objects layer (each rank's actor rows, bg white, an upstream gradient on its alpha as the
object-accumulation loss gives it: sgr_sharded_forward_layers / _backward_layers).  The two variants alternate step by step after two
warm-up steps each; CUDA events around each whole step, median and p10-p90 of --steps steps.  All ranks share one H100, so a time is the
sum of the ranks' work (and their barrier waits) on one card, not what N cards reach together.  The card's name and power limit are read
in the same run.  Extra peer memory per rank, by arithmetic: 48 B x P_total per layer + 1 B x P_total."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import sharded as SH  # noqa: E402
from street_gaussians_b200 import synthetic  # noqa: E402
from street_gaussians_b200.rasterizer import _forward_impl  # noqa: E402
import util  # noqa: E402


def run_world(scene, st, world, steps, dev):
    P = int(scene["means3D"].shape[0])
    n_bkgd = P - 8 * 50_000
    chunk = -(-P // world)
    P_r = [max(0, min(chunk, P - r * chunk)) for r in range(world)]
    offs = [r * chunk for r in range(world)]
    keys = ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")
    part = lambda k, lo, hi: None if scene.get(k) is None else scene[k][lo:hi].to(dev).contiguous()
    locs = [SH._local_tensors(*(part(k, offs[r], offs[r] + P_r[r]) for k in keys[:3]), None, *(part(k, offs[r], offs[r] + P_r[r]) for k in keys[3:]))
            for r in range(world)]
    ranges = [(min(P_r[r], max(0, n_bkgd - offs[r])), P_r[r]) for r in range(world)]
    with torch.no_grad():
        R = int(_forward_impl(*(part(k, 0, P) for k in keys[:3]), None, *(part(k, 0, P) for k in keys[3:]), st, None, None)[5].num_instances)
    capacity = R + R // 4 + 4096
    wss = SH.PeerWorkspace.emulate(st, chunk, world, dev, layers=1)
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    up = [scene[k].to(dev) for k in ("grad_color", "grad_depth", "grad_alpha")]
    zc, zd = torch.zeros_like(up[0]), torch.zeros_like(up[1])
    white = torch.ones(3, device=dev)
    sinks = [torch.empty((e - b, 3), device=dev) for b, e in ranges]
    band = lambda r: SH.cyclic_band(int(st.image_height), r, world) if world > 1 else None

    def step(layered):
        outs = []
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                lay = [(ranges[r][0], ranges[r][1], white)] if layered else None
                outs.append(SH.sharded_forward_raw(st, band(r), wss[r], locs[r], P_r[r], capacity, -1, layers=lay))
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                o = outs[r]
                lay = [(ranges[r][0], ranges[r][1], white, o[4][0][2], (zc, zd, up[2]), sinks[r])] if layered else None
                SH.sharded_backward_raw(st, band(r), wss[r], locs[r], P_r[r], capacity, o[2], *up, layers=lay)

    times = {False: [], True: []}
    with torch.no_grad():
        for i in range(2 * steps + 4):
            layered = bool(i % 2)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(layered)
            for s in streams:
                torch.cuda.current_stream().wait_stream(s)
            b.record()
            torch.cuda.synchronize()
            if i >= 4:
                times[layered].append(a.elapsed_time(b))
    q = lambda v: dict(median_ms=round(statistics.median(v), 3), p10_ms=round(sorted(v)[len(v) // 10], 3),
                       p90_ms=round(sorted(v)[(9 * len(v)) // 10], 3))
    P_total = chunk * world
    return dict(world=world, chunk=chunk, plain=q(times[False]), objects_layer=q(times[True]),
                extra_peer_bytes_per_rank=48 * P_total + P_total)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    scene = synthetic.make_config("C", seed=0)
    st = util.settings_from(sgb, scene["cam"], dev)
    res = dict(card=card, note="ranks emulated on streams of ONE GPU; a step = every rank's fused forward + backward",
               worlds=[run_world(scene, st, w, args.steps, dev) for w in (1, 2, 4, 8)])
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
