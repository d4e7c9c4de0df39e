"""Time of the composer's forward + backward under Gaussian sharding on one GPU, on a config-C-sized scene (1.5 M background + 8 x 50 k
actor Gaussians, SH degree 3, fourier_dim 5, flip mask, background pose correction):

  single      compose() of the whole scene (the single-GPU call, no reduction)
  p2p w1      compose(rasterizer=) at world 1: the accumulator rows staged and summed through a peer workspace of one rank
  nccl w1     compose(group=) at world 1: the rows, the (identity) all-reduce, the finalize
  p2p wN      N ranks emulated on N streams of this one GPU, each composing its 1/N of the rows, summed over emulated peer workspaces with
              device-side barriers; the time is for all N ranks together on one GPU, so it says nothing about N GPUs

    python tools/sharded_compose_bench.py [--reps 20] [--worlds 2 8] [--out sharded_compose_bench.json]

Times are CUDA events around forward + backward (after a synchronise), median over the repetitions after warm-up.  The card's name and
power limit are printed with the numbers.  No multi-GPU figure comes from this tool.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import compose_case as CC  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import sharded as SH  # noqa: E402

NAMES = ("xyz", "rotation", "scaling", "opacity", "features")
N_BG, ACTORS, M, FOURIER = 1_500_000, (50_000,) * 8, 16, 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def scene(dev):
    models = [{k: v.to(dev) for k, v in m.items()} for m in CC.make_case(0, N_BG, list(ACTORS), M, FOURIER)]
    g = torch.Generator().manual_seed(1)
    P = N_BG + sum(ACTORS)
    return dict(models=models, poses=torch.randn(len(ACTORS), 7, generator=g).to(dev), idft=torch.randn(len(ACTORS), FOURIER, generator=g).to(dev),
                flip=(torch.rand(sum(ACTORS), generator=g) < 0.5).to(dev), fq=torch.tensor([0.0, 0.0, 1.0, 0.0], device=dev),
                corr=((torch.tensor([1.0, 0, 0, 0]) + 0.1 * torch.randn(4, generator=g)).to(dev), torch.randn(3, generator=g).to(dev)),
                up={k: v.to(dev) for k, v in CC.upstream(2, P, M).items()}, P=P)


def rank_inputs(sc, B, r):
    """Leaves of rank r's rows [B[r], B[r+1]) of the model-major composed array, its flip rows and upstream rows."""
    loc, flip, at = [], [], 0
    for m, mod in enumerate(sc["models"]):
        n = int(mod["xyz"].shape[0])
        lo, hi = min(max(B[r] - at, 0), n), min(max(B[r + 1] - at, 0), n)
        loc.append({k: v[lo:hi].detach().clone().requires_grad_(True) for k, v in mod.items()})
        if m:
            flip.append(sc["flip"][at - N_BG + lo: at - N_BG + hi])
        at += n
    return loc, torch.cat(flip), [sc["up"][k][B[r]:B[r + 1]] for k in NAMES]


def step(sc, inputs, **kw):
    loc, flip, up = inputs
    poses = sc["poses"].clone().requires_grad_(True)
    cr, ct = (t.clone().requires_grad_(True) for t in sc["corr"])
    out = sgb.compose(loc, poses, sc["idft"], flip, sc["fq"], pose_correction=(cr, ct), **kw)
    torch.autograd.backward(list(out), up)


def settings(dev):
    z = torch.zeros(3, device=dev)
    return sgb.GaussianRasterizationSettings(32, 32, 0.5, 0.5, z, 1.0, torch.eye(4, device=dev), torch.eye(4, device=dev), 0, z, False, False)


def timed(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--worlds", type=int, nargs="*", default=[2, 8])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda")
    sc = scene(dev)
    res = dict(card=card(), P=sc["P"], actors=len(ACTORS))
    whole = rank_inputs(sc, [0, sc["P"]], 0)
    res["single_ms"] = timed(lambda: step(sc, whole), a.reps)
    ws1 = SH.PeerWorkspace.emulate(settings(dev), 8, 1, dev)[0]
    res["p2p_w1_ms"] = timed(lambda: step(sc, whole, rasterizer=types.SimpleNamespace(exchange="p2p", group=None, pose_workspace=lambda: ws1)),
                             a.reps)
    res["nccl_w1_ms"] = timed(lambda: step(sc, whole, group=types.SimpleNamespace()), a.reps)
    for world in a.worlds:
        wss = SH.PeerWorkspace.emulate(settings(dev), 8, world, dev)
        streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
        B = [sc["P"] * r // world for r in range(world + 1)]
        ins = [rank_inputs(sc, B, r) for r in range(world)]
        main_stream = torch.cuda.current_stream(dev)

        def emulated():
            for r in range(world):  # one thread issues every rank: nothing on the host waits, the barriers wait on the device
                streams[r].wait_stream(main_stream)
                with torch.cuda.stream(streams[r]):
                    step(sc, ins[r], rasterizer=types.SimpleNamespace(exchange="p2p", group=None, pose_workspace=lambda r=r: wss[r]))
            for s in streams:
                main_stream.wait_stream(s)

        res[f"p2p_w{world}_emulated_ms"] = timed(emulated, a.reps)
    print(f"card: {res['card']}")
    for k, v in res.items():
        if k.endswith("_ms"):
            print(f"{k:24s} {v:8.3f} ms")
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
