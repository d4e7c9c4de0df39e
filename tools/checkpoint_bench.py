"""Time sharded.save_checkpoint and sharded.load_checkpoint of config C (1.5M background + 8 x 50k actors, SH degree 3, every parameter
with Adam moments) with the ranks emulated by threads on ONE GPU (tests/rank_threads.py), and report the device bytes the save adds at
its peak.  The emulated ranks share one device and one stream, so these times include no cross-GPU traffic: they measure the packing, the
device-to-host copies, the host assembly, torch.save and the sliced torch.load.

    python tools/checkpoint_bench.py [--world 8] [--piece-mib 1024] [--dir /tmp]
"""
import argparse
import os
import sys
import tempfile
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from rank_threads import run_ranks  # noqa: E402
from street_gaussians_b200 import sharded as SH, training  # noqa: E402

NAMES = training.PARAM_NAMES


def config_c(world, dev):
    """Per rank, the even split of config C's rows, with FusedAdam state and statistics filled."""
    sizes = [1_500_000] + [50_000] * 8
    slices = SH.even_slices(sizes, world)
    shards, opts = [], []
    for r in range(world):
        objs = []
        for k, n in enumerate(sizes):
            lo, hi = slices[r][k]
            m = hi - lo
            o = types.SimpleNamespace(_xyz=torch.randn(m, 3, device=dev), _features_dc=torch.randn(m, 1, 3, device=dev),
                                      _features_rest=torch.randn(m, 15, 3, device=dev), _opacity=torch.randn(m, 1, device=dev),
                                      _scaling=torch.randn(m, 3, device=dev), _rotation=torch.randn(m, 4, device=dev),
                                      _semantic=torch.zeros(m, 0, device=dev), max_radii2D=torch.rand(m, device=dev),
                                      xyz_gradient_accum=torch.rand(m, 2, device=dev), denom=torch.rand(m, 1, device=dev), spatial_lr_scale=1.0,
                                      active_sh_degree=3)
            for a in NAMES:
                setattr(o, a, torch.nn.Parameter(getattr(o, a)))
            objs.append(o)
        opt = training.FusedAdam([{"params": [getattr(o, a)], "lr": 1e-3, "name": a} for o in objs for a in NAMES], eps=1e-15)
        for o in objs:
            for a in NAMES:
                p = getattr(o, a)
                opt.state[p] = dict(step=100, exp_avg=torch.randn_like(p), exp_avg_sq=torch.rand_like(p))
        shards.append(objs)
        opts.append(opt)
    return [f"m{k}" for k in range(len(sizes))], shards, opts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--piece-mib", type=int, default=1024)
    ap.add_argument("--dir", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    names, shards, opts = config_c(args.world, dev)
    with tempfile.TemporaryDirectory(dir=args.dir) as tmp:
        path = os.path.join(tmp, "iteration_1.pth")
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        run_ranks(args.world, lambda r, tr: SH.save_checkpoint(path, dict(zip(names, shards[r])), 1, opts[r], transport=tr,
                                                               piece_bytes=args.piece_mib << 20))
        torch.cuda.synchronize()
        t_save = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated() - base
        size = os.path.getsize(path)
        t0 = time.perf_counter()
        run_ranks(args.world, lambda r, tr: SH.load_checkpoint(path, dict(zip(names, shards[r])), opts[r], transport=tr))
        torch.cuda.synchronize()
        t_load = time.perf_counter() - t0
    print(f"config C, {args.world} emulated ranks on {torch.cuda.get_device_name()}, pieces of {args.piece_mib} MiB: file {size / 2**20:.0f} MiB, "
          f"save {t_save:.2f} s, load {t_load:.2f} s, peak extra device bytes of the save (all emulated ranks) {peak / 2**20:.0f} MiB")


if __name__ == "__main__":
    main()
