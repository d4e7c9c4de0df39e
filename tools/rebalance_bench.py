"""Cost of rebalancing Gaussian ownership (sharded.rebalance) on one GPU: a config-C-sized partition (1.5 M background + 8 x 50 k actor
Gaussians, SH degree 3, Adam moments on every tensor) split 2:1 over two ranks emulated by threads, as densification leaves it when one
rank's half of the scene grows twice as fast.  rebalance() moves a sixth of the rows: one sgr_rebalance_pack launch on the heavy rank,
the in-process copy standing in for NCCL, and one sgr_rebalance_splice launch per rank.

    python tools/rebalance_bench.py [--reps 5] [--out rebalance_bench.json]

Kernel times come from torch.profiler (CUDA activities): the first copy_spans_kernel of a repetition is the pack, the others the
splices.  The bytes each kernel must move (a read and a write per float) are computed from the plan, and the rate is those bytes over the
kernel time.  The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
from street_gaussians_b200 import sharded as SH  # noqa: E402
from street_gaussians_b200 import training  # noqa: E402
from rank_threads import run_ranks  # noqa: E402

COUNTS = [1_500_000] + [50_000] * 8
WIDTHS = (3, 3, 45, 1, 3, 4, 0)  # floats per row of PARAM_NAMES at SH degree 3, no semantics


def global_models(dev):
    g = torch.Generator(device=dev).manual_seed(0)
    out = []
    for n in COUNTS:
        m = {a: torch.randn((n, w), device=dev, generator=g) for a, w in zip(training.PARAM_NAMES, WIDTHS)}
        m.update({a + "/m": torch.randn((n, w), device=dev, generator=g) for a, w in zip(training.PARAM_NAMES, WIDTHS)})
        m.update({a + "/v": torch.rand((n, w), device=dev, generator=g) for a, w in zip(training.PARAM_NAMES, WIDTHS)})
        m.update(max_radii2D=torch.rand(n, device=dev, generator=g), xyz_gradient_accum=torch.rand(n, 2, device=dev, generator=g),
                 denom=torch.rand(n, 1, device=dev, generator=g))
        out.append(m)
    return out


def shards_2_to_1(models):
    """Rank 0 owns the first two thirds of the global rows, rank 1 the rest; each with a FusedAdam whose state is set."""
    P = sum(COUNTS)
    B = [0, 2 * P // 3, P]
    shards, opts = [], []
    for r in range(2):
        objs, at = [], 0
        for m, n in zip(models, COUNTS):
            lo, hi = min(max(B[r] - at, 0), n), min(max(B[r + 1] - at, 0), n)
            o = {a: torch.nn.Parameter(m[a][lo:hi].clone()) for a in training.PARAM_NAMES}
            o.update({s: m[s][lo:hi].clone() for s in training.STAT_NAMES})
            objs.append(o)
            at += n
        opt = training.FusedAdam([{"params": [o[a] for o in objs for a in training.PARAM_NAMES]}], lr=1e-3)
        for o, m in zip(objs, models):
            for a in training.PARAM_NAMES:
                n = o[a].shape[0]
                opt.state[o[a]] = dict(step=1, exp_avg=m[a + "/m"][:n].clone(), exp_avg_sq=m[a + "/v"][:n].clone())
        shards.append(objs)
        opts.append(opt)
    return shards, opts


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rebalance_bench needs a CUDA device")
    dev = torch.device("cuda")
    models = global_models(dev)
    row_floats = sum(WIDTHS) * 3 + 4
    P = sum(COUNTS)
    moved = 2 * P // 3 - (P + 1) // 2   # rows rank 0 sends to rank 1
    bytes_pack = 2 * 4 * row_floats * moved
    bytes_splice = 2 * 4 * row_floats * P  # every row of both new shards is written once (kept or received)
    pack_ms, splice_ms = [], []
    for rep in range(args.reps + 1):
        shards, opts = shards_2_to_1(models)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            got = run_ranks(2, lambda r, tr: SH.rebalance(shards[r], opts[r], transport=tr))
            torch.cuda.synchronize()
        assert got == [(P + 1) // 2, P // 2], got
        ks = sorted((e for e in prof.events() if "copy_spans_kernel" in e.name), key=lambda e: e.time_range.start)
        assert len(ks) == 3, [e.name for e in ks]
        if rep == 0:
            continue  # warm-up: module loading and the caching allocator's first blocks
        dur = [(e.time_range.end - e.time_range.start) / 1e3 for e in ks]
        pack_ms.append(dur[0])
        splice_ms.append(sum(dur[1:]))
        del shards, opts
    med = lambda v: sorted(v)[len(v) // 2]
    res = dict(card=card(), rows_total=P, rows_moved=moved, floats_per_row=row_floats, reps=args.reps,
               pack_ms_median=round(med(pack_ms), 3), splice_ms_median=round(med(splice_ms), 3),
               pack_GBps=round(bytes_pack / (med(pack_ms) * 1e-3) / 1e9, 1), splice_GBps=round(bytes_splice / (med(splice_ms) * 1e-3) / 1e9, 1),
               pack_ms=[round(v, 3) for v in pack_ms], splice_ms=[round(v, 3) for v in splice_ms])
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
