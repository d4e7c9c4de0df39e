"""Cost of rebalancing Gaussian ownership (sharded.rebalance) on one GPU: a config-C-sized partition (1.5 M background + 8 x 50 k actor
Gaussians, SH degree 3, Adam moments on every tensor) split 2:1 over two ranks emulated by threads, as densification leaves it when one
rank's half of the scene grows twice as fast.  rebalance() moves a sixth of the rows: one sgr_rebalance_pack launch on the heavy rank,
the in-process copy standing in for NCCL, and one sgr_rebalance_splice launch per rank.

    python tools/rebalance_bench.py [--reps 5] [--out rebalance_bench.json]

Kernel times come from torch.profiler (CUDA activities): the first copy_spans_kernel of a repetition is the pack, the others the
splices.  The bytes each kernel must move (a read and a write per float) are computed from the plan, and the rate is those bytes over the
kernel time.  The card's name and power limit are printed with the numbers.

The p2p arm runs the same rebalance through sharded.PeerTransport on two peer workspaces emulated on the one GPU (PeerWorkspace.emulate,
one stream per rank, the workspace of a 1920 x 1280 frame at the old chunk), alternating with the in-process arm repetition by repetition.
Its copy_pieces_kernel launches (the table's stage and pull on both ranks, the rows' stage on the sending rank and their pull on the
receiving one) are timed the same way; their bytes are a read and a write per moved float for the stage and again for the pull.  The
"pull" reads the other rank's staging region in the same card's memory, so these are EMULATED numbers: they say what the copies cost on
one H100, not what NVLink or a multi-GPU rebalance takes.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import ctypes as C  # noqa: E402

import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import _capi  # noqa: E402
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


def peer_rasterizers(dev, chunk):
    """Two GaussianShardedRasterizer(exchange="p2p") of a 1920 x 1280 frame holding emulated peer workspaces of `chunk` slots per rank (what
    their last forward set up), and one stream per rank."""
    z = torch.zeros(3, device=dev)
    st = sgb.GaussianRasterizationSettings(1280, 1920, 0.5, 0.4, z, 1.0, torch.eye(4, device=dev), torch.eye(4, device=dev), 3, z, False, False)
    wss = SH.PeerWorkspace.emulate(st, chunk, 2, dev)
    rasts = []
    for ws in wss:
        r = SH.GaussianShardedRasterizer(st, chunk=chunk, exchange="p2p")
        r._ws = ws
        rasts.append(r)
    return rasts, [torch.cuda.Stream(device=dev) for _ in range(2)]


def load_peer_kernels(dev, rasts, streams):
    """The piece copy and the barrier kernel loaded before a rank spins in an emulated barrier (a first launch under lazy module loading
    waits for the spinning kernel): one round on a world-1 workspace, then one barrier per rank enqueued from this thread."""
    ws = SH.PeerWorkspace.emulate(rasts[0].raster_settings, 64, 1, dev)[0]
    a, b = torch.randn(64, device=dev), torch.empty(64, device=dev)
    P = _capi.SgrPeerPiece
    _capi.call("sgr_peer_exchange_round", dev, C.byref(ws.peers), 4096, (P * 1)(P(0, 0, 0, 64, a.data_ptr())), 1,
               (P * 1)(P(0, 0, 0, 64, b.data_ptr())), 1)
    torch.cuda.synchronize()
    for r in range(2):
        with torch.cuda.stream(streams[r]):
            _capi.call("sgr_peer_barrier", dev, C.byref(rasts[r]._ws.peers), 0)
            rasts[r]._ws.next_epochs(1)
    torch.cuda.synchronize()


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
    bytes_p2p = 2 * 2 * 4 * row_floats * moved  # stage and pull: a read and a write per moved float each
    rasts, streams = peer_rasterizers(dev, 2 * P // 3)
    load_peer_kernels(dev, rasts, streams)
    pack_ms, splice_ms, p2p_ms, rounds = [], [], [], []
    for rep in range(args.reps + 1):
        for arm in ("in_process", "p2p"):
            shards, opts = shards_2_to_1(models)
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                if arm == "in_process":
                    got = run_ranks(2, lambda r, tr: SH.rebalance(shards[r], opts[r], transport=tr))
                else:
                    def rank(r, _tr):
                        with torch.cuda.stream(streams[r]):
                            return SH.rebalance(shards[r], opts[r], rasterizer=rasts[r], transport=SH.PeerTransport(rasts[r]))
                    got = run_ranks(2, rank)
                torch.cuda.synchronize()
            assert got == [(P + 1) // 2, P // 2], (arm, got)
            ks = sorted((e for e in prof.events() if "copy_spans_kernel" in e.name), key=lambda e: e.time_range.start)
            assert len(ks) == 3, [e.name for e in ks]
            pieces = [e for e in prof.events() if "copy_pieces_kernel" in e.name]
            if arm == "p2p":
                for r in rasts:  # the next repetition's rebalance finds its workspace at the old chunk again
                    r.chunk = 2 * P // 3
            if rep == 0:
                continue  # warm-up: module loading and the caching allocator's first blocks
            dur = [(e.time_range.end - e.time_range.start) / 1e3 for e in ks]
            if arm == "in_process":
                pack_ms.append(dur[0])
                splice_ms.append(sum(dur[1:]))
            else:
                p2p_ms.append(sum((e.time_range.end - e.time_range.start) / 1e3 for e in pieces))
                rounds.append(len(SH.peer_rounds([[0, row_floats * moved], [0, 0]], SH.PeerTransport(rasts[0]).staging_bytes // 4)))
            del shards, opts
    med = lambda v: sorted(v)[len(v) // 2]
    res = dict(card=card(), rows_total=P, rows_moved=moved, floats_per_row=row_floats, reps=args.reps,
               pack_ms_median=round(med(pack_ms), 3), splice_ms_median=round(med(splice_ms), 3),
               pack_GBps=round(bytes_pack / (med(pack_ms) * 1e-3) / 1e9, 1), splice_GBps=round(bytes_splice / (med(splice_ms) * 1e-3) / 1e9, 1),
               pack_ms=[round(v, 3) for v in pack_ms], splice_ms=[round(v, 3) for v in splice_ms],
               p2p_emulated_on_one_gpu=dict(copy_ms_median=round(med(p2p_ms), 3), copy_GBps=round(bytes_p2p / (med(p2p_ms) * 1e-3) / 1e9, 1),
                                            rounds=rounds[0], copy_ms=[round(v, 3) for v in p2p_ms]))
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
