"""Blocks, bytes and kernel times of the sky cube gradient's exchange over peer memory (sgr_band_sky_composite_backward_marked +
sgr_sky_grad_peer_sum), with the ranks EMULATED on ONE GPU, beside the dense all-reduce it replaces.

    python tools/sky_p2p_bench.py [--H 1280 --W 1920 --R 1024 --steps 10]

Two cameras with Waymo front-camera intrinsics: tools/sky_bench.py's camera that sees three cube faces (sky mask over half the frame,
jittered), and a level street camera facing a face centre with the sky mask over the top 40 % of the rows.  For world 1, 2, 4 and 8
(cyclic bands):
  blocks  the union and per-rank counts of the 32 x 32-texel blocks, read from the marking backward's own maps;
  bytes   what each rank reads from the other ranks' sections (as owner: the other ranks' copies of its marked blocks; in the gather:
          the union blocks other ranks own), next to the dense ring all-reduce's 2 (N - 1) / N x 6 R^2 3 x 4 bytes per rank;
  times   torch.profiler kernel records, per rank and call: the band backward with and without marking (ranks one after the other),
          and the exchange's stage, owner-sum and gather kernels and its barriers (ranks as threads on streams of the one GPU).
Emulated "peer" reads are reads of this card's own HBM and the barriers mostly wait for the other emulated ranks: no NVLink time and
no time across GPUs is measured here.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
from street_gaussians_b200 import _capi, sky  # noqa: E402
from street_gaussians_b200 import sharded as SH  # noqa: E402
from street_gaussians_b200._capi import ptr  # noqa: E402
from street_gaussians_b200.rasterizer import GaussianRasterizationSettings, TileRowBand  # noqa: E402
from rank_threads import run_ranks  # noqa: E402

BLOCK = 32
KERNELS = (("bwd_unmarked", "sky_composite_bwd_kernel<true, false>"), ("bwd_marked", "sky_composite_bwd_kernel<true, true>"),
           ("stage", "sky_stage_kernel"), ("owner_sum", "sky_owner_sum_kernel"), ("gather", "sky_gather_kernel"),
           ("barrier", "peer_barrier_kernel"))


def kernel_ms(fn):
    """Run fn under torch.profiler; {group: total device ms} from the trace's kernel records."""
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
            for g, name in KERNELS:
                if name in e["name"]:
                    out[g] += e.get("dur", 0.0) / 1000.0
    return out


def look_at(target, dev):
    """tools/sky_bench.py's camera: looking along `target` with world y as up."""
    z = torch.tensor(target)
    z = z / z.norm()
    x = torch.linalg.cross(torch.tensor([0.0, 1.0, 0.0]), z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    w2c = torch.eye(4)
    w2c[:3, :3] = torch.stack([x, y, z], 1).T
    return w2c.to(dev)


def block_bytes(R, dev):
    nb = -(-R // BLOCK)
    f, r, c = torch.meshgrid(torch.arange(6), torch.arange(R), torch.arange(R), indexing="ij")
    return torch.bincount(((f * nb + r // BLOCK) * nb + c // BLOCK).reshape(-1), minlength=6 * nb * nb).to(dev, torch.int64) * 12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=1280)
    ap.add_argument("--W", type=int, default=1920)
    ap.add_argument("--R", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sky_p2p_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    H, W, R, K = args.H, args.W, args.R, args.steps
    g = torch.Generator(device=dev).manual_seed(0)
    Kin = torch.tensor([[2055.6, 0.0, 939.7], [0.0, 2051.3, 641.1], [0.0, 0.0, 1.0]], device=dev)
    cube = 0.5 * torch.ones(6, R, R, 3, device=dev)
    acc = torch.rand(1, H, W, generator=g, device=dev)
    up = torch.randn(3, H, W, generator=g, device=dev)
    top = torch.zeros(1, H, W, dtype=torch.uint8, device=dev)
    top[:, : int(0.4 * H)] = 1
    cams = {"three_faces_half_mask_jitter": (look_at([1.0, -1.0, 1.0], dev), (torch.rand(1, H, W, generator=g, device=dev) < 0.5).to(torch.uint8),
                                            (torch.rand(H, W, generator=g, device=dev), torch.rand(H, W, generator=g, device=dev))),
            "level_face_centre_top40": (look_at([1.0, 0.0, 0.0], dev), top, (None, None))}
    z = torch.zeros(3, device=dev)
    st = GaussianRasterizationSettings(H, W, 0.5, 0.5, z, 1.0, torch.eye(4, device=dev), torch.eye(4, device=dev), 0, z, False, False)
    nblk = int(_capi.lib().sgr_sky_grad_blocks(R))
    sizes = block_bytes(R, dev)
    dense = 6 * R * R * 3 * 4

    def band_bwd(w2c, mask, jit, band, gcube, gacc, bmap):
        """The band backward on the whole-frame inputs (a rank reads only its band's pixels), marked when bmap is given."""
        common = (H, W, *band, R, _capi.SKY_MASK_GIVEN, 1.0, ptr(acc), ptr(mask), ptr(cube), ptr(Kin), ptr(w2c), ptr(jit[0]), ptr(jit[1]), ptr(up),
                  ptr(gacc), ptr(gcube))
        if bmap is None:
            _capi.call("sgr_band_sky_composite_backward", dev, *common)
        else:
            _capi.call("sgr_band_sky_composite_backward_marked", dev, *common, ptr(bmap))

    # every kernel loaded before emulated ranks spin: the backward both ways and the exchange at world 1, then two ranks' exchanges
    # enqueued one after the other from this thread (tests/test_sky_p2p_gpu._warm_up)
    w2c, mask, jit = cams["level_face_centre_top40"]
    g1 = torch.zeros_like(cube)
    ga = torch.zeros_like(acc)
    for world in (1, 2):
        wss, skys = SH.PeerWorkspace.emulate(st, 8, world, dev), SH.SkyWorkspace.emulate(R, world, dev)
        streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
        torch.cuda.synchronize()
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                b = SH.cyclic_band(H, r, world)
                band_bwd(w2c, mask, jit, b, g1, ga, None)
                band_bwd(w2c, mask, jit, b, g1, ga, skys[r].block_map)
                sky.sky_grad_peer_sum(wss[r], skys[r], g1)
        torch.cuda.synchronize()

    report = []
    for cam, (w2c, mask, jit) in cams.items():
        for world in (1, 2, 4, 8):
            bands = [SH.cyclic_band(H, r, world) if world > 1 else TileRowBand(0, (H + 15) // 16, 1) for r in range(world)]
            wss, skys = SH.PeerWorkspace.emulate(st, 8, world, dev), SH.SkyWorkspace.emulate(R, world, dev)
            gcubes = [torch.zeros_like(cube) for _ in range(world)]
            gaccs = [torch.zeros_like(acc) for _ in range(world)]
            bwd = []
            for r in range(world):
                band_bwd(w2c, mask, jit, bands[r], gcubes[r], gaccs[r], skys[r].block_map)
                un = kernel_ms(lambda: [band_bwd(w2c, mask, jit, bands[r], gcubes[r], gaccs[r], None) for _ in range(K)])
                mk = kernel_ms(lambda: [band_bwd(w2c, mask, jit, bands[r], gcubes[r], gaccs[r], skys[r].block_map) for _ in range(K)])
                bwd.append((un["bwd_unmarked"] / K, mk["bwd_marked"] / K))
            maps = torch.stack([s.block_map.bool() for s in skys])
            union = maps.any(0)
            owner = torch.arange(nblk, device=dev) % world
            reads = []
            for r in range(world):
                mine = owner == r
                others = maps.sum(0) - maps[r].long()
                reads.append(int((others * sizes * mine).sum()) + int((sizes * (union & ~mine)).sum()))
            streams = [torch.cuda.Stream(device=dev) for _ in range(world)]

            def steps(n):
                def rank(r, _tr):
                    with torch.cuda.stream(streams[r]):
                        for _ in range(n):
                            sky.sky_grad_peer_sum(wss[r], skys[r], gcubes[r])
                torch.cuda.synchronize()
                run_ranks(world, rank)
                torch.cuda.synchronize()

            steps(2)
            ms = kernel_ms(lambda: steps(K))
            report.append(dict(camera=cam, world=world, union_blocks=int(union.sum()), blocks=nblk,
                               rank_blocks=[int(m.sum()) for m in maps], peer_read_MB_per_rank=[round(b / 1e6, 3) for b in reads],
                               dense_allreduce_MB_per_rank=round(2 * (world - 1) / world * dense / 1e6, 3),
                               bwd_unmarked_ms_per_rank=[round(u, 4) for u, _ in bwd], bwd_marked_ms_per_rank=[round(m, 4) for _, m in bwd],
                               **{f"{k}_ms_per_rank_call": round(ms[k] / (K * world), 4) for k in ("stage", "owner_sum", "gather", "barrier")}))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu, tool="torch.profiler kernel records", H=H, W=W, R=R, steps=K, block=f"{BLOCK}x{BLOCK} texels",
                          rows=report, nvlink_time="not measured: emulated peer reads are reads of this card's HBM, and the barriers "
                          "mostly wait for the other emulated ranks"), indent=1))


if __name__ == "__main__":
    main()
