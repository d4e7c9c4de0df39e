"""CPU: the sky cube gradient's exchange over peer memory and the colour correction's sums over it (include/sgr.h sgr_sky_grad_blocks,
sgr_sky_peer_bytes, sgr_band_sky_composite_backward_marked, sgr_sky_grad_peer_sum; sky.sky_composite / corrections.color_correct with
rasterizer=).  A numpy model of the block map, the union, the owner rule and each rank's peer reads against the size queries; the new
struct's layout against ctypes; argument checks before anything is enqueued; rasterizer= resolution; and a gloo world-2 run of the
autograd entries with the C calls stubbed: the p2p backward makes one exchange call per stage and no collective, the nccl one still
all-reduces once per backward, and world 1 takes the whole-frame entries."""
import ctypes as C
import os
import socket
import subprocess
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi, corrections, sky
from street_gaussians_b200 import sharded as SH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK = C.c_void_p(1 << 20)  # a 16-byte aligned address: validation fails before anything dereferences it
BLOCK = 32


def _err():
    return _capi.lib().sgr_last_error().decode()


# ---- the block model ---------------------------------------------------------------------------------------------------------
def block_of_texel(R: int) -> np.ndarray:
    """Block index of every texel of [6, R, R]: (face * nb + row // 32) * nb + column // 32, nb = ceil(R / 32)."""
    nb = -(-R // BLOCK)
    f, r, c = np.meshgrid(np.arange(6), np.arange(R), np.arange(R), indexing="ij")
    return ((f * nb + r // BLOCK) * nb + c // BLOCK).reshape(-1)


def block_bytes(R: int) -> np.ndarray:
    """fp32 bytes of every block's texels (3 channels); clipped blocks at the last rows and columns are smaller."""
    return np.bincount(block_of_texel(R), minlength=6 * (-(-R // BLOCK)) ** 2) * 12


def peer_reads(maps: np.ndarray, sizes: np.ndarray):
    """Per rank, the bytes it reads from other ranks' sections: as owner of block b (b % world == rank) the block of every other rank
    that marked it, and in the gather every union block whose owner is another rank.  maps [world, blocks] bool."""
    world, nblk = maps.shape
    union = maps.any(0)
    owner = np.arange(nblk) % world
    reads = np.zeros(world, dtype=np.int64)
    for r in range(world):
        mine = owner == r
        others = maps.sum(0) - maps[r]
        reads[r] = int((others * sizes * mine).sum()) + int((sizes * (union & ~mine)).sum())
    return union, reads


@pytest.mark.parametrize("R", [1, 16, 100, 1024])
def test_block_model_matches_the_size_queries(R):
    L = _capi.lib()
    nb = -(-R // BLOCK)
    assert int(L.sgr_sky_grad_blocks(R)) == 6 * nb * nb
    sizes = block_bytes(R)
    assert sizes.size == 6 * nb * nb and int(sizes.sum()) == 6 * R * R * 12 and (sizes > 0).all()
    assert int(sizes.max()) == min(R, BLOCK) ** 2 * 12
    cube = -(-(6 * R * R * 12) // 256) * 256
    assert int(L.sgr_sky_peer_bytes(R)) == -(-(cube + 6 * nb * nb) // 256) * 256
    # the union, the owner rule and the read set on a random map: every union block is read once per rank that does not own it,
    # and the owner reads every other rank's copy of its blocks
    rng = np.random.default_rng(R)
    for world in (1, 2, 3, 8):
        maps = rng.random((world, sizes.size)) < 0.3
        union, reads = peer_reads(maps, sizes)
        owned = np.arange(sizes.size) % world
        for r in range(world):
            want = sum(int(sizes[b]) * (int(maps[:, b].sum()) - int(maps[r, b])) for b in range(sizes.size) if owned[b] == r)
            want += sum(int(sizes[b]) for b in np.flatnonzero(union) if owned[b] != r)
            assert reads[r] == want
        if world == 1:
            assert reads[0] == 0
    for bad in (0, -1, 16385):
        assert L.sgr_sky_grad_blocks(bad) == 0 and L.sgr_sky_peer_bytes(bad) == 0


def test_struct_layout_compiled_from_the_header(tmp_path):
    src = tmp_path / "layout.c"
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "sgr.h"', 'int main(void) {',
            '  printf("size %zu\\n", sizeof(SgrSkyPeers));']
    body += [f'  printf("{f[0]} %zu\\n", offsetof(SgrSkyPeers, {f[0]}));' for f in _capi.SgrSkyPeers._fields_] + ['  return 0;', '}']
    src.write_text("\n".join(body))
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(line.rsplit(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["size"]) == C.sizeof(_capi.SgrSkyPeers)
    for f in _capi.SgrSkyPeers._fields_:
        assert int(out[f[0]]) == getattr(_capi.SgrSkyPeers, f[0]).offset, f[0]
    for name in ("sgr_sky_grad_blocks", "sgr_sky_peer_bytes", "sgr_band_sky_composite_backward_marked", "sgr_sky_grad_peer_sum"):
        assert name in _capi.SYMBOLS


def _peers(world=2, rank=1, flags=True):
    pe = _capi.SgrPeers()
    pe.world, pe.rank, pe.chunk = world, rank, 8
    for p in range(min(world, _capi.MAX_PEERS)):
        pe.flags[p] = OK.value if flags else None
    return pe


def _sky_peers(world=2, sec=OK.value, nbytes=1 << 40):
    sp = _capi.SgrSkyPeers()
    for p in range(min(world, _capi.MAX_PEERS)):
        sp.sec[p] = sec
    sp.bytes = nbytes
    return sp


def test_exchange_validates_before_launch():
    L = _capi.lib()
    R = 100
    need = int(L.sgr_sky_peer_bytes(R))

    def call(pe=_peers(), sp=_sky_peers(), R=R, m=OK, g=OK):
        return L.sgr_sky_grad_peer_sum(C.byref(pe) if pe is not None else None, C.byref(sp) if sp is not None else None, R, m, g, None)

    assert call(pe=None) == -1 and "peers is NULL" in _err()
    assert call(sp=None) == -1 and "sky_peers is NULL" in _err()
    assert call(pe=_peers(world=0, rank=0)) == -1 and "bad peer table" in _err()
    assert call(pe=_peers(world=_capi.MAX_PEERS + 1, rank=0)) == -1 and "bad peer table" in _err()
    assert call(pe=_peers(rank=2)) == -1 and "bad peer table" in _err()
    assert call(pe=_peers(flags=False)) == -1 and "barrier pad" in _err()
    assert call(sp=_sky_peers(sec=None)) == -1 and "sky section" in _err()
    assert call(sp=_sky_peers(sec=OK.value + 4)) == -1 and "16-byte aligned" in _err()
    assert call(sp=_sky_peers(nbytes=need - 1)) == -3 and f"{need} needed" in _err()
    for bad in (0, 16385):
        assert call(R=bad) == -1 and "R=" in _err()
    assert call(m=None) == -1 and "NULL" in _err()
    assert call(g=None) == -1 and "NULL" in _err()
    assert call(g=C.c_void_p(OK.value + 4)) == -1 and "dL_dcube is not 16-byte aligned" in _err()


def test_marked_backward_validates_before_launch():
    L = _capi.lib()

    def call(band=(0, 1, 1), R=4, g_cube=OK, block_map=OK):
        return L.sgr_band_sky_composite_backward_marked(40, 8, *band, R, 0, 1.0, OK, None, OK, OK, OK, None, None, OK, OK, g_cube, block_map, None)

    assert call(band=(0, 4, 1)) == -1 and "band" in _err()
    assert call(R=0) == -1 and "R=" in _err()
    assert call(g_cube=None) == -1 and "NULL" in _err()
    assert call(block_map=None) == -1 and "NULL" in _err()


def _st(H=96, W=128):
    return sgb.GaussianRasterizationSettings(H, W, 0.5, 0.4, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)


def test_sky_workspace_emulation_wires_the_sections():
    R, world = 100, 3
    wss = SH.SkyWorkspace.emulate(R, world, torch.device("cpu"))
    bases = [ws.buf.data_ptr() for ws in wss]
    for r, ws in enumerate(wss):
        assert (ws.R, ws.world, ws.rank) == (R, world, r) and ws.bytes == int(_capi.lib().sgr_sky_peer_bytes(R))
        assert [ws.peers.sec[p] for p in range(world)] == bases and ws.peers.bytes == ws.bytes
        assert ws.block_map.dtype == torch.uint8 and ws.block_map.numel() == 6 * 4 * 4
    r = SH.GaussianShardedRasterizer(_st(), exchange="p2p")
    with pytest.raises(_capi.SgrError, match="device"):
        r.sky_workspace(R)
    a = r.sky_workspace(R, torch.device("cpu"))
    r.repartition(10, chunk=16)
    assert r.sky_workspace(R) is a  # kept across repartition()
    assert r.sky_workspace(16, torch.device("cpu")).R == 16  # a new R: a new section


def _raster(exchange="p2p", group=None, band=None, ws=None, sky_ws=None):
    def loss_workspace():
        if ws is None:
            raise _capi.SgrError("no forward")
        return ws
    return types.SimpleNamespace(exchange=exchange, group=group, band=band, loss_workspace=loss_workspace,
                                 sky_workspace=lambda R, device=None: sky_ws)


def test_rasterizer_resolution_refuses_mismatches():
    H, W = 96, 128
    band = SH.cyclic_band(H, 1, 2)
    ws = SH.PeerWorkspace.emulate(_st(), 8, 2, torch.device("cpu"))[1]
    img, acc = torch.rand(3, H, W), torch.rand(1, H, W)
    cube, K, w2c = torch.zeros(6, 4, 4, 3), torch.eye(3), torch.eye(4)
    ri = _raster(band=band, ws=ws)
    with pytest.raises(ValueError, match="band"):
        sky.sky_composite(img, acc, cube, K, w2c, band=SH.cyclic_band(H, 0, 2), rasterizer=ri)
    with pytest.raises(ValueError, match="group"):
        sky.sky_composite(img, acc, cube, K, w2c, group=object(), rasterizer=ri)
    with pytest.raises(ValueError, match="band"):
        corrections.color_correct(img, torch.zeros(3, 4), band=SH.cyclic_band(H, 0, 2), rasterizer=ri)
    with pytest.raises(ValueError, match="group"):
        corrections.color_correct(img, torch.zeros(3, 4), group=object(), rasterizer=ri)
    # the rasterizer's forward must run first
    with pytest.raises(_capi.SgrError, match="forward"):
        sky.sky_composite(img, acc, cube, K, w2c, rasterizer=_raster(band=band))
    with pytest.raises(_capi.SgrError, match="forward"):
        corrections.color_correct(img, torch.zeros(3, 4), rasterizer=SH.GaussianShardedRasterizer(_st(), exchange="p2p"))
    # the matching band, and the group, pass resolution (then CPU tensors are refused)
    with pytest.raises(_capi.SgrError, match="CUDA"):
        sky.sky_composite(img, acc, cube, K, w2c, band=band, rasterizer=ri)
    rows, xfer = sky._resolve(None, None, ri, H)
    assert rows == (band.begin, band.end, band.step) and xfer.kind == "p2p" and xfer.ws is ws
    g = object()
    rows, xfer = sky._resolve(band, g, _raster("nccl", group=g, band=band), H)
    assert xfer.kind == "nccl" and xfer.group is g
    assert sky._resolve(None, None, _raster(band=None, ws=ws), H)[0] is None  # world 1: the whole-frame entries


# ---- gloo world 2, C calls stubbed -------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _floats(p, n, ctype=C.c_float):
    return np.ctypeslib.as_array((ctype * n).from_address(p.value))


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        H, W, R = 40, 8, 4
        band = SH.cyclic_band(H, rank, world)
        cpu = torch.device("cpu")
        ws = SH.PeerWorkspace.emulate(_st(H, W), 8, world, cpu)[rank]
        sky_ws = SH.SkyWorkspace.emulate(R, world, cpu)[rank]
        calls, reduces = [], []

        def stub(name, device, *args):
            calls.append(name)
            if name in ("sgr_band_sky_composite_forward", "sgr_sky_composite_forward", "sgr_band_color_correct_forward", "sgr_color_correct_forward"):
                _floats(args[-1], 3 * H * W)[:] = 1.0
            elif name in ("sgr_band_sky_composite_backward", "sgr_band_sky_composite_backward_marked", "sgr_sky_composite_backward"):
                k = -3 if name.endswith("marked") else -2
                _floats(args[k + 1], 6 * R * R * 3)[:] += rank + 1
                if name.endswith("marked"):
                    assert args[-1].value == sky_ws.block_map.data_ptr()
            elif name == "sgr_sky_grad_peer_sum":
                assert args[2] == R and args[3].value == sky_ws.block_map.data_ptr()
            elif name in ("sgr_band_color_correct_backward", "sgr_band_peer_sum"):
                pass
            elif name == "sgr_color_correct_backward":
                _floats(args[6], 12)[:] = 3.0
            elif name == "sgr_band_color_correct_affine_grad":
                _floats(args[1], 12)[:] = 2.0
            else:
                raise AssertionError(f"unexpected call {name}")

        real_all_reduce = dist.all_reduce

        def counting_all_reduce(t, *a, **k):
            reduces.append((calls[-1], tuple(t.shape), t.dtype))
            return real_all_reduce(t, *a, **k)

        _capi.call = stub
        dist.all_reduce = counting_all_reduce
        sky._check = lambda rgb, acc, cube_map, K, w2c, sky_mask: (H, W, R)
        corrections._check_cuda = lambda t, what: None

        def step(ri):
            calls.clear()
            reduces.clear()
            rgb = torch.rand(3, H, W, requires_grad=True)
            acc = torch.rand(1, H, W, requires_grad=True)
            cube = torch.zeros(6, R, R, 3, requires_grad=True)
            affine = torch.eye(4)[:3].clone().requires_grad_(True)
            out = sky.sky_composite(rgb, acc, cube, torch.eye(3), torch.eye(4), rasterizer=ri)
            col = corrections.color_correct(out, affine, rasterizer=ri)
            col.backward(torch.rand(3, H, W))
            return list(calls), list(reduces), cube.grad

        # p2p: the marked backward and one exchange for the cube, one peer sum for the affine; no collective
        epochs = ws.epoch
        c, red, _ = step(_raster(band=band, ws=ws, sky_ws=sky_ws))
        assert red == [], red
        assert c == ["sgr_band_sky_composite_forward", "sgr_band_color_correct_forward", "sgr_band_color_correct_backward", "sgr_band_peer_sum",
                     "sgr_band_color_correct_affine_grad", "sgr_band_sky_composite_backward_marked", "sgr_sky_grad_peer_sum"], c
        assert ws.epoch == epochs + 2 + 3  # the peer sum's two barriers and the exchange's three
        # nccl: one all-reduce per backward, over the rasterizer's group
        c, red, g = step(_raster("nccl", band=band))
        assert red == [("sgr_band_color_correct_backward", (12,), torch.float64), ("sgr_band_sky_composite_backward", (6, R, R, 3), torch.float32)], red
        assert "sgr_sky_grad_peer_sum" not in c and bool((g == sum(range(1, world + 1))).all())
        # world 1 (the rasterizer has no band): the whole-frame entries, nothing to exchange
        c, red, g = step(_raster(band=None, ws=ws, sky_ws=sky_ws))
        assert red == [] and c == ["sgr_sky_composite_forward", "sgr_color_correct_forward", "sgr_color_correct_backward",
                                   "sgr_sky_composite_backward"], c
        assert bool((g == rank + 1).all())
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, repr(e) + traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_backward_transports_gloo_world2():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
