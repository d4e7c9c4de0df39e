"""GPU: sharded.rebalance through sharded.PeerTransport (the table all-gather and the row moves over the peer workspace,
sgr_peer_exchange_round) on 2, 3, 5 and 8 ranks emulated by threads (tests/rank_threads.py), one stream per rank, on workspaces of
PeerWorkspace.emulate poisoned with 0x7f before the rebalance.  Every kernel of the path is loaded before any rank spins in an emulated
barrier (_warm_up).

The same uneven shards as tests/test_rebalance_gpu.py (with_raw scene, 4 sub-models, 2 semantic floats per row, three FusedAdam steps,
filled statistics) are rebalanced twice, once through rank_threads.InProcessTransport and once through PeerTransport.  Checked:
  * parameters, both Adam moments, steps and the three densification statistics are bit-identical between the two, and so are the
    new counts and the rasterizers' chunks;
  * every rank took the same rounds and 1 + 1 + 2 rounds barriers; with a workspace set up at an eighth of the chunk the moves exceed
    the staging region and take several rounds;
  * with the workspace the transport staged through, a fused Gaussian-sharded forward and backward (sgr_sharded_forward /
    sgr_sharded_backward) renders colour, depth and alpha bit-identically to the same step after the in-process rebalance, on fresh
    workspaces, with no barrier timeout; the gradients agree up to the blend backward's float atomics."""
import ctypes as C

import pytest
import torch

import util
import street_gaussians_b200 as sgb
from rank_threads import run_ranks
from street_gaussians_b200 import _capi
from street_gaussians_b200 import sharded as SH
from test_rebalance_gpu import NAMES, make_global, make_optimizer, set_grads, shard_model, snapshot, split
from test_sharded64_gpu import _single, _warm_up_fused_path

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
CASES = [(2, 1), (3, 1), (5, 1), (8, 1), (2, 8), (3, 8)]  # (world, workspace chunk divisor)
_cache, _warm = {}, []


def _global():
    if not _cache:
        _cache["g"] = make_global()
    return _cache["g"]


def _warm_up(st):
    """The fused step's kernels and the barrier kernel (test_sharded64_gpu), and the piece copy, before any rank spins; the pack and
    splice kernels are loaded by the in-process rebalance each test runs first."""
    if _warm:
        return
    _warm_up_fused_path(DEV)
    ws = SH.PeerWorkspace.emulate(st, 64, 1, DEV)[0]
    a, b = torch.randn(37, device=DEV), torch.empty(40, device=DEV)
    P = _capi.SgrPeerPiece
    _capi.call("sgr_peer_exchange_round", DEV, C.byref(ws.peers), 4096, (P * 1)(P(0, 0, 0, 37, a.data_ptr())), 1,
               (P * 1)(P(0, 0, 0, 37, b.data_ptr())), 1)
    torch.cuda.synchronize()
    assert torch.equal(a, b[:37])
    _warm.append(True)


def _shards(models, grads, world):
    cuts = split(models, world)
    shards = [[shard_model(k, m, *cuts[r][k]) for k, m in enumerate(models)] for r in range(world)]
    opts = [make_optimizer(objs) for objs in shards]
    for it in range(3):
        for objs, opt, rows in zip(shards, opts, cuts):
            set_grads(objs, [[g * (1 + it) for g in gk] for gk in grads], rows)
            opt.step()
    return shards, opts


def _fused_step(st, poses, idft, shards, wss, streams, capacity, up):
    """Every rank's sgr_sharded_forward, then every rank's sgr_sharded_backward, each on its stream: (colour, depth, alpha summed over
    the bands, the ranks' gradients concatenated rank-major)."""
    world, H = len(shards), int(st.image_height)
    locs = []
    for objs in shards:
        xyz, rot, scale, opac, sh = sgb.compose(objs, poses, idft)
        locs.append(SH._local_tensors(xyz.detach(), sh.detach(), None, None, opac.detach(), scale.detach(), rot.detach(), None))
    status = [torch.zeros(8, dtype=torch.int32).pin_memory() for _ in range(world)]
    torch.cuda.synchronize()
    outs, grads = [], []
    with torch.no_grad():
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                outs.append(SH.sharded_forward_raw(st, SH.cyclic_band(H, r, world), wss[r], locs[r], int(locs[r]["means3D"].shape[0]), capacity,
                                                   -1, status[r]))
        torch.cuda.synchronize()
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                grads.append(SH.sharded_backward_raw(st, SH.cyclic_band(H, r, world), wss[r], locs[r], int(locs[r]["means3D"].shape[0]), capacity,
                                                     outs[r][2], *up))
        torch.cuda.synchronize()
    for r in range(world):
        assert int(status[r][4]) == 0 and int(status[r][1]) == 0, (r, status[r].tolist())  # no barrier timeout, no overflow
    imgs = tuple(sum(o[i] for o in outs) for i in range(3))
    g = [torch.cat([gr[i] for gr in grads]) if grads[0][i] is not None else None for i in range(8)]
    return imgs, g


@pytest.mark.parametrize("world,div", CASES)
def test_peer_transport_rebalance_is_the_in_process_one(world, div, monkeypatch):
    cam, poses, idft, models, grads, up = _global()
    st = util.settings_from(sgb, cam, DEV)
    _warm_up(st)
    shA, optA = _shards(models, grads, world)
    shB, optB = _shards(models, grads, world)
    counts0 = [sum(o._xyz.shape[0] for o in objs) for objs in shA]
    assert max(counts0) - min(counts0) > 1
    c0 = max(counts0)
    rastA = [SH.GaussianShardedRasterizer(st, chunk=c0) for _ in range(world)]
    P_A = run_ranks(world, lambda r, tr: SH.rebalance(shA[r], optA[r], rasterizer=rastA[r], transport=tr))
    torch.cuda.synchronize()

    ws_chunk = c0 // div
    wss = SH.PeerWorkspace.emulate(st, ws_chunk, world, DEV)
    for ws in wss:
        ws.buf[: ws.off_flags].fill_(0x7f)  # all but the barrier pads: the transport reads only what it staged
    rastB = []
    for r in range(world):
        ra = SH.GaussianShardedRasterizer(st, chunk=ws_chunk, exchange="p2p")
        ra._ws = wss[r]  # the workspace the rasterizer's last forward set up
        rastB.append(ra)
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    seen = []
    rounds = SH.peer_rounds
    monkeypatch.setattr(SH, "peer_rounds", lambda sizes, cap: seen.append(rounds(sizes, cap)) or seen[-1])
    torch.cuda.synchronize()

    def rank(r, _tr):
        with torch.cuda.stream(streams[r]):
            return SH.rebalance(shB[r], optB[r], rasterizer=rastB[r], transport=SH.PeerTransport(rastB[r]))

    P_B = run_ranks(world, rank)
    torch.cuda.synchronize()
    assert P_B == P_A and [r.chunk for r in rastB] == [r.chunk for r in rastA] == [max(P_A)] * world
    assert len(seen) == world and all(s == seen[0] for s in seen)
    n_rounds = len(seen[0])
    assert n_rounds >= (2 if div > 1 else 1), n_rounds
    assert [ws.epoch for ws in wss] == [2 + 2 * n_rounds] * world  # all_gather's barrier, the leading one, two per round
    assert all(rb._ws is ws and not ws.fwd_pending for rb, ws in zip(rastB, wss))
    for k, (a, b) in enumerate(zip(snapshot(shA, optA), snapshot(shB, optB))):
        for key in a:
            assert torch.equal(a[key], b[key]), (world, div, k, key)
    for objs_a, objs_b, oa, ob in zip(shA, shB, optA, optB):
        for a_m, b_m in zip(objs_a, objs_b):
            for a in NAMES:
                assert oa.state[getattr(a_m, a)]["step"] == ob.state[getattr(b_m, a)]["step"] == 3
    if div > 1:
        return  # the workspace is smaller than the new chunk: the next forward sets up a new one
    # the fused step on the workspaces the transport staged through renders as after the in-process rebalance
    H = int(cam["image_height"])
    glob = sgb.compose([{a[1:]: torch.cat([getattr(objs[k], a).detach() for objs in shA]) for a in NAMES[:6]} for k in range(len(models))],
                       poses, idft)
    scene = dict(means3D=glob[0], rotations=glob[1], scales=glob[2], opacities=glob[3], shs=glob[4])
    capacity = int(_single(scene, st)[5].num_instances) + 1000
    upd = [up[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
    imgs_b, g_b = _fused_step(st, poses, idft, shB, wss, streams, capacity, upd)
    fresh = SH.PeerWorkspace.emulate(st, ws_chunk, world, DEV)
    for ws in fresh:
        ws.buf[: ws.off_flags].fill_(0x7f)
    imgs_a, g_a = _fused_step(st, poses, idft, shA, fresh, streams, capacity, upd)
    for x, y, name in zip(imgs_a, imgs_b, ("color", "depth", "alpha")):
        assert torch.equal(x, y), name
    assert float(imgs_a[2].max()) > 0 and H > 0
    for i, (x, y) in enumerate(zip(g_a, g_b)):
        if x is not None:
            assert float((x - y).abs().max()) <= 1e-4 * float(x.abs().max()) + 1e-12, i
