"""GPU: the band losses over peer memory (band_losses.frame_losses / lidar_depth_loss and the losses.py wrappers with rasterizer= of a
GaussianShardedRasterizer(exchange="p2p"); include/sgr.h sgr_band_halo_exchange_peers / sgr_band_peer_sum), with 1, 2, 3, 5 and 8 ranks
emulated by threads (tests/rank_threads.py) on streams of one GPU through PeerWorkspace.emulate and a stand-in rasterizer.

Every kernel is loaded before any rank spins in an emulated barrier (_warm_up), and every rank's loss section is poisoned with 0x7f
before each exchange, so no call reads bytes it did not write in that call.

Checked per case, through the real autograd entries: every rank's values are bit-identical to every other rank's; each value is within
the bound test_band_losses_gpu.py states against the single-GPU call (one fp32 ulp for the photometric and LiDAR values, the photometric
one plus the rounding of adding lambda_dssim; VALUE_RTOL_ACC for sky and object accumulation); n, k and the LiDAR selection are exact;
each rank's gradient rows are bit-identical to the single-GPU gradient and its other rows are zero.  Two frames with different inputs run
back to back through the same workspaces.
Sensitivity: partials whose fp64 sum depends on the order give the ascending-rank sum on every rank (the descending one differs); an
int32 sum at world 8 is exact; a halo that drops one side fails the gradient check."""
import types

import numpy as np
import pytest
import torch

from rank_threads import run_ranks
from street_gaussians_b200 import _capi, band_losses, losses
from street_gaussians_b200 import sharded as SH
from street_gaussians_b200.rasterizer import GaussianRasterizationSettings, TileRowBand
from test_band_losses_gpu import (VALUE_RTOL_ACC, W_OF, _banded, _bits_equal, _inputs, _lidar_inputs, _rows, _single_lidar,
                                  _ulp_close)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
LAMBDA_DSSIM, SKY_W, OBJ_W, LIDAR_W, KEEP = 0.2, 0.5, 0.3, 0.7, 0.95
CASES = [(world, "cyclic", H) for world in (1, 2, 3, 5, 8) for H in (375, 1280)] + [(8, "cyclic", 80)] + \
        [(world, "contiguous", 375) for world in (2, 3, 5)] + [(8, "contiguous", 40)]
_warm = []


def _settings(H, W):
    z = torch.zeros(3, device=DEV)
    return GaussianRasterizationSettings(H, W, 0.5, 0.5, z, 1.0, torch.eye(4, device=DEV), torch.eye(4, device=DEV), 0, z, False, False)


def _band(H, r, world, layout):
    if world == 1:
        return None  # what GaussianShardedRasterizer.band is at world 1: the losses take the whole image
    return (SH.cyclic_band if layout == "cyclic" else SH.contiguous_band)(H, r, world)


def _stand_in(ws, band):
    """What the band losses read of a GaussianShardedRasterizer(exchange="p2p"), around an emulated workspace."""
    return types.SimpleNamespace(exchange="p2p", group=None, band=band, loss_workspace=lambda: ws)


@pytest.fixture(autouse=True)
def _poison_loss_sections(monkeypatch):
    """Fill the calling rank's loss section with 0x7f on its stream before every exchange.  Safe between calls: each call ends with a
    barrier after which no peer reads the section."""
    halo, psum = band_losses.peer_exchange_halo, band_losses.peer_sum

    def poison(ws):
        ws.buf[ws.off_loss: ws.off_loss + ws.loss_bytes].fill_(0x7f)

    def halo_poisoned(ws, image, band):
        poison(ws)
        return halo(ws, image, band)

    def sum_poisoned(ws, t):
        poison(ws)
        return psum(ws, t)

    monkeypatch.setattr(band_losses, "peer_exchange_halo", halo_poisoned)
    monkeypatch.setattr(band_losses, "peer_sum", sum_poisoned)


def _frame_inputs(H, W, seed):
    img, gt, m = _inputs(H, W, seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 100)
    acc = torch.rand(1, H, W, device=DEV, generator=g)
    acc.view(-1)[:: 97] = 0.0  # clamped: zero gradient
    acc_obj = torch.rand(1, H, W, device=DEV, generator=g)
    sky = torch.rand(1, H, W, device=DEV, generator=g) > 0.5
    bound = torch.rand(1, H, W, device=DEV, generator=g) > 0.6
    depth, dacc, lidar, lm = _lidar_inputs(H, W, seed + 7, "ties" if seed % 2 else "plain")
    return dict(img=img, gt=gt, mask=m.view(1, H, W).bool(), acc=acc, acc_obj=acc_obj, sky=sky, bound=bound, depth=depth, dacc=dacc,
                lidar=lidar, lmask=lm.view(1, H, W).bool())


LEAVES = ("img", "acc", "acc_obj", "depth", "dacc")


def _single(x):
    """The whole-frame calls: values, gradients, and the LiDAR n and k."""
    lv = {k: x[k].clone().requires_grad_(True) for k in LEAVES}
    v = dict(photometric=losses.photometric_loss(lv["img"], x["gt"], x["mask"], lambda_dssim=LAMBDA_DSSIM),
             sky=losses.sky_loss(lv["acc"], x["sky"], SKY_W), obj_acc=losses.obj_acc_loss(lv["acc_obj"], x["bound"], OBJ_W),
             lidar=losses.lidar_depth_loss(lv["depth"], lv["dacc"], x["lidar"], x["lmask"], LIDAR_W, KEEP))
    grads = torch.autograd.grad([v["photometric"], v["sky"], v["obj_acc"], v["lidar"]], [lv[k] for k in LEAVES])
    _, _, s = _single_lidar(x["depth"], x["dacc"], x["lidar"], x["lmask"].reshape(-1).to(torch.uint8), KEEP, LIDAR_W)
    return {k: t.detach() for k, t in v.items()}, dict(zip(LEAVES, grads)), s


def _rank_step(x, rows, ri, ws):
    """One rank's losses of one frame, through frame_losses / lidar_depth_loss and through the losses.py wrappers, and the LiDAR n and
    k through the stages over the same transport.  Returns (values, leaves) per form; gradients are taken after the ranks joined."""
    out = {}
    for form in ("entry", "wrapper"):
        lv = {k: _banded(x[k], rows).requires_grad_(True) for k in LEAVES}
        if form == "entry":
            v = band_losses.frame_losses(lv["img"], x["gt"], x["mask"], lambda_dssim=LAMBDA_DSSIM, acc=lv["acc"], sky_mask=x["sky"],
                                         sky_weight=SKY_W, acc_obj=lv["acc_obj"], obj_bound=x["bound"], obj_weight=OBJ_W, rasterizer=ri)
            v["lidar"] = band_losses.lidar_depth_loss(lv["depth"], lv["dacc"], x["lidar"], x["lmask"], LIDAR_W, KEEP, rasterizer=ri)
        else:
            v = dict(photometric=losses.photometric_loss(lv["img"], x["gt"], x["mask"], lambda_dssim=LAMBDA_DSSIM, rasterizer=ri),
                     sky=losses.sky_loss(lv["acc"], x["sky"], SKY_W, rasterizer=ri),
                     obj_acc=losses.obj_acc_loss(lv["acc_obj"], x["bound"], OBJ_W, rasterizer=ri),
                     lidar=losses.lidar_depth_loss(lv["depth"], lv["dacc"], x["lidar"], x["lmask"], LIDAR_W, KEEP, rasterizer=ri))
        out[form] = (v, lv)
    band, xfer = band_losses.resolve(None, None, ri, x["depth"].shape[-2])
    H, W = (int(s) for s in x["depth"].shape[-2:])
    d, a = _banded(x["depth"], rows), _banded(x["dacc"], rows)
    state, scratch = band_losses.lidar_keys(d, a, x["lidar"], x["lmask"].reshape(-1).to(torch.uint8), band)
    for level in (1, 2):
        xfer.sum(band_losses.lidar_level_words(state, level - 1))
        band_losses.lidar_select(level, KEEP, H, W, band, state, scratch)
    xfer.sum(band_losses.lidar_level_words(state, 2))
    sums = band_losses.lidar_select(3, KEEP, H, W, band, state, scratch)
    xfer.sum(sums)
    out["lidar_scalars"] = band_losses.lidar_grad(d, a, x["lidar"], LIDAR_W, band, state, sums, scratch, False, False)[2]
    return out


def _emulate(world, layout, H, frames):
    """Every frame of `frames` through `world` emulated ranks, back to back on the same workspaces: per rank, per frame, _rank_step."""
    W = int(frames[0]["img"].shape[-1])
    wss = SH.PeerWorkspace.emulate(_settings(H, W), 8, world, DEV)
    ris = [_stand_in(wss[r], _band(H, r, world, layout)) for r in range(world)]
    rows = [_rows(H, r, world, layout) for r in range(world)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    torch.cuda.synchronize()

    def rank(r, _tr):
        with torch.cuda.stream(streams[r]):
            return [_rank_step(x, rows[r], ris[r], wss[r]) for x in frames]

    res = run_ranks(world, rank)
    torch.cuda.synchronize()
    return res, rows


def _warm_up():
    """Every kernel of the path loaded before ranks spin in emulated barriers (see test_sharded64_gpu._warm_up_fused_path): the whole
    path at world 1 (no barrier, no halo message), the halo copies, then two ranks enqueued one after the other from this thread, so the
    barrier kernel is loaded while nothing spins."""
    if _warm:
        return
    H, W = 375, W_OF[375]
    x = _frame_inputs(H, W, 1)
    _emulate(1, "cyclic", H, [x])
    _single(x)
    b = SH.cyclic_band(H, 0, 2)
    for side in (band_losses.SEND_UP, band_losses.SEND_DOWN):
        band_losses.halo_pack(x["img"], b, side)
    for side in (band_losses.RECV_UP, band_losses.RECV_DOWN):
        band_losses.halo_unpack(x["img"].clone(), b, side, torch.zeros(3, band_losses.halo_rows(H, b, side), W, device=DEV))
    pair = SH.PeerWorkspace.emulate(_settings(H, W), 8, 2, DEV)
    streams = [torch.cuda.Stream(device=DEV) for _ in range(2)]
    t = [torch.zeros(5, device=DEV, dtype=torch.float64) for _ in range(2)]
    u = [torch.zeros(5, device=DEV, dtype=torch.int32) for _ in range(2)]
    torch.cuda.synchronize()
    for r in range(2):
        with torch.cuda.stream(streams[r]):
            band_losses.peer_sum(pair[r], t[r])
            band_losses.peer_sum(pair[r], u[r])
    torch.cuda.synchronize()
    _warm.append(True)


def _check_case(world, layout, H, frames, res, rows):
    for f, x in enumerate(frames):
        ref_v, ref_g, ref_s = _single(x)
        for form in ("entry", "wrapper"):
            vals = [res[r][f][form][0] for r in range(world)]
            for key in ("photometric", "sky", "obj_acc", "lidar"):
                for r in range(1, world):
                    assert _bits_equal(vals[r][key].reshape(1), vals[0][key].reshape(1)), (f, form, key, r)
            got = vals[0]
            raw_g, raw_r = float(got["photometric"].detach()) - LAMBDA_DSSIM, float(ref_v["photometric"]) - LAMBDA_DSSIM
            bound = np.spacing(np.float32(max(abs(raw_g), abs(raw_r)))) + np.spacing(np.float32(abs(float(ref_v["photometric"]))))
            assert abs(float(got["photometric"]) - float(ref_v["photometric"])) <= bound, (f, form)
            for key in ("sky", "obj_acc"):
                assert abs(float(got[key]) - float(ref_v[key])) <= VALUE_RTOL_ACC * abs(float(ref_v[key])), (f, form, key)
            assert _ulp_close(got["lidar"], ref_v["lidar"]), (f, form, float(got["lidar"]), float(ref_v["lidar"]))
            sel = torch.zeros_like(ref_g["depth"], dtype=torch.bool)
            for r in range(world):
                v, lv = res[r][f][form]
                grads = torch.autograd.grad([v["photometric"], v["sky"], v["obj_acc"], v["lidar"]], [lv[k] for k in LEAVES])
                for k, g in zip(LEAVES, grads):
                    own = rows[r]
                    assert _bits_equal(g[:, own], ref_g[k][:, own]), (f, form, k, r)
                    if (~own).any():
                        assert not bool(g[:, ~own].any()), (f, form, k, r)
                sel |= grads[LEAVES.index("depth")] != 0
            assert torch.equal(sel, ref_g["depth"] != 0), (f, form)  # the LiDAR selection
        for r in range(world):
            s = res[r][f]["lidar_scalars"]
            assert float(s[2]) == float(ref_s[2]) and float(s[3]) == float(ref_s[3]), (f, r, "n / k")


@pytest.mark.parametrize("world,layout,H", CASES)
def test_band_losses_over_peer_memory_are_the_frame_on_every_rank(world, layout, H):
    _warm_up()
    W = W_OF[H]
    frames = [_frame_inputs(H, W, 20 + world), _frame_inputs(H, W, 41 + world)]  # two frames through the same sections
    res, rows = _emulate(world, layout, H, frames)
    _check_case(world, layout, H, frames, res, rows)


def _sum_ranks(world, locals_):
    wss = SH.PeerWorkspace.emulate(_settings(80, 64), 8, world, DEV)
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    ts = [t.clone() for t in locals_]
    torch.cuda.synchronize()

    def rank(r, _tr):
        with torch.cuda.stream(streams[r]):
            band_losses.peer_sum(wss[r], ts[r])

    run_ranks(world, rank)
    torch.cuda.synchronize()
    return ts


def test_peer_sum_adds_the_ranks_in_ascending_order():
    """2^53 + 1 rounds back to 2^53: from rank 0 up the sum is 1, from rank 3 down it is 2.  Every rank gets the ascending one."""
    _warm_up()
    parts = [2.0 ** 53, 1.0, -2.0 ** 53, 1.0]
    asc, desc = 0.0, 0.0
    for p in parts:
        asc += p
    for p in reversed(parts):
        desc += p
    assert asc == 1.0 and desc == 2.0
    locs = [torch.tensor([p, -p, 0.5], device=DEV, dtype=torch.float64) for p in parts]
    out = _sum_ranks(4, locs)
    for t in out:
        assert float(t[0]) == asc and float(t[0]) != desc
        assert float(t[1]) == -asc and float(t[2]) == 2.0


def test_peer_sum_int32_is_exact_at_world_8():
    _warm_up()
    g = torch.Generator(device=DEV).manual_seed(3)
    locs = [torch.randint(-(1 << 27), 1 << 27, (4096 + 6,), device=DEV, generator=g, dtype=torch.int32) for _ in range(8)]
    want = sum(t.long() for t in locs)
    assert int(want.abs().max()) < (1 << 31)
    for t in _sum_ranks(8, locs):
        assert torch.equal(t.long(), want)


@pytest.mark.parametrize("world,layout", [(2, "cyclic"), (3, "contiguous"), (5, "cyclic")])
@pytest.mark.parametrize("dropped", ["up", "down"])
def test_halo_without_one_side_fails_the_gradient_check(world, layout, dropped, monkeypatch):
    """Mutation check: the real exchange runs on every rank, then the rows it received from one side are put back to the rank's own
    (zero) rows.  The photometric gradient near those band edges then differs from the single-GPU one."""
    _warm_up()
    H, W = 375, W_OF[375]
    exchange = band_losses.peer_exchange_halo  # the poisoning wrapper of the autouse fixture

    def one_sided(ws, image, band):
        out = exchange(ws, image, band)
        side = band_losses.RECV_UP if dropped == "up" else band_losses.RECV_DOWN
        idx = band_losses.halo_row_indices(H, band, side).to(image.device)
        out[:, idx] = image.detach()[:, idx].to(out.dtype)
        return out

    monkeypatch.setattr(band_losses, "peer_exchange_halo", one_sided)
    x = _frame_inputs(H, W, 5)
    ref = x["img"].clone().requires_grad_(True)
    ref_g, = torch.autograd.grad(losses.photometric_loss(ref, x["gt"], x["mask"]), [ref])
    wss = SH.PeerWorkspace.emulate(_settings(H, W), 8, world, DEV)
    rows = [_rows(H, r, world, layout) for r in range(world)]
    leaves = [_banded(x["img"], rows[r]).requires_grad_(True) for r in range(world)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    torch.cuda.synchronize()

    def rank(r, _tr):
        with torch.cuda.stream(streams[r]):
            return losses.photometric_loss(leaves[r], x["gt"], x["mask"], rasterizer=_stand_in(wss[r], _band(H, r, world, layout)))

    vals = run_ranks(world, rank)
    torch.cuda.synchronize()
    wrong = 0
    for r in range(world):
        g, = torch.autograd.grad(vals[r], [leaves[r]])
        wrong += int((g[:, rows[r]] != ref_g[:, rows[r]]).sum())
    assert wrong > 0


def test_world_one_band_is_the_whole_image():
    """At world 1 (the rasterizer has no band) the losses take the whole image: the single-GPU gradient bit for bit."""
    _warm_up()
    H, W = 375, W_OF[375]
    x = _frame_inputs(H, W, 9)
    ws = SH.PeerWorkspace.emulate(_settings(H, W), 8, 1, DEV)[0]
    band, xfer = band_losses.resolve(None, None, _stand_in(ws, None), H)
    assert tuple(band) == (0, (H + 15) // 16, 1) and xfer.kind == "p2p"
    assert tuple(band_losses.resolve(TileRowBand(0, (H + 15) // 16, 1), None, _stand_in(ws, None), H)[0]) == tuple(band)
