"""GPU: the sky cube gradient and the colour correction's sums over peer memory (sky.sky_composite / corrections.color_correct with
rasterizer= of a GaussianShardedRasterizer(exchange="p2p"); include/sgr.h sgr_band_sky_composite_backward_marked, sgr_sky_grad_peer_sum),
with 1, 2, 3, 5 and 8 ranks emulated by threads (tests/rank_threads.py) on streams of one GPU through PeerWorkspace.emulate,
SkyWorkspace.emulate and a stand-in rasterizer.

Every kernel is loaded before any rank spins in an emulated barrier (_warm_up), and every rank's sky section is filled with NaN before
each exchange, so no call reads bytes it did not stage in that call.

Checked through the real autograd entries, two frames with different touched blocks back to back through the same sections: every
rank's cube_map.grad has the same bytes; it is within tests/sky_oracle.py's per-texel bound of the whole-frame float64 gradient (and
within the atomic-order bound of the whole-frame fp32 one); rgb_out, dL/drgb and dL/dacc rows are bit-identical to the whole-frame
call's; each rank's block map, poisoned with 0xff first, holds exactly the blocks of the texels its band's sampled pixels tap.
The exchange alone: chosen partials and maps give torch's ascending-rank sum bit for bit (a descending one differs) and zeros outside
the union.  The colour correction's affine gradient is the ascending fp64 sum of the band partials, rounded once, on every rank.  Both
backwards pass with synchronising CUDA calls made errors, and one emulated iteration (sky -> colour correction -> frame losses)
matches the band semantics."""
import types

import pytest
import torch

import sky_oracle as SO
import street_gaussians_b200 as sgb
from rank_threads import run_ranks
from street_gaussians_b200 import _capi, band_losses, corrections, losses, sky
from street_gaussians_b200 import sharded as SH
from street_gaussians_b200._capi import ptr
from street_gaussians_b200.rasterizer import GaussianRasterizationSettings, TileRowBand
from test_sky_gpu import _look_at

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
F64 = torch.float64
U = 2.0 ** -24
W_OF = {375: 200, 1280: 1920}
BLOCK = 32
VIEWS = {"edge": ([1.0, -0.15, 1.0], 0.1), "corner": ([1.0, -1.0, 1.0], 0.2)}
# (sky mask given, fill, jitter)
VARIANTS = [(False, 1.0, False), (True, 0.0, True), (True, 1.0, False), (False, 0.0, True)]
_warm = []


def _settings(H, W):
    z = torch.zeros(3, device=DEV)
    return GaussianRasterizationSettings(H, W, 0.5, 0.5, z, 1.0, torch.eye(4, device=DEV), torch.eye(4, device=DEV), 0, z, False, False)


def _stand_in(ws, sky_ws, band):
    """What sky_composite / color_correct read of a GaussianShardedRasterizer(exchange="p2p"), around emulated workspaces."""
    return types.SimpleNamespace(exchange="p2p", group=None, band=band, loss_workspace=lambda: ws, sky_workspace=lambda R, device=None: sky_ws)


def _rows_of(H, band):
    if band is None:
        return torch.ones(H, dtype=torch.bool, device=DEV)
    rows = torch.arange((H + 15) // 16)
    own = (rows >= band.begin) & (rows < band.end) & (((rows - band.begin) % band.step) == 0)
    return own.repeat_interleave(16)[:H].to(DEV)


def _banded(x, rows):
    return torch.where(rows.view(1, -1, 1), x, torch.zeros_like(x))


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.fixture(autouse=True)
def _poison_sky_sections(monkeypatch):
    """Fill the calling rank's sky section with NaN (0xff bytes) on its stream before every exchange.  Safe between calls: each call
    ends with a barrier after which no peer reads the section."""
    exchange = sky.sky_grad_peer_sum

    def poisoned(ws, sky_ws, g_cube):
        sky_ws.buf.fill_(0xff)
        return exchange(ws, sky_ws, g_cube)

    monkeypatch.setattr(sky, "sky_grad_peer_sum", poisoned)


# ---- frames and the whole-frame reference ---------------------------------------------------------------------------------------
def _frame(H, R, seed, view, variant):
    W = W_OF[H]
    masked, fill, jitter = variant
    g = torch.Generator(device=DEV).manual_seed(seed)
    cube = -0.2 + 1.4 * torch.rand(6, R, R, 3, generator=g, device=DEV)
    rgb = torch.rand(3, H, W, generator=g, device=DEV)
    acc = torch.rand(1, H, W, generator=g, device=DEV)
    acc = torch.where(torch.rand(1, H, W, generator=g, device=DEV) < 0.5, torch.zeros_like(acc), acc)
    up = torch.randn(3, H, W, generator=g, device=DEV)
    mask = torch.rand(1, H, W, generator=g, device=DEV) < 0.3 if masked else None
    f = 1.07 * W
    K = torch.tensor([[f, 0.0, W / 2], [0.0, f, H / 2], [0.0, 0.0, 1.0]], device=DEV)
    return dict(cube=cube, rgb=rgb, acc=acc, up=up, mask=mask, K=K, w2c=_look_at(*VIEWS[view]).to(DEV), fill=fill, jitter=jitter,
                seed=seed)


def _composite(x, rgb, acc, cube, rasterizer=None):
    if x["jitter"]:
        torch.manual_seed(x["seed"])  # the same [H, W] jitter pair on every rank and in the whole-frame call
    return sgb.sky_composite(rgb, acc, cube, x["K"], x["w2c"], sky_mask=x["mask"], perturb=x["jitter"], white_background=x["fill"] == 1.0,
                             rasterizer=rasterizer)


def _whole(x):
    rgb, acc, cube = (x[k].clone().requires_grad_(True) for k in ("rgb", "acc", "cube"))
    out = _composite(x, rgb, acc, cube)
    out.backward(x["up"])
    jx = jy = None
    if x["jitter"]:
        torch.manual_seed(x["seed"])
        H, W = x["rgb"].shape[1:]
        jx, jy = torch.rand(H, W, device=DEV), torch.rand(H, W, device=DEV)
    return dict(out=out.detach(), rgb=rgb.grad, acc=acc.grad, cube=cube.grad, jx=jx, jy=jy)


def _texel_terms(x, ref):
    """Per texel: n, the number of per-pixel terms its atomics add, and sum |term| (the fp64 restatement of the kernel's terms)."""
    H, W = x["rgb"].shape[1:]
    R = x["cube"].shape[1]
    d = SO.rays(H, W, x["K"].to(F64), x["w2c"].to(F64), ref["jx"], ref["jy"])
    face, gx, gy = SO.face_coords(d)
    idx, w = SO.effective(*SO.taps(face, *SO.tex_xy(gx, gy, R), R))
    sampled = SO.sky_mask_of(x["acc"], x["mask"])
    gt = (x["up"].to(F64) * (1 - x["acc"].to(F64))).permute(1, 2, 0) * sampled.unsqueeze(-1)
    term = (w.unsqueeze(-1) * gt.unsqueeze(-2)).abs()
    live = (w > 0) & sampled.unsqueeze(-1)
    n = torch.zeros(6 * R * R, dtype=F64, device=DEV).index_add_(0, idx.reshape(-1), live.reshape(-1).to(F64))
    sabs = torch.zeros(6 * R * R, 3, dtype=F64, device=DEV).index_add_(0, idx.reshape(-1), term.reshape(-1, 3))
    return n.view(6, R, R, 1), sabs.view(6, R, R, 3)


def _block_ids(idx, R):
    nb = -(-R // BLOCK)
    idx = idx[idx >= 0]
    f, rem = idx // (R * R), idx % (R * R)
    return ((f * nb + (rem // R) // BLOCK) * nb + (rem % R) // BLOCK).unique()


def _map_bounds(x, ref, rows):
    """(blocks every restated tap set marks, blocks any marks): the band's sampled pixels' taps at (x, y) and at (x +- e, y +- e), e =
    1e-3 texel, so a tap the fp32 kernel puts on the other side of a texel edge is allowed."""
    H, W = x["rgb"].shape[1:]
    R = x["cube"].shape[1]
    d = SO.rays(H, W, x["K"].to(F64), x["w2c"].to(F64), ref["jx"], ref["jy"])
    face, gx, gy = SO.face_coords(d)
    tx, ty = SO.tex_xy(gx, gy, R)
    sel = SO.sky_mask_of(x["acc"], x["mask"]) & rows.view(-1, 1)
    sets = []
    for ex, ey in ((0, 0), (-1, -1), (-1, 1), (1, -1), (1, 1)):
        xs, ys = (tx + 1e-3 * ex).clamp(-0.5, R - 0.5), (ty + 1e-3 * ey).clamp(-0.5, R - 0.5)
        idx, _ = SO.taps(face[sel], xs[sel], ys[sel], R)
        sets.append(set(_block_ids(idx.reshape(-1), R).tolist()))
    return set.intersection(*sets), set.union(*sets)


def _chain(x, gt, rgb, acc, cube, A, ri):
    """sky_composite -> color_correct -> the photometric and sky losses, whole-frame (ri None) or with rasterizer=ri."""
    s = _composite(x, rgb, acc, cube, ri)
    s.retain_grad()
    col = corrections.color_correct(s, A, rasterizer=ri)
    col.retain_grad()
    if ri is None:
        vals = [losses.photometric_loss(col, gt, None, 1.0, 0.2), losses.sky_loss(acc, x["mask"], 1.0)]
    else:
        fl = band_losses.frame_losses(col, gt, None, 1.0, 0.2, acc=acc, sky_mask=x["mask"], rasterizer=ri)
        vals = [fl["photometric"], fl["sky"]]
    return vals, s, col


# ---- emulated ranks through the autograd entry ----------------------------------------------------------------------------------
def _emulate(world, H, R, frames, check_map=True):
    """Every frame of `frames` through `world` emulated ranks, back to back on the same workspaces.  Forwards are issued from this thread
    (the jitter comes from the global generator); the backwards, which are collective, from one thread per rank."""
    W = W_OF[H]
    wss = SH.PeerWorkspace.emulate(_settings(H, W), 8, world, DEV)
    skys = SH.SkyWorkspace.emulate(R, world, DEV) if world > 1 else [None]
    bands = [SH.cyclic_band(H, r, world) if world > 1 else None for r in range(world)]
    ris = [_stand_in(wss[r], skys[r], bands[r]) for r in range(world)]
    rows = [_rows_of(H, b) for b in bands]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    res = []
    for x in frames:
        torch.cuda.synchronize()
        per = []
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                lv = dict(rgb=_banded(x["rgb"], rows[r]).requires_grad_(True), acc=_banded(x["acc"], rows[r]).requires_grad_(True),
                          cube=x["cube"].clone().requires_grad_(True))
                out = _composite(x, lv["rgb"], lv["acc"], lv["cube"], ris[r])
                if skys[r] is not None and check_map:
                    skys[r].block_map.fill_(0xff)
                per.append((lv, out, _banded(x["up"], rows[r])))
        torch.cuda.synchronize()

        def rank(r, _tr):
            with torch.cuda.stream(streams[r]):
                lv, out, up = per[r]
                torch.autograd.backward([out], [up])

        run_ranks(world, rank)
        torch.cuda.synchronize()
        res.append([dict(out=o.detach(), rgb=lv["rgb"].grad, acc=lv["acc"].grad, cube=lv["cube"].grad,
                         map=skys[r].block_map.clone() if skys[r] is not None else None) for r, (lv, o, _) in enumerate(per)])
    return res, rows


def _warm_up():
    """Every kernel of the path loaded before ranks spin in emulated barriers: the whole chain once on the band entries with a
    whole-image band at world 1 (no barrier), the whole-frame calls, the halo copies, then two ranks' exchanges enqueued one after the
    other from this thread, so the barrier kernel loads while nothing spins."""
    if _warm:
        return
    H, W, R = 375, W_OF[375], 16
    x = _frame(H, R, 1, "edge", VARIANTS[1])
    gt = torch.rand(3, H, W, device=DEV)
    ri = _stand_in(SH.PeerWorkspace.emulate(_settings(H, W), 8, 1, DEV)[0], SH.SkyWorkspace.emulate(R, 1, DEV)[0],
                   TileRowBand(0, (H + 15) // 16, 1))
    for r in (ri, None):
        leaves = [t.clone().requires_grad_(True) for t in (x["rgb"], x["acc"], x["cube"], torch.eye(4, device=DEV)[:3])]
        torch.autograd.backward(_chain(x, gt, *leaves, r)[0])
    b = SH.cyclic_band(H, 0, 2)
    for side in (band_losses.SEND_UP, band_losses.SEND_DOWN):
        band_losses.halo_pack(x["rgb"], b, side)
    for side in (band_losses.RECV_UP, band_losses.RECV_DOWN):
        band_losses.halo_unpack(x["rgb"].clone(), b, side, torch.zeros(3, band_losses.halo_rows(H, b, side), W, device=DEV))
    wss = SH.PeerWorkspace.emulate(_settings(H, W), 8, 2, DEV)
    skys = SH.SkyWorkspace.emulate(R, 2, DEV)
    g = [torch.zeros(6, R, R, 3, device=DEV) for _ in range(2)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(2)]
    torch.cuda.synchronize()
    for r in range(2):
        with torch.cuda.stream(streams[r]):
            skys[r].block_map.zero_()
            sky.sky_grad_peer_sum(wss[r], skys[r], g[r])
            band_losses.peer_sum(wss[r], torch.zeros(12, device=DEV, dtype=F64))
    torch.cuda.synchronize()
    _warm.append(True)


CASES = [(world, H) for world in (1, 2, 3, 5, 8) for H in (375, 1280)]


@pytest.mark.parametrize("R", [16, 100, 1024])
@pytest.mark.parametrize("world,H", CASES)
def test_sky_over_peer_memory_is_the_frame_on_every_rank(world, H, R):
    _warm_up()
    k = (world + H + R) % len(VARIANTS)
    # two frames whose touched blocks differ (a face edge, then a cube corner), both mask modes, both fills and jitter over the cases
    frames = [_frame(H, R, 10 * world + R, "edge", VARIANTS[k]), _frame(H, R, 11 * world + R + 1, "corner", VARIANTS[(k + 1) % len(VARIANTS)])]
    res, rows = _emulate(world, H, R, frames)
    for f, x in enumerate(frames):
        ref = _whole(x)
        got = res[f]
        for r in range(world):
            own = rows[r]
            for key in ("out", "rgb", "acc"):
                assert _bits_equal(got[r][key][:, own], ref[key][:, own]), (f, r, key)
                if bool((~own).any()):
                    assert not bool(got[r][key][:, ~own].any()), (f, r, key)
            assert _bits_equal(got[r]["cube"], got[0]["cube"]), (f, r, "cube bytes differ between ranks")
        gc = got[0]["cube"].to(F64)
        n, sabs = _texel_terms(x, ref)
        bound = 2 * n * U * sabs * (1 + 1e-3) + 1e-30
        err = (gc - ref["cube"].to(F64)).abs()
        assert bool((err <= bound).all()), (f, int((err > bound).sum()), float((err / bound).max()))
        assert int((ref["cube"] != 0).sum()) > 10
        if H == 375 or world == 8:  # the fp64 restatement (memory-heavy at 1280 x 1920)
            o = SO.sky64(x["rgb"], x["acc"], x["cube"], x["K"], x["w2c"], x["up"], x["mask"], ref["jx"], ref["jy"], x["fill"])
            e64 = (gc - o["dcube"]).abs()
            assert bool((e64 <= o["b_dcube"]).all()), (f, int((e64 > o["b_dcube"]).sum()))
        if world > 1:
            for r in range(world):
                lo, hi = _map_bounds(x, ref, rows[r])
                m = got[r]["map"]
                assert int(m.max()) <= 1, (f, r, "the map's 0xff fill survived")
                marked = set(torch.nonzero(m).view(-1).tolist())
                assert lo <= marked <= hi and len(hi - lo) <= max(4, len(hi) // 20), (f, r, len(lo - marked), len(marked - hi), len(hi - lo))


# ---- the exchange alone ---------------------------------------------------------------------------------------------------------
def _exchange(parts, maps, R):
    world = len(parts)
    wss = SH.PeerWorkspace.emulate(_settings(80, 64), 8, world, DEV)
    skys = SH.SkyWorkspace.emulate(R, world, DEV)
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    gs = [p.clone() for p in parts]
    for r in range(world):
        skys[r].block_map.copy_(maps[r])
    torch.cuda.synchronize()

    def rank(r, _tr):
        with torch.cuda.stream(streams[r]):
            sky.sky_grad_peer_sum(wss[r], skys[r], gs[r])

    run_ranks(world, rank)
    torch.cuda.synchronize()
    return gs


def _texel_blocks(R):
    nb = -(-R // BLOCK)
    f, r, c = torch.meshgrid(torch.arange(6), torch.arange(R), torch.arange(R), indexing="ij")
    return ((f * nb + r // BLOCK) * nb + c // BLOCK).to(DEV)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("R", [37, 100])  # 37: clipped blocks and rows that start off 16-byte alignment
def test_exchange_is_the_ascending_rank_sum(world, R):
    """Values 2^24 and 1 make the order visible: 2^24 + 1 rounds back to 2^24, so summing from rank 0 up and from the last rank down
    differ.  Each rank's partial is zero outside its marked blocks; blocks nobody marked come back zero."""
    _warm_up()
    nblk = int(_capi.lib().sgr_sky_grad_blocks(R))
    g = torch.Generator(device=DEV).manual_seed(R + world)
    tb = _texel_blocks(R)
    maps, parts = [], []
    scale = [2.0 ** 24 if p % 2 == 0 else 1.0 for p in range(world)]
    for p in range(world):
        m = (torch.rand(nblk, generator=g, device=DEV) < 0.4).to(torch.uint8)
        m[0] = 1  # block 0: marked everywhere, the order shows there for certain
        m[nblk - 1] = 0  # the last block: nobody's
        part = (1.0 + torch.rand(6, R, R, 3, generator=g, device=DEV)) * scale[p] * (1 if p % 4 < 2 else -1)
        part = torch.where(m.bool()[tb].unsqueeze(-1), part, torch.zeros_like(part))
        maps.append(m * (1 + p))  # any non-zero byte marks
        parts.append(part)
    got = _exchange(parts, maps, R)
    asc = torch.zeros_like(parts[0])
    for p in range(world):
        asc = asc + parts[p]
    desc = torch.zeros_like(parts[0])
    for p in reversed(range(world)):
        desc = desc + parts[p]
    if world > 2:  # two terms add alike in either order
        assert not _bits_equal(asc, desc)
    union = torch.stack(maps).bool().any(0)[tb]
    for r in range(world):
        assert _bits_equal(got[r], asc), r
        assert not bool(got[r][~union].any()) and not bool(torch.isnan(got[r]).any())


# ---- the colour correction ------------------------------------------------------------------------------------------------------
def _cc_partials(img, A, up, band):
    H, W = img.shape[1:]
    nb = int(_capi.lib().sgr_band_color_correct_scratch_bytes(H, W))
    scratch = torch.empty(nb, device=DEV, dtype=torch.uint8)
    sums = torch.empty(12, device=DEV, dtype=F64)
    _capi.call("sgr_band_color_correct_backward", DEV, H, W, *band, ptr(img), ptr(A), ptr(up), None, ptr(sums), ptr(scratch), nb)
    return sums


@pytest.mark.parametrize("world", [2, 5, 8])
def test_color_correct_over_peer_memory(world):
    _warm_up()
    H, W = 375, W_OF[375]
    g = torch.Generator(device=DEV).manual_seed(world)
    img = torch.rand(3, H, W, generator=g, device=DEV)
    A = torch.eye(4, device=DEV)[:3] + 0.1 * torch.randn(3, 4, generator=g, device=DEV)
    up = torch.randn(3, H, W, generator=g, device=DEV)
    wss = SH.PeerWorkspace.emulate(_settings(H, W), 8, world, DEV)
    bands = [SH.cyclic_band(H, r, world) for r in range(world)]
    rows = [_rows_of(H, b) for b in bands]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    leaves = [(_banded(img, rows[r]).requires_grad_(True), A.clone().requires_grad_(True)) for r in range(world)]
    torch.cuda.synchronize()

    def rank(r, _tr):
        with torch.cuda.stream(streams[r]):
            out = corrections.color_correct(leaves[r][0], leaves[r][1], rasterizer=_stand_in(wss[r], None, bands[r]))
            torch.autograd.backward([out], [_banded(up, rows[r])])

    run_ranks(world, rank)
    torch.cuda.synchronize()
    total = torch.zeros(12, dtype=F64)
    for r in range(world):  # ascending rank order, in fp64
        total = total + _cc_partials(_banded(img, rows[r]), A, _banded(up, rows[r]), tuple(bands[r])).cpu()
    want = total.to(torch.float32).view(3, 4).to(DEV)
    for r in range(world):
        assert _bits_equal(leaves[r][1].grad, want), r


# ---- no host synchronisation ------------------------------------------------------------------------------------------------------
def test_p2p_backwards_make_no_host_synchronisation():
    _warm_up()
    world, H, R = 2, 375, 100
    x = _frame(H, R, 5, "corner", VARIANTS[1])
    wss = SH.PeerWorkspace.emulate(_settings(H, W_OF[H]), 8, world, DEV)
    skys = SH.SkyWorkspace.emulate(R, world, DEV)
    bands = [SH.cyclic_band(H, r, world) for r in range(world)]
    rows = [_rows_of(H, b) for b in bands]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    per = []
    for r in range(world):
        with torch.cuda.stream(streams[r]):
            ri = _stand_in(wss[r], skys[r], bands[r])
            rgb, acc = _banded(x["rgb"], rows[r]).requires_grad_(True), _banded(x["acc"], rows[r]).requires_grad_(True)
            cube, A = x["cube"].clone().requires_grad_(True), torch.eye(4, device=DEV)[:3].clone().requires_grad_(True)
            out = corrections.color_correct(_composite(x, rgb, acc, cube, ri), A, rasterizer=ri)
            per.append((out, _banded(x["up"], rows[r]), cube, A))
    torch.cuda.synchronize()

    def rank(r, _tr):
        with torch.cuda.stream(streams[r]):
            torch.autograd.backward([per[r][0]], [per[r][1]])

    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        run_ranks(world, rank)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    assert _bits_equal(per[0][2].grad, per[1][2].grad) and _bits_equal(per[0][3].grad, per[1][3].grad)


# ---- one emulated iteration ---------------------------------------------------------------------------------------------------------
def test_one_iteration_at_world_two():
    """sky_composite -> color_correct -> frame_losses with rasterizer= of a p2p stand-in, then backward, against the whole-frame calls:
    dL/drgb and dL/dacc rows bit-identical, the cube gradient the same bytes on both ranks and within the atomic-order bound, the affine
    gradient the ascending fp64 sum of the band partials of the ranks' own upstream gradients, rounded once."""
    _warm_up()
    world, H, R = 2, 375, 100
    W = W_OF[H]
    x = _frame(H, R, 21, "edge", VARIANTS[2])
    g = torch.Generator(device=DEV).manual_seed(4)
    gt = torch.rand(3, H, W, generator=g, device=DEV)
    A0 = torch.eye(4, device=DEV)[:3] + 0.05 * torch.randn(3, 4, generator=g, device=DEV)
    rgb0, acc0, cube0, Aw = (t.clone().requires_grad_(True) for t in (x["rgb"], x["acc"], x["cube"], A0))
    vals, s0, _ = _chain(x, gt, rgb0, acc0, cube0, Aw, None)
    torch.autograd.backward(vals)
    wss = SH.PeerWorkspace.emulate(_settings(H, W), 8, world, DEV)
    skys = SH.SkyWorkspace.emulate(R, world, DEV)
    bands = [SH.cyclic_band(H, r, world) for r in range(world)]
    rows = [_rows_of(H, b) for b in bands]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    leaves = [tuple(t.clone().requires_grad_(True) for t in (_banded(x["rgb"], rows[r]), _banded(x["acc"], rows[r]), x["cube"], A0))
              for r in range(world)]
    torch.cuda.synchronize()

    def rank(r, _tr):  # the band losses' forward is collective too: the whole chain runs per rank thread
        with torch.cuda.stream(streams[r]):
            if x["jitter"]:
                raise AssertionError("this test's variant draws no jitter (threads share the generator)")
            vals, s, col = _chain(x, gt, *leaves[r], _stand_in(wss[r], skys[r], bands[r]))
            torch.autograd.backward(vals)
            return s, col

    res = run_ranks(world, rank)
    torch.cuda.synchronize()
    total = torch.zeros(12, dtype=F64)
    for r in range(world):
        own = rows[r]
        rgb, acc, cube, A = leaves[r]
        assert _bits_equal(rgb.grad[:, own], rgb0.grad[:, own]) and _bits_equal(acc.grad[:, own], acc0.grad[:, own]), r
        assert _bits_equal(cube.grad, leaves[0][2].grad) and _bits_equal(A.grad, leaves[0][3].grad), r
        s, col = res[r]
        total = total + _cc_partials(s.detach(), A0, col.grad, tuple(bands[r])).cpu()
    assert _bits_equal(leaves[0][3].grad, total.to(torch.float32).view(3, 4).to(DEV))
    ref = dict(jx=None, jy=None)
    n, sabs = _texel_terms(dict(x, up=s0.grad), ref)
    err = (leaves[0][2].grad.to(F64) - cube0.grad.to(F64)).abs()
    assert bool((err <= 2 * n * U * sabs * (1 + 1e-3) + 1e-30).all())
