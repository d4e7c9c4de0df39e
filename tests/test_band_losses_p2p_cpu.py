"""CPU: the band losses' exchanges over peer memory (include/sgr.h sgr_band_peer_bytes, sgr_band_halo_exchange_peers,
sgr_band_peer_sum; band_losses.resolve and the rasterizer= keyword).  The entries validate their arguments before anything is enqueued,
the loss section is large enough for every halo message and every summed array, PeerWorkspace wires the section for every rank, and
rasterizer= picks the transport and the band, refusing what does not match before any launch."""
import ctypes as C
import types

import pytest
import torch

import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi, band_losses, losses
from street_gaussians_b200 import sharded as SH
from street_gaussians_b200.rasterizer import TileRowBand

OK = C.c_void_p(1 << 20)  # a 16-byte aligned address: validation fails before anything dereferences it


def _err():
    return _capi.lib().sgr_last_error().decode()


def test_symbols_exported():
    L = _capi.lib()
    for name in ("sgr_band_peer_bytes", "sgr_band_halo_exchange_peers", "sgr_band_peer_sum"):
        assert name in _capi.SYMBOLS
        assert getattr(L, name) is not None
    names = [f[0] for f in _capi.SgrPeers._fields_]
    assert names[-2:] == ["loss", "loss_bytes"]  # appended after pose_acc: the earlier offsets are unchanged
    assert _capi.SgrPeers.pose_acc.offset < _capi.SgrPeers.loss.offset < _capi.SgrPeers.loss_bytes.offset


def _peers(world=2, rank=1, loss=True, flags=True, nbytes=1 << 40):
    pe = _capi.SgrPeers()
    pe.world, pe.rank, pe.chunk = world, rank, 8
    for p in range(min(world, _capi.MAX_PEERS)):
        pe.loss[p] = OK.value if loss else None
        pe.flags[p] = OK.value if flags else None
    pe.loss_bytes = nbytes
    return pe


def test_halo_exchange_validates_before_launch():
    L = _capi.lib()
    H, W = 375, 200
    need = int(L.sgr_band_peer_bytes(3, H, W))

    def call(pe=None, Cn=3, H=H, W=W, band=(1, 24, 2), image=OK, out=OK):
        return L.sgr_band_halo_exchange_peers(C.byref(pe) if pe is not None else None, Cn, H, W, *band, image, out, None)

    assert call(None) == -1 and "peers is NULL" in _err()
    assert call(_peers(world=0, rank=0)) == -1 and "bad peer table" in _err()
    assert call(_peers(world=_capi.MAX_PEERS + 1, rank=0)) == -1 and "bad peer table" in _err()
    assert call(_peers(rank=2)) == -1 and "bad peer table" in _err()
    assert call(_peers(loss=False)) == -1 and "no loss section" in _err()
    assert call(_peers(flags=False)) == -1 and "no barrier pad" in _err()
    assert call(_peers(nbytes=need - 1)) == -3 and f"{need} needed" in _err()
    assert call(_peers(), band=(0, 25, 1)) == -1 and "bad tile-row band" in _err()
    assert call(_peers(), band=(3, 2, 1)) == -1 and "bad tile-row band" in _err()
    assert call(_peers(), band=(0, 4, 0)) == -1 and "bad tile-row band" in _err()
    assert call(_peers(), H=0) == -1 and "bad image size" in _err()
    assert call(_peers(), Cn=0) == -1 and "bad channel count" in _err()
    assert call(_peers(), image=None) == -1 and "NULL pointer" in _err()
    assert call(_peers(), out=None) == -1 and "NULL pointer" in _err()
    # a 4-channel image needs more than the 3-channel section
    assert call(_peers(nbytes=need), Cn=4) == -3 and "needed" in _err()


def test_peer_sum_validates_before_launch():
    L = _capi.lib()

    def call(pe=None, kind=_capi.PEER_SUM_FLOAT64, count=5, local=OK, out=OK):
        return L.sgr_band_peer_sum(C.byref(pe) if pe is not None else None, kind, count, local, out, None)

    assert call(None) == -1 and "peers is NULL" in _err()
    assert call(_peers(world=0, rank=0)) == -1 and "bad peer table" in _err()
    assert call(_peers(world=_capi.MAX_PEERS + 1, rank=0)) == -1 and "bad peer table" in _err()
    assert call(_peers(loss=False)) == -1 and "no loss section" in _err()
    assert call(_peers(flags=False)) == -1 and "no barrier pad" in _err()
    assert call(_peers(nbytes=39)) == -3 and "40 needed" in _err()
    assert call(_peers(nbytes=19), kind=_capi.PEER_SUM_INT32) == -3 and "20 needed" in _err()
    assert call(_peers(), count=-1) == -1 and "negative count" in _err()
    assert call(_peers(), kind=2) == -1 and "unknown element type" in _err()
    assert call(_peers(), kind=-1) == -1 and "unknown element type" in _err()
    assert call(_peers(), local=None) == -1 and "NULL pointer" in _err()
    assert call(_peers(), out=None) == -1 and "NULL pointer" in _err()


def test_peer_bytes_covers_every_message_and_sum():
    """At least the largest pair of halo messages (sgr_band_halo_rows of SEND_UP and SEND_DOWN of one rank's band, [3][rows][W] fp32) over
    2-8 ranks in both layouts, and at least the largest array the band losses sum."""
    L = _capi.lib()
    assert L.sgr_band_peer_bytes(0, 40, 48) == 0 and L.sgr_band_peer_bytes(3, 0, 48) == 0 and L.sgr_band_peer_bytes(3, 40, 0) == 0
    for H, W in ((40, 48), (80, 64), (375, 200), (1280, 1920)):
        n = int(L.sgr_band_peer_bytes(3, H, W))
        assert n % 256 == 0
        rows = (H + 15) // 16
        largest_sum = max(4 * _capi.LIDAR_LEVEL0_WORDS, 4 * _capi.LIDAR_BINS, 8 * (1 + rows), 8 * 5)
        assert n >= largest_sum
        pair = 0
        for world in range(2, 9):
            for mk in (SH.cyclic_band, SH.contiguous_band):
                for r in range(world):
                    b = mk(H, r, world)
                    msgs = [int(L.sgr_band_halo_rows(H, *b, side)) for side in (band_losses.SEND_UP, band_losses.SEND_DOWN)]
                    pair = max(pair, 3 * sum(msgs) * W * 4)
        assert n >= pair > 0
    # 1920 x 1280, two ranks, cyclic: 40 strips of 10 rows per message, two messages of 3 x 1920 fp32 rows
    assert int(L.sgr_band_peer_bytes(3, 1280, 1920)) == 2 * 10 * 40 * 1920 * 3 * 4


def _st():
    return sgb.GaussianRasterizationSettings(96, 128, 0.5, 0.4, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)


def test_peer_workspace_wires_the_loss_section():
    """PeerWorkspace.emulate on CPU buffers: the section sits 256-aligned after the composer's accumulator section and before the
    barrier pad, holds sgr_band_peer_bytes(3, H, W), and every rank's table points at every rank's section."""
    st = _st()
    need = int(_capi.lib().sgr_band_peer_bytes(3, 96, 128))
    for S in (0, 5):
        wss = SH.PeerWorkspace.emulate(st, 11, 3, torch.device("cpu"), S)
        bases = [ws.buf.data_ptr() for ws in wss]
        for ws in wss:
            assert ws.off_loss % 256 == 0 and ws.off_loss >= ws.off_pose + 64 * _capi.POSE_ACC_ROWS
            assert ws.loss_bytes == need and ws.peers.loss_bytes == need
            assert ws.off_flags >= ws.off_loss + need and ws.total == ws.off_flags + 256
            assert [ws.peers.loss[p] for p in range(3)] == [b + ws.off_loss for b in bases]
            assert ws.layout(st, ws.P_total, torch.device("cpu"), S)[4] == ws.off_flags


def _raster(exchange="p2p", group=None, band=None, ws=None):
    def loss_workspace():
        if ws is None:
            raise _capi.SgrError("no forward")
        return ws
    return types.SimpleNamespace(exchange=exchange, group=group, band=band, loss_workspace=loss_workspace)


def test_rasterizer_resolution():
    H = 375
    g = object()
    band = SH.cyclic_band(H, 1, 3)
    # nccl: the rasterizer's group and band
    b, t = band_losses.resolve(None, None, _raster("nccl", group=g, band=band), H)
    assert t.kind == "nccl" and t.group is g and tuple(b) == tuple(band)
    b, t = band_losses.resolve(band, g, _raster("nccl", group=g, band=band), H)
    assert t.kind == "nccl" and t.group is g
    # no rasterizer: band= / group= as given
    b, t = band_losses.resolve(band, g, None, H)
    assert t.kind == "nccl" and t.group is g and b is band
    # p2p: the workspace of the rasterizer's forward; world 1 (no band) takes the whole image
    ws = object()
    b, t = band_losses.resolve(None, None, _raster(band=None, ws=ws), H)
    assert t.kind == "p2p" and t.ws is ws and tuple(b) == (0, 24, 1)
    # mismatches
    with pytest.raises(ValueError, match="group"):
        band_losses.resolve(None, object(), _raster("nccl", group=g, band=band), H)
    with pytest.raises(ValueError, match="band"):
        band_losses.resolve(SH.cyclic_band(H, 0, 3), None, _raster(band=band, ws=ws), H)
    with pytest.raises(_capi.SgrError):
        band_losses.resolve(None, None, _raster(band=band), H)


def test_real_rasterizer_needs_a_forward_first():
    r = SH.GaussianShardedRasterizer(_st(), exchange="p2p")
    with pytest.raises(_capi.SgrError, match="forward"):
        r.loss_workspace()
    img = torch.rand(3, 96, 128)
    with pytest.raises(_capi.SgrError, match="forward"):
        band_losses.frame_losses(img, img, rasterizer=r)
    with pytest.raises(_capi.SgrError, match="forward"):
        losses.lidar_depth_loss(img[:1], img[:1], img[:1], rasterizer=r)


def test_entries_refuse_before_any_launch():
    """On CPU tensors nothing can launch: each refusal below comes first."""
    H, W = 96, 128
    band = SH.cyclic_band(H, 0, 2)
    ws = SH.PeerWorkspace.emulate(_st(), 8, 2, torch.device("cpu"))[0]
    img4 = torch.rand(4, H, W)
    with pytest.raises(ValueError, match="3-channel"):
        band_losses.frame_losses(img4, img4, rasterizer=_raster(band=band, ws=ws))
    with pytest.raises(ValueError, match="3-channel"):
        losses.photometric_loss(img4, img4, rasterizer=_raster(band=band, ws=ws))
    with pytest.raises(ValueError, match="band"):
        losses.l1_loss(torch.rand(3, H, W), torch.rand(3, H, W), band=SH.cyclic_band(H, 1, 2), rasterizer=_raster(band=band, ws=ws))
    with pytest.raises(ValueError, match="group"):
        losses.sky_loss(torch.rand(1, H, W), torch.rand(1, H, W) > 0.5, group=object(), rasterizer=_raster(band=band, ws=ws))
    with pytest.raises(ValueError, match="band"):
        band_losses.lidar_depth_loss(torch.rand(1, H, W), torch.rand(1, H, W), torch.rand(1, H, W), band=TileRowBand(0, 6, 1),
                                     rasterizer=_raster(band=band, ws=ws))
    # a 4-channel image on the NCCL transport is not refused for its channels (the CPU tensors are)
    with pytest.raises(_capi.SgrError, match="CUDA"):
        band_losses.frame_losses(img4, img4, rasterizer=_raster("nccl", band=band))
