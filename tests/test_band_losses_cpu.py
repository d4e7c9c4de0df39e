"""CPU-side checks of the losses on a tile-row band (include/sgr.h, band_losses.py): a numpy restatement of the halo row sets and of the
LiDAR tie bookkeeping for both layouts, the SgrLidarState layout against the header, and bad bands rejected before any launch."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from street_gaussians_b200 import _capi, band_losses, losses
from street_gaussians_b200.rasterizer import TileRowBand
from street_gaussians_b200.sharded import band_of_rows, contiguous_band, cyclic_band

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("sgr_band_halo_rows", "sgr_band_halo_pack", "sgr_band_halo_unpack", "sgr_band_image_loss_stats", "sgr_band_image_loss_grad",
       "sgr_band_sky_loss", "sgr_band_obj_acc_loss", "sgr_band_acc_loss_value", "sgr_band_lidar_scratch_bytes", "sgr_band_lidar_keys",
       "sgr_band_lidar_select", "sgr_band_lidar_grad")
CASES = [(H, world, layout) for H in (7, 16, 40, 375, 1280) for world in (1, 2, 3, 5, 8) for layout in ("cyclic", "contiguous")]


def _band(H, rank, world, layout):
    return (cyclic_band if layout == "cyclic" else contiguous_band)(H, rank, world)


def _owner_of_rows(H, world, layout):
    owner = np.full(H, -1)
    for r in range(world):
        owner[band_of_rows(H, r, world, layout).numpy()] = r
    assert (owner >= 0).all()
    return owner


def test_band_symbols_exported():
    lib = C.CDLL(_capi.LIB_PATH)
    for s in NEW:
        assert s in _capi.SYMBOLS and hasattr(lib, s), s
    assert _capi.lib().sgr_abi_version() == 7


@pytest.mark.parametrize("H,world,layout", CASES)
def test_halo_rows_restated(H, world, layout):
    """Every rank needs exactly the foreign rows within 10 px of its own; each arrives from their owner, sent as the owner's
    SEND_DOWN / SEND_UP rows in the receiver's RECV_UP / RECV_DOWN order, with matching buffer sizes."""
    owner = _owner_of_rows(H, world, layout)
    for r in range(world):
        own = np.flatnonzero(owner == r)
        near = set()
        for y in own:
            near.update(range(max(0, y - 10), min(H, y + 11)))
        need = sorted(y for y in near if owner[y] != r)
        got = band_losses.halo_of_rows(H, r, world, layout)
        flat = sorted({int(y) for _, rows in got for y in rows})  # (a 16-row tile between two owned ones arrives in two 10-row pieces)
        assert flat == need, (r, flat, need)
        for src, rows in got:
            assert (owner[rows.numpy()] == src).all()
        band = _band(H, r, world, layout)
        up, down = band_losses.halo_peers(r, world)
        for side, peer, peer_side in ((band_losses.RECV_UP, up, band_losses.SEND_DOWN), (band_losses.RECV_DOWN, down, band_losses.SEND_UP)):
            rows = band_losses.halo_row_indices(H, band, side)
            assert band_losses.halo_rows(H, band, side) == rows.numel()  # the library's count
            sent = band_losses.halo_row_indices(H, _band(H, peer, world, layout), peer_side)
            assert torch.equal(rows, sent), (r, side)
            assert band_losses.halo_rows(H, _band(H, peer, world, layout), peer_side) == rows.numel()
        if band.begin == band.end:
            assert all(band_losses.halo_rows(H, band, s) == 0 for s in range(4))


@pytest.mark.parametrize("layout", ["cyclic", "contiguous"])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_tie_prefix_bookkeeping_restated(world, layout):
    """The ties a rank takes: those whose count of ties at a lower flat index (the summed ties of the tile rows above its own, plus its
    own earlier ones in the row) is below `take`.  Over all ranks that is the `take` ties of lowest flat index."""
    rng = np.random.default_rng(world)
    H, W = 375, 24
    keys = rng.integers(0, 6, size=(H, W))
    t = 3
    tie = keys == t
    rows = (H + 15) // 16
    per_row = np.array([tie[16 * r: 16 * r + 16].sum() for r in range(rows)])
    for take in (0, 1, int(tie.sum()) // 2, int(tie.sum())):
        chosen = np.zeros_like(tie)
        for r in range(world):
            own = band_of_rows(H, r, world, layout).numpy()
            local = np.where(own[:, None], tie, False)
            row_ties = np.array([local[16 * u: 16 * u + 16].sum() for u in range(rows)])
            summed = per_row  # the sum of every rank's row_ties
            assert np.array_equal(sum(np.array([np.where(band_of_rows(H, q, world, layout).numpy()[:, None], tie, False)[16 * u: 16 * u + 16].sum()
                                                 for u in range(rows)]) for q in range(world)), summed)
            for u in np.flatnonzero(row_ties):
                before = summed[:u].sum()
                flat = np.flatnonzero(local[16 * u: 16 * u + 16].reshape(-1))
                for j, f in enumerate(flat):
                    if before + j < take:
                        chosen[16 * u + f // W, f % W] = True
        want = np.zeros(H * W, bool)
        want[np.flatnonzero(tie.reshape(-1))[:take]] = True
        assert np.array_equal(chosen.reshape(-1), want), take


def test_lidar_state_layout_matches_header(tmp_path):
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "sgr.h"', 'int main(void) {',
            '  printf("SgrLidarState %zu\\n", sizeof(SgrLidarState));',
            '  printf("LEVEL0 %d\\n", SGR_LIDAR_LEVEL0_WORDS);', '  printf("BINS %d\\n", SGR_LIDAR_BINS);',
            '  printf("HALO %d %d %d %d\\n", SGR_HALO_SEND_UP, SGR_HALO_SEND_DOWN, SGR_HALO_RECV_UP, SGR_HALO_RECV_DOWN);']
    body += [f'  printf("SgrLidarState.{f[0]} %zu\\n", offsetof(SgrLidarState, {f[0]}));' for f in _capi.SgrLidarState._fields_]
    body += ['  return 0;', '}']
    src, exe = tmp_path / "lidar.c", tmp_path / "lidar"
    src.write_text("\n".join(body))
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(line.split(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    ct = _capi.SgrLidarState
    assert int(out["SgrLidarState"]) == C.sizeof(ct)
    for f in ct._fields_:
        assert int(out[f"SgrLidarState.{f[0]}"]) == getattr(ct, f[0]).offset, f[0]
    assert int(out["LEVEL0"]) == _capi.LIDAR_LEVEL0_WORDS and int(out["BINS"]) == _capi.LIDAR_BINS
    assert out["HALO"] == "0 1 2 3"
    # the level-0 words end where level 1's histogram begins
    assert 4 * _capi.LIDAR_LEVEL0_WORDS == ct.hist.offset + 4 * _capi.LIDAR_BINS


BAD = [TileRowBand(-1, 2, 1), TileRowBand(2, 1, 1), TileRowBand(0, 4, 1), TileRowBand(0, 2, 0)]  # 40 px: 3 tile rows


@pytest.mark.parametrize("band", BAD)
def test_wrappers_reject_bad_bands_before_touching_the_gpu(band):
    img = torch.zeros(3, 40, 8)
    acc = torch.zeros(1, 40, 8)
    with pytest.raises(ValueError, match="band"):
        band_losses.halo_pack(img, band, band_losses.SEND_UP)
    with pytest.raises(ValueError, match="band"):
        band_losses.image_loss_stats(img, img, None, band)
    with pytest.raises(ValueError, match="band"):
        band_losses.acc_loss_band("sgr_band_sky_loss", acc, acc.bool(), 1.0, band)
    with pytest.raises(ValueError, match="band"):
        band_losses.lidar_keys(acc, acc, acc, None, band)
    with pytest.raises(ValueError, match="band"):
        losses.photometric_loss(img, img, band=band)
    with pytest.raises(ValueError, match="band"):
        losses.lidar_depth_loss(acc, acc, acc, band=band)
    L = _capi.lib()
    b, e, s = band
    assert L.sgr_band_halo_rows(40, b, e, s, 0) == -1
    assert L.sgr_band_image_loss_stats(3, 40, 8, b, e, s, None, None, None, None, None, 0, None) == -1
    assert "band" in L.sgr_last_error().decode()
    assert L.sgr_band_sky_loss(40, 8, b, e, s, None, None, 1.0, None, None, None) == -1
    assert L.sgr_band_lidar_select(1, 0.95, 40, 8, b, e, s, None, None, None, 0, None) == -1


def test_cpu_tensors_and_bad_sides_fail_loudly():
    band = TileRowBand(0, 1, 2)
    with pytest.raises(_capi.SgrError, match="CUDA"):
        losses.sky_loss(torch.zeros(1, 40, 8), torch.zeros(1, 40, 8, dtype=torch.bool), band=band)
    with pytest.raises(ValueError, match="side"):
        band_losses.halo_rows(40, band, 7)
    L = _capi.lib()
    assert L.sgr_band_halo_pack(3, 40, 8, 0, 1, 2, band_losses.RECV_UP, None, None, None) == -1
    assert "side" in L.sgr_last_error().decode()
    assert L.sgr_band_lidar_select(4, 0.95, 40, 8, 0, 1, 2, C.c_void_p(16), None, C.c_void_p(16), 1 << 30, None) == -1
    assert L.sgr_band_lidar_select(1, 0.0, 40, 8, 0, 1, 2, C.c_void_p(16), None, C.c_void_p(16), 1 << 30, None) == -1
