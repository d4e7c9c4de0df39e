"""CPU-side checks of the evaluation metrics (include/sgr.h "Evaluation metrics", street_gaussians_b200/metrics.py): the entries are
exported under ABI 7, bad sizes, bands, flags and NULL buffers are rejected before any CUDA call, CPU tensors raise, the float64
restatement (eval_oracle.py) gives the hand-computed values, and under gloo at world 2 with the C calls stubbed `ViewMetrics.result()`
all-reduces exactly once whatever the number of views."""
import ctypes as C
import multiprocessing as mp
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist

import eval_oracle as EO
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi, metrics
from street_gaussians_b200.rasterizer import TileRowBand
from street_gaussians_b200.sharded import cyclic_band

NEW = ("sgr_eval_metrics_scratch_bytes", "sgr_eval_metrics_accumulate", "sgr_band_eval_metrics_accumulate", "sgr_eval_metrics_finish")
P = C.c_void_p(256)  # a non-NULL address that must never be dereferenced: every call below fails validation first


def test_symbols_exported_and_abi_unchanged():
    lib = C.CDLL(_capi.LIB_PATH)
    for s in NEW:
        assert s in _capi.SYMBOLS and hasattr(lib, s), s
    assert _capi.lib().sgr_abi_version() == 7
    assert sgb.metrics is metrics and "ViewMetrics" in dir(sgb) and "psnr" in dir(metrics)


@pytest.mark.parametrize("V,Cn,H,W", [(0, 3, 40, 48), (1, 0, 40, 48), (1, 3, 0, 48), (1, 3, 40, 0), (1, 3, -4, 48), (65536, 1, 40, 48),
                                      (22000, 3, 40, 48), (1, 3, 1 << 16, 1 << 15)])
def test_bad_sizes_rejected(V, Cn, H, W):
    L = _capi.lib()
    assert L.sgr_eval_metrics_scratch_bytes(V, Cn, H, W) == 0
    assert L.sgr_eval_metrics_accumulate(V, Cn, H, W, 0, P, P, None, P, P, 1 << 40, None) == -1
    assert "bad sizes" in L.sgr_last_error().decode()


@pytest.mark.parametrize("band", [TileRowBand(-1, 2, 1), TileRowBand(2, 1, 1), TileRowBand(0, 4, 1), TileRowBand(0, 2, 0)])
def test_bad_bands_rejected(band):
    L = _capi.lib()
    b, e, s = band
    assert L.sgr_band_eval_metrics_accumulate(1, 3, 40, 48, b, e, s, 0, P, P, None, P, P, 1 << 40, None) == -1
    assert "band" in L.sgr_last_error().decode()
    with pytest.raises(ValueError, match="band"):
        metrics.accumulate(torch.zeros(1, 3, 40, 48), torch.zeros(1, 3, 40, 48), None, torch.zeros(1, 5, dtype=torch.float64), 0, band)


@pytest.mark.parametrize("flags", [16, -1, 2, 2 | 4, 32 | 1])
def test_bad_flags_rejected(flags):
    L = _capi.lib()
    assert L.sgr_eval_metrics_accumulate(1, 3, 40, 48, flags, P, P, None, P, P, 1 << 40, None) == -1
    assert "flags" in L.sgr_last_error().decode()


def test_null_buffers_rejected():
    L = _capi.lib()
    need = L.sgr_eval_metrics_scratch_bytes(1, 3, 40, 48)
    assert need > 0
    for args in ((None, P, P, P), (P, None, P, P), (P, P, None, P)):
        img, gt, sums, scratch = args
        assert L.sgr_eval_metrics_accumulate(1, 3, 40, 48, 1, img, gt, None, sums, scratch, need, None) == -1
        assert "NULL" in L.sgr_last_error().decode()
    for scratch, nbytes in ((None, need), (P, need - 1)):  # SGR_ENOMEM, like the other entries' scratch checks
        assert L.sgr_eval_metrics_accumulate(1, 3, 40, 48, 1, P, P, None, P, scratch, nbytes, None) == -3
        assert "scratch" in L.sgr_last_error().decode()
    assert L.sgr_eval_metrics_finish(0, P, P, None) == -1
    assert L.sgr_eval_metrics_finish(1, None, P, None) == -1
    assert L.sgr_eval_metrics_finish(1, P, None, None) == -1


def test_cpu_tensors_and_bad_options_raise():
    x = torch.zeros(3, 40, 48)
    with pytest.raises(_capi.SgrError, match="CUDA"):
        metrics.psnr(x, x)
    with pytest.raises(_capi.SgrError, match="CUDA"):
        metrics.ViewMetrics().add(x, x)
    with pytest.raises(ValueError, match="clamp"):
        metrics.ViewMetrics(clamp=False, quantize8=True)
    with pytest.raises(ValueError, match="mask"):
        metrics._mask_u8(torch.zeros(2, 40, 48, dtype=torch.bool), 40, 48, "cpu")
    with pytest.raises(ValueError, match="mask"):
        metrics._mask_u8(torch.zeros(40, 48), 40, 48, "cpu")
    r = metrics.ViewMetrics().result()  # no views: nothing to read
    assert r["psnr"].numel() == 0 and np.isnan(r["mean"]["psnr"])


# ---- the float64 restatement on hand-computed cases -----------------------------------------------------------------------------
def _rand(shape, seed):
    return np.random.default_rng(seed).random(shape, dtype=np.float32)


def test_oracle_identical_images():
    x = _rand((3, 40, 48), 0)
    r = EO.view_metrics(x, x.copy())
    assert r["psnr"] == np.inf and r["l1"] == 0.0 and r["n"] == 3 * 40 * 48
    assert abs(r["ssim"] - 1.0) < 1e-12  # S = 1 exactly at every pixel when x == y


def test_oracle_one_pixel_difference():
    x = np.full((3, 40, 48), 0.5, np.float32)
    y = x.copy()
    y[1, 7, 9] = 0.25
    r = EO.view_metrics(x, y, clamp=False)
    n = 3 * 40 * 48
    assert r["l1"] == pytest.approx(0.25 / n, rel=1e-15)
    assert r["psnr"] == pytest.approx(20 * np.log10(1 / np.sqrt(0.0625 / n)), rel=1e-15)
    # masked to that pixel: n = 3 elements, mse = 0.0625 / 3
    m = np.zeros((40, 48), bool)
    m[7, 9] = True
    r = EO.view_metrics(x, y, m, clamp=False)
    assert r["n"] == 3 and r["l1"] == pytest.approx(0.25 / 3, rel=1e-15)
    assert r["psnr"] == pytest.approx(20 * np.log10(1 / np.sqrt(0.0625 / 3)), rel=1e-15)
    # the SSIM map differs from 1 only within the 11x11 window of the pixel, in channel 1
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    smap = EO.ssim_map(x64, y64)
    off = np.argwhere(np.abs(smap - 1) > 1e-12)
    assert set(off[:, 0]) == {1} and off[:, 1].min() >= 2 and off[:, 1].max() <= 12 and off[:, 2].min() >= 4 and off[:, 2].max() <= 14


def test_oracle_all_false_mask():
    x, y = _rand((3, 40, 48), 1), _rand((3, 40, 48), 2)
    m = np.zeros((40, 48), bool)
    r = EO.view_metrics(x, y, m)
    assert r["n"] == 0 and np.isnan(r["psnr"]) and np.isnan(r["l1"])
    assert r["ssim"] == 1.0  # both images zeroed: S = C1 C2 / (C1 C2) everywhere
    r = EO.view_metrics(x, y, m, ssim_masked=False)
    assert r["ssim"] < 0.5  # the unmasked images of independent noise


def test_oracle_quantize8_is_the_save_image_round_trip():
    """x -> trunc(clamp(fp32(fp32(255 x) + 0.5), 0, 255)) / 255: torchvision's save_image rounding, halves up, read back / 255."""
    v = EO.quant_boundary_values()
    q = EO.prepare(v, True, True)
    t = (v * np.float32(255)).astype(np.float32) + np.float32(0.5)
    assert np.array_equal(q, (np.trunc(np.clip(t, 0, 255)).astype(np.float32) / np.float32(255)).astype(np.float32))
    # torch's own round trip of the same values, as save_image and to_tensor do it
    tt = torch.from_numpy(v).mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).float().div(255)
    assert np.array_equal(q, tt.numpy())
    # levels are kept, and the result is always one of the 256 levels, the nearest one up to fp32 ties
    lv = np.arange(256, dtype=np.float32) / np.float32(255)
    assert np.array_equal(EO.prepare(lv, True, True), lv)
    k = np.rint(q.astype(np.float64) * 255)
    assert np.array_equal((k.astype(np.float32) / np.float32(255)), q)
    assert np.all(np.abs(k - v.astype(np.float64) * 255) <= 0.5 + 1e-4)
    # the set tells the save_image rounding apart from truncation and from a 255 x formed in fp64
    trunc = (np.trunc(v * np.float32(255)) / np.float32(255)).astype(np.float32)
    f64 = (np.trunc(np.clip(v.astype(np.float64) * 255 + 0.5, 0, 255)) / 255).astype(np.float32)
    assert not np.array_equal(q, trunc) and not np.array_equal(q, f64)
    assert EO.prepare(np.float32(1.5), True, True) == 1.0 and EO.prepare(np.float32(-0.5), True, True) == 0.0


# ---- gloo world 2, C calls stubbed -------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, views, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        H, W = 40, 24
        band = cyclic_band(H, rank, world)
        calls, reduces = [], []

        def stub(name, device, *args):
            """Stands in for the library on CPU memory: view i's slot gets (rank + 1) (i + 1) in every sum; finish copies the sums."""
            calls.append(name)
            if name == "sgr_band_eval_metrics_accumulate":
                assert tuple(args[4:7]) == tuple(band), args[4:7]
                sums = np.ctypeslib.as_array((C.c_double * 5).from_address(args[11].value))
                sums += (rank + 1) * (calls.count(name))
            elif name == "sgr_eval_metrics_finish":
                V = args[0]
                s = np.ctypeslib.as_array((C.c_double * (5 * V)).from_address(args[1].value)).reshape(V, 5)
                out = np.ctypeslib.as_array((C.c_float * (4 * V + 4)).from_address(args[2].value)).reshape(V + 1, 4)
                out[:V] = s[:, :4]
                out[V] = [s[:, k].mean() for k in range(3)] + [V]
            elif name not in ("sgr_band_halo_pack", "sgr_band_halo_unpack"):
                raise AssertionError(f"unexpected call {name}")

        real_all_reduce = dist.all_reduce

        def counting_all_reduce(t, *a, **k):
            reduces.append((tuple(t.shape), t.dtype))
            return real_all_reduce(t, *a, **k)

        _capi.call = stub
        dist.all_reduce = counting_all_reduce
        metrics._check_cuda = lambda *ts: None
        vm = metrics.ViewMetrics(band=band)
        for _ in range(views):
            vm.add(torch.rand(3, H, W), torch.rand(3, H, W), torch.ones(1, H, W, dtype=torch.bool))
        assert reduces == []  # the adds exchange halos point to point only
        r = vm.result()
        assert reduces == [((views, 5), torch.float64)], reduces
        tot = sum(range(1, world + 1))
        assert torch.equal(r["psnr"], torch.tensor([tot * (i + 1) for i in range(views)], dtype=torch.float32))
        assert torch.equal(r["n"], torch.tensor([tot * (i + 1) for i in range(views)], dtype=torch.int64))
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, repr(e) + traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("views", [1, 3, 37])
def test_result_all_reduces_once_gloo_world2(views):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, views, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
