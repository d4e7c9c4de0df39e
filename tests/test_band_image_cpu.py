"""CPU-side checks of the sky composite and the colour correction on a tile-row band (include/sgr.h, sky.py, corrections.py): the new entries
reject bad arguments before any CUDA call, a numpy restatement of the band's pixel set in both layouts, and a gloo world-2 run of the
autograd entries with the C calls stubbed, which shows each backward all-reduces its parameter partial exactly once and leaves the image
gradients band-local."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from street_gaussians_b200 import _capi, band_losses
from street_gaussians_b200.rasterizer import TileRowBand
from street_gaussians_b200.sharded import band_of_rows, contiguous_band, cyclic_band

NEW = ("sgr_band_sky_composite_forward", "sgr_band_sky_composite_backward", "sgr_band_color_correct_forward", "sgr_band_color_correct_scratch_bytes",
       "sgr_band_color_correct_backward", "sgr_band_color_correct_affine_grad")
P = C.c_void_p(256)  # a non-NULL pointer that is never dereferenced: every call below fails its checks first
BAD = [(-1, 2, 1), (2, 1, 1), (0, 4, 1), (0, 2, 0)]  # 40 px: 3 tile rows


def test_band_image_symbols_exported():
    lib = C.CDLL(_capi.LIB_PATH)
    for s in NEW:
        assert s in _capi.SYMBOLS and hasattr(lib, s), s
    assert _capi.lib().sgr_abi_version() == 7


def _sky(L, fwd, H=40, W=8, band=(0, 1, 1), R=4, mode=0, ptrs=None, jitter=(None, None)):
    p = dict(rgb=P, acc=P, mask=None, cube=P, K=P, w2c=P, g=P, out=P)
    p.update(ptrs or {})
    if fwd:
        return L.sgr_band_sky_composite_forward(H, W, *band, R, mode, 1.0, p["rgb"], p["acc"], p["mask"], p["cube"], p["K"], p["w2c"], *jitter,
                                                p["out"], None)
    return L.sgr_band_sky_composite_backward(H, W, *band, R, mode, 1.0, p["acc"], p["mask"], p["cube"], p["K"], p["w2c"], *jitter, p["g"], p["out"],
                                             p["out"], None)


def _rejects(rc, word):
    """SGR_EINVAL with `word` in the message."""
    return rc == -1 and word in _capi.lib().sgr_last_error().decode()


@pytest.mark.parametrize("fwd", [True, False], ids=["forward", "backward"])
def test_sky_entries_validate_before_cuda(fwd):
    """SGR_EINVAL (-1), not SGR_ECUDA: every check runs before the library touches CUDA (this machine may have no GPU)."""
    L = _capi.lib()
    for b in BAD:
        assert _rejects(_sky(L, fwd, band=b), "band"), b
    assert _rejects(_sky(L, fwd, H=0), "size")
    for R in (0, -3, 16385):
        assert _rejects(_sky(L, fwd, R=R), "R="), R
    assert _rejects(_sky(L, fwd, mode=2), "mode")
    assert _rejects(_sky(L, fwd, mode=_capi.SKY_MASK_GIVEN), "sky_mask")
    for k in ("acc", "cube", "K", "w2c") + (("rgb",) if fwd else ("g",)):
        assert _rejects(_sky(L, fwd, ptrs={k: None}), "NULL"), k
    assert _rejects(_sky(L, fwd, jitter=(P, None)), "jitter")


def test_color_correct_entries_validate_before_cuda():
    L = _capi.lib()
    nb = int(L.sgr_band_color_correct_scratch_bytes(40, 8))
    assert nb > 0 and L.sgr_band_color_correct_scratch_bytes(0, 8) == 0 and L.sgr_band_color_correct_scratch_bytes(1 << 16, 1 << 15) == 0
    for b in BAD:
        assert _rejects(L.sgr_band_color_correct_forward(40, 8, *b, P, P, P, None), "band"), b
        assert _rejects(L.sgr_band_color_correct_backward(40, 8, *b, P, P, P, P, P, P, nb, None), "band"), b
    assert _rejects(L.sgr_band_color_correct_forward(40, 0, 0, 1, 1, P, P, P, None), "size")
    for i in range(3):
        args = [P, P, P]
        args[i] = None
        assert _rejects(L.sgr_band_color_correct_forward(40, 8, 0, 1, 1, *args, None), "NULL"), i
    for i in (0, 1, 2, 4):  # image, affine, dL_dout, partials (dL_dimage may be NULL)
        args = [P, P, P, P, P]
        args[i] = None
        assert _rejects(L.sgr_band_color_correct_backward(40, 8, 0, 1, 1, *args, P, nb, None), "NULL"), i
    assert L.sgr_band_color_correct_backward(40, 8, 0, 1, 1, P, P, P, None, P, P, nb - 1, None) == -3  # SGR_ENOMEM
    assert L.sgr_band_color_correct_backward(40, 8, 0, 1, 1, P, P, P, None, P, None, nb, None) == -3
    assert _rejects(L.sgr_band_color_correct_affine_grad(None, P, None), "NULL")
    assert _rejects(L.sgr_band_color_correct_affine_grad(P, None, None), "NULL")


def test_wrappers_reject_bad_bands_and_cpu_tensors():
    from street_gaussians_b200 import corrections, sky
    img, acc = torch.zeros(3, 40, 8), torch.zeros(1, 40, 8)
    cube, K, w2c = torch.zeros(6, 4, 4, 3), torch.eye(3), torch.eye(4)
    for b in BAD:
        with pytest.raises(ValueError, match="band"):
            sky.sky_composite(img, acc, cube, K, w2c, band=TileRowBand(*b))
        with pytest.raises(ValueError, match="band"):
            corrections.color_correct(img, torch.zeros(3, 4), band=TileRowBand(*b))
    with pytest.raises(_capi.SgrError, match="CUDA"):
        sky.sky_composite(img, acc, cube, K, w2c, band=TileRowBand(0, 1, 2))
    with pytest.raises(_capi.SgrError, match="CUDA"):
        corrections.color_correct(img, torch.zeros(3, 4), band=TileRowBand(0, 1, 2))


# ---- the band's pixel set ----------------------------------------------------------------------------------------------------
def band_items(H: int, W: int, band, per: int = 1) -> np.ndarray:
    """The kernels' work items restated (sgr_common.cuh band_pixel): items of `per` pixels, item t of the band_rows * strip items of the
    band's tile rows in order (strip = 16 W / per) is item (begin + (t // strip) step) strip + t % strip of the frame; those past the
    image are skipped.  Returns the frame's pixel indices the items cover, in item order."""
    b, e, s = band_losses.check_band(band, H)
    n_rows = len(range(b, e, s))
    strip = 16 * W // per
    t = np.arange(n_rows * strip, dtype=np.int64)
    item = (b + (t // strip) * s) * strip + t % strip
    item = item[item < H * W // per]
    return (item[:, None] * per + np.arange(per)[None, :]).reshape(-1)


@pytest.mark.parametrize("layout", ["cyclic", "contiguous"])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("H,W", [(375, 200), (40, 48), (80, 64), (16, 8), (7, 12), (1280, 24)])
def test_band_pixel_set_restated(H, W, world, layout):
    """Each rank's items cover exactly the pixels of band_of_rows, once each, in ascending order (also in float4 items when H W % 4 == 0):
    a partial last tile row is clipped at H, an empty band has no items, and the ranks' sets partition the frame."""
    mk = cyclic_band if layout == "cyclic" else contiguous_band
    seen = np.zeros(H * W, dtype=np.int64)
    for r in range(world):
        band = mk(H, r, world)
        rows = band_of_rows(H, r, world, layout).numpy()
        want = np.flatnonzero(np.repeat(rows, W))
        for per in (1, 4) if (H * W) % 4 == 0 else (1,):
            got = band_items(H, W, band, per)
            assert np.array_equal(got, want), (r, per)
        if band.begin == band.end:
            assert want.size == 0
        seen[want] += 1
    assert (seen == 1).all()


# ---- gloo world 2, C calls stubbed -------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _floats(p, n, ctype=C.c_float):
    return np.ctypeslib.as_array((ctype * n).from_address(p.value))


def _worker(rank, world, port, layout, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from street_gaussians_b200 import corrections, sky
        H, W, R = 40, 8, 4
        band = (cyclic_band if layout == "cyclic" else contiguous_band)(H, rank, world)
        own = np.repeat(band_of_rows(H, rank, world, layout).numpy(), W)
        calls, reduces = [], []

        def stub(name, device, *args):
            """Stands in for the library on CPU memory: band rows of the outputs get recognisable values, the parameter partials
            (rank + 1) (k + 1)."""
            calls.append(name)
            if name != "sgr_band_color_correct_affine_grad":
                assert tuple(args[2:5]) == tuple(band), (name, args[2:5])
            if name == "sgr_band_sky_composite_forward":
                out = _floats(args[-1], 3 * H * W).reshape(3, -1)
                out[:, own] = 5.0
            elif name == "sgr_band_sky_composite_backward":
                gacc, gcube = args[-2], args[-1]
                _floats(gacc, H * W)[own] = -1.0
                _floats(gcube, 6 * R * R * 3)[:] += (rank + 1) * (1 + np.arange(6 * R * R * 3))
            elif name == "sgr_band_color_correct_forward":
                _floats(args[-1], 3 * H * W).reshape(3, -1)[:, own] = 7.0
            elif name == "sgr_band_color_correct_backward":
                _floats(args[8], 3 * H * W).reshape(3, -1)[:, own] = 2.0
                _floats(args[9], 12, C.c_double)[:] = (rank + 1) * (1 + np.arange(12))
            elif name == "sgr_band_color_correct_affine_grad":
                _floats(args[1], 12)[:] = _floats(args[0], 12, C.c_double)
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

        rgb = torch.rand(3, H, W, requires_grad=True)
        acc = torch.rand(1, H, W, requires_grad=True)
        cube = torch.zeros(6, R, R, 3, requires_grad=True)
        affine = torch.eye(4)[:3].clone().requires_grad_(True)
        out = sky.sky_composite(rgb, acc, cube, torch.eye(3), torch.eye(4), band=band)
        assert bool((out.detach().reshape(3, -1)[:, ~own] == 0).all()) and bool((out.detach().reshape(3, -1)[:, own] == 5).all())
        col = corrections.color_correct(out, affine, band=band)
        assert bool((col.detach().reshape(3, -1)[:, ~own] == 0).all())
        assert reduces == []  # nothing collective in the forwards
        up = torch.rand(3, H, W)
        col.backward(up)
        # one all-reduce per backward, of the parameter partial: the 12 doubles, then the dense cube gradient
        assert reduces == [("sgr_band_color_correct_backward", (12,), torch.float64),
                           ("sgr_band_sky_composite_backward", (6, R, R, 3), torch.float32)], reduces
        tot = sum(range(1, world + 1))
        assert torch.equal(affine.grad.reshape(-1), torch.tensor([tot * (k + 1) for k in range(12)], dtype=torch.float32))
        assert torch.equal(cube.grad.reshape(-1), tot * (1 + torch.arange(6 * R * R * 3, dtype=torch.float32)))
        # the image gradients stay band-local: dL/drgb = dL/dout (the colour correction's band-local dL/dimage), dL/dacc on the band's rows
        g_img = torch.zeros(3, H * W)
        g_img[:, own] = 2.0
        assert torch.equal(rgb.grad.reshape(3, -1), g_img)
        assert bool((acc.grad.reshape(-1)[own] == -1).all()) and bool((acc.grad.reshape(-1)[~own] == 0).all())
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, repr(e) + traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("layout", ["cyclic", "contiguous"])
def test_band_image_backward_reduces_once_gloo_world2(layout):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, layout, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res
