"""CPU-side checks of the feature maps' finishing on a tile-row band (include/sgr.h sgr_band_finish_features_*, features.finish_features(band=)):
the new entries reject bad arguments before any CUDA call, the wrapper rejects a bad band before anything is launched, band=None makes
exactly the whole-frame call it made before, and a numpy restatement of the finishing kernels' band pixel set in both layouts."""
import ctypes as C

import numpy as np
import pytest
import torch

from street_gaussians_b200 import _capi, band_losses, features
from street_gaussians_b200.rasterizer import TileRowBand
from street_gaussians_b200.sharded import band_of_rows, contiguous_band, cyclic_band

NEW = ("sgr_band_finish_features_forward", "sgr_band_finish_features_backward")
P = C.c_void_p(256)  # a non-NULL pointer that is never dereferenced: every call below fails its checks first
BAD = [(-1, 2, 1), (2, 1, 1), (0, 4, 1), (0, 2, 0)]  # 40 px: 3 tile rows


def _rejects(rc, word):
    """SGR_EINVAL with `word` in the message."""
    return rc == -1 and word in _capi.lib().sgr_last_error().decode()


def test_band_feature_symbols_exported():
    lib = C.CDLL(_capi.LIB_PATH)
    for s in NEW:
        assert s in _capi.SYMBOLS and hasattr(lib, s), s


def _fwd(L, S=5, H=40, W=8, nc=3, mode=0, band=(0, 1, 1), ptrs=(P, P, P)):
    return L.sgr_band_finish_features_forward(S, H, W, nc, mode, *band, *ptrs, None)


def _bwd(L, S=5, H=40, W=8, nc=3, mode=0, band=(0, 1, 1), ptrs=(P, P, P, P)):
    return L.sgr_band_finish_features_backward(S, H, W, nc, mode, *band, *ptrs, None)


@pytest.mark.parametrize("call", [_fwd, _bwd], ids=["forward", "backward"])
def test_entries_validate_before_cuda(call):
    """SGR_EINVAL (-1), not SGR_ECUDA: every check runs before the library touches CUDA (this machine may have no GPU)."""
    L = _capi.lib()
    for b in BAD:
        assert _rejects(call(L, band=b), "band"), b
    assert _rejects(call(L, H=0), "size")
    assert _rejects(call(L, W=0), "size")
    assert _rejects(call(L, S=0), "size")
    assert _rejects(call(L, H=1 << 16, W=1 << 15), "size")  # H W >= 2^31
    assert _rejects(call(L, nc=2), "normal_channels")
    assert _rejects(call(L, S=2, nc=3), "normal channels")
    assert _rejects(call(L, mode=2), "mode")


def test_entries_reject_null_pointers():
    L = _capi.lib()
    assert _rejects(_fwd(L, ptrs=(None, P, P)), "NULL")
    assert _rejects(_fwd(L, ptrs=(P, None, P)), "NULL")  # normals needed with 3 normal channels
    assert _rejects(_fwd(L, ptrs=(P, P, None)), "NULL")  # semantic needed with S > 3
    assert _rejects(_bwd(L, ptrs=(None, P, P, P)), "NULL")
    assert _rejects(_bwd(L, ptrs=(P, P, P, None)), "NULL")


def test_empty_band_launches_nothing():
    """An empty band passes its checks and returns before any launch: no stream, no device is touched."""
    L = _capi.lib()
    before = L.sgr_launch_count()
    assert _fwd(L, band=(2, 2, 1)) == 0
    assert _bwd(L, band=(3, 3, 4), ptrs=(P, None, None, P)) == 0
    assert L.sgr_launch_count() == before


def test_wrapper_rejects_bad_bands_before_any_launch(monkeypatch):
    calls = []
    monkeypatch.setattr(_capi, "call", lambda *a: calls.append(a))
    for b in BAD:
        with pytest.raises(ValueError, match="band"):
            features.finish_features(torch.zeros(5, 40, 8), 3, "logits", band=TileRowBand(*b))
    assert calls == []
    with pytest.raises(_capi.SgrError, match="CUDA"):  # a good band reaches the CUDA check
        features.finish_features(torch.zeros(5, 40, 8), 3, "logits", band=TileRowBand(0, 3, 2))
    assert calls == []


@pytest.mark.parametrize("nc,mode", [(3, "logits"), (0, "probabilities")])
def test_band_none_makes_the_whole_frame_call(monkeypatch, nc, mode):
    """band=None: the entry, arguments and output shapes of the whole-frame call, in both directions."""
    calls = []
    monkeypatch.setattr(_capi, "call", lambda name, dev, *a: calls.append((name, a[:5])))
    monkeypatch.setattr(features, "_cuda_f32", lambda *a, **k: None)
    x = torch.rand(5, 40, 8, requires_grad=True)
    n, s = features.finish_features(x, nc, mode)
    assert calls == [("sgr_finish_features_forward", (5, 40, 8, nc, features.MODES[mode]))]
    assert (n is None) == (nc == 0) and tuple(s.shape) == (5 - nc, 40, 8)
    s.backward(torch.ones_like(s))
    assert calls[1] == ("sgr_finish_features_backward", (5, 40, 8, nc, features.MODES[mode]))
    assert len(calls) == 2


def test_band_call_passes_the_band_and_zeroes_foreign_rows(monkeypatch):
    """band=: the band entries with (begin, end, step) after the whole-frame arguments, into zero-filled outputs and dL/drendered."""
    calls = []

    def stub(name, dev, *a):
        calls.append((name, a[:8]))
        out = a[-2] if name.endswith("forward") else a[-1]  # semantic / dL_drendered: the call writes nothing here
        assert out is not None

    monkeypatch.setattr(_capi, "call", stub)
    monkeypatch.setattr(features, "_cuda_f32", lambda *a, **k: None)
    x = torch.rand(5, 40, 8, requires_grad=True)
    n, s = features.finish_features(x, 3, "probabilities", band=TileRowBand(1, 3, 2))
    assert calls == [("sgr_band_finish_features_forward", (5, 40, 8, 3, 1, 1, 3, 2))]
    assert not n.any() and not s.any()
    (g,) = torch.autograd.grad(s.sum() + n.sum(), x)
    assert calls[1] == ("sgr_band_finish_features_backward", (5, 40, 8, 3, 1, 1, 3, 2))
    assert not g.any()


# ---- the band's pixel set ----------------------------------------------------------------------------------------------------
def finish_pixels(H: int, W: int, band) -> np.ndarray:
    """The finishing kernels' work items restated (features.cu, sgr_common.cuh band_pixel): M = band_rows * 16 W items, item t is frame
    pixel (begin + (t // (16 W)) step) 16 W + t % (16 W), and items at or past H W do nothing.  Returns the pixels, in item order."""
    b, e, s = band_losses.check_band(band, H)
    strip = 16 * W
    t = np.arange(len(range(b, e, s)) * strip, dtype=np.int64)
    p = (b + (t // strip) * s) * strip + t % strip
    return p[p < H * W]


@pytest.mark.parametrize("layout", ["cyclic", "contiguous"])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("H,W", [(375, 200), (1280, 24), (40, 48), (16, 8), (7, 12)])
def test_finish_pixel_set_restated(H, W, world, layout):
    """Each rank's items cover exactly the pixels of band_of_rows, once each, in ascending order: a partial last tile row is clipped at
    H, an empty band has no items, and the ranks' sets partition the frame."""
    mk = cyclic_band if layout == "cyclic" else contiguous_band
    seen = np.zeros(H * W, dtype=np.int64)
    for r in range(world):
        band = mk(H, r, world)
        want = np.flatnonzero(np.repeat(band_of_rows(H, r, world, layout).numpy(), W))
        assert np.array_equal(finish_pixels(H, W, band), want), r
        seen[want] += 1
    assert (seen == 1).all()
