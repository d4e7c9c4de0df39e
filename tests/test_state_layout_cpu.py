"""sgr_state_layout against the library's own sizes, and rasterizer.state_views against sgr_state_layout, without a GPU: every section
of the geom, img and binning states starts 256-B aligned, the sections follow one another in carve order with room for what the views
read, each state ends where sgr_state_sizes / sgr_binning_bytes say, the tile ids are 16 bits exactly where the binning uses them, and
each named view starts at the offset the C entry reports."""
import ctypes as C

import pytest
import torch

import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi
from street_gaussians_b200 import rasterizer as R

P_VALUES = (0, 1, 255, 257, 100_000)
R_VALUES = (0, 1, 12_345)
# (width, height, tiles, key_bytes exact, key_bytes bounded); some frames end in partial tiles
FRAMES = [(13, 9, 1, 2, 2), (2048, 2048, 16_384, 2, 2), (1805, 2320, 16_385, 2, 2), (4079, 4097, 65_535, 2, 2),
          (4096, 4096, 65_536, 2, 4), (4112, 4112, 66_049, 4, 4)]


def settings(W, H):
    return sgb.GaussianRasterizationSettings(H, W, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)


def frame(W, H, P):
    fr = _capi.SgrFrame()
    fr.P, fr.width, fr.height, fr.tan_fovx, fr.tan_fovy, fr.scale_modifier = P, W, H, 0.5, 0.5, 1.0
    return fr


def layout(W, H, P, R_, bounded):
    lay = _capi.SgrStateLayout()
    assert _capi.lib().sgr_state_layout(C.byref(frame(W, H, P)), R_, bounded, C.byref(lay)) == 0, _capi.lib().sgr_last_error()
    return lay


def section_bytes(W, H, P, R_, ntile):
    """The least size of each section: what state_views and the kernels address in it."""
    u32 = 4 * P
    geom = dict(rec=48 * P, tiles_touched=u32, depth_key=u32, iota=u32, depth_sorted=u32, perm=u32, offsets=u32, big_list=u32, status=256,
                jac=48 * P, ckey=u32, cval=u32)
    img = dict(ranges=8 * ntile, tile_max_contrib=4 * ntile, n_contrib=4 * W * H, blend_T=4 * W * H, far_ranges=8 * ntile, split=8 * ntile)
    binning = dict(keys_in=4 * R_, keys_out=4 * R_, vals_in=4 * R_, vals_out=4 * R_, sort_temp=4 * R_, bucket=0)
    return geom, img, binning


@pytest.mark.parametrize("bounded", [0, 1])
@pytest.mark.parametrize("W,H,ntile,kb_exact,kb_bounded", FRAMES)
def test_layout_matches_sizes_and_carve_order(W, H, ntile, kb_exact, kb_bounded, bounded):
    assert ((W + 15) // 16) * ((H + 15) // 16) == ntile
    L = _capi.lib()
    for P in P_VALUES:
        gb, ib = C.c_size_t(), C.c_size_t()
        assert L.sgr_state_sizes(C.byref(frame(W, H, P)), C.byref(gb), C.byref(ib)) == 0
        for R_ in R_VALUES:
            lay = layout(W, H, P, R_, bounded)
            assert lay.key_bytes == (kb_bounded if bounded else kb_exact)
            sizes = section_bytes(W, H, P, R_, ntile)
            ends = (lay.geom_bytes, lay.img_bytes, lay.binning_bytes)
            for names, need, end in zip((_capi.GEOM_SECTIONS, _capi.IMG_SECTIONS, _capi.BIN_SECTIONS), sizes, ends):
                offs = [getattr(lay, k) for k in names]
                assert offs[0] == 0 and all(o % 256 == 0 for o in offs) and end % 256 == 0, (names, offs, end)
                for k, o, nxt in zip(names, offs, offs[1:] + [end]):
                    assert nxt >= o + need[k], (P, R_, k, o, nxt)
            assert (lay.geom_bytes, lay.img_bytes) == (gb.value, ib.value)
            assert lay.binning_bytes == L.sgr_binning_bytes(R_)


@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("W,H,ntile,kb_exact,kb_bounded", FRAMES)
def test_state_views_read_at_the_reported_offsets(W, H, ntile, kb_exact, kb_bounded, bounded):
    """A marker written at each section's offset in CPU byte buffers is the first element of that section's view.  Every marker is
    new, so a stale one left in reused memory cannot pass."""
    st = settings(W, H)
    n = 0
    for P in P_VALUES:
        for R_ in R_VALUES:
            lay = layout(W, H, P, R_, int(bounded))
            fs = R._ForwardState()
            fs.geom, fs.img, fs.binning = (torch.empty(n, dtype=torch.uint8) for n in (lay.geom_bytes, lay.img_bytes, lay.binning_bytes))
            fs.num_instances, fs.bounded = R_, bounded
            marks = {}
            for buf, names in ((fs.geom, _capi.GEOM_SECTIONS), (fs.img, _capi.IMG_SECTIONS), (fs.binning, _capi.BIN_SECTIONS)):
                for k in names:
                    n += 1
                    marks[k] = n
                    buf[getattr(lay, k):getattr(lay, k) + 4] = torch.tensor([marks[k]], dtype=torch.int32).view(torch.uint8)
            v = R.state_views(st, fs, P)
            expect = dict(rec=(P, 12), status=(64,), ranges=(ntile, 2), tile_max_contrib=(ntile,), n_contrib=(H, W))
            expect.update({k: (P,) for k in _capi.GEOM_SECTIONS if k not in expect and k != "jac"})
            expect.update({k: (R_,) for k in ("keys_in", "keys_out", "vals_in", "vals_out")})
            assert {k: tuple(t.shape) for k, t in v.items()} == expect
            assert v["rec"].dtype == torch.float32 and v["keys_in"].element_size() == lay.key_bytes
            for k, t in v.items():
                if t.numel():
                    first = t.reshape(-1)[:1]
                    assert int(first.view(torch.int32) if first.dtype == torch.float32 else first) == marks[k], k


def test_layout_rejects_bad_arguments():
    L = _capi.lib()
    lay = _capi.SgrStateLayout()
    assert L.sgr_state_layout(C.byref(frame(64, 64, 10)), -1, 0, C.byref(lay)) == -1 and b"num_instances" in L.sgr_last_error()
    assert L.sgr_state_layout(C.byref(frame(0, 64, 10)), 5, 0, C.byref(lay)) == -1 and b"bad sizes" in L.sgr_last_error()
    assert L.sgr_state_layout(C.byref(frame(64, 64, 10)), 5, 0, None) == -1
