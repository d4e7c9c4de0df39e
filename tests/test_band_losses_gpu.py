"""The losses on a tile-row band (band_losses.py) against the single-GPU calls, with N ranks emulated on one GPU: every rank's stages run
on its banded inputs, the halo moves through the library's pack / unpack, and the test sums the partial buffers as the all-reduce does.

Per case: each rank's gradient rows equal the single-GPU gradient bit for bit and its other rows are zero; n, k and the LiDAR selection
are exact.  Values: the photometric and LiDAR partial sums are the single-GPU block sums regrouped in fp64, so the fp32 value is within
one ulp of the single-GPU one; the sky and object-accumulation kernels sum fp32 per thread in another grouping, whose error bound for
these positive terms is below VALUE_RTOL_ACC of the value (at most 10 terms per thread at 1280 x 1920: 10 * 2^-24 < 1e-6)."""
import numpy as np
import pytest
import torch

from street_gaussians_b200 import _capi, band_losses, losses
from street_gaussians_b200._capi import ptr
from street_gaussians_b200.rasterizer import TileRowBand
from street_gaussians_b200.sharded import band_of_rows, contiguous_band, cyclic_band

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
VALUE_RTOL_ACC = 4e-6
CASES = [(world, layout, H) for world in (1, 2, 3, 5, 8) for layout in ("cyclic", "contiguous") for H in (375, 1280)] + \
        [(8, "cyclic", 80), (8, "contiguous", 40)]  # more ranks than tile rows: empty bands
W_OF = {375: 200, 1280: 1920, 80: 64, 40: 48}


def _bands(H, world, layout):
    mk = cyclic_band if layout == "cyclic" else contiguous_band
    return [mk(H, r, world) for r in range(world)]


def _rows(H, r, world, layout):
    return band_of_rows(H, r, world, layout).to(DEV)


def _banded(x, rows):
    return torch.where(rows.view(1, -1, 1), x, torch.zeros_like(x))


def _bits_equal(a, b):
    """Equal bit for bit (NaN included)."""
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _ulp_close(a, b):
    a, b = float(a), float(b)
    if np.isnan(a) or np.isnan(b):
        return np.isnan(a) and np.isnan(b)
    return abs(a - b) <= float(np.spacing(np.float32(max(abs(a), abs(b)))))


def _single_image(img, gt, m, w_l1, w_ssim):
    Cn, H, W = img.shape
    grad = torch.empty_like(img)
    scalars = torch.empty(4, device=DEV)
    nb = int(_capi.lib().sgr_image_loss_scratch_bytes(Cn, H, W))
    scratch = torch.empty(nb, device=DEV, dtype=torch.uint8)
    _capi.call("sgr_image_loss", DEV, Cn, H, W, ptr(img), ptr(gt), ptr(m), w_l1, w_ssim, ptr(grad), ptr(scalars), ptr(scratch), nb)
    return grad, scalars


def _emulated_image(img, gt, m, w_l1, w_ssim, H, world, layout, halo=True):
    bands = _bands(H, world, layout)
    xs = [_banded(img, _rows(H, r, world, layout)) for r in range(world)]
    filled = [x.clone() for x in xs]
    if halo:
        for r in range(world):
            up, down = band_losses.halo_peers(r, world)
            b = bands[r]
            for side, src, src_side in ((band_losses.RECV_UP, up, band_losses.SEND_DOWN), (band_losses.RECV_DOWN, down, band_losses.SEND_UP)):
                buf = band_losses.halo_pack(xs[src], bands[src], src_side)
                if buf.numel():
                    band_losses.halo_unpack(filled[r], b, side, buf)
    stats = [band_losses.image_loss_stats(filled[r], gt, m, bands[r]) for r in range(world)]
    total = sum(p for p, _ in stats)
    outs = [band_losses.image_loss_grad(filled[r], gt, m, bands[r], w_l1, w_ssim, total.clone(), stats[r][1]) for r in range(world)]
    return outs, filled


def _inputs(H, W, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    img = torch.rand(3, H, W, device=DEV, generator=g)
    gt = torch.rand(3, H, W, device=DEV, generator=g)
    m = (torch.rand(H * W, device=DEV, generator=g) > 0.2).to(torch.uint8)
    return img, gt, m


@pytest.mark.parametrize("world,layout,H", CASES)
def test_photometric_band_bit_equal(world, layout, H):
    W = W_OF[H]
    img, gt, m = _inputs(H, W, 11 + world)
    w_l1, w_ssim = 0.8, -0.2
    ref_g, ref_s = _single_image(img, gt, m, w_l1, w_ssim)
    outs, filled = _emulated_image(img, gt, m, w_l1, w_ssim, H, world, layout)
    covered = torch.zeros(H, dtype=torch.bool, device=DEV)
    for r, (g, s) in enumerate(outs):
        rows = _rows(H, r, world, layout)
        covered |= rows
        assert _bits_equal(g[:, rows], ref_g[:, rows]), f"rank {r}: gradient rows differ"
        assert float(g[:, ~rows].abs().max()) == 0.0 if (~rows).any() else True
        assert float(s[3]) == float(ref_s[3])  # the mask count is exact
        for i in range(3):
            assert _ulp_close(s[i], ref_s[i]), (r, i, float(s[i]), float(ref_s[i]))
    assert bool(covered.all())


@pytest.mark.parametrize("world,layout", [(2, "cyclic"), (3, "contiguous"), (5, "cyclic")])
def test_photometric_band_needs_the_halo(world, layout):
    """Mutation check: without the halo rows the gradient near every band edge is wrong."""
    H, W = 375, 200
    img, gt, m = _inputs(H, W, 5)
    ref_g, _ = _single_image(img, gt, m, 0.8, -0.2)
    outs, _ = _emulated_image(img, gt, m, 0.8, -0.2, H, world, layout, halo=False)
    wrong = sum(int((g[:, _rows(H, r, world, layout)] != ref_g[:, _rows(H, r, world, layout)]).sum()) for r, (g, _) in enumerate(outs))
    assert wrong > 0


def _single_acc(entry, acc, flag, weight):
    grad = torch.empty_like(acc)
    scalars = torch.empty(2, device=DEV)
    scratch = torch.empty(64, device=DEV, dtype=torch.uint8)
    _capi.call(entry, DEV, acc.numel(), ptr(acc), ptr(flag), weight, ptr(grad), ptr(scalars), ptr(scratch))
    return grad, scalars


@pytest.mark.parametrize("world,layout,H", CASES)
@pytest.mark.parametrize("which", ["sky", "obj"])
def test_acc_losses_band_bit_equal(world, layout, H, which):
    W = W_OF[H]
    g = torch.Generator(device=DEV).manual_seed(world * 7 + H)
    acc = torch.rand(1, H, W, device=DEV, generator=g)
    acc.view(-1)[:: 97] = 0.0  # clamped: zero gradient
    acc.view(-1)[1:: 101] = 1.0
    flag = (torch.rand(H * W, device=DEV, generator=g) > 0.5).to(torch.uint8)
    entry = "sgr_sky_loss" if which == "sky" else "sgr_obj_acc_loss"
    ref_g, ref_s = _single_acc(entry, acc, flag, 0.3)
    bands = _bands(H, world, layout)
    parts = [band_losses.acc_loss_band("sgr_band_" + entry[4:], _banded(acc, _rows(H, r, world, layout)), flag, 0.3, bands[r]) for r in range(world)]
    total = sum(p for _, p in parts)
    s = band_losses.acc_loss_value(H * W, 0.3, total)
    for r, (gr, _) in enumerate(parts):
        rows = _rows(H, r, world, layout)
        assert _bits_equal(gr[:, rows], ref_g[:, rows])
        assert float(gr[:, ~rows].abs().max()) == 0.0 if (~rows).any() else True
    assert abs(float(s[0]) - float(ref_s[0])) <= VALUE_RTOL_ACC * abs(float(ref_s[0]))


def _single_lidar(depth, acc, lidar, m, keep, weight):
    N = depth.numel()
    gd, ga = torch.empty_like(depth), torch.empty_like(acc)
    scalars = torch.empty(4, device=DEV)
    nb = int(_capi.lib().sgr_lidar_depth_loss_scratch_bytes(N))
    scratch = torch.empty(nb, device=DEV, dtype=torch.uint8)
    _capi.call("sgr_lidar_depth_loss", DEV, N, ptr(depth), ptr(acc), ptr(lidar), ptr(m), keep, weight, ptr(gd), ptr(ga), ptr(scalars), ptr(scratch), nb)
    return gd, ga, scalars


def _emulated_lidar(depth, acc, lidar, m, keep, weight, H, world, layout, sum_ties=True):
    W = depth.shape[-1]
    bands = _bands(H, world, layout)
    rows = [_rows(H, r, world, layout) for r in range(world)]
    d = [_banded(depth, rows[r]) for r in range(world)]
    a = [_banded(acc, rows[r]) for r in range(world)]
    st = [band_losses.lidar_keys(d[r], a[r], lidar, m, bands[r]) for r in range(world)]

    def reduce(views):
        tot = sum(v.long() for v in views)
        for v in views:
            v.copy_(tot.to(torch.int32))

    for level in (1, 2):
        reduce([band_losses.lidar_level_words(s, level - 1) for s, _ in st])
        for r in range(world):
            band_losses.lidar_select(level, keep, H, W, bands[r], st[r][0], st[r][1])
    reduce([band_losses.lidar_level_words(s, 2) for s, _ in st])
    sums = [band_losses.lidar_select(3, keep, H, W, bands[r], st[r][0], st[r][1]) for r in range(world)]
    total = sum(sums)
    if not sum_ties:  # mutation: each rank's own tie counts instead of the summed ones (the value's sum stays summed)
        for r in range(world):
            sums[r][0] = total[0]
    outs = []
    for r in range(world):
        outs.append(band_losses.lidar_grad(d[r], a[r], lidar, weight, bands[r], st[r][0], total.clone() if sum_ties else sums[r], st[r][1]))
    return outs


def _lidar_inputs(H, W, seed, kind):
    g = torch.Generator(device=DEV).manual_seed(seed)
    lidar = torch.rand(1, H, W, device=DEV, generator=g) * 50
    lidar[torch.rand(1, H, W, device=DEV, generator=g) < 0.3] = 0.0  # invalid
    acc = torch.rand(1, H, W, device=DEV, generator=g) * 0.5 + 0.5
    depth = (lidar + torch.randn(1, H, W, device=DEV, generator=g)) * acc
    m = (torch.rand(H * W, device=DEV, generator=g) > 0.1).to(torch.uint8)
    if kind == "ties":  # errors in a few integer values: the k-th one is tied across many tile rows and ranks
        acc = torch.ones_like(acc)
        depth = lidar + torch.randint(1, 6, lidar.shape, device=DEV, generator=g).float()
    elif kind == "nan":
        depth.view(-1)[:: 13] = float("nan")
    elif kind == "k0":
        lidar = torch.zeros_like(lidar)
        lidar.view(-1)[H * W // 2] = 3.0
        m = None
    elif kind == "all_masked":
        m = torch.zeros(H * W, device=DEV, dtype=torch.uint8)
    return depth, acc, lidar, m


LIDAR_CASES = [c + (kind,) for c in CASES for kind in ("plain", "ties", "nan", "k0", "all_masked")
               if kind in ("plain", "ties") or c[2] != 1280]  # the edge inputs at the small sizes


@pytest.mark.parametrize("world,layout,H,kind", LIDAR_CASES)
def test_lidar_band_selection_exact(world, layout, H, kind):
    W = W_OF[H]
    depth, acc, lidar, m = _lidar_inputs(H, W, 3 + world, kind)
    keep, weight = 0.95, 0.7
    rd, ra, rs = _single_lidar(depth, acc, lidar, m, keep, weight)
    outs = _emulated_lidar(depth, acc, lidar, m, keep, weight, H, world, layout)
    for r, (gd, ga, s) in enumerate(outs):
        rows = _rows(H, r, world, layout)
        assert _bits_equal(gd[:, rows], rd[:, rows]) and _bits_equal(ga[:, rows], ra[:, rows]), f"rank {r}"
        if (~rows).any():
            assert not bool(gd[:, ~rows].any()) and not bool(ga[:, ~rows].any())
        assert float(s[2]) == float(rs[2]) and float(s[3]) == float(rs[3]), "n / k"
        assert _ulp_close(s[0], rs[0]) and _ulp_close(s[1], rs[1])
    sel_ref = rd != 0
    sel = sum((gd != 0).long() for gd, _, _ in outs) > 0
    assert torch.equal(sel, sel_ref)
    if kind in ("k0", "all_masked"):
        assert float(rs[3]) == 0 and np.isnan(float(rs[0]))


@pytest.mark.parametrize("world,layout", [(2, "cyclic"), (3, "contiguous"), (5, "cyclic")])
def test_lidar_band_needs_the_summed_tie_prefix(world, layout):
    """Mutation check: with each rank's own tie counts in place of the summed ones, the tied pixels taken are not the single-GPU ones."""
    H, W = 375, 200
    depth, acc, lidar, m = _lidar_inputs(H, W, 1, "ties")
    rd, _, _ = _single_lidar(depth, acc, lidar, m, 0.95, 1.0)
    outs = _emulated_lidar(depth, acc, lidar, m, 0.95, 1.0, H, world, layout, sum_ties=False)
    sel = sum((gd != 0).long() for gd, _, _ in outs) > 0
    assert not torch.equal(sel, rd != 0)


def test_autograd_entries_one_rank():
    """The autograd entries with the whole-image band and no process group: the single-GPU values and gradients, bit for bit."""
    H, W = 375, 200
    band = TileRowBand(0, (H + 15) // 16, 1)
    img, gt, m = _inputs(H, W, 2)
    mask = m.view(1, H, W).bool()
    acc = torch.rand(1, H, W, device=DEV)
    sky = torch.rand(1, H, W, device=DEV) > 0.5
    x1, x2 = img.clone().requires_grad_(True), img.clone().requires_grad_(True)
    a1, a2 = acc.clone().requires_grad_(True), acc.clone().requires_grad_(True)
    ref = losses.photometric_loss(x1, gt, mask) + losses.sky_loss(a1, sky, 0.5)
    out = losses.photometric_loss(x2, gt, mask, band=band) + losses.sky_loss(a2, sky, 0.5, band=band)
    ref.backward()
    out.backward()
    assert _ulp_close(ref, out)
    assert _bits_equal(x1.grad, x2.grad) and _bits_equal(a1.grad, a2.grad)
    fl = band_losses.frame_losses(img, gt, mask, acc=acc, sky_mask=sky, acc_obj=acc, obj_bound=sky, band=band)
    assert _ulp_close(fl["photometric"], losses.photometric_loss(img, gt, mask))
    assert _ulp_close(fl["obj_acc"], losses.obj_acc_loss(acc, sky))
    depth, acc2, lidar, lm = _lidar_inputs(H, W, 9, "ties")
    d1, d2 = depth.clone().requires_grad_(True), depth.clone().requires_grad_(True)
    l1 = losses.lidar_depth_loss(d1, acc2, lidar, lm.view(1, H, W).bool())
    l2 = losses.lidar_depth_loss(d2, acc2, lidar, lm.view(1, H, W).bool(), band=band)
    l1.backward()
    l2.backward()
    assert _ulp_close(l1, l2) and _bits_equal(d1.grad, d2.grad)
