"""CPU half of the near-threshold tier: the scene builders put their pairs where they claim, blend64's `decisions` argument
changes nothing when it restates fp64's own decisions, and power_interval's bound holds for fp32 evaluations of `power`."""
import numpy as np
import torch

import threshold_case as TC
from oracle import raster64 as R64

F64 = torch.float64


def _ring_rel(sc, ring_pix):
    pre = R64.preprocess64(sc)
    rec = pre["rec"]
    rel = []
    for k, pp in enumerate(ring_pix):
        if pp:
            xy = torch.tensor(pp, dtype=F64)
            p, _, _ = R64.power_interval(rec[k][None], xy[:, 0], xy[:, 1])
            rel.append(rec[k, 5] * torch.exp(p) / R64.ALPHA_MIN - 1)
    return torch.cat(rel), pre


def test_rings_are_in_the_band():
    """Every returned ring pair has o exp(power) within +-3e-6 of 1/255 (fp64), most targeted pixels survive, and both sides
    of the threshold are populated; rings of different splats never share an ambiguous pixel."""
    for kind, minimum in (("iso", 300), ("aniso", 100), ("rot", 50)):
        sc, rp = TC.rings(seed=10, kind=kind)
        rel, pre = _ring_rel(sc, rp)
        assert len(rel) >= minimum, (kind, len(rel))
        assert float(rel.abs().max()) <= TC.BAND, kind
        assert int((rel > 0).sum()) >= len(rel) // 5 and int((rel < 0).sum()) >= len(rel) // 5, kind
        amb = R64.ambiguous_pairs(pre["rec"], pre["radii"], 176, 160)
        assert len(amb["pix"]) >= minimum // 2 and int(torch.bincount(amb["pix"]).max()) == 1, kind
        assert float(sc["opacities"].max()) < 1.0
    sc, rp = TC.stacked_rings(seed=20, front=True)
    rel, pre = _ring_rel(sc, rp)
    assert float(rel.abs().max()) <= TC.BAND
    # T at each ring pair >= 0.1 behind the two wide splats
    res = R64.blend64(pre["rec"], pre["radii"], 176, 160, pre["cam"]["bg"])
    assert float(res["T_final"].min()) >= 0.1


def test_centre_pixels_have_zero_offset():
    sc = TC.centre_pixels()
    pre = R64.preprocess64(sc)
    assert torch.equal(pre["rec"][:, 0], torch.full_like(pre["rec"][:, 0], 16.0))
    assert torch.equal(pre["rec"][:, 1], torch.full_like(pre["rec"][:, 1], 15.0))
    # the fp32 projection of a centre on the optical axis is exact as well
    m = sc["means3D"]
    assert bool((m[:, :2] == 0).all())


def test_needles_reach_the_stated_kappa():
    sc, info = TC.needles()
    pre = R64.preprocess64(sc)
    r = pre["cond"] / info["kappa"]
    assert float(r.min()) > 0.99 and float(r.max()) < 1.01
    assert bool(pre["vis"].all())
    x0, y0, x1, y1 = R64.tile_rect(pre["rec"][:, 0], pre["rec"][:, 1], pre["radii"], 256, 192)
    area = (x1 - x0) * (y1 - y0)
    assert bool((area[info["kappa"] >= 1e4] > 64).all())
    assert bool(((pre["rec"][:, 0] < 0) | (pre["rec"][:, 0] > 256) | (pre["rec"][:, 1] < 0) | (pre["rec"][:, 1] > 192)).any())


def test_blend64_natural_decisions_are_identity():
    """decisions = fp64's own decisions on every ambiguous pair (and on a sample of clear ones) is bit-identical to none."""
    sc, _ = TC.stacked_rings(seed=3, front=False, semantics=2)
    pre = R64.preprocess64(sc)
    rec, radii = pre["rec"], pre["radii"]
    pix, gid, take = [], [], []
    for ch in R64.instance_pixels(rec, radii, 176, 160):
        d = ch["dec"]
        o = rec[ch["gid"], 5][:, None]
        nat = ~(d["power"] > 0) & ~(torch.clamp(o * torch.exp(torch.clamp(d["power"], max=0.0)), max=R64.ALPHA_CAP) < R64.ALPHA_MIN)
        sel = ch["inside"] & ((d["may"] & ~d["must"]) | (torch.rand(d["may"].shape, generator=torch.Generator().manual_seed(1)) < 0.05))
        n, i = torch.nonzero(sel, as_tuple=True)
        pix.append(ch["pix"][n, i]); gid.append(ch["gid"][n]); take.append(nat[n, i])
    pix, gid, take = torch.cat(pix), torch.cat(gid), torch.cat(take)
    assert int(take.sum()) > 100 and int((~take).sum()) > 100
    up = dict(color=sc["grad_color"], depth=sc["grad_depth"], alpha=sc["grad_alpha"], semantic=sc["grad_semantic"])
    a = R64.blend64(rec, radii, 176, 160, pre["cam"]["bg"], semantics=sc["semantics"], upstream=up)
    b = R64.blend64(rec, radii, 176, 160, pre["cam"]["bg"], semantics=sc["semantics"], upstream=up, decisions=(pix, gid, take))
    for key in ("color", "depth", "alpha", "semantic", "grad2d", "grad_semantics", "kmass_grad2d", "n_blend", "last_id"):
        assert torch.equal(a[key], b[key]), key
    # and a flipped decision does change the result
    c = R64.blend64(rec, radii, 176, 160, pre["cam"]["bg"], decisions=(pix[:1], gid[:1], ~take[:1]))
    assert not torch.equal(a["alpha"], c["alpha"])


def _fma(x, y, z):
    """fp32 fused multiply-add: the fp64 product of two fp32 values is exact, the sum then rounds (to fp64, then fp32)."""
    return (x.double() * y.double() + z.double()).float()


def test_power_interval_contains_fp32_power():
    """Random pairs over round, thin and diagonal conics (condition numbers up to 1e6), offsets up to the 3-sigma ellipse and
    beyond: the fp32 power, plain or contracted to FMAs in three orders, lies within power_interval's bound; the bound is used
    (largest error / bound above 1e-2)."""
    g = torch.Generator().manual_seed(0)
    n = 200_000
    kap = 10 ** (torch.rand(n, generator=g, dtype=F64) * 6)
    ang = torch.rand(n, generator=g, dtype=F64) * np.pi
    lmin = 0.3 + torch.rand(n, generator=g, dtype=F64) * 3
    lmax = lmin * kap
    c_, s_ = torch.cos(ang), torch.sin(ang)
    # covariance -> conic
    sxx, syy, sxy = c_ * c_ * lmax + s_ * s_ * lmin, s_ * s_ * lmax + c_ * c_ * lmin, c_ * s_ * (lmax - lmin)
    det = sxx * syy - sxy * sxy
    a, b, c = (syy / det).float(), (-sxy / det).float(), (sxx / det).float()
    t = (torch.rand(n, generator=g, dtype=F64) * 2 - 1) * 4
    u = (torch.rand(n, generator=g, dtype=F64) * 2 - 1) * 4
    mx = (torch.rand(n, generator=g, dtype=F64) * 2000 - 500).float()
    my = (torch.rand(n, generator=g, dtype=F64) * 2000 - 500).float()
    # pixel = centre + t sqrt(lmax) along the axis + u sqrt(lmin) across it, rounded to the pixel grid
    px = torch.round(mx.double() + t * torch.sqrt(lmax) * c_ - u * torch.sqrt(lmin) * s_)
    py = torch.round(my.double() + t * torch.sqrt(lmax) * s_ + u * torch.sqrt(lmin) * c_)
    rec = torch.zeros(n, 12, dtype=torch.float32)
    rec[:, 0], rec[:, 1], rec[:, 2], rec[:, 3], rec[:, 4] = mx, my, a, b, c
    power, err, _ = R64.power_interval(rec, px, py)
    dx, dy = mx - px.float(), my - py.float()
    half = torch.tensor(-0.5, dtype=torch.float32)
    variants = {
        "plain": half * (a * dx * dx + c * dy * dy) - b * dx * dy,
        "fma_acc": _fma(-b * dx, dy, half * _fma(c * dy, dy, (a * dx) * dx)),
        "fma_b_first": half * _fma(a * dx, dx, c * dy * dy) - (b * dx) * dy,
        "fma_all": _fma(-b, dx * dy, half * _fma(a, dx * dx, _fma(c, dy * dy, torch.zeros_like(a)))),
    }
    worst = 0.0
    for name, p32 in variants.items():
        e = (p32.double() - power).abs()
        assert bool((e <= err).all()), (name, float((e / err).max()))
        worst = max(worst, float((e / (err + 1e-300)).max()))
    assert worst > 1e-2, worst
