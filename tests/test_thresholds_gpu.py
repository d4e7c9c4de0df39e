"""The rasterizer at its thresholds (tests/threshold_case.py builds the scenes): pairs placed ON the reference's per-pair tests
(alpha < 1/255, power > 0) and thin needles whose fp32 `power` is too coarse for a constant culling slack.

A pair is ambiguous when the fp32 evaluation of the reference's expressions may take either decision (oracle/raster64.py
pair_decisions: the fp64 power within EPS_POWER 2^-24 pm, alpha within EPS_ALPHA 2^-24).  Three checks:

  forward read-back   the forward's decision on each ambiguous pair is read from its alpha image: blend64 with the pair forced
                      in and forced out differ by alpha T >= 0.36 / 255 at that pixel, against a rounding bound near 1e-6, and the
                      kernel's alpha must sit next to one of the two (never near a tie);
  backward agreement  the kernel's grad2d (and dL/dsemantics) must lie within the per-element bound of blend64 given the
                      FORWARD's decisions — a backward that re-decides a pair differently drops or invents that pair's gradient and
                      moves T for every pair in front of it;
  conservative cull   every tile of the reference's rectangle holding a pixel where the pair MAY blend is emitted, and there
                      fp64 power - err >= the record's power_min (the blend loops skip pairs below it before expf); edge
                      rings make a ring's extreme pixel the only may-blend pixel of its tile, so the row spans must reach it;
  vs the reference    tests/golden/live/thresholds.npz (make_threshold_golden.py): the compiled reference's radii, images and
                      records on the near-threshold scenes; bit-equal images wherever the contributing records are bit-equal."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_raster64_gpu as T64
import threshold_case as TC
import util
from oracle import raster64 as R64
from street_gaussians_b200 import rasterizer as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPORT = {}


def ring_scenes(S=0):
    """the ring families (one splat per pixel; behind and in front of wide splats) and the centre-pixel stack"""
    out = []
    for i, kind in enumerate(("iso", "aniso", "rot")):
        out.append((f"ring_{kind}", TC.rings(seed=10 + i, kind=kind, semantics=S)[0]))
    out.append(("ring_behind", TC.stacked_rings(seed=20, front=True, semantics=S)[0]))
    out.append(("ring_front", TC.stacked_rings(seed=21, front=False, semantics=S, bg=(0.25, 0.5, 0.75))[0]))
    out.append(("centre_pixel", TC.centre_pixels(seed=22, semantics=S)))
    return out


def decisions_check(name, scene, band=None, capacity=None):
    """Forward read-back and backward agreement on one scene; returns (ambiguous, taken, skipped) counts."""
    k = T64.run_kernels(scene, band, capacity)
    cam = scene["cam"]
    W, H = cam["image_width"], cam["image_height"]
    rec, radii = k["rec"].double(), k["radii"]
    sem = scene.get("semantics")
    S = 0 if sem is None else sem.shape[1]
    up = dict(color=scene["grad_color"], depth=scene["grad_depth"], alpha=scene["grad_alpha"], semantic=scene.get("grad_semantic"))
    rows = torch.ones(H, dtype=torch.bool)
    if band is not None:
        rows = torch.zeros(H, dtype=torch.bool)
        for r in range(band.begin, band.end, band.step):
            rows[r * 16:min(H, r * 16 + 16)] = True
        up = {kk: (v * rows[None, :, None].to(v.dtype)) if v is not None else None for kk, v in up.items()}
    rows = rows.to(DEV)
    amb = R64.ambiguous_pairs(rec, radii, W, H)
    inb = rows[amb["pix"] // W]
    pix, gid = amb["pix"][inb], amb["gid"][inb]
    if len(pix):
        assert int(torch.bincount(pix).max()) == 1, (name, "more than one ambiguous pair at a pixel: the read-back is not a two-way choice")
    bg = cam["bg"]
    semd = sem.to(DEV) if S else None
    a_in = R64.blend64(rec, radii, W, H, bg, decisions=(pix, gid, torch.ones_like(pix, dtype=torch.bool)))["alpha"].reshape(-1)[pix]
    a_out = R64.blend64(rec, radii, W, H, bg, decisions=(pix, gid, torch.zeros_like(pix, dtype=torch.bool)))["alpha"].reshape(-1)[pix]
    ka = k["alpha"].double().reshape(-1)[pix]
    d_in, d_out = (ka - a_in).abs(), (ka - a_out).abs()
    sep = (a_in - a_out).abs()
    take = d_in < d_out
    worst = {}
    if len(pix):
        assert float(sep.min()) >= 3e-4, (name, "an ambiguous pair at T < 0.1", float(sep.min()))
        worst["tie"] = float((torch.minimum(d_in, d_out) / sep).max())
        assert worst["tie"] <= 0.05, (name, "the kernel's alpha is near a tie of the two decisions", worst["tie"])
    bl = R64.blend64(rec, radii, W, H, bg, semantics=semd, upstream=up, alpha_img=k["alpha"], decisions=(pix, gid, take))
    pxmask = rows[:, None].expand(H, W)
    for key in ("color", "depth", "alpha") + (("semantic",) if S else ()):
        err = (k[key].double() - bl[key]).abs()[:, pxmask]
        bnd = R64.bound(bl["kmass_" + key])[:, pxmask] + 1e-30
        worst[key] = float((err / bnd).max())
        assert (err <= bnd).all(), (name, key, worst[key])
    err = (k["grad2d"].double() - bl["grad2d"]).abs()[:, :11]
    bnd = R64.bound(bl["kmass_grad2d"], bl["mass_grad2d"], bl["ntiles"])[:, :11] + 1e-30
    worst["grad2d"] = float((err / bnd).max())
    bad = torch.nonzero((err > bnd).any(1)).reshape(-1)
    assert len(bad) == 0, (name, "grad2d disagrees with the forward's decisions", worst["grad2d"], f"{len(bad)} Gaussians", bad[:8].tolist())
    if S:
        err = (k["gsem"].double() - bl["grad_semantics"]).abs()
        bnd = R64.bound(bl["kmass_grad_semantics"], bl["mass_grad_semantics"], bl["ntiles"]) + 1e-30
        worst["grad_semantics"] = float((err / bnd).max())
        assert (err <= bnd).all(), (name, "grad_semantics", worst["grad_semantics"])
    n_take = int(take.sum())
    REPORT[name] = dict(ambiguous=len(pix), taken=n_take, skipped=len(pix) - n_take, **{kk: round(v, 4) for kk, v in worst.items()})
    print(name, REPORT[name])
    return len(pix), n_take, len(pix) - n_take


@pytest.mark.parametrize("S", [0, 1, 17])
def test_backward_takes_the_forward_decision(S):
    """S = 0 runs blend_bwd2 (ex2.approx with the expf fall-back near 1/255), S = 1 and 17 run blend_bwd<4> / blend_bwd<32>.
    The scenes straddle the threshold: >= 500 ambiguous pairs, each outcome >= 100 times."""
    tot = [0, 0, 0]
    for name, sc in ring_scenes(S):
        n = decisions_check(f"{name}_S{S}", sc)
        tot = [a + b for a, b in zip(tot, n)]
    print(f"S={S}: ambiguous {tot[0]}, taken {tot[1]}, skipped {tot[2]}")
    assert tot[0] >= 500 and tot[1] >= 100 and tot[2] >= 100, tot


def test_decisions_band_and_bounded():
    """A cyclic tile-row band and the bounded (sync-free) binning, once each."""
    sc = TC.stacked_rings(seed=30, front=True)[0]
    n1 = decisions_check("band", sc, band=R.TileRowBand(0, 10, 2))
    n2 = decisions_check("bounded", sc, capacity=R.InstanceCapacity(initial=200_000))
    assert n1[0] >= 50 and n2[0] >= 100, (n1, n2)


VARIANT_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import test_thresholds_gpu as T
T.test_backward_takes_the_forward_decision(0)
print("OK")
"""


def test_backward_expf_variant():
    """SGR_BWD2_EXPF=1 (expf everywhere in blend_bwd2) is read once per process: the S = 0 check in a fresh interpreter."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = VARIANT_SCRIPT.format(root=os.path.dirname(here), tests=here)
    p = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, SGR_BWD2_EXPF="1"), capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]


# ------------------------------------------------------------------------------------------------ culling and power_min
def emitted_keys(k, P):
    """tile * P + Gaussian of every instance the binning emitted (the kernel's ranges and list)."""
    rg = k["ranges"].long()
    lengths = (rg[:, 1] - rg[:, 0]).clamp(min=0)
    total = int(lengths.sum())
    if total == 0:
        return torch.zeros(0, dtype=torch.int64, device=DEV)
    tiles = torch.repeat_interleave(torch.arange(len(rg), device=DEV), lengths)
    first = torch.repeat_interleave(rg[:, 0], lengths)
    offs = torch.arange(total, device=DEV) - torch.repeat_interleave(torch.cumsum(lengths, 0) - lengths, lengths)
    ids = k["list"].long()[first + offs]
    return torch.sort(tiles * P + ids).values


def cull_check(name, scene, group=None):
    """Every (tile, Gaussian) of the reference's rectangle with a may-blend pixel is emitted; power_min <= fp64 power - err at
    every may-blend pixel.  group: per-Gaussian labels (e.g. kappa) for the report of what was lost."""
    k = T64.run_kernels(scene, backward=False)
    cam = scene["cam"]
    W, H = cam["image_width"], cam["image_height"]
    rec, radii = k["rec"].double(), k["radii"]
    P = rec.shape[0]
    emitted = emitted_keys(k, P)
    need = missing = pmin_bad = 0
    lost = torch.zeros(P, dtype=torch.int64, device=DEV)
    lost_pmin = torch.zeros(P, dtype=torch.int64, device=DEV)
    for ch in R64.instance_pixels(rec, radii, W, H):
        may = ch["dec"]["may"]
        req = may.any(1)
        key = ch["tile"] * P + ch["gid"]
        if len(emitted):
            pos = torch.searchsorted(emitted, key).clamp(max=len(emitted) - 1)
            got = emitted[pos] == key
        else:
            got = torch.zeros_like(req)
        miss = req & ~got
        need += int(req.sum())
        missing += int(miss.sum())
        lost.index_add_(0, ch["gid"], miss.to(torch.int64))
        lo = ch["dec"]["power"] - ch["dec"]["err"]
        pm_bad = may & (lo < rec[ch["gid"], 6][:, None])
        pmin_bad += int(pm_bad.sum())
        lost_pmin.index_add_(0, ch["gid"], pm_bad.any(1).to(torch.int64))
    info = dict(emitted=int(len(emitted)), needed=need, missing=missing, power_min_below=pmin_bad)
    if group is not None:
        g = torch.as_tensor(group, device=DEV)
        info["missing_by_group"] = {float(v): int(lost[g == v].sum()) for v in torch.unique(g)}
        info["power_min_by_group"] = {float(v): int(lost_pmin[g == v].sum()) for v in torch.unique(g)}
    REPORT[name] = info
    print(name, info)
    assert missing == 0, (name, "tiles with may-blend pixels were culled", info)
    assert pmin_bad == 0, (name, "may-blend pixels below power_min", info)
    return info


def test_needles_culling_and_power_min():
    """Needles of kappa 1e3 .. 1e6 at 0, 30, 45, 89 degrees with opacities (1 + 1e-3) / 255 .. 0.999, centred on tile corners,
    off screen and at random; kappa >= 1e4 rectangles take the warp-cooperative walk and emit_big_kernel."""
    sc, info = TC.needles(seed=40)
    k = T64.run_kernels(sc, backward=False)
    x0, y0, x1, y1 = R64.tile_rect(k["rec"][:, 0].double(), k["rec"][:, 1].double(), k["radii"], 256, 192)
    assert int(((x1 - x0) * (y1 - y0)).max()) > 64
    cull_check("needles", sc, group=info["kappa"])
    sc2, info2 = TC.needles(seed=41, W=320, H=176)
    cull_check("needles_b", sc2, group=info2["kappa"])


def test_rings_culling_and_power_min():
    """The ring pixels sit on alpha = 1/255: exactly where culling and power_min draw their line."""
    for name, sc in ring_scenes(0):
        cull_check(f"cull_{name}", sc)


def test_edge_rings_culling():
    """Rings whose extreme pixel is the first / last column or row of a tile and the tile's only may-blend pixel: the row
    spans of tile_visit.cuh must reach exactly that pixel (24 such tiles)."""
    sc, _ = TC.edge_rings(seed=60)
    info = cull_check("cull_edge_rings", sc)
    assert info["needed"] >= 40


# ------------------------------------------------------------------------------------------------ vs the compiled reference
def test_forward_vs_reference_at_thresholds():
    """tests/golden/live/thresholds.npz (make_threshold_golden.py: the compiled reference on golden_scenes()).  Radii are equal;
    every pixel whose contributing records (pairs that may blend there) are all bit-equal to the reference's has bit-equal colour
    and alpha; every other pixel differs by at most 1e-4 or by at most two threshold flips, at a pixel holding a pair that
    power_interval marks ambiguous on this library's records or on the reference's."""
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live", "thresholds.npz"))
    total = dict(pixels=0, bit_equal_pixels=0, differing=0, ambiguous_pixels=0, records_equal=0, records=0)
    for name, scene in TC.golden_scenes().items():
        k = T64.run_kernels(scene, backward=False)
        cam = scene["cam"]
        W, H = cam["image_width"], cam["image_height"]
        P = scene["means3D"].shape[0]
        radii = k["radii"].cpu().numpy()
        assert (radii == z[f"{name}/radii"]).all(), (name, "radii")
        rec = k["rec"].cpu().numpy()
        vis = radii > 0
        same = ((rec[:, 0:2].view(np.uint32) == z[f"{name}/xy"].view(np.uint32)).all(1)
                & (rec[:, 2:6].view(np.uint32) == z[f"{name}/conic_opacity"].view(np.uint32)).all(1)
                & (rec[:, 7].view(np.uint32) == z[f"{name}/depth"].view(np.uint32))
                & (rec[:, 8:11].view(np.uint32) == z[f"{name}/rgb"].view(np.uint32)).all(1))
        total["records"] += int(vis.sum())
        total["records_equal"] += int((same & vis).sum())
        ref_rec = k["rec"].double().clone()
        ref_rec[:, 0:2] = torch.from_numpy(z[f"{name}/xy"]).double().to(DEV)
        ref_rec[:, 2:6] = torch.from_numpy(z[f"{name}/conic_opacity"]).double().to(DEV)
        # per pixel: does a pair with a non-bit-equal record, or an ambiguous pair, touch it
        same_t = torch.from_numpy(same).to(DEV)
        foreign = torch.zeros(H * W, dtype=torch.bool, device=DEV)
        amb = torch.zeros(H * W, dtype=torch.bool, device=DEV)
        for r_ in (k["rec"].double(), ref_rec):
            for ch in R64.instance_pixels(r_, k["radii"], W, H):
                d = ch["dec"]
                pm = ch["pix"][d["may"]]
                foreign[pm[~same_t[ch["gid"][:, None].expand_as(d["may"])[d["may"]]]]] = True
                amb[ch["pix"][d["may"] & ~d["must"]]] = True
        mine = torch.cat([k["color"].reshape(3, -1), k["alpha"].reshape(1, -1)]).cpu().numpy()
        theirs = np.concatenate([z[f"{name}/color"].reshape(3, -1), z[f"{name}/alpha"].reshape(1, -1)])
        diff_bits = (mine.view(np.uint32) != theirs.view(np.uint32)).any(0)
        foreign, amb = foreign.cpu().numpy(), amb.cpu().numpy()
        clean = ~foreign
        assert not (diff_bits & clean).any(), (name, "pixels with bit-equal records differ", np.flatnonzero(diff_bits & clean)[:10])
        d = np.abs(mine.astype(np.float64) - theirs.astype(np.float64)).max(0)
        big = d > 1e-4
        assert (amb[big]).all(), (name, "a pixel differs by more than 1e-4 without an ambiguous pair", np.flatnonzero(big & ~amb)[:10])
        vmax = max(1.0, float(np.abs(theirs).max()))
        assert (d[big] <= 2 * util.flip_bound(vmax) * 1.05).all(), (name, float(d.max()))
        total["pixels"] += H * W
        total["bit_equal_pixels"] += int((~diff_bits).sum())
        total["differing"] += int(diff_bits.sum())
        total["ambiguous_pixels"] += int(amb.sum())
    REPORT["vs_reference"] = total
    print("vs_reference", total)
    assert total["ambiguous_pixels"] >= 100
