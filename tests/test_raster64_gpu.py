"""The fp64 per-element tier on the GPU: the blend kernels against oracle/raster64.py's blend64 fed the kernels' own fp32 records,
per pixel and per Gaussian component, on margin scenes built around the edges the kernels branch on.

Bound of an element: 2^-24 (kmass + ntiles mass), the derivation is blend64's docstring:
  per pair, kappa = 64 + 2 n_p + pm + sum_j alpha_j / (1 - alpha_j) (pm_j + 4): the pixel's T recurrence (forward product or
  backward division, 2 roundings per factor), the relative error of each alpha (pm = the magnitude of the terms of `power`, +4 for
  expf and the opacity product) amplified in 1 - alpha, and the n_p-term running sums; 64 covers the constant-depth steps (warp
  and chunk reductions, exp / ex2.approx, the reciprocal);  + ntiles(g) for the one float atomic per tile per component.
The backward reads T_final from the kernel's own alpha image, as the reference's does, so 1 - sum(w) is not amplified.
Every scene is passed through margin_scene (fp64) and then checked with margins on the kernel's records, so that both sides take
the same discrete decision on every pair: what remains is rounding, and nothing is allowed to flip."""
import os
import subprocess
import sys

import pytest
import torch

import raster64_case as RC
import util
from oracle import raster64 as R64
import street_gaussians_b200 as sgb
from street_gaussians_b200 import rasterizer as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPORT = {}


def run_kernels(scene, band=None, capacity=None, backward=True):
    """Forward + backward stage 1 through the library; returns the images, grad2d and the kernel's own records / lists."""
    cam = scene["cam"]
    st = util.settings_from(sgb, cam, DEV)
    dv = lambda k: scene[k].to(DEV) if scene.get(k) is not None else None
    P = scene["means3D"].shape[0]
    with torch.no_grad():
        col, rad, dep, alp, sem, fst, tens = R._forward_impl(dv("means3D"), dv("shs"), dv("colors_precomp"), dv("semantics"),
                                                            dv("opacities"), dv("scales"), dv("rotations"), dv("cov3D_precomp"), st,
                                                            band, capacity)
        S = 0 if scene.get("semantics") is None else scene["semantics"].shape[1]
        gs = scene["grad_semantic"].to(DEV) if S else torch.zeros(0, cam["image_height"], cam["image_width"], device=DEV)
        g2d = gsem = None
        if backward:
            g2d, gsem = R._backward_blend_impl(st, band, fst, tens, alp, scene["grad_color"].to(DEV), scene["grad_depth"].to(DEV),
                                               scene["grad_alpha"].to(DEV), gs)
    torch.cuda.synchronize()
    v = R.state_views(st, fst, P)
    vals_out = v["vals_out"].clone() if fst.num_instances else torch.zeros(0, dtype=torch.int32, device=DEV)
    return dict(color=col, depth=dep, alpha=alp, semantic=sem, radii=rad, grad2d=g2d, gsem=gsem, rec=v["rec"].clone(), ranges=v["ranges"].clone(),
                n_contrib=v["n_contrib"].clone(), list=vals_out, state=fst, tensors=tens, settings=st)


def check(name, scene, band=None, capacity=None, delta=R64.margins.__defaults__[0], backward=True, max_removed=0.1, kept=None):
    """margin_scene -> kernels -> margins on the kernel's records -> blend64 on those records -> per-element comparison.
    kept: a dict that receives the margin scene, for the caller's assertions on what survived."""
    P0 = scene["means3D"].shape[0]
    scene, removed, _ = R64.margin_scene(scene, delta=delta, device=DEV)
    if kept is not None:
        kept["scene"] = scene
    assert removed <= max_removed * P0, (removed, P0)
    k = run_kernels(scene, band, capacity, backward)
    cam = scene["cam"]
    W, H = cam["image_width"], cam["image_height"]
    rec = k["rec"].double()
    assert len(R64.margins(rec, k["radii"], W, H, delta / 4)) == 0, "a decision of the kernel's own records lies within the margin"
    # radii and clamp bits: the fp64 preprocess agrees exactly (margin scene)
    pre = R64.preprocess64(scene, DEV)
    assert torch.equal(pre["radii"].to(torch.int32), k["radii"]), "radii"
    vis = k["radii"] > 0
    assert torch.equal(k["rec"][vis, 11].view(torch.int32), pre["rec"][vis, 11].to(torch.int32)), "clamp bits"
    sem = scene.get("semantics")
    S = 0 if sem is None else sem.shape[1]
    up = dict(color=scene["grad_color"], depth=scene["grad_depth"], alpha=scene["grad_alpha"], semantic=scene.get("grad_semantic"))
    rows = None
    if band is not None:  # compare on the band's pixels; zero upstream elsewhere makes the full-image sums the band's partial sums
        rows = torch.zeros(H, dtype=torch.bool)
        for r in range(band.begin, band.end, band.step):
            rows[r * 16:min(H, r * 16 + 16)] = True
        up = {kk: (v * rows[None, :, None].to(v.dtype)) if v is not None else None for kk, v in up.items()}
    bl = R64.blend64(rec, k["radii"], W, H, cam["bg"], semantics=sem.to(DEV) if S else None, upstream=up if backward else None,
                     alpha_img=k["alpha"])
    worst = {}
    pxmask = torch.ones(H, W, dtype=torch.bool, device=DEV) if rows is None else rows.to(DEV)[:, None].expand(H, W)
    # A. forward, per pixel
    for key in ("color", "depth", "alpha") + (("semantic",) if S else ()):
        err = (k[key].double() - bl[key]).abs()[:, pxmask]
        bnd = R64.bound(bl["kmass_" + key])[:, pxmask] + 1e-30
        worst[key] = float((err / bnd).max())
        assert (err <= bnd).all(), (name, key, worst[key])
    # contributor count: the kernel's last contributor (its own culled list) is the Gaussian blend64 blends last
    nc = k["n_contrib"]
    tile = (torch.arange(H, device=DEV)[:, None] // 16) * ((W + 15) // 16) + torch.arange(W, device=DEV)[None, :] // 16
    pos = k["ranges"][tile, 0].long() + nc.long() - 1
    lid = torch.where(nc > 0, k["list"][pos.clamp(min=0, max=max(len(k["list"]) - 1, 0))].long() if len(k["list"]) else torch.zeros_like(pos),
                      torch.full_like(pos, -1))
    assert torch.equal(lid[pxmask], bl["last_id"][pxmask]), (name, "last contributor")
    if backward:
        # B. backward stage 1, per Gaussian and component (column 11 is padding)
        err = (k["grad2d"].double() - bl["grad2d"]).abs()[:, :11]
        bnd = R64.bound(bl["kmass_grad2d"], bl["mass_grad2d"], bl["ntiles"])[:, :11] + 1e-30
        r = err / bnd
        worst["grad2d"] = float(r.max())
        assert (err <= bnd).all(), (name, "grad2d", worst["grad2d"], torch.nonzero(err > bnd)[:8].tolist())
        if S:
            err = (k["gsem"].double() - bl["grad_semantics"]).abs()
            bnd = R64.bound(bl["kmass_grad_semantics"], bl["mass_grad_semantics"], bl["ntiles"]) + 1e-30
            worst["grad_semantics"] = float((err / bnd).max())
            assert (err <= bnd).all(), (name, "grad_semantics", worst["grad_semantics"])
    REPORT[name] = dict(removed=removed, P=P0, **{kk: round(v, 4) for kk, v in worst.items()})
    print(name, REPORT[name])
    return bl, k


# ------------------------------------------------------------------------------------------------ list depths
@pytest.mark.parametrize("K", [31, 32, 33, 64, 65, 255, 256, 257, 513])
def test_list_depth(K):
    """K faint splats stacked over tile (1, 1): every pixel of that tile blends exactly K of them (blend_bwd2 batches of 32,
    blend_bwd batches of 64, blend_fwd batches of 256)."""
    # margin_scene may drop a few of the stack; add a surplus until exactly K survive
    for extra in range(16):
        sc = RC.stack(48, 48, 24, 24, K + extra, seed=K)
        sc, _, _ = R64.margin_scene(sc, device=DEV)
        pre = R64.preprocess64(sc, DEV)
        nb = R64.blend64(pre["rec"], pre["radii"], 48, 48, pre["cam"]["bg"])["n_blend"][16:32, 16:32]
        if int(nb.min()) == int(nb.max()) == K:
            break
    bl, _ = check(f"depth{K}", sc)
    assert int(bl["n_blend"][16:32, 16:32].min()) == int(bl["n_blend"][16:32, 16:32].max()) == K
    assert not bool(bl["stopped"][16:32, 16:32].any())


def test_early_termination():
    """Tile (0, 0): 300 opaque-ish splats, every pixel stops in the middle of the first 256-record batch (the num_done == 256
    break skips the second batch) and in the middle of a 32-splat batch of the backward.  Tile (3, 0): an opaque stack covers
    only its left half, so some pixels stop and some do not."""
    a = RC.stack(64, 32, 8, 8, 300, seed=1, opac=(0.25, 0.45), sigma=10.0)
    g = torch.Generator().manual_seed(2)
    b = RC.screen_scene(64, 32, 49.0 + torch.rand(40, generator=g, dtype=torch.float64), 8.0 + torch.rand(40, generator=g, dtype=torch.float64),
                        1.2, 1.0 + 0.01 * torch.arange(40, dtype=torch.float64), 0.5 + 0.2 * torch.rand(40, generator=g, dtype=torch.float64), seed=2)
    bl, _ = check("termination", RC.cat_scenes(RC.cat_scenes(a, b), RC.filler(64, 32, 20, seed=3)))
    t0 = bl["stopped"][:16, :16]
    assert bool(t0.all()) and int(bl["n_list"][0, 0]) > 256
    nb = bl["n_blend"][:16, :16]
    assert int(nb.max()) % 32 != 0 and int(nb.max()) < 256
    t2 = bl["stopped"][:16, 48:64]
    assert bool(t2.any()) and not bool(t2.all())


def test_capped_pairs_and_background():
    """Opacity 0.999 splats: pairs past the 0.99 cap (value capped, gradient uncapped); non-zero background."""
    g = torch.Generator().manual_seed(4)
    n = 60
    r = lambda lo, hi: torch.rand(n, generator=g, dtype=torch.float64) * (hi - lo) + lo
    sc = RC.screen_scene(80, 48, r(0, 80), r(0, 48), r(4.0, 8.0), r(2, 20), torch.full((n,), 0.999, dtype=torch.float64), seed=4,
                         bg=(0.25, 0.5, 0.75))
    bl, _ = check("capped_bg", RC.cat_scenes(sc, RC.filler(80, 48, 60, seed=4, bg=(0.25, 0.5, 0.75))))
    assert int(bl["n_capped"].sum()) > 20


def test_large_distant_thin_splats_white_bg():
    """1920 x 48 strip: splats whose band-owned rectangle spans more than 64 tiles (emit_big_kernel), splats covering the whole
    image, centres left of / above the image (negative rectangle truncation), centres hundreds of pixels from the tiles they
    touch (large D, E in blend_bwd2's moment re-centring), thin splats with a conic condition number ~1e4; white background."""
    W, H = 1920, 48
    bgw = (1.0, 1.0, 1.0)
    # (sizes chosen so that 3 sqrt(lambda_max) sits well away from an integer: the radius margin is relative)
    big = RC.screen_scene(W, H, [300.0, 1200.0, 960.0], [20.0, 30.0, 24.0], [110.13, 90.17, 700.2], [5.0, 6.0, 40.0], [0.3, 0.4, 0.2], seed=5, bg=bgw)
    off = RC.screen_scene(W, H, [-40.0, 100.0, -300.0, 2400.0], [-30.0, -45.0, 20.0, 60.0], [25.1, 20.1, 140.1, 130.2],
                          [3.0, 3.5, 8.0, 9.0], [0.6, 0.5, 0.7, 0.7], seed=6, bg=bgw)
    g = torch.Generator().manual_seed(7)
    n = 40
    thin = RC.screen_scene(W, H, torch.rand(n, generator=g, dtype=torch.float64) * W, torch.rand(n, generator=g, dtype=torch.float64) * H,
                           55.0, 2.0 + torch.rand(n, generator=g, dtype=torch.float64) * 10, 0.6, thin=1e-3, seed=7, bg=bgw)
    sc = RC.cat_scenes(RC.cat_scenes(RC.cat_scenes(big, off), thin), RC.filler(W, H, 300, seed=8, bg=bgw))
    kept = {}
    bl, k = check("large_distant_thin", sc, kept=kept)
    x0, y0, x1, y1 = bl["rect"]
    assert int(((x1 - x0) * (y1 - y0)).max()) > 64
    pre = R64.preprocess64(kept["scene"], DEV)
    vis = pre["vis"]
    px, py = pre["rec"][:, 0], pre["rec"][:, 1]
    assert bool(((px < 0) & vis).any()) and bool(((py < 0) & vis).any()), "centres left of and above the image"
    assert bool(((px < -200) & vis).any()), "a centre hundreds of pixels from the tiles it touches"
    assert bool(((pre["clamped_x"] | pre["clamped_y"]) & vis).any()), "a centre past the 1.3 tan(fov) Jacobian clamp"
    gx, gy = (W + 15) // 16, (H + 15) // 16
    assert bool(((x0 == 0) & (y0 == 0) & (x1 == gx) & (y1 == gy)).any()), "a splat covering the whole image"
    rec = k["rec"].double()
    a, b_, c = rec[:, 2], rec[:, 3], rec[:, 4]
    tr, det = a + c, a * c - b_ * b_
    lmax = 0.5 * tr + torch.sqrt(torch.clamp(0.25 * tr * tr - det, min=0))
    cond = lmax / torch.clamp(det / torch.clamp(lmax, min=1e-30), min=1e-30)
    assert float(cond[k["radii"] > 0].max()) > 3e3


@pytest.mark.parametrize("W,H", [(97, 61), (13, 11), (200, 1)])
def test_image_sizes(W, H):
    """Partial tiles (odd W and H), a single-tile image, a 1-pixel-high strip."""
    check(f"size{W}x{H}", RC.filler(W, H, max(40, W * H // 60), seed=W + H, sh_degree=1))


@pytest.mark.parametrize("S", [1, 4, 5, 8, 9, 16, 17, 32])
def test_feature_channels_backward(S):
    """blend_bwd<SCH>: one S at each boundary of every instantiation (4, 8, 16, 32), with a 70-deep stack (two 64-batches)."""
    sc = RC.cat_scenes(RC.stack(64, 48, 40, 24, 70, seed=S, semantics=S), RC.filler(64, 48, 80, seed=S, semantics=S))
    check(f"S{S}", sc)


@pytest.mark.parametrize("S", [33, 64, 65])
def test_feature_channels_forward_chunks(S):
    """blend_fwd's semantic-only chunk passes (S > 32)."""
    check(f"S{S}_fwd", RC.filler(64, 48, 120, seed=S, semantics=S), backward=False)


def test_band_and_bounded_modes():
    """A cyclic tile-row band and the bounded (sync-free) binning, per element on the band's pixels."""
    sc = RC.cat_scenes(RC.filler(96, 80, 200, seed=11, sh_degree=2), RC.stack(96, 80, 40, 40, 40, seed=11, sh_degree=2))
    check("band", sc, band=R.TileRowBand(1, 5, 2))
    check("bounded", sc, capacity=R.InstanceCapacity(initial=200_000))


# ------------------------------------------------------------------------------------------------ C. preprocess
def preprocess_scene(D, seed, colors_precomp=False, cov3d=False, cam=None, sh_coeffs=None):
    """Splats on screen plus centres outside 1.3 tan(fov) whose splats reach into the image (the Jacobian clamp and its zero
    gradient), SH colours driven below 0 (clamp bits), anisotropic covariances from raw, non-normalised quaternions.
    cam: a 96 x 64 camera (synthetic.make_camera; its sh_degree replaces D) — the clamp cases are then placed by tx/tz against
    1.3 tan(fov / 2), wherever that falls in the image.  sh_coeffs: coefficients stored beyond the active degree's."""
    W, H = 96, 64
    g = torch.Generator().manual_seed(seed)
    n = 80
    r = lambda lo, hi, m=n: torch.rand(m, generator=g, dtype=torch.float64) * (hi - lo) + lo
    kw = dict(sh_degree=D) if cam is None else dict(cam=cam, sh_coeffs=sh_coeffs)
    a = RC.screen_scene(W, H, r(0, W), r(0, H), r(2.0, 7.0), r(3.0, 20.0), r(0.1, 0.9), seed=seed, **kw)
    # |tx/tz| between 1.45 and 1.9 tan (clamped at 1.3 tan) with splats of 25-40 px reaching in: left, right, above, below
    m = 8
    ndc = r(1.45, 1.9, m)
    sx = torch.tensor([1, -1, 0, 0, 1, -1, 1, -1], dtype=torch.float64)
    sy = torch.tensor([0, 0, 1, -1, 1, 1, -1, -1], dtype=torch.float64)
    if cam is None:
        cx = torch.where(sx != 0, ((sx * ndc + 1) * W - 1) / 2, r(10, W - 10, m))
        cy = torch.where(sy != 0, ((sy * ndc + 1) * H - 1) / 2, r(10, H - 10, m))
    else:
        u0, v0 = RC.ratio_of(cam, r(10, W - 10, m), r(10, H - 10, m))
        u = torch.where(sx != 0, sx * ndc * cam["tanfovx"], u0)
        v = torch.where(sy != 0, sy * ndc * cam["tanfovy"], v0)
        cx, cy = RC.pixel_of(cam, u, v)
    b = RC.screen_scene(W, H, cx, cy, r(25.0, 40.0, m), r(4.0, 8.0, m), r(0.3, 0.8, m), seed=seed + 1, **kw)
    c = RC.screen_scene(W, H, r(0, W, 12), r(0, H, 12), r(2.0, 5.0, 12), r(3.0, 20.0, 12), r(0.3, 0.8, 12), seed=seed + 2,
                        rgb=torch.tensor([-0.4, 0.6, -0.3], dtype=torch.float64), **kw)
    sc = RC.cat_scenes(RC.cat_scenes(a, b), c)
    if cam is not None:
        # centres past the x clamp that still lie inside the image, where the camera puts 1.3 tan(fov / 2) inside it
        limx = 1.3 * cam["tanfovx"]
        u_edge = float(RC.ratio_of(cam, W - 4.0, H / 2)[0])
        if u_edge > 1.1 * limx:
            k = 10
            vv = RC.ratio_of(cam, r(0, W, k), r(8, H - 8, k))[1]
            uu = limx * 1.02 + r(0, 1, k) * (u_edge - limx * 1.05)
            ix, iy = RC.pixel_of(cam, uu, vv)
            d = RC.screen_scene(W, H, ix, iy, r(3.0, 8.0, k), r(3.0, 20.0, k), r(0.3, 0.8, k), seed=seed + 3, **kw)
            sc = RC.cat_scenes(sc, d)
    P = sc["means3D"].shape[0]
    q = torch.randn(P, 4, generator=g)
    sc["rotations"] = (q / q.norm(dim=1, keepdim=True) * (0.8 + 0.4 * torch.rand(P, 1, generator=g))).float()
    sc["scales"] = (sc["scales"] * (0.5 + torch.rand(P, 3, generator=g))).float()
    if colors_precomp:
        sc["colors_precomp"] = torch.rand(P, 3, generator=g).float()
        sc.pop("shs")
    if cov3d:
        s_ = sc["scales"].double(); qq = sc["rotations"].double()
        rr, x, y, z = qq.unbind(1)
        Rm = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + rr * z), 2 * (x * z - rr * y)], -1),
                          torch.stack([2 * (x * y - rr * z), 1 - 2 * (x * x + z * z), 2 * (y * z + rr * x)], -1),
                          torch.stack([2 * (x * z + rr * y), 2 * (y * z - rr * x), 1 - 2 * (x * x + y * y)], -1)], -2)
        Mm = s_[:, :, None] * Rm
        Sg = Mm.transpose(1, 2) @ Mm
        sc["cov3D_precomp"] = torch.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]], 1).float()
        sc.pop("scales"); sc.pop("rotations")
    return sc


def check_preprocess(name, scene):
    """Preprocess forward per Gaussian against preprocess64 (pixel position, conic, RGB, depth within a derived bound; radius and
    clamp bits exact), and _backward_geom_impl fed the kernel's own grad2d against chain64 applied to that same grad2d.
    Bounds (2^-24 units, 64 = the fp32 steps of each quantity, rounded up):
      px, py   64 (1 + |p| + W/2 ndc_mass): ndc_mass = sum |proj_i m_i| / |w| + |ndc| is what the projection sums;
      depth    64 sum |view_i m_i|;
      conic    64 x 2 cov_mass / lambda_min^2: the 2D covariance carries 64 roundings of its largest summed magnitude, and
               d(C^-1) = -C^-1 dC C^-1 amplifies that by at most 1 / lambda_min^2;
      rgb      64 (sum of |SH terms| + 0.5);
      gradients chain_bound (oracle/raster64.py)."""
    P0 = scene["means3D"].shape[0]
    scene, removed, _ = R64.margin_scene(scene, device=DEV)
    assert removed <= 0.1 * P0, (removed, P0)
    k = run_kernels(scene)
    pre = R64.preprocess64(scene, DEV, requires_grad=True)
    cam = pre["cam"]
    vis = pre["vis"]
    assert torch.equal(pre["radii"].to(torch.int32), k["radii"]), "radii"
    rec, ref = k["rec"].double(), pre["rec"]
    assert torch.equal(k["rec"][vis, 11].view(torch.int32), ref[vis, 11].to(torch.int32)), "clamp bits"
    e = R64.EPS32 * 64.0
    bounds = {
        "px": e * (1 + ref[:, 0].abs() + 0.5 * cam["W"] * pre["ndc_mass"][:, 0]),
        "py": e * (1 + ref[:, 1].abs() + 0.5 * cam["H"] * pre["ndc_mass"][:, 1]),
        "depth": e * pre["depth_mass"],
        "conic": e * 2 * pre["cov_mass"] / pre["lmin"] ** 2,
        "rgb": e * pre["sh_mass"].amax(1),
    }
    cols = {"px": [0], "py": [1], "depth": [7], "conic": [2, 3, 4], "rgb": [8, 9, 10]}
    worst = {}
    for key, cs in cols.items():
        err = (rec[vis][:, cs] - ref[vis][:, cs]).abs()
        bnd = bounds[key][vis][:, None] + 1e-300
        worst[key] = float((err / bnd).max())
        assert (err <= bnd).all(), (name, key, worst[key])
    # backward stage 2 on the kernel's own grad2d
    g2d = k["grad2d"]
    out = R._backward_geom_impl(k["settings"], None, k["state"], k["tensors"], k["radii"], g2d)
    kg = dict(zip(["g_means3D", "g_means2D", "g_shs", "g_colors_precomp", "g_opacities", "g_scales", "g_rotations", "g_cov3D_precomp"], out))
    torch.cuda.synchronize()
    ch = R64.chain64(pre, g2d.double())
    assert torch.equal(kg["g_means2D"][vis], g2d[vis, 0:3]), "means2D is grad2d[0..2]"
    n = 0
    for key in ("g_means3D", "g_shs", "g_colors_precomp", "g_opacities", "g_scales", "g_rotations", "g_cov3D_precomp"):
        if kg[key] is None:
            continue
        assert key in ch, key
        err = (kg[key].double().reshape(ch[key].shape) - ch[key]).abs()
        bnd = R64.chain_bound(ch, key) + 1e-300
        worst[key] = float((err / bnd).max())
        assert (err <= bnd).all(), (name, key, worst[key], torch.nonzero(err > bnd)[:6].tolist())
        n += 1
    assert n >= 3
    REPORT[name] = dict(removed=removed, P=P0, **{kk: round(v, 4) for kk, v in worst.items()})
    print(name, REPORT[name])
    return pre, k


PRE_CASES = [("sh0_M1", dict(D=0)), ("sh1_M4", dict(D=1)), ("sh2_M9", dict(D=2)), ("sh3_M16", dict(D=3)),
             ("colors_precomp", dict(D=0, colors_precomp=True)), ("cov3D_precomp", dict(D=3, cov3d=True))]


@pytest.mark.parametrize("name,kw", PRE_CASES, ids=[c[0] for c in PRE_CASES])
def test_preprocess_per_element(name, kw):
    """Preprocess forward and backward per element: SH with M = 1, 4, 9, 16 (the TMA and staged preprocess_bwd paths),
    colors_precomp, cov3D_precomp.  Every scene holds Jacobian-clamped Gaussians; the SH ones hold colours clamped at 0."""
    pre, k = check_preprocess(name, preprocess_scene(seed=len(name), **kw))
    vis = pre["vis"]
    assert bool(((pre["clamped_x"] | pre["clamped_y"]) & vis).sum() >= 3), "Jacobian-clamped Gaussians"
    if not kw.get("colors_precomp"):
        assert int(k["tensors"]["sh"].shape[1]) == (kw["D"] + 1) ** 2
        assert bool(((k["rec"][:, 11].view(torch.int32) != 0) & vis).any()), "SH colours clamped at 0"


# ------------------------------------------------------------------------------------------------ D. end to end
def test_end_to_end_autograd():
    """GaussianRasterizer + autograd against render64 (the kernel's alpha image feeds T_final on both sides), per row:
    error <= chain_bound + t_rec max|row of render64|, images error <= 2^-24 kmass + t_rec mass.  t_rec covers the blend being fed
    fp32 records rather than fp64 ones: the records differ by the bounds of check_preprocess, which move a pair's power by at most
    64 2^-24 (1 + cond) (1 + max(W, H)) relative to the terms it sums.  Catches plumbing errors: argument order, the means2D leaf,
    semantics, bands of the result tuple."""
    check_end_to_end("end_to_end", RC.cat_scenes(preprocess_scene(D=3, seed=31), preprocess_scene(D=3, seed=32)))


def check_end_to_end(name, sc):
    """test_end_to_end_autograd on the 96 x 64 scene `sc` (4 semantic channels and a background are added)."""
    gen = torch.Generator().manual_seed(33)
    sc["semantics"] = torch.rand(sc["means3D"].shape[0], 4, generator=gen)
    sc["grad_semantic"] = torch.randn(4, 64, 96, generator=gen) / (64 * 96)
    sc["cam"] = dict(sc["cam"], bg=torch.tensor([0.1, 0.2, 0.3]))
    sc, removed, _ = R64.margin_scene(sc, device=DEV)
    mine = util.run_api(sgb, sc)
    r = R64.render64(sc, DEV, alpha_img=torch.from_numpy(mine["alpha"]))
    assert (r["radii"].cpu().numpy() == mine["radii"]).all()
    cond = float(r["pre"]["cond"][r["pre"]["vis"]].max())
    t_rec = R64.EPS32 * 64.0 * (1 + cond) * (1 + 96)
    worst = {}
    bl = r["blend"]
    for key in ("color", "depth", "alpha", "semantic"):
        err = (torch.from_numpy(mine[key]).to(DEV).double() - r[key]).abs()
        bnd = R64.bound(bl["kmass_" + key]) + t_rec * bl["mass_" + key] + 1e-300
        worst[key] = float((err / bnd).max())
        assert (err <= bnd).all(), (key, worst[key])
    for key in ("g_means3D", "g_means2D", "g_shs", "g_opacities", "g_scales", "g_rotations", "g_semantics"):
        ref = r[key]
        got = torch.from_numpy(mine[key]).to(DEV).double().reshape(ref.shape)
        if key == "g_means2D":
            got, ref = got[:, :2], ref[:, :2]
            bnd0 = (R64.EPS32 * r["kmass_g_means2D"])[:, :2]
        else:
            bnd0 = R64.chain_bound(r, key)
        rowmax = ref.abs().reshape(ref.shape[0], -1).amax(1).reshape((-1,) + (1,) * (ref.dim() - 1))
        bnd = bnd0 + t_rec * rowmax + 1e-300
        err = (got - ref).abs()
        worst[key] = float((err / bnd).max())
        assert (err <= bnd).all(), (key, worst[key])
    REPORT[name] = dict(removed=removed, t_rec=t_rec, **{kk: round(v, 4) for kk, v in worst.items()})
    print(name, REPORT[name])


VARIANT_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import test_raster64_gpu as T
{calls}
print("OK")
"""


@pytest.mark.parametrize("var", ["SGR_NO_TMA", "SGR_BWD2_EXPF"])
def test_kernel_variants_read_once_per_process(var):
    """SGR_NO_TMA=1 (staged instead of TMA row loads in preprocess_bwd at M = 16) and SGR_BWD2_EXPF=1 (expf instead of ex2.approx
    in blend_bwd2) are read once per process: run the per-element check each one changes in a fresh interpreter."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, **{var: "1"})
    calls = {"SGR_NO_TMA": 'T.test_preprocess_per_element("sh3_M16", dict(D=3))',  # the staged M = 16 preprocess_bwd path
             "SGR_BWD2_EXPF": "T.test_list_depth(65)"}[var]  # blend_bwd2 with expf
    code = VARIANT_SCRIPT.format(root=os.path.dirname(here), tests=here, calls=calls)
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
