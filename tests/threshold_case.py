"""Near-threshold scene builders for the rasterizer's decision tier (tests/test_thresholds_*.py), on top of
raster64_case.screen_scene.  Unlike margin scenes, these put pairs ON the reference's thresholds on purpose:

  rings         splats centred on pixel centres whose opacity puts o exp(power) within +-3e-6 (relative, fp64) of 1/255 on a
                ring of pixels at the same distance: the alpha < 1/255 test is left to fp32 rounding on every ring pixel;
  centre pixels splats centred exactly on a pixel (fp32 record px, py integers), where power = -0: the power > 0 test;
  needles       thin splats of conic condition number kappa = 1e3 .. 1e6 at several angles and opacities, for the tile culling
                and the power_min skip, whose fp32 `power` error grows with the magnitude of the conic's terms.
"""
from __future__ import annotations

import math

import torch

import raster64_case as RC
from oracle import raster64 as R64

F64 = torch.float64
RING_R2 = (25, 50, 65)  # squared ring radii with 12, 12 and 16 integer pixel offsets
BAND = 3e-6  # relative half-width of the band around 1/255 the rings are placed in (fp64)
ROT_DEG = 30.0  # axis angle of the 'rot' ring family


def ring_offsets(r2):
    n = int(math.isqrt(r2)) + 1
    return [(i, j) for i in range(-n, n + 1) for j in range(-n, n + 1) if i * i + j * j == r2]


def _flat_z(sc):
    """Screen-space splats without extent along the view axis (screen_scene's z scale would stretch off-centre splats
    radially through the Jacobian's third column)."""
    s = sc["scales"].clone()
    s[:, 2] = s[:, 0] * 1e-5
    sc["scales"] = s
    return sc


def _rot_z(ang):
    ang = torch.as_tensor(ang, dtype=F64)
    z = torch.zeros_like(ang)
    return torch.stack([torch.cos(ang / 2), z, z, torch.sin(ang / 2)], 1).float()


def _grid(W, H, spacing, seed):
    """integer centres on a grid of the given spacing, each shifted by up to +-2 px so that rings meet tile edges anywhere."""
    g = torch.Generator().manual_seed(seed)
    xs = torch.arange(spacing // 2 + 2, W - spacing // 2 - 1, spacing)
    ys = torch.arange(spacing // 2 + 2, H - spacing // 2 - 1, spacing)
    cx = xs[None, :].expand(len(ys), -1).reshape(-1)
    cy = ys[:, None].expand(-1, len(xs)).reshape(-1)
    n = len(cx)
    cx = cx + torch.randint(-2, 3, (n,), generator=g)
    cy = cy + torch.randint(-2, 3, (n,), generator=g)
    return cx.to(F64), cy.to(F64)


def calibrate(sc, ring_pix, seed, band=BAND):
    """Set each splat's opacity so that o exp(power) = (1/255) (1 + j), j uniform in +-band/2, at the median fp64 power of its
    ring pixels (preprocess64's records).  ring_pix: per splat a list of (x, y) pixels.  The fp32 means put the record's centre
    up to ~5e-6 px off the pixel grid, which spreads a ring's powers: returns (scene, the ring pixels whose o exp(power) lies
    within +-band of 1/255 relative, per splat)."""
    g = torch.Generator().manual_seed(seed + 77)
    pre = R64.preprocess64(sc)
    rec = pre["rec"]
    n = rec.shape[0]
    o = sc["opacities"].double().clone()
    for k in range(n):
        if not ring_pix[k]:
            continue
        xy = torch.tensor(ring_pix[k], dtype=F64)
        p, _, _ = R64.power_interval(rec[k][None], xy[:, 0], xy[:, 1])
        j = (float(torch.rand(1, generator=g, dtype=F64)) - 0.5) * band
        o[k, 0] = R64.ALPHA_MIN * math.exp(-float(p.median())) * (1 + j)
    assert float(o.max()) < 1.0
    sc["opacities"] = o.float()
    o32 = sc["opacities"].double()[:, 0]
    kept = []
    for k in range(n):
        if not ring_pix[k]:
            kept.append([])
            continue
        xy = torch.tensor(ring_pix[k], dtype=F64)
        p, _, _ = R64.power_interval(rec[k][None], xy[:, 0], xy[:, 1])
        rel = o32[k] * torch.exp(p) / R64.ALPHA_MIN - 1
        kept.append([ring_pix[k][i] for i in range(len(ring_pix[k])) if abs(float(rel[i])) <= band])
    return sc, kept


def rings(W=176, H=160, spacing=22, seed=0, kind="iso", semantics=0, bg=(0.0, 0.0, 0.0), z=5.0):
    """One family of ring splats on a grid, a single splat per pixel (rings of neighbours never share a pixel).
    kind: 'iso' (isotropic, a whole ring of 12-16 pixels at one distance), 'aniso' (axis-aligned, the 4 mirror images of one
    offset), 'rot' (rotated by ROT_DEG, the 2 point reflections).  Returns (scene, ring_pix): per splat its pixels in the band."""
    g = torch.Generator().manual_seed(seed)
    cx, cy = _grid(W, H, spacing, seed)
    n = len(cx)
    r2 = torch.tensor(RING_R2)[torch.randint(0, len(RING_R2), (n,), generator=g)]
    pw = 2.0 + 1.5 * torch.rand(n, generator=g, dtype=F64)  # -power at the ring: opacity exp(pw) / 255 in [0.03, 0.13]
    ring_pix, sig_x, sig_y = [], [], []
    for k in range(n):
        offs = ring_offsets(int(r2[k]))
        if kind == "iso":
            s2 = float(r2[k]) / (2 * float(pw[k]))  # dilated variance
            sig_x.append(s2); sig_y.append(s2)
            sel = offs
        else:
            i, j = offs[int(torch.randint(0, len(offs), (1,), generator=g))]
            i, j = abs(i) or 1, abs(j) or 1  # a genuinely 2D offset
            ratio = 1.7
            # dilated variances (vx, vy = ratio^2 vx) along the splat's axes, rotated by ROT_DEG for 'rot' as preprocess64 does
            # (Sigma = R^T diag R, R = [[c, s], [-s, c]]):  d^T Sigma^-1 d / 2 = pw at d = (i, j)
            th = math.radians(ROT_DEG) if kind == "rot" else 0.0
            u, v = math.cos(th) * i + math.sin(th) * j, -math.sin(th) * i + math.cos(th) * j  # R d
            vx = (u * u + v * v / ratio ** 2) / (2 * float(pw[k]))
            sig_x.append(vx); sig_y.append(vx * ratio ** 2)
            sel = [(i, j), (-i, -j)] if kind == "rot" else [(i, j), (-i, j), (i, -j), (-i, -j)]
        ring_pix.append([(float(cx[k]) + a, float(cy[k]) + b) for a, b in sel])
    sx = torch.sqrt(torch.tensor(sig_x, dtype=F64) - 0.3)
    sy = torch.sqrt(torch.tensor(sig_y, dtype=F64) - 0.3)
    sc = RC.screen_scene(W, H, cx, cy, sx, z + 0.01 * torch.arange(n, dtype=F64), 0.05, seed=seed, semantics=semantics, bg=bg)
    fx = W / (2 * sc["cam"]["tanfovx"])
    zz = sc["means3D"][:, 2].double()
    sc["scales"] = torch.stack([sx * zz / fx, sy * zz / fx, sx * zz / fx * 1e-5], 1).float()
    if kind == "rot":
        sc["rotations"] = _rot_z(torch.full((n,), math.radians(ROT_DEG), dtype=F64))
    return calibrate(sc, ring_pix, seed)


def stacked_rings(W=176, H=160, spacing=22, seed=0, front=True, semantics=0, bg=(0.0, 0.0, 0.0)):
    """The iso ring family behind (front=True) or in front of two wide splats of opacity 0.2-0.4 that cover the image:
    T >= 0.36 at every ring pair, and the ring's decision moves T for the pairs behind it."""
    zr = 5.0
    sc, ring_pix = rings(W, H, spacing, seed, "iso", semantics=semantics, bg=bg, z=zr)
    g = torch.Generator().manual_seed(seed + 5)
    zo = torch.tensor([2.0, 2.5] if front else [20.0, 25.0], dtype=F64)
    wide = RC.screen_scene(W, H, torch.tensor([W * 0.4, W * 0.6], dtype=F64), torch.tensor([H * 0.45, H * 0.55], dtype=F64),
                           torch.tensor([2.0 * W, 2.2 * W], dtype=F64), zo, 0.2 + 0.2 * torch.rand(2, generator=g, dtype=F64),
                           seed=seed + 5, semantics=semantics, bg=bg)
    _flat_z(wide)
    return RC.cat_scenes(sc, wide), ring_pix + [[], []]


def centre_pixels(W=33, H=31, n=4, seed=0, semantics=0):
    """n splats centred exactly on the image's centre pixel ((W - 1) / 2, (H - 1) / 2 with W, H odd: the fp32 projection of a
    centre on the optical axis is exact), at increasing depths: dx = dy = 0 and power = -0 there."""
    assert W % 2 == 1 and H % 2 == 1
    g = torch.Generator().manual_seed(seed)
    sc = RC.screen_scene(W, H, torch.full((n,), (W - 1) / 2, dtype=F64), (H - 1) / 2, 1.0 + 3.0 * torch.rand(n, generator=g, dtype=F64),
                         3.0 + torch.arange(n, dtype=F64), 0.1 + 0.3 * torch.rand(n, generator=g, dtype=F64), seed=seed, semantics=semantics)
    m = sc["means3D"].clone()
    m[:, 0] = 0.0
    m[:, 1] = 0.0
    sc["means3D"] = m
    return _flat_z(sc)


KAPPAS = (1e3, 1e4, 1e5, 1e6)
ANGLES = (0.0, 30.0, 45.0, 89.0)
OPACITIES = ((1 + 1e-3) / 255, 0.02, 0.5, 0.999)


def needles(W=256, H=192, seed=0, z=4.0):
    """One needle per (kappa, angle, opacity): dilated screen variances 0.3 kappa along the needle and 0.3 across it (conic
    condition number kappa).  Centres cycle through tile corners (between four pixels), points off screen whose needle
    reaches in, and random points; kappa >= 1e4 rectangles span more than 64 tiles (the warp-cooperative walk and
    emit_big_kernel)."""
    g = torch.Generator().manual_seed(seed)
    combos = [(k, a, o) for k in KAPPAS for a in ANGLES for o in OPACITIES]
    n = len(combos)
    kap = torch.tensor([c[0] for c in combos], dtype=F64)
    ang = torch.tensor([math.radians(c[1]) for c in combos], dtype=F64)
    op = torch.tensor([c[2] for c in combos], dtype=F64)
    cx, cy = torch.empty(n, dtype=F64), torch.empty(n, dtype=F64)
    for i in range(n):
        r = torch.rand(2, generator=g, dtype=F64)
        kind = i % 3
        if kind == 0:  # a tile corner
            cx[i] = 16 * (1 + int(r[0] * (W // 16 - 1))) - 0.5
            cy[i] = 16 * (1 + int(r[1] * (H // 16 - 1))) - 0.5
        elif kind == 1:  # off screen (left / right / above / below), 10-40 px out
            side = int(r[0] * 4)
            d = 10 + 30 * float(r[1])
            cx[i] = [-d, W + d, W * float(r[1]), W * float(r[0])][side]
            cy[i] = [H * float(r[1]), H * float(r[0]), -d, H + d][side]
        else:
            cx[i], cy[i] = r[0] * W, r[1] * H
    s_long = torch.sqrt(0.3 * (kap - 1.0))
    sc = RC.screen_scene(W, H, cx, cy, s_long, z + 0.01 * torch.arange(n, dtype=F64), op, seed=seed)
    fx = W / (2 * sc["cam"]["tanfovx"])
    zz = sc["means3D"][:, 2].double()
    s = s_long * zz / fx
    sc["scales"] = torch.stack([s, s * 1e-6, s * 1e-6], 1).float()
    sc["rotations"] = _rot_z(ang)
    return sc, dict(kappa=kap, angle=ang, opacity=op)


def golden_scenes():
    """The small near-threshold scenes whose reference output tests/golden/make_threshold_golden.py stores
    (tests/golden/live/thresholds.npz): name -> scene, regenerated from seeds on the CPU."""
    out = {}
    for i, kind in enumerate(("iso", "aniso", "rot")):
        out[f"ring_{kind}"] = rings(W=112, H=96, seed=50 + i, kind=kind)[0]
    out["ring_behind"] = stacked_rings(W=112, H=96, seed=53, front=True)[0]
    out["ring_front"] = stacked_rings(W=112, H=96, seed=54, front=False, bg=(0.25, 0.5, 0.75))[0]
    out["centre_pixel"] = centre_pixels(seed=55)
    out["needles"] = needles(W=128, H=96, seed=56)[0]
    return out


def edge_rings(W=128, H=96, seed=0):
    """Isotropic r^2 = 25 rings whose extreme pixel (+-5, 0) or (0, +-5) is the first or last pixel column / row of a tile: that
    pixel is the only one of its tile where the splat may blend, so the tile is kept only if the culled x- (or y-) extent
    reaches exactly that pixel.  Returns (scene, ring_pix)."""
    g = torch.Generator().manual_seed(seed)
    cx, cy, sel = [], [], []
    for ty in range(1, H // 16 - 1):
        for tx in range(1, W // 16 - 1):
            side = (tx + ty) % 4
            if side == 0:    # right extreme on the first column of tile tx + 1
                x, y, o = 16 * (tx + 1) - 5, 16 * ty + 7, (5, 0)
            elif side == 1:  # left extreme on the last column of tile tx - 1
                x, y, o = 16 * tx + 4, 16 * ty + 8, (-5, 0)
            elif side == 2:  # lower extreme on the first row of tile row ty + 1
                x, y, o = 16 * tx + 7, 16 * (ty + 1) - 5, (0, 5)
            else:            # upper extreme on the last row of tile row ty - 1
                x, y, o = 16 * tx + 8, 16 * ty + 4, (0, -5)
            cx.append(float(x)); cy.append(float(y)); sel.append(o)
    n = len(cx)
    pw = 2.0 + 1.5 * torch.rand(n, generator=g, dtype=F64)
    s2 = 25.0 / (2 * pw)
    sc = RC.screen_scene(W, H, torch.tensor(cx, dtype=F64), torch.tensor(cy, dtype=F64), torch.sqrt(s2 - 0.3),
                         5.0 + 0.01 * torch.arange(n, dtype=F64), 0.05, seed=seed)
    _flat_z(sc)
    ring_pix = [[(cx[k] + sel[k][0], cy[k] + sel[k][1])] for k in range(n)]
    return calibrate(sc, ring_pix, seed)
