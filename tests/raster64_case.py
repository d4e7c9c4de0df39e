"""Screen-space scene builders for the fp64 per-element tier (tests/test_raster64_*.py): each edge the kernels branch on is
placed on purpose — list depths, early termination, capped pairs, large / distant / thin splats — instead of left to chance."""
from __future__ import annotations

import math

import torch

from oracle import raster64 as R64
from street_gaussians_b200 import synthetic


def screen_scene(W, H, px, py, sigma, z, opac, rgb=None, sh_degree=0, seed=0, thin=None, bg=(0.0, 0.0, 0.0), semantics=0, fovx=50.0):
    """Gaussians given in pixels under an identity camera: centre (px, py), isotropic screen std-dev `sigma` (before the 0.3
    dilation), view depth z, opacity.  thin: per-Gaussian ratio of the short to the long axis (with a random rotation)."""
    gen = torch.Generator().manual_seed(seed)
    cam = synthetic.make_camera(W, H, fovx, None, sh_degree, bg)
    t = lambda v: torch.as_tensor(v, dtype=torch.float64).reshape(-1)
    px, py, sigma, z, opac = t(px), t(py), t(sigma), t(z), t(opac)
    n = len(px)
    py, sigma, z, opac = py.expand(n), sigma.expand(n), z.expand(n), opac.expand(n)
    ndcx, ndcy = (2 * px + 1) / W - 1, (2 * py + 1) / H - 1
    fx = W / (2 * cam["tanfovx"])
    means = torch.stack([ndcx * cam["tanfovx"] * z, ndcy * cam["tanfovy"] * z, z], 1)
    s = sigma * z / fx
    scales = torch.stack([s, s, s], 1)
    rot = torch.zeros(n, 4, dtype=torch.float64); rot[:, 0] = 1
    if thin is not None:
        thin = t(thin).expand(n)
        scales[:, 1] = s * thin
        ang = torch.rand(n, generator=gen, dtype=torch.float64) * math.pi
        rot = torch.stack([torch.cos(ang / 2), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), torch.sin(ang / 2)], 1)
    M = (sh_degree + 1) ** 2
    shs = torch.randn(n, M, 3, generator=gen, dtype=torch.float64) * 0.15
    rgb = torch.rand(n, 3, generator=gen, dtype=torch.float64) * 0.8 + 0.1 if rgb is None else torch.as_tensor(rgb, dtype=torch.float64).expand(n, 3)
    shs[:, 0] = (rgb - 0.5) / R64.SH_C0
    sc = dict(cam=cam, means3D=means.float(), scales=scales.float(), rotations=rot.float(), opacities=opac[:, None].float(),
              shs=shs.float().contiguous())
    if semantics:
        sc["semantics"] = torch.rand(n, semantics, generator=gen).float()
    npx = W * H
    sc["grad_color"] = torch.randn(3, H, W, generator=gen) / npx
    sc["grad_depth"] = torch.randn(1, H, W, generator=gen) / npx
    sc["grad_alpha"] = torch.randn(1, H, W, generator=gen) / npx
    if semantics:
        sc["grad_semantic"] = torch.randn(semantics, H, W, generator=gen) / npx
    return sc


def cat_scenes(a, b):
    out = dict(a)
    for k in R64._SCENE_PER_GAUSSIAN:
        if a.get(k) is not None:
            out[k] = torch.cat([a[k], b[k]]).contiguous()
    return out


def filler(W, H, n, seed, **kw):
    """n random small Gaussians over the image (keeps the other tiles busy)."""
    g = torch.Generator().manual_seed(seed + 1000)
    r = lambda lo, hi: torch.rand(n, generator=g, dtype=torch.float64) * (hi - lo) + lo
    return screen_scene(W, H, r(0, W), r(0, H), r(1.5, 6.0), r(3.0, 30.0), r(0.05, 0.9), seed=seed, **kw)


def stack(W, H, cx, cy, K, seed, opac=(0.006, 0.010), sigma=40.0, z0=2.0, **kw):
    """K wide, faint Gaussians stacked over the tile around (cx, cy), in strictly increasing depth: every pixel of that tile
    blends all K of them."""
    g = torch.Generator().manual_seed(seed)
    o = torch.rand(K, generator=g, dtype=torch.float64) * (opac[1] - opac[0]) + opac[0]
    jit = lambda: (torch.rand(K, generator=g, dtype=torch.float64) - 0.5) * 2.0
    z = z0 + 0.01 * torch.arange(K, dtype=torch.float64) + 0.001 * torch.rand(K, generator=g, dtype=torch.float64)
    return screen_scene(W, H, cx + jit(), cy + jit(), sigma, z, o, seed=seed, **kw)
