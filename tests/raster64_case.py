"""Screen-space scene builders for the fp64 per-element tier (tests/test_raster64_*.py): each edge the kernels branch on is
placed on purpose — list depths, early termination, capped pairs, large / distant / thin splats — instead of left to chance.

Every builder takes `cam=`: a camera dict of synthetic.make_camera (any pose, intrinsics, sh_degree, scale_modifier).  Without
it the scene is built under the identity camera of fovx 50 degrees, as the existing per-element cases are."""
from __future__ import annotations

import math

import torch

from oracle import raster64 as R64
from street_gaussians_b200 import synthetic

F64 = torch.float64


def _projection(cam):
    """The camera's projection matrix P (4 x 4, fp64, column-vector convention: ndc = (P c)[:3] / (P c)[3] for a view-space c)."""
    view_t = cam["viewmatrix"].to(F64)
    return (torch.linalg.inv(view_t) @ cam["projmatrix"].to(F64)).T


def pixel_of(cam, u, v):
    """Pixel position (px, py) of the view-space direction with tx/tz = u, ty/tz = v (ndc2Pix of the projection)."""
    P = _projection(cam)
    W, H = cam["image_width"], cam["image_height"]
    ndcx = P[0, 0] * u + P[0, 1] * v + P[0, 2]
    ndcy = P[1, 0] * u + P[1, 1] * v + P[1, 2]
    return ((ndcx + 1) * W - 1) / 2, ((ndcy + 1) * H - 1) / 2


def ratio_of(cam, px, py):
    """Inverse of pixel_of: (tx/tz, ty/tz) of the view-space ray through pixel (px, py)."""
    P = _projection(cam)
    W, H = cam["image_width"], cam["image_height"]
    ndcx = (2 * torch.as_tensor(px, dtype=F64) + 1) / W - 1 - P[0, 2]
    ndcy = (2 * torch.as_tensor(py, dtype=F64) + 1) / H - 1 - P[1, 2]
    det = P[0, 0] * P[1, 1] - P[0, 1] * P[1, 0]
    return (P[1, 1] * ndcx - P[0, 1] * ndcy) / det, (P[0, 0] * ndcy - P[1, 0] * ndcx) / det


def _rotmat_quat(Rm):
    """(w, x, y, z) of a proper rotation matrix (fp64)."""
    t = float(Rm[0, 0] + Rm[1, 1] + Rm[2, 2])
    if t > 0:
        s = math.sqrt(t + 1.0) * 2
        q = [0.25 * s, (Rm[2, 1] - Rm[1, 2]) / s, (Rm[0, 2] - Rm[2, 0]) / s, (Rm[1, 0] - Rm[0, 1]) / s]
    else:
        i = int(torch.argmax(torch.diagonal(Rm)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(float(1.0 + Rm[i, i] - Rm[j, j] - Rm[k, k])) * 2
        q = [0.0] * 4
        q[0] = float(Rm[k, j] - Rm[j, k]) / s
        q[1 + i] = 0.25 * s
        q[1 + j] = float(Rm[j, i] + Rm[i, j]) / s
        q[1 + k] = float(Rm[k, i] + Rm[i, k]) / s
    return torch.tensor([float(v) for v in q], dtype=F64)


def to_world(cam, means_view, rot_view):
    """View-space means and quaternions -> world space through the inverse of the camera's view (a rotation R_cw turns the
    covariance R S^2 R^T into R_cw R S^2 R^T R_cw^T, i.e. the quaternion q into q_cw q)."""
    w2c = cam["viewmatrix"].to(F64).T
    c2w = torch.linalg.inv(w2c)
    means = means_view @ c2w[:3, :3].T + c2w[:3, 3]
    q_cw = _rotmat_quat(c2w[:3, :3])
    return means, synthetic._quat_mul(q_cw.expand_as(rot_view), rot_view)


def screen_scene(W, H, px, py, sigma, z, opac, rgb=None, sh_degree=0, seed=0, thin=None, bg=(0.0, 0.0, 0.0), semantics=0, fovx=50.0,
                 cam=None, sh_coeffs=None):
    """Gaussians given in pixels: centre (px, py), isotropic world std-dev sigma z / fx (screen std-dev `sigma` before the 0.3
    dilation on a square-pixel camera; fx = W / (2 tanfovx), the rasterizer's x focal length), view depth z, opacity.
    thin: per-Gaussian ratio of the short to the long axis (with a random rotation).  cam: the camera (synthetic.make_camera,
    image W x H); the view-space centres and quaternions go to world space through its inverse view.  Its sh_degree is the active
    degree; sh_coeffs (default (sh_degree + 1)^2) coefficients are stored, the inactive ones random like the others."""
    gen = torch.Generator().manual_seed(seed)
    if cam is None:
        cam = synthetic.make_camera(W, H, fovx, None, sh_degree, bg)
        posed = False
    else:
        assert (cam["image_width"], cam["image_height"]) == (W, H), "the camera's image is W x H"
        cam = dict(cam, bg=torch.tensor(bg, dtype=torch.float32))
        sh_degree = cam["sh_degree"]
        posed = True
    t = lambda v: torch.as_tensor(v, dtype=F64).reshape(-1)
    px, py, sigma, z, opac = t(px), t(py), t(sigma), t(z), t(opac)
    n = len(px)
    py, sigma, z, opac = py.expand(n), sigma.expand(n), z.expand(n), opac.expand(n)
    fx = W / (2 * cam["tanfovx"])
    if not posed:
        ndcx, ndcy = (2 * px + 1) / W - 1, (2 * py + 1) / H - 1
        means = torch.stack([ndcx * cam["tanfovx"] * z, ndcy * cam["tanfovy"] * z, z], 1)
    else:
        u, v = ratio_of(cam, px, py)
        means = torch.stack([u * z, v * z, z], 1)
    s = sigma * z / fx
    scales = torch.stack([s, s, s], 1)
    rot = torch.zeros(n, 4, dtype=F64); rot[:, 0] = 1
    if thin is not None:
        thin = t(thin).expand(n)
        scales[:, 1] = s * thin
        ang = torch.rand(n, generator=gen, dtype=F64) * math.pi
        rot = torch.stack([torch.cos(ang / 2), torch.zeros(n, dtype=F64), torch.zeros(n, dtype=F64), torch.sin(ang / 2)], 1)
    if posed:
        means, rot = to_world(cam, means, rot)
    M = (sh_degree + 1) ** 2 if sh_coeffs is None else int(sh_coeffs)
    shs = torch.randn(n, M, 3, generator=gen, dtype=F64) * 0.15
    rgb = torch.rand(n, 3, generator=gen, dtype=F64) * 0.8 + 0.1 if rgb is None else torch.as_tensor(rgb, dtype=F64).expand(n, 3)
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
    r = lambda lo, hi: torch.rand(n, generator=g, dtype=F64) * (hi - lo) + lo
    return screen_scene(W, H, r(0, W), r(0, H), r(1.5, 6.0), r(3.0, 30.0), r(0.05, 0.9), seed=seed, **kw)


def stack(W, H, cx, cy, K, seed, opac=(0.006, 0.010), sigma=40.0, z0=2.0, **kw):
    """K wide, faint Gaussians stacked over the tile around (cx, cy), in strictly increasing depth: every pixel of that tile
    blends all K of them."""
    g = torch.Generator().manual_seed(seed)
    o = torch.rand(K, generator=g, dtype=F64) * (opac[1] - opac[0]) + opac[0]
    jit = lambda: (torch.rand(K, generator=g, dtype=F64) - 0.5) * 2.0
    z = z0 + 0.01 * torch.arange(K, dtype=F64) + 0.001 * torch.rand(K, generator=g, dtype=F64)
    return screen_scene(W, H, cx + jit(), cy + jit(), sigma, z, o, seed=seed, **kw)
