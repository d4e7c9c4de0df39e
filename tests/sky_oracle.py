"""Torch and float64 restatements of the reference's sky cube map composite — TEST INFRASTRUCTURE.

  composite   lib/models/sky_cubemap.py:77-123 and street_gaussian_renderer.py:107-111 in torch, in the dtype of its inputs:
              rays Rm^T K^-1 (i + a, j + b, 1) (graphics_utils.py:186-207), the mask (the given sky mask or rows 0-49; else
              1 - acc > 1e-3 on the detached acc), the cube lookup below, the clamp to [0, 1], the fill and rgb + sky (1 - acc).
              Differentiable in rgb, acc and the cube map.  In fp32 it is the "torch restatement" the benchmark times.
  lookup      what dr.texture(cube, dirs, filter_mode='linear', boundary_mode='cube') computes, restated (nvdiffrast is not
              installed here): the face of the largest |component| (z only if strictly largest, then y if |y| > |x|, else x;
              faces 0:+x 1:-x 2:+y 3:-y 4:+z 5:-z), face coordinates inverting cube_to_dir (sky_cubemap.py:154-161),
              u = clamp((g + 1) / 2, 0, 1), bilinear over the four taps around (u R - 0.5, v R - 0.5) with texel (col, row)
              centred at ((col + 0.5) / R, (row + 0.5) / R).  A tap past a face edge reads the adjacent face's edge texel at the
              same position along the shared edge (ADJ).  A tap past a cube corner has no texel; it takes the mean of the three taps
              that exist.  That corner rule is this project's: nvdiffrast's own rule at corners is not verified against.
  texture     the dr.texture signature over lookup, for tests/golden/make_sky_golden.py.
  sky64       float64 values by autograd of `composite`, with per-element bounds for rgb_out, dL/dacc and every texel of dL/dcube.

Pinned by tests/golden/callsite/sky.npz (tests/golden/make_sky_golden.py runs the reference's own SkyCubeMap.forward).
Bounds follow oracle/step64.py's conventions: u = 2^-24, first order, each constant a count of roundings derived at sky64.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

U = 2.0 ** -24
TINY = 1e-30
F64 = torch.float64
TOP_ROWS = 50  # sky_cubemap.py:83

# cube_to_dir's face frames: direction = N + gx U + gy V
FACE_N = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
FACE_U = [(0, 0, -1), (0, 0, 1), (1, 0, 0), (1, 0, 0), (1, 0, 0), (-1, 0, 0)]
FACE_V = [(0, -1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1), (0, -1, 0), (0, -1, 0)]

# ADJ[face][edge] = (neighbour face, its column, its row) for a tap past edge 0: column -1, 1: column R, 2: row -1, 3: row R, at
# position t along the edge (the row for edges 0 and 1, the column for 2 and 3).  "0" / "R-1": the neighbour's first / last
# column or row; "t" / "R-1-t": the same / the reversed position along the shared edge.
ADJ = [
    [(4, "R-1", "t"), (5, "0", "t"), (2, "R-1", "R-1-t"), (3, "R-1", "t")],
    [(5, "R-1", "t"), (4, "0", "t"), (2, "0", "t"), (3, "0", "R-1-t")],
    [(1, "t", "0"), (0, "R-1-t", "0"), (5, "R-1-t", "0"), (4, "t", "0")],
    [(1, "R-1-t", "R-1"), (0, "t", "R-1"), (4, "t", "R-1"), (5, "R-1-t", "R-1")],
    [(1, "R-1", "t"), (0, "0", "t"), (2, "t", "R-1"), (3, "t", "0")],
    [(0, "R-1", "t"), (1, "0", "t"), (2, "R-1-t", "0"), (3, "R-1-t", "R-1")],
]
_SPEC = {"0": 0, "R-1": 1, "t": 2, "R-1-t": 3}


def cube_to_dir(s: int, x, y):
    """sky_cubemap.py:154-161."""
    one = torch.ones_like(x)
    return torch.stack({0: (one, -y, -x), 1: (-one, -y, x), 2: (x, one, y), 3: (x, -one, -y), 4: (x, -y, one), 5: (-x, -y, -one)}[s], dim=-1)


def face_coords(d):
    """Face and face coordinates (gx, gy) of directions d [..., 3]."""
    a = d.abs()
    zf = (a[..., 2] > a[..., 0]) & (a[..., 2] > a[..., 1])
    yf = ~zf & (a[..., 1] > a[..., 0])
    axis = torch.where(zf, 2, torch.where(yf, 1, 0))
    comp = d.gather(-1, axis.unsqueeze(-1)).squeeze(-1)
    face = 2 * axis + (comp < 0).long()
    Ut = torch.tensor(FACE_U, dtype=d.dtype, device=d.device)[face]
    Vt = torch.tensor(FACE_V, dtype=d.dtype, device=d.device)[face]
    ma = comp.abs()
    return face, (d * Ut).sum(-1) / ma, (d * Vt).sum(-1) / ma


def tex_xy(gx, gy, R: int):
    """Continuous texel coordinates (column, row) whose integer values are texel centres."""
    u = ((gx + 1) * 0.5).clamp(0, 1)
    v = ((gy + 1) * 0.5).clamp(0, 1)
    return u * R - 0.5, v * R - 0.5


def _adj_tensors(device):
    f = torch.tensor([[e[0] for e in row] for row in ADJ], device=device)
    c = torch.tensor([[_SPEC[e[1]] for e in row] for row in ADJ], device=device)
    r = torch.tensor([[_SPEC[e[2]] for e in row] for row in ADJ], device=device)
    return f, c, r


def _spec(code, t, R):
    return torch.where(code == 0, torch.zeros_like(t), torch.where(code == 1, torch.full_like(t, R - 1), torch.where(code == 2, t, R - 1 - t)))


def tap_texels(face, c, r, R: int):
    """Flat texel index into [6, R, R] of integer taps (c, r) in [-1, R] on `face`, by ADJ past an edge; -1 past a cube corner."""
    oc, orow = (c < 0) | (c >= R), (r < 0) | (r >= R)
    af, ac, ar = _adj_tensors(face.device)
    edge = torch.where(oc, (c >= R).long(), 2 + (r >= R).long())
    t = torch.where(oc, r, c)
    nf, ncode, rcode = af[face, edge], ac[face, edge], ar[face, edge]
    wc, wr = _spec(ncode, t, R), _spec(rcode, t, R)
    inside = (face * R + r.clamp(0, R - 1)) * R + c.clamp(0, R - 1)
    wrapped = (nf * R + wr) * R + wc
    idx = torch.where(oc | orow, wrapped, inside)
    return torch.where(oc & orow, torch.full_like(idx, -1), idx)


def taps(face, x, y, R: int):
    """Texels [..., 4] (-1 for a corner tap) and bilinear weights [..., 4] of the taps around (x, y), in the order (x0, y0),
    (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1)."""
    x0, y0 = torch.floor(x), torch.floor(y)
    fx, fy = x - x0, y - y0
    c0, r0 = x0.long(), y0.long()
    idx = torch.stack([tap_texels(face, c0 + (k & 1), r0 + (k >> 1), R) for k in range(4)], -1)
    w = torch.stack([(1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy], -1)
    return idx, w


def effective(idx, w):
    """A corner tap's weight shared by thirds among the three taps that exist: (texels with the corner's replaced by 0, weights)."""
    corner = idx < 0
    wc = (w * corner).sum(-1, keepdim=True)
    has = corner.any(-1, keepdim=True)
    w_eff = torch.where(corner, torch.zeros_like(w), w + torch.where(has, wc / 3, torch.zeros_like(wc)))
    return idx.clamp(min=0), w_eff


def lookup(cube, d):
    """The restated dr.texture(linear, cube) of cube [6, R, R, C] along directions d [..., 3] -> [..., C]; differentiable in cube."""
    R = cube.shape[1]
    face, gx, gy = face_coords(d)
    x, y = tex_xy(gx, gy, R)
    idx, w = effective(*taps(face, x, y, R))
    flat = cube.reshape(6 * R * R, -1)
    return (flat[idx.reshape(-1)].reshape(*idx.shape, -1) * w.unsqueeze(-1).to(cube.dtype)).sum(-2)


def texture(tex, uv, filter_mode="linear", boundary_mode="cube", **_):
    """nvdiffrast.torch.texture's signature for a cube map tex [1, 6, R, R, C] and directions uv [1, ..., 3]."""
    assert filter_mode == "linear" and boundary_mode == "cube" and tex.shape[0] == 1
    return lookup(tex[0], uv[0]).unsqueeze(0)


def rays(H: int, W: int, K, w2c, jx=None, jy=None):
    """Unnormalised ray directions [H, W, 3] = Rm^T K^-1 (i + a, j + b, 1), Rm = w2c[:3, :3]; a = b = 0.5 without jitter."""
    dt, dev = K.dtype, K.device
    j, i = torch.meshgrid(torch.arange(H, dtype=dt, device=dev), torch.arange(W, dtype=dt, device=dev), indexing="ij")
    px = i + (jx.to(dt) if jx is not None else 0.5)
    py = j + (jy.to(dt) if jy is not None else 0.5)
    p = torch.stack([px, py, torch.ones_like(px)], -1)
    M = w2c[:3, :3].T @ torch.linalg.inv(K)
    return p @ M.T


def sky_mask_of(acc, sky_mask):
    """The pixels that sample the cube [H, W]: the given mask and rows 0-49 (not written back), or 1 - acc > 1e-3."""
    if sky_mask is not None:
        m = sky_mask.reshape(acc.shape[-2:]).clone()
        m[:TOP_ROWS] = True
        return m
    return (1 - acc.detach()[0].float()) > 1e-3


def composite(rgb, acc, cube, K, w2c, sky_mask=None, jx=None, jy=None, fill: float = 1.0):
    """rgb + sky (1 - acc) in the dtype of rgb; differentiable in rgb, acc and cube."""
    H, W = rgb.shape[1:]
    dt = rgb.dtype
    d = rays(H, W, K.to(dt), w2c.to(dt), jx, jy)
    mask = sky_mask_of(acc, sky_mask)
    s = lookup(cube.to(dt), d).clamp(0, 1)  # [H, W, 3]
    sky = torch.where(mask.unsqueeze(-1), s, torch.full_like(s, fill)).permute(2, 0, 1)
    return rgb + sky * (1 - acc)


def sky64(rgb, acc, cube, K, w2c, g, sky_mask=None, jx=None, jy=None, fill: float = 1.0) -> Dict[str, torch.Tensor]:
    """float64 rgb_out, dL/dacc, dL/dcube for the upstream g [3, H, W], with per-element bounds b_out, b_dacc, b_dcube (u = 2^-24).

    The kernel's ray (K^-1 by the adjugate, then Rm^T K^-1, then the product with p = fl(i + a)):
      dK^-1_mn <= 8 u (|adj|_mn + |adj_mn| |det|_abs / |det|) / |det|   (2 roundings per cofactor, 5 in det, the reciprocal and product)
      dd_k     <= sum_m |Rm_mk| sum_n dK^-1_mn |p_n| + 8 u sum_m |Rm_mk| sum_n |K^-1_mn| |p_n|   (3 + 3 roundings, 1 in p, 1 spare)
    The face coordinate g = c * fl(1 / a) (2 roundings): dg <= (dc + |g| da) / a + 2 u |g|; the texel coordinate x = fl(fl(fl(g + 1) / 2) R
    - 0.5): dx <= R dg / 2 + 3 u R.  The lookup is continuous and piecewise bilinear in (x, y), also across face edges and corners, so
    the kernel's value lies within Lx dx + Ly dy of the exact one, Lx, Ly its largest slopes over the box (x +- dx, y +- dy) (taken at the
    box's corners: a slope is linear in the other coordinate within a cell).  Rounding of the lookup: the weights 2 u, the corner mean
    4 u, 4 products and 3 adds: 8 u sum w |t|.  So ds = Lx dx + Ly dy + 8 u sum w |t|, and the clamp does not increase it.
      out    ds |1 - acc| + 2 u |sky (1 - acc)| + u |out|          (1 - acc, the product, the sum)
      dacc   sum_c ds_c |g_c| + 3 u sum_c |sky_c g_c|
      dcube  per term w_eff g (1 - acc): 6 u (1 - acc, its product with g, the corner share, its add, the product with w), plus
             n u sum |term| for the n terms of a texel added in any order; the weights move by at most 4/3 (dx + dy) (1-Lipschitz
             bilinear weights plus a third of the corner's), on the texels of any of the box's tap sets; and where s_c is within ds_c
             of 0 or 1 the clamp's gate may differ: the whole term.
    """
    dev = rgb.device
    d64 = lambda t: t.detach().to(dev, F64)
    H, W = rgb.shape[1:]
    R = cube.shape[1]
    r64, a64, c64 = d64(rgb).requires_grad_(True), d64(acc).requires_grad_(True), d64(cube).requires_grad_(True)
    K64, T64 = d64(K), d64(w2c)
    out = composite(r64, a64, c64, K64, T64, sky_mask, jx, jy, fill)
    gg = d64(g)
    da, dc = torch.autograd.grad(out, [a64, c64], gg)
    res = dict(out=out.detach(), dacc=da, dcube=dc)

    # the ray's error
    k = K64
    adj = torch.stack([torch.stack([k[1, 1] * k[2, 2] - k[1, 2] * k[2, 1], k[0, 2] * k[2, 1] - k[0, 1] * k[2, 2], k[0, 1] * k[1, 2] - k[0, 2] * k[1, 1]]),
                       torch.stack([k[1, 2] * k[2, 0] - k[1, 0] * k[2, 2], k[0, 0] * k[2, 2] - k[0, 2] * k[2, 0], k[0, 2] * k[1, 0] - k[0, 0] * k[1, 2]]),
                       torch.stack([k[1, 0] * k[2, 1] - k[1, 1] * k[2, 0], k[0, 1] * k[2, 0] - k[0, 0] * k[2, 1], k[0, 0] * k[1, 1] - k[0, 1] * k[1, 0]])])
    ka = k.abs()
    adj_abs = torch.stack([torch.stack([ka[1, 1] * ka[2, 2] + ka[1, 2] * ka[2, 1], ka[0, 2] * ka[2, 1] + ka[0, 1] * ka[2, 2], ka[0, 1] * ka[1, 2] + ka[0, 2] * ka[1, 1]]),
                           torch.stack([ka[1, 2] * ka[2, 0] + ka[1, 0] * ka[2, 2], ka[0, 0] * ka[2, 2] + ka[0, 2] * ka[2, 0], ka[0, 2] * ka[1, 0] + ka[0, 0] * ka[1, 2]]),
                           torch.stack([ka[1, 0] * ka[2, 1] + ka[1, 1] * ka[2, 0], ka[0, 1] * ka[2, 0] + ka[0, 0] * ka[2, 1], ka[0, 0] * ka[1, 1] + ka[0, 1] * ka[1, 0]])])
    det = (k[0] * adj[:, 0]).sum()
    det_abs = (ka[0] * adj_abs[:, 0]).sum()
    kinv = adj / det
    d_kinv = 8 * U * (adj_abs + adj.abs() * det_abs / det.abs()) / det.abs()
    Ra = T64[:3, :3].abs()
    j_, i_ = torch.meshgrid(torch.arange(H, dtype=F64, device=dev), torch.arange(W, dtype=F64, device=dev), indexing="ij")
    px = i_ + (jx.to(dev, F64) if jx is not None else 0.5)
    py = j_ + (jy.to(dev, F64) if jy is not None else 0.5)
    pa = torch.stack([px.abs(), py.abs(), torch.ones_like(px)], -1)
    dd = pa @ (Ra.T @ d_kinv).T + 8 * U * (pa @ (Ra.T @ kinv.abs()).T)  # [H, W, 3]
    dirs = rays(H, W, K64, T64, jx, jy)
    face, gx, gy = face_coords(dirs)
    Ut = torch.tensor(FACE_U, dtype=F64, device=dev)[face].abs()
    Vt = torch.tensor(FACE_V, dtype=F64, device=dev)[face].abs()
    Nt = torch.tensor(FACE_N, dtype=F64, device=dev)[face].abs()
    ma = (dirs.abs() * Nt).sum(-1)
    dma, dcu, dcv = (dd * Nt).sum(-1), (dd * Ut).sum(-1), (dd * Vt).sum(-1)
    dgx = (dcu + gx.abs() * dma) / ma + 2 * U * gx.abs()
    dgy = (dcv + gy.abs() * dma) / ma + 2 * U * gy.abs()
    dx, dy = R * dgx / 2 + 3 * U * R, R * dgy / 2 + 3 * U * R
    x, y = tex_xy(gx, gy, R)
    flat = d64(cube).reshape(6 * R * R, 3)

    def slopes(xs, ys):
        idx, w = taps(face, xs, ys, R)
        ie, _ = effective(idx, w)
        t = flat[ie.reshape(-1)].reshape(*ie.shape, 3)  # [H, W, 4, 3]
        corner = (idx < 0).unsqueeze(-1)
        mean = (t * ~corner).sum(-2, keepdim=True) / 3
        t = torch.where(corner, mean, t)
        fx, fy = (xs - torch.floor(xs)).unsqueeze(-1), (ys - torch.floor(ys)).unsqueeze(-1)
        lx = (1 - fy) * (t[..., 1, :] - t[..., 0, :]).abs() + fy * (t[..., 3, :] - t[..., 2, :]).abs()
        ly = (1 - fx) * (t[..., 2, :] - t[..., 0, :]).abs() + fx * (t[..., 3, :] - t[..., 1, :]).abs()
        return lx, ly, idx, t

    lx, ly, idx0, t0 = slopes(x, y)
    box = []
    for sx in (-1, 1):
        for sy in (-1, 1):
            xs = (x + sx * dx).clamp(-0.5, R - 0.5)
            ys = (y + sy * dy).clamp(-0.5, R - 0.5)
            bx, by, bidx, _ = slopes(xs, ys)
            lx, ly = torch.maximum(lx, bx), torch.maximum(ly, by)
            box.append(bidx)
    _, w0 = taps(face, x, y, R)
    w_eff_idx, w_eff = effective(idx0, w0)
    sum_wt = (w0.unsqueeze(-1) * t0.abs()).sum(-2)  # [H, W, 3]
    ds = lx * dx.unsqueeze(-1) + ly * dy.unsqueeze(-1) + 8 * U * sum_wt
    mask = sky_mask_of(d64(acc), sky_mask).unsqueeze(-1)
    s = (w_eff.unsqueeze(-1) * flat[w_eff_idx.reshape(-1)].reshape(*w_eff_idx.shape, 3)).sum(-2)
    sky = torch.where(mask, s.clamp(0, 1), torch.full_like(s, fill))
    dsky = torch.where(mask, ds, torch.zeros_like(ds)).permute(2, 0, 1)
    sky = sky.permute(2, 0, 1)
    tm = (1 - d64(acc)).abs()
    res["b_out"] = dsky * tm + 2 * U * (sky * tm).abs() + U * res["out"].abs() + TINY
    res["b_dacc"] = (dsky * gg.abs()).sum(0, keepdim=True) + 3 * U * (sky * gg).abs().sum(0, keepdim=True) + TINY

    # dL/dcube
    gt = (gg * tm).permute(1, 2, 0) * mask  # [H, W, 3] |g (1 - acc)| where sampled
    gate_amb = mask & ((s.abs() <= ds) | ((s - 1).abs() <= ds))
    gate = mask & (s >= 0) & (s <= 1)
    term = w_eff.unsqueeze(-1) * (gt * gate).unsqueeze(-2)  # [H, W, 4, 3]
    n = torch.zeros(6 * R * R, dtype=F64, device=dev).index_add_(0, w_eff_idx.reshape(-1), (w_eff > 0).reshape(-1).to(F64) * mask[..., 0].unsqueeze(-1).expand_as(w_eff).reshape(-1))
    sabs = torch.zeros(6 * R * R, 3, dtype=F64, device=dev).index_add_(0, w_eff_idx.reshape(-1), term.abs().reshape(-1, 3))
    b = (6 * U + n.unsqueeze(-1) * U) * sabs
    amb = w_eff.unsqueeze(-1) * (gt.abs() * gate_amb).unsqueeze(-2)
    b = b.index_add_(0, w_eff_idx.reshape(-1), amb.reshape(-1, 3))
    move = (4.0 / 3.0) * (dx + dy).unsqueeze(-1) * gt.abs()  # [H, W, 3]
    for bidx in [idx0] + box:
        valid = bidx >= 0
        contrib = (move.unsqueeze(-2) * valid.unsqueeze(-1)).reshape(-1, 3)
        b = b.index_add_(0, bidx.clamp(min=0).reshape(-1), contrib)
    res["b_dcube"] = b.reshape(6, R, R, 3) + TINY
    res["face"], res["x"], res["y"] = face, x, y
    return res
