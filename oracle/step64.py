"""float64 restatements of the per-step kernels around the rasterizer, each with a per-element error bound — TEST
INFRASTRUCTURE, not product code (nothing under street_gaussians_b200/ may import it).  Runs on the CPU or on a CUDA device.

  compose64     the scene-graph composer, forward and backward (csrc/compose.cu; reference lib/models/street_gaussian_model.py:
                287-449, lib/models/gaussian_model.py:224-251, lib/models/gaussian_model_actor.py:71-80, lib/utils/general_utils.py:
                125-146 and 220-238; the values come from oracle/compose_oracle.py run in fp64)
  image_loss64  (1 - l) l1w L1 + l (1 - SSIM) and dL/dimage in closed form (csrc/losses.cu; reference lib/utils/loss_utils.py:21-37
                and :84-126, train.py:101-104)
  adam64        one torch.optim.Adam step without weight decay / amsgrad (csrc/optim.cu adam_kernel; reference
                lib/models/gaussian_model.py:300-303, 316-318)
  stats64       the densification statistics (csrc/optim.cu densify_stats_kernel; reference lib/models/street_gaussian_model.py:
                551-571)
  acc_loss64    the sky loss and the object-accumulation loss, value and dL/dacc (csrc/losses.cu acc_loss_kernel<SkyForm / ObjForm>;
                reference train.py:107-122)
  lidar64       the LiDAR depth loss: the exact top-k selection, value and fp32 gradients in the kernel's order (csrc/losses.cu
                lidar_*_kernel; reference train.py:124-132)

Every function returns, for each output element, the fp64 value and an absolute bound on |fp32 kernel - fp64 value| (lidar64's
gradients are instead an fp32 restatement the kernel must match bit for bit), built from the
magnitudes the fp32 code actually combines.  u = 2^-24 is the unit roundoff of fp32; a rounding whose result can be subnormal adds
an absolute 2^-149.  The bounds are first order (products of two error terms are dropped); each constant is a count of roundings,
derived in the docstring of the function that uses it and rounded up, never fitted to observed errors.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from oracle import compose_oracle as CO

F64 = torch.float64
U = 2.0 ** -24
TINY = 2.0 ** -149
KEYS = ("xyz", "rotation", "scaling", "opacity", "features_dc", "features_rest")


def _absmul(a, b):
    """|a| (x) |b|: for each component of the Hamilton product, the sum of the magnitudes of its four terms."""
    a0, a1, a2, a3 = torch.unbind(a.abs(), -1)
    b0, b1, b2, b3 = torch.unbind(b.abs(), -1)
    return torch.stack((a0 * b0 + a1 * b1 + a2 * b2 + a3 * b3, a0 * b1 + a1 * b0 + a2 * b3 + a3 * b2,
                        a0 * b2 + a1 * b3 + a2 * b0 + a3 * b1, a0 * b3 + a1 * b2 + a2 * b1 + a3 * b0), -1)


def _rot_poly(q):
    """R of a unit quaternion as the polynomial general_utils.py:125-146 evaluates after normalising: [..., 9]."""
    w, x, y, z = torch.unbind(q, -1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y), 2 * (x * y + w * z), 1 - 2 * (x * x + z * z),
                        2 * (y * z - w * x), 2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)


# ----------------------------------------------------------------------------------------------- composer
def compose64(models: Sequence[dict], poses, idft, flip, flip_quat, up: dict) -> Dict[str, torch.Tensor]:
    """models: [background, actor...] dicts of the fp32 raw tensors (compose_case.KEYS); poses [A, 7], idft [A, C], flip bool [sum of
    actor counts] or None, flip_quat [4]; up: fp32 upstream gradients of the composed xyz, rotation, scaling, opacity, features.
    Returns {name: value} and {"b_" + name: bound} for the forward outputs (xyz, rotation, scaling, opacity, features), every raw
    gradient ("g{i}_{key}") and the actor pose gradients ("dposes", [A, 7]).

    Bounds (u = 2^-24; the composer rounds on every operation, FMA contraction only removes roundings):
      xyz        posed: u (16 sum_j |x_j| + 6 (sum_j |R_ij x_j| + |t_i|)).  R is formed from q / |q|: the norm carries 3 u (a positive
                 four-term sum, halved by the square root, plus the sqrt), the division 1 u, and each entry 1 - 2 (y^2 + z^2) etc.
                 adds 4 roundings on terms of size <= 2, so |dR_ij| <= 16 u; the product R x + t is a 4-term sum (6 u on its
                 magnitudes).  Background rows are copies: bound 0.
      rotation   unposed: 6 u |n_k| (the 4 u of one normalisation, rounded up).  posed: y = q_obj (x) b with b = [flip (x)] n, z = y/|y|:
                 |dy| <= 14 u |q_obj| (x) |b| (6 u from n, 4 u per Hamilton product) and the projection onto the sphere passes at
                 most sum_j |dy_j| / |y| to each component, the final normalisation 4 u |z_k|:  u (16 sum_j mass(y)_j / |y| + 6 |z_k|).
      scaling    expf is within 2 ulp <= 4 u |v|, plus 2^-149.
      opacity    1 / (1 + expf(-o)): 4 u from expf, 1 u each for the add and the division: 6 u |v|, plus 2^-149.
      features   DC of an actor: C products summed sequentially, 2C roundings on sum_c |dc_c w_c|; every other element is a copy (0).
    Gradients:
      scaling    6 u |v| (expf and one product);  opacity |v| (10 u + 8 u o / (1 - o)): 1 - o inherits o's 6 u absolute error, which
                 is relative to 1 - o;  features_dc: actor u |v| (one product), background a copy (0);  features_rest a copy (0).
      xyz        posed: u (16 sum_j |g_j| + 6 sum_j |R_ji g_j|) (R^T g, the same R as above); background a copy (0).
      rotation   K u M_k with the magnitude chain M of  gy = (g - z (z.g)) / |y|,  gb = conj(q_obj) (x) gy [conj(flip) (x) gb],
                 out = (gb - n (n.gb)) / |raw|:  M(gy)_k = (|g_k| + |z_k| sum_j |z_j g_j|) / |y|, M(gb) = |q_obj| (x) M(gy) [|flip| (x) ..],
                 M_k = (M(gb)_k + |n_k| sum_j |n_j| M(gb)_j) / |raw|.  K = 64 posed (z's forward error, <= 16 u of the mass, enters
                 twice, through z and through |y|; 8 further stages of at most 4 roundings each), K = 32 unposed (g = gb directly).
                 The 1/|raw| and 1/|y| factors are what a small raw quaternion amplifies.
      dposes     per actor, a sum of per-Gaussian terms: the 9 products g_xyz (x) x_local, the rotation terms ga = gy (x) conj(b) and
                 g_xyz itself.  Each warp adds its 32 terms in a 5-level tree, then float atomics add at most n_atom = n / 32 + 66
                 partial sums in any order (one per whole warp, up to 32 per lane from each of the two boundary warps), so a sum
                 carries (5 + n_atom) u sum |term|.  The matrix part goes through the finalize kernel's linear map c (dR/dq at
                 q / |q| projected on the tangent space, over |q|), which adds 16 roundings on sum |c| |G|:
                   quaternion k: u [(7 + n_atom) sum |ga_k| + 64 sum M(ga)_k + (22 + n_atom) sum_ij |c_kij| sum |G_ij|]
                   translation i: (5 + n_atom) u sum |g_xyz_i|.
    """
    dev = models[0]["xyz"].device
    d = lambda t: t.detach().to(dev, F64)
    m64 = [{k: d(v).requires_grad_(True) for k, v in m.items()} for m in models]
    A = len(models) - 1
    fq = d(flip_quat) if flip_quat is not None else torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=F64, device=dev)
    p64 = d(poses).requires_grad_(True) if A else torch.zeros(0, 7, dtype=F64, device=dev)
    i64 = d(idft) if A else torch.zeros(0, 1, dtype=F64, device=dev)
    fl = flip.to(dev).bool() if flip is not None else None
    out = CO.compose(m64, p64, i64, fl, fq)
    names = ("xyz", "rotation", "scaling", "opacity", "features")
    res = {k: out[k].detach() for k in names}
    ins = [m[k] for m in m64 for k in KEYS] + ([p64] if A else [])
    grads = torch.autograd.grad([out[k] for k in names], ins, [d(up[k]) for k in names], allow_unused=True)
    for i, m in enumerate(m64):
        for j, k in enumerate(KEYS):
            g = grads[i * 6 + j]
            res[f"g{i}_{k}"] = g if g is not None else torch.zeros_like(m[k])
    if A:
        res["dposes"] = grads[-1]

    # per-Gaussian inputs in composed order
    counts = [int(m["xyz"].shape[0]) for m in models]
    P = sum(counts)
    seg = torch.repeat_interleave(torch.arange(len(models), device=dev), torch.tensor(counts, device=dev))
    posed = seg > 0
    raw = lambda k: torch.cat([d(m[k]) for m in models])
    x_l, r_raw, ls = raw("xyz"), raw("rotation"), raw("scaling")
    qo_tab = torch.cat([torch.tensor([[1.0, 0, 0, 0, 0, 0, 0]], dtype=F64, device=dev), d(poses) if A else torch.zeros(0, 7, dtype=F64, device=dev)])
    qo, t_obj = qo_tab[seg, :4], qo_tab[seg, 4:7]
    fm = torch.zeros(P, dtype=torch.bool, device=dev)
    if fl is not None:
        fm[counts[0]:] = fl
    x_l = torch.where(fm[:, None], x_l * torch.tensor([1.0, -1.0, 1.0], dtype=F64, device=dev), x_l)
    qhat = qo / qo.norm(dim=1, keepdim=True)
    R = _rot_poly(qhat).reshape(P, 3, 3)
    pz = posed[:, None]
    # forward
    res["b_xyz"] = torch.where(pz, U * (16 * x_l.abs().sum(1, keepdim=True) + 6 * ((R.abs() * x_l.abs()[:, None, :]).sum(2) + t_obj.abs())),
                               torch.zeros(P, 3, dtype=F64, device=dev))
    rn = r_raw.norm(dim=1, keepdim=True).clamp(min=1e-12)
    n = r_raw / rn
    massb = torch.where(fm[:, None], _absmul(fq.expand(P, 4), n), n.abs())
    b = torch.where(fm[:, None], CO.quat_mul(fq.expand(P, 4), n), n)
    y = CO.quat_mul(qo, b)
    yn = y.norm(dim=1, keepdim=True).clamp(min=1e-12)
    z = y / yn
    mass_y = _absmul(qo, massb)
    res["b_rotation"] = torch.where(pz, U * (16 * mass_y.sum(1, keepdim=True) / yn + 6 * z.abs()), 6 * U * n.abs()) + TINY
    res["b_scaling"] = 4 * U * res["scaling"].abs() + TINY
    res["b_opacity"] = 6 * U * res["opacity"].abs() + TINY
    M = res["features"].shape[1]
    bf = torch.zeros(P, M, 3, dtype=F64, device=dev)
    off = counts[0]
    for a in range(A):
        nA = counts[a + 1]
        if nA:
            dc = d(models[a + 1]["features_dc"])
            Cd = dc.shape[1]
            bf[off:off + nA, 0] = 2 * Cd * U * (dc * i64[a][None, :Cd, None]).abs().sum(1)
        off += nA
    res["b_features"] = bf
    # backward
    gx, gq = d(up["xyz"]), d(up["rotation"])
    bg = {}
    o = torch.cat([torch.sigmoid(d(m["opacity"])) for m in models])
    bg["scaling"] = 6 * U * torch.cat([res[f"g{i}_scaling"] for i in range(len(models))]).abs() + TINY
    gop = torch.cat([res[f"g{i}_opacity"] for i in range(len(models))])
    bg["opacity"] = gop.abs() * (10 * U + 8 * U * o / (1 - o)) + TINY
    bg["xyz"] = torch.where(pz, U * (16 * gx.abs().sum(1, keepdim=True) + 6 * (R.abs() * gx.abs()[:, :, None]).sum(1)),
                            torch.zeros(P, 3, dtype=F64, device=dev))
    zz = torch.where(pz, z, n)
    yy = torch.where(pz, yn, torch.ones_like(yn))
    m_gy = (gq.abs() + zz.abs() * (zz * gq).abs().sum(1, keepdim=True)) / yy
    m_gb = torch.where(pz, _absmul(qo, m_gy), m_gy)
    m_gb = torch.where(fm[:, None], _absmul(fq.expand(P, 4), m_gb), m_gb)
    m_out = (m_gb + n.abs() * (n.abs() * m_gb).sum(1, keepdim=True)) / rn
    bg["rotation"] = torch.where(pz, 64.0, 32.0) * U * m_out + TINY
    off = 0
    for i, m in enumerate(models):
        c = counts[i]
        for k in ("xyz", "rotation", "scaling", "opacity"):
            res[f"b_g{i}_{k}"] = bg[k][off:off + c].reshape(res[f"g{i}_{k}"].shape)
        res[f"b_g{i}_features_dc"] = (U * res[f"g{i}_features_dc"].abs() + TINY) if i > 0 else torch.zeros_like(res[f"g{i}_features_dc"])
        res[f"b_g{i}_features_rest"] = torch.zeros_like(res[f"g{i}_features_rest"])
        off += c
    if A:
        gy = (gq - z * (z * gq).sum(1, keepdim=True)) / yn
        ga = CO.quat_mul(gy, b * torch.tensor([1.0, -1.0, -1.0, -1.0], dtype=F64, device=dev))
        m_ga = _absmul(m_gy, massb)
        G = (gx[:, :, None] * x_l[:, None, :]).reshape(P, 9)
        sums = lambda t: torch.zeros(A + 1, t.shape[1], dtype=F64, device=dev).index_add_(0, seg, t)[1:]
        s_ga, s_mga, s_G, s_gx = sums(ga.abs()), sums(m_ga), sums(G.abs()), sums(gx.abs())
        # c_kij = (D_k,ij - qh_k sum_m qh_m D_m,ij) / |q|, D = dR/dqh of the polynomial at qh = q / |q|
        q = d(poses)[:, :4]
        nq = q.norm(dim=1, keepdim=True)
        qh = q / nq
        D = torch.stack([torch.autograd.functional.jacobian(_rot_poly, qh[a]) for a in range(A)])  # [A, 9, 4]
        Dk = D.transpose(1, 2)  # [A, 4, 9]
        cabs = (Dk.abs() + qh.abs()[:, :, None] * (qh.abs()[:, :, None] * Dk.abs()).sum(1, keepdim=True)) / nq[:, :, None]
        n_atom = torch.tensor(counts[1:], dtype=F64, device=dev)[:, None] // 32 + 66
        bq = U * ((7 + n_atom) * s_ga + 64 * s_mga + (22 + n_atom) * (cabs * s_G[:, None, :]).sum(2))
        bt = (5 + n_atom) * U * s_gx
        res["b_dposes"] = torch.cat([bq, bt], 1) + TINY
    return res


# ----------------------------------------------------------------------------------------------- image loss
C1_32 = float(np.float32(np.float32(0.01) * np.float32(0.01)))  # the kernel's constants: 0.01f * 0.01f, 0.03f * 0.03f
C2_32 = float(np.float32(np.float32(0.03) * np.float32(0.03)))


def window_1d() -> np.ndarray:
    """The kernel's 1D window (make_window in csrc/losses.cu): (float)exp(-(k - 5)^2 / 4.5) in double, divided in fp32 by the fp32
    rounding of their exact sum (loss_utils.py:84-86: torch.Tensor([...]) / sum)."""
    g = np.array([np.float32(math.exp(-float((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5))) for k in range(11)], np.float32)
    s = np.float32(g.astype(np.float64).sum())
    return (g / s).astype(np.float32)


def window_2d(dev="cpu") -> torch.Tensor:
    """The 2D window the kernel's two separable passes apply: the outer product of window_1d, exact in fp64."""
    w = torch.from_numpy(window_1d().astype(np.float64)).to(dev)
    return w[:, None] * w[None, :]


def _pixel(m1, m2, s11, s22, s12, nodes):
    """The kernel's per-pixel SSIM arithmetic (ssim_stats_kernel) in its own order; every rounded intermediate goes to `nodes`."""
    def r(t):
        nodes.append(t)
        return t
    mu1_sq, mu2_sq, mu12 = r(m1 * m1), r(m2 * m2), r(m1 * m2)
    sig1, sig2, sig12 = r(s11 - mu1_sq), r(s22 - mu2_sq), r(s12 - mu12)
    A1, A2 = r(2.0 * mu12 + C1_32), r(2.0 * sig12 + C2_32)
    B1, B2 = r(r(mu1_sq + mu2_sq) + C1_32), r(r(sig1 + sig2) + C2_32)
    inv = r(1.0 / r(B1 * B2))
    S = r(r(A1 * A2) * inv)
    d_mu = r(r(r(2.0 * m2 * r(A2 - A1)) * inv) - r(r(S * 2.0 * m1) * r(r(1.0 / B1) - r(1.0 / B2))))
    d_xx = r(-S / B2)
    d_xy = r(r(2.0 * A1) * inv)
    return dict(S=S, d_mu=d_mu, d_xx=d_xx, d_xy=d_xy, B2=B2)


def image_loss64(img, gt, mask, w_l1: float, w_ssim: float) -> Dict[str, torch.Tensor]:
    """img, gt [C, H, W] fp32; mask [1, H, W] bool or None.  The kernel's grad (dL/dimage of w_l1 L1 + w_ssim SSIM) and scalars
    (value, L1, SSIM, masked pixel count), each with a bound ("b_" + name), plus "premise" = bound(B2) / B2 per pixel.

    Conventions of the reference: with a mask both images are zeroed outside it; the SSIM mean runs over all C H W pixels, L1 over
    the masked pixels times C; torch.abs's backward takes sign(0) = 0; an empty mask gives a NaN L1 (and a zero L1 gradient).
    Bounds, first-order propagation evaluated in fp64 (u = 2^-24):
      moments    mu_x, mu_y, E[x^2], E[y^2], E[xy]: two 11-tap passes, at most 24 roundings per term (two products and 10 additions
                 per pass, rounded up): 24 u conv(|term|).  The window is the kernel's own, so it adds no error.
      per pixel  S, d_mu, d_xx, d_xy (and B2) are evaluated as the kernel does; their error is  sum_j |df/dmoment_j| err_j  +
                 u sum_v |df/dv| |v| over every rounded intermediate v (both derivatives taken by fp64 autograd of `_pixel`).  This is
                 where sig = E[x^2] - mu^2 cancels in flat regions: |df/dv| |v| keeps the size of the cancelled terms.
      gradient   a, b, d = conv(d_mu), conv(d_xx), conv(d_xy): conv(err) + 24 u conv(|.|);  w_ssim / (C H W) (a + 2 x b + y d): 4 u
                 on |a| + 2 |x b| + |y d|, 3 u on the result (the fp32 coefficient and weight, the product); w_l1 sign / (n C): 2 u;
                 the sum: u.  Zero outside the mask, exactly.
      scalars    sums of fp32 per-pixel values through a 5-level warp tree (6 u on sum |.|, plus each value's own bound), then fp64;
                 the division and mix in fp64, one rounding to fp32 (u |.|); the count is exact.
    The linearisation assumes each relative perturbation is small; the caller asserts premise < 1e-2 on every pixel."""
    dev = img.device
    x, yv = img.detach().to(F64), gt.detach().to(F64)
    C, H, W = x.shape
    if mask is not None:
        mk = mask.reshape(1, H, W).to(dev).bool()
        x, yv = torch.where(mk, x, 0.0), torch.where(mk, yv, 0.0)
    else:
        mk = torch.ones(1, H, W, dtype=torch.bool, device=dev)
    win = window_2d(dev)[None, None].expand(C, 1, 11, 11).contiguous()
    conv = lambda t: F.conv2d(t[None], win, padding=5, groups=C)[0]
    terms = (x, yv, x * x, yv * yv, x * yv)
    mom = [conv(t) for t in terms]
    err_mom = [24 * U * conv(t.abs()) for t in terms]
    leaves = [m.clone().requires_grad_(True) for m in mom]
    with torch.enable_grad():
        nodes = []
        px = _pixel(*leaves, nodes)
        val, err = {}, {}
        for key in ("S", "d_mu", "d_xx", "d_xy", "B2"):
            gs = torch.autograd.grad(px[key].sum(), leaves + nodes, retain_graph=True, allow_unused=True)
            e = sum(gs[j].abs() * err_mom[j] for j in range(5) if gs[j] is not None)
            e = e + U * sum(g.abs() * v.detach().abs() for g, v in zip(gs[5:], nodes) if g is not None)
            val[key], err[key] = px[key].detach(), e.detach()
    n_el = float(C * H * W)
    cnt = float(mk.sum())
    a, b_, dd = conv(val["d_mu"]), conv(val["d_xx"]), conv(val["d_xy"])
    ea = conv(err["d_mu"]) + 24 * U * conv(val["d_mu"].abs())
    eb = conv(err["d_xx"]) + 24 * U * conv(val["d_xx"].abs())
    ed = conv(err["d_xy"]) + 24 * U * conv(val["d_xy"].abs())
    xo, yo = img.detach().to(F64), gt.detach().to(F64)  # the kernel multiplies by the unmasked x, y (zero gradient off the mask)
    inner = a + 2 * xo * b_ + yo * dd
    mass = a.abs() + 2 * (xo * b_).abs() + (yo * dd).abs()
    cs = w_ssim / n_el
    g_s = cs * inner
    e_s = abs(cs) * (ea + 2 * xo.abs() * eb + yo.abs() * ed + 4 * U * mass) + 3 * U * g_s.abs()
    sgn = torch.sign(xo - yo)
    n_l1 = cnt * C
    g_l = (w_l1 / n_l1) * sgn if n_l1 > 0 else torch.zeros_like(xo)
    grad = torch.where(mk, g_s + g_l, 0.0)
    b_grad = torch.where(mk, e_s + 2 * U * g_l.abs() + U * (g_s + g_l).abs(), 0.0) + torch.where(mk, TINY, 0.0)
    # scalars
    S = val["S"]
    ssim = float(S.sum()) / n_el
    b_ssim = (float(err["S"].sum()) + 6 * U * float(S.abs().sum())) / n_el + U * abs(ssim)
    ad = torch.where(mk, (xo - yo).abs(), 0.0)
    l1 = float(ad.sum()) / n_l1 if n_l1 > 0 else float("nan")
    b_l1 = 7 * U * float(ad.sum()) / n_l1 + U * abs(l1) if n_l1 > 0 else 0.0
    value = (w_l1 * l1 if w_l1 != 0 else 0.0) + w_ssim * ssim  # a weight-0 term is absent: ssim() of an empty mask is 1
    b_value = (abs(w_l1) * b_l1 if w_l1 != 0 else 0.0) + abs(w_ssim) * b_ssim + 2 * U * abs(value)
    return dict(grad=grad, b_grad=b_grad, l1=l1, b_l1=b_l1, ssim=ssim, b_ssim=b_ssim, value=value, b_value=b_value, count=cnt,
                premise=err["B2"] / val["B2"].abs(), S=S, b_S=err["S"])


# ----------------------------------------------------------------------------------------------- Adam
def adam64(p, g, m, v, lr: float, step: int, beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-15) -> Dict[str, torch.Tensor]:
    """One Adam step from the fp32 state (p, g, m, v) in fp64, with beta1, beta2, lr and the bias corrections in double exactly as
    torch.optim.Adam forms them (lr / (1 - beta1^step), sqrt(1 - beta2^step)):
        m' = m + (g - m)(1 - beta1);  v' = beta2 v + (1 - beta2) g^2;  p' = p - lr / bc1 * m' / (sqrt(v') / sqrt(bc2) + eps).
    Bounds (u = 2^-24; the kernel hands 1 - beta1, beta2, 1 - beta2, eps, lr / bc1 and 1 / sqrt(bc2) over as fp32):
      m'   u |m'| (the add) + 3 u (1 - beta1) |g - m| (the difference, the fp32 constant, the product), + 3 2^-149;
      v'   u |v'| + 2 u beta2 |v| + 3 u (1 - beta2) g^2 (a constant and two products), + 4 2^-149;
      p'   the update U = lr/bc1 m'/den, den = sqrt(v') ibc2 + eps: its error relative to itself is 8 u (lr and lr/bc1 to fp32, 1/sqrt(bc2)
           to fp32, sqrt, product, add, division, product) plus what the kernel's own m', v' carry: |U| err(den)/den +
           lr/bc1 err(m')/den with err(den) = ibc2 min(err(v') / (2 sqrt v'), sqrt(err(v'))) + u eps;  then u |p'| for the
           subtraction, + 2^-149."""
    p, g, m, v = (t.detach().to(F64) for t in (p, g, m, v))
    omb1, omb2 = 1.0 - beta1, 1.0 - beta2
    m1 = m + (g - m) * omb1
    v1 = beta2 * v + omb2 * g * g
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    ss, ibc2 = lr / bc1, 1.0 / math.sqrt(bc2)
    den = torch.sqrt(v1) * ibc2 + eps
    upd = ss * m1 / den
    p1 = p - upd
    bm = U * m1.abs() + 3 * U * omb1 * (g - m).abs() + 3 * TINY
    bv = U * v1.abs() + 2 * U * beta2 * v.abs() + 3 * U * omb2 * g * g + 4 * TINY
    sq = torch.sqrt(v1)
    eden = ibc2 * torch.minimum(bv / (2 * sq).clamp(min=1e-300), torch.sqrt(bv)) + U * eps
    bu = 8 * U * upd.abs() + upd.abs() * eden / den + ss * bm / den
    bp = bu + U * p1.abs() + TINY
    return dict(p=p1, m=m1, v=v1, b_p=bp, b_m=bm, b_v=bv)


# ----------------------------------------------------------------------------------------------- densification statistics
def stats64(max_radii2D, grad_accum, denom, radii, grad2d) -> Dict[str, torch.Tensor]:
    """One call of the statistics on ONE model's slice (street_gaussian_model.py:551-571): where radii > 0,
    max_radii2D = max(max_radii2D, radii), grad_accum[:, 0] += |grad2d[:, :2]|, [:, 1] += |grad2d[:, 2]|, denom += 1.
    max_radii2D and denom are exact (a max, and an integer-valued add below 2^24).  grad_accum: the hypot sqrtf(x^2 + y^2) is
    within 3 u of itself (two products and a sum of positives, halved by the root, plus the root) and the add rounds once:
    3 u |hypot| + u |result|, + 2 2^-149."""
    mr, ga, dn = (t.detach().to(F64) for t in (max_radii2D, grad_accum, denom))
    r = radii.to(F64)
    g = grad2d.detach().to(F64)
    vis = radii > 0
    hyp = torch.sqrt(g[:, 0] ** 2 + g[:, 1] ** 2)
    add = torch.stack([hyp, g[:, 2].abs()], 1)
    ga1 = torch.where(vis[:, None], ga.reshape(-1, 2) + add, ga.reshape(-1, 2))
    b = torch.where(vis[:, None], 3 * U * torch.stack([hyp, torch.zeros_like(hyp)], 1) + U * ga1.abs() + 2 * TINY, 0.0)
    return dict(max_radii2D=torch.where(vis, torch.maximum(mr, r), mr), denom=torch.where(vis[:, None], dn.reshape(-1, 1) + 1, dn.reshape(-1, 1)),
                xyz_gradient_accum=ga1, b_xyz_gradient_accum=b)


# ----------------------------------------------------------------------------------------------- sky / object accumulation losses
ACC_LO = float(np.float32(1e-6))                               # the kernel's clamp edges 1e-6f and 1.f - 1e-6f; torch.clamp casts
ACC_HI = float(np.float32(np.float32(1.0) - np.float32(1e-6)))  # min=1e-6, max=1 - 1e-6 to the same two floats
ACC_MAX_BLOCKS = 1056                                           # launch_acc_loss: min(ceil(N / 256), kNumSMs * 8) blocks


def acc_blocks(N: int) -> int:
    return max(1, min(-(-N // 256), ACC_MAX_BLOCKS))


def acc_loss64(kind: str, acc, flag, weight: float) -> Dict[str, torch.Tensor]:
    """kind "sky" (train.py:107-113): mean(flag ? -log(1 - a) : -log(a)); kind "obj" (train.py:114-122): mean(flag ? -(a log a +
    (1 - a) log(1 - a)) : -log(1 - a)); a = clamp(acc, 1e-6, 1 - 1e-6), times weight.  acc fp32, flag bool, any shape.
    Returns grad (dL/dacc, flat), value and their bounds b_grad, b_value; "inside" marks the pixels where the clamp passes the
    gradient (a in [1e-6f, 1 - 1e-6f], inclusive like torch.clamp's backward).  A NaN in acc is kept by the clamp, as torch.clamp
    keeps it: the value is NaN and that pixel's gradient is 0.

    Everything is computed in fp64 from the fp32 acc (the clamp is exact in fp32).  Bounds (u = 2^-24; CUDA's logf is within 1 ulp,
    i.e. 2 u of its result; om = 1 - ac is one fp32 rounding, exact for ac >= 0.5, and log(om (1 + d)) = log(om) + d moves a log by
    at most u absolutely):
      gradient   the kernel forms (weight / (float)N) * deriv:  the fp32 weight, (float)N, the division and the product are 4 u on
                 |grad|; deriv adds  sky: 1 / (1 - ac) 2 u |deriv| (om, the division), -1 / ac  u |deriv|;  obj: logf(om) - logf(ac)
                 2 u (|log om| + |log ac|) + u (om's rounding) + u |deriv| (the subtraction) - absolute, since the two logs cancel
                 near ac = 0.5 -, 1 / om 2 u |deriv|.  Each times |weight| / N; plus 2^-149.
                 The obj entropy bound also covers autograd's order of the same expression, so that the fp32 torch restatement can
                 stand in for the kernel on the CPU: with G the incoming gradient, torch adds -G log ac (3 u |G log ac|), -(G ac) / ac
                 (2 u |G|), G log om (|G| (3 u |log om| + u)) and (G om) / om (2 u |G|), whose +-G cancel, in 3 additions of partial
                 sums up to |G| (|log ac| + |log om| + 2) (3 u each): in all |G| u (6 (|log om| + |log ac|) + 11), which is larger
                 than the kernel's count and is the one used.
      values     per pixel  sky: -logf(om) u + 2 u |v|, -logf(ac) 2 u |v|;  obj: -(ac logf(ac) + om logf(om)) with t1 = ac log ac,
                 t2 = om log om: 3 u |t1| (logf, product) + 4 u |t2| + u om (om's rounding, through both factors of t2) + u |v| (the
                 sum), rounded up to 4 u (|t1| + |t2|) + u om + u |v|;  -logf(om) u + 2 u |v|.
      value      each thread adds its m = ceil(N / (blocks 256)) values in fp32 ((m - 1) u on sum |v|), then 5 shuffle levels (5 u),
                 then fp64 (the 8 warp sums and one atomic per block: (blocks + 8) 2^-53); the mean and weight in fp64 and one
                 rounding to fp32, with the fp32 weight: 2 u |value|."""
    a = acc.detach().reshape(-1).to(F64)
    f = flag.detach().reshape(-1).to(a.device).bool()
    N = a.numel()
    nan = torch.isnan(a)
    ac = torch.where(nan, a, a.clamp(ACC_LO, ACC_HI))
    inside = (a >= ACC_LO) & (a <= ACC_HI)
    om = 1.0 - ac
    la, lo = torch.log(ac), torch.log(om)
    if kind == "sky":
        v = torch.where(f, -lo, -la)
        dv = torch.where(f, 1.0 / om, -1.0 / ac)
        e_v = torch.where(f, U + 2 * U * v.abs(), 2 * U * v.abs())
        e_d = torch.where(f, 2 * U * dv.abs(), U * dv.abs())
    elif kind == "obj":
        t1, t2 = ac * la, om * lo
        v = torch.where(f, -(t1 + t2), -lo)
        dv = torch.where(f, lo - la, 1.0 / om)
        e_v = torch.where(f, 4 * U * (t1.abs() + t2.abs()) + U * om + U * v.abs(), U + 2 * U * v.abs())
        e_d = torch.where(f, 6 * U * (la.abs() + lo.abs()) + 11 * U, 2 * U * dv.abs())
    else:
        raise ValueError(kind)
    c = weight / N
    grad = torch.where(inside, c * dv, 0.0)
    b_grad = torch.where(inside, abs(c) * e_d + 4 * U * grad.abs() + TINY, 0.0)
    blocks = acc_blocks(N)
    m = -(-N // (blocks * 256))
    s_abs = float(v.abs().sum())
    value = weight * float(v.sum()) / N
    b_value = abs(weight) / N * (float(e_v.sum()) + (m - 1 + 5) * U * s_abs + (blocks + 8) * 2.0 ** -53 * s_abs) + 2 * U * abs(value) + TINY
    return dict(grad=grad, b_grad=b_grad, value=value, b_value=b_value, inside=inside, blocks=blocks, terms_per_thread=m)


# ----------------------------------------------------------------------------------------------- LiDAR depth loss
LIDAR_MAX_BLOCKS = 528         # lidar_grid: min(ceil(N / 256), kNumSMs * 4) blocks of contiguous pixel ranges
NAN_KEY = 0x7FC00000           # every NaN key, whatever its bits, as one class above +inf (0x7F800000)


def lidar_grid(N: int):
    """(blocks, chunk): chunk = ceil(tiles / blocks) 256 pixels per block; blocks past ceil(N / chunk) are empty."""
    tiles = -(-N // 256)
    blocks = max(1, min(tiles, LIDAR_MAX_BLOCKS))
    return blocks, -(-tiles // blocks) * 256


def _f32(t):
    return np.ascontiguousarray(t.detach().cpu().reshape(-1).numpy() if torch.is_tensor(t) else np.asarray(t).reshape(-1), np.float32)


def lidar_keys(depth, acc, lidar):
    """err = |depth / (acc + 1e-10f) - lidar| in fp32 (numpy's fp32 add, division and subtraction are IEEE and keep subnormals, as
    the library's build does) and the sort key of each pixel: err's bit pattern, NaN mapped to NAN_KEY.  CUDA writes the canonical NaN
    0x7FFFFFFF and x86 does not, so only NaN-ness, not the bits, is comparable."""
    d, a, l = _f32(depth), _f32(acc), _f32(lidar)
    with np.errstate(all="ignore"):
        b = a + np.float32(1e-10)
        e = d / b
        df = e - l
        err = np.abs(df)
    key = np.where(np.isnan(err), NAN_KEY, err.view(np.uint32).astype(np.int64))
    return dict(b=b, e=e, df=df, err=err, key=key, lidar=l)


def lidar64(depth, acc, lidar, mask, weight: float, keep: float) -> dict:
    """The LiDAR depth loss, weight * mean of the k = int(keep n) smallest err over the n pixels with lidar > 0 and mask.

    Selection: the first k of the valid pixels stably sorted by (key, flat index) - exactly the kernel's radix select with ties taken
    at the lowest flat indices.  value: the fp64 mean of the selected err times the fp32 weight the kernel receives; the kernel sums in
    fp64 (at most k roundings of 2^-53 on a sum of non-negative terms, then the division and the weight) and rounds once to fp32, which
    can be subnormal:  b_value = (u + (k + 2) 2^-53) |value| + 2^-149.
    NaN for k = 0, and for a selected NaN.  Gradients (flat fp32, 0 off the selection) restate lidar_grad_kernel in its own order:
    gk = w32 / (float)k, g = sign(df) gk with sign(0) = sign(NaN) = 0, gd = g / b, ga = -g (e / b); the kernel must match them bit
    for bit."""
    r = lidar_keys(depth, acc, lidar)
    l, key = r["lidar"], r["key"]
    valid = l > 0
    if mask is not None:
        valid &= _f32(mask.to(torch.float32) if torch.is_tensor(mask) else mask) != 0
    n = int(valid.sum())
    k = int(keep * n)
    idx = np.nonzero(valid)[0]
    order = idx[np.argsort(key[idx], kind="stable")]
    sel = np.zeros(key.size, bool)
    sel[order[:k]] = True
    w32 = np.float32(weight)
    gd = np.zeros(key.size, np.float32)
    ga = np.zeros(key.size, np.float32)
    if k:
        t = int(key[order[k - 1]])
        mean = float(r["err"][order[:k]].astype(np.float64).sum()) / k
        value = float(w32) * mean
        gk = w32 / np.float32(k)
        df, b, e = r["df"][sel], r["b"][sel], r["e"][sel]
        sg = np.where(df > 0, np.float32(1), np.where(df < 0, np.float32(-1), np.float32(0))).astype(np.float32)
        g = sg * gk
        with np.errstate(all="ignore"):
            gd[sel] = g / b
            ga[sel] = -g * (e / b)
    else:
        t, value = None, float("nan")
    lt = int((valid & (key < t)).sum()) if k else 0
    ties = int((valid & (key == t)).sum()) if k else 0
    b_value = (U + (k + 2) * 2.0 ** -53) * abs(value) + TINY
    return dict(valid=valid, n=n, k=k, sel=sel, key=key, t=t, lt=lt, ties=ties, take=k - lt, value=value, b_value=b_value, gd=gd, ga=ga,
                err=r["err"], df=r["df"])
