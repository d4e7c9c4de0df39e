"""Torch and float64 restatements of the reference's background pose correction and colour correction — TEST INFRASTRUCTURE.

  compose       oracle/compose_oracle.compose plus the pose correction of the background, as the reference applies it:
                lib/models/camera_pose.py:89-104 correct_gaussian_xyz ([xyz, 1] @ [[R, t], [0, 0, 0, 1]]^T with
                R = quaternion_to_matrix(F.normalize(q))), :106-114 correct_gaussian_rotation (F.normalize(q) (x) rotation, with no final
                normalisation), called from lib/models/street_gaussian_model.py:311-312, 340-341.
  color / reg   lib/models/color_correction.py:129-132 (einsum + bias) and :134-140 (mean |A - I| + |A_sky - I|).
  compose64     oracle/step64.compose64 with the correction: values by fp64 autograd of `compose`, the correction's gradient also in
                closed form (the finalize kernel's chain), and per-element bounds for the background rows and the correction.
  color64       the colour correction in fp64 in closed form with per-element bounds; reg64 likewise for the regularisation.

Pinned by tests/golden/callsite/correction_sh{1,3}.npz (tests/golden/make_correction_golden.py runs the reference's own code).
Bounds follow oracle/step64.py's conventions: u = 2^-24, first order, each constant a count of roundings derived below.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle import compose_oracle as CO
from oracle import step64 as S64

F64 = torch.float64
U, TINY = S64.U, S64.TINY
NAMES = ("xyz", "rotation", "scaling", "opacity", "features")
KCC_THREADS, KCC_MAX_BLOCKS = 256, 4 * 132  # csrc/corrections.cu: block size and grid cap


def compose(models, poses, idft, flip, flip_quat, correction: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
    """compose_oracle.compose, then the background rows moved by correction = (rot [4], trans [3]) like the reference."""
    out = CO.compose(models, poses, idft, flip, flip_quat)
    if correction is None:
        return out
    rot, trans = correction
    bk = models[0]
    nb = bk["xyz"].shape[0]
    q = F.normalize(rot.unsqueeze(0), dim=-1)                                                          # camera_pose.py:95-96
    R = CO.quat_to_matrix(q)[0]
    Mx = torch.cat([torch.cat([R, trans[:, None]], -1), torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=R.dtype, device=R.device)], 0)
    xyz_b = (torch.cat([bk["xyz"], torch.ones_like(bk["xyz"][..., :1])], -1) @ Mx.T)[:, :3]           # :100-102
    rot_b = CO.quat_mul(q.expand(nb, 4), F.normalize(bk["rotation"]))                                  # :110-111
    out = dict(out)
    out["xyz"] = torch.cat([xyz_b, out["xyz"][nb:]])
    out["rotation"] = torch.cat([rot_b, out["rotation"][nb:]])
    return out


def color(image, affine):
    """color_correction.py:131: einsum('ij, jhw -> ihw', A[:3, :3], image) + A[:3, 3]."""
    return torch.einsum("ij, jhw -> ihw", affine[:3, :3], image) + affine[:3, 3].unsqueeze(-1).unsqueeze(-1)


def reg(affine, affine_sky=None, weight: float = 1.0):
    """weight * mean(|A - I| + |A_sky - I|) (color_correction.py:134-140; train.py:135-138 multiplies by the weight)."""
    eye = torch.eye(4, dtype=affine.dtype, device=affine.device)[:3]
    t = torch.abs(affine - eye)
    if affine_sky is not None:
        t = t + torch.abs(affine_sky - eye)
    return weight * t.mean()


def dcorrection_closed_form(q_raw, G, ga_sum, gx_sum):
    """The finalize kernel's chain in fp64: G = sum g (x) x [3, 3], ga_sum = sum g_rot (x) conj(n) [4] (d / d q-hat),
    gx_sum = sum g_xyz [3].  d/d q_raw through F.normalize, then quaternion_to_matrix's own normalisation on the matrix path."""
    qh = q_raw / q_raw.norm().clamp(min=1e-12)
    u = qh / qh.norm()
    D = torch.autograd.functional.jacobian(S64._rot_poly, u)             # [9, 4] = dR/du
    du = (D * G.reshape(9, 1)).sum(0)
    dqh = ga_sum + (du - u * (u * du).sum()) / qh.norm()
    n = q_raw.norm()
    dq = (dqh - qh * (qh * dqh).sum()) / n if n >= 1e-12 else dqh / 1e-12
    return torch.cat([dq, gx_sum])


def compose64(models: Sequence[dict], poses, idft, flip, flip_quat, up: dict, correction) -> Dict[str, torch.Tensor]:
    """step64.compose64 with the pose correction (rot [4], trans [3]) on the background.  Returns the values of every output and raw
    gradient, "dcorrection" [7] by autograd and "dcorrection_closed" by the finalize kernel's chain, and "b_" + name bounds.

    Actor rows and their pose gradients are untouched by the correction: their bounds are step64.compose64's.  Background rows
    (u = 2^-24, nb background Gaussians):
      q-hat = c / max(|c|, 1e-12): 3 u in the norm (a common scale that quaternion_to_matrix's second normalisation removes) and
             1 u per component from the division, so R carries at most 16 u + 8 u of the direction error: |dR_ij| <= 24 u.
      xyz    u (24 sum_j |x_j| + 6 (sum_j |R_ij x_j| + |t_i|)) — the actor formula with 24 for 16.
      rot    q-hat (x) n, not normalised: q-hat 6 u, n 6 u (step64's unposed bound), 4 roundings of the product:
             16 u (|q-hat| (x) |n|)_k.
      g_xyz  R^T g: u (24 sum_j |g_j| + 6 sum_j |R_ji g_j|).
      g_rot  gb = conj(q-hat) (x) g (4 roundings on |q-hat| (x) |g|, 6 u from q-hat), then step64's unposed chain (K = 32) on gb:
             K = 48 on M_k = (M(gb)_k + |n_k| sum_j |n_j| M(gb)_j) / |raw| with M(gb) = |q-hat| (x) |g|.
      dcorrection  the per-row terms ga = g (x) conj(n) (4 roundings, n's 6 u: 10 u), the 9 products g (x) x (1 u) and g itself are
             summed by warp trees and float atomics: (5 + n_atom) u sum |term|, n_atom = nb / 32 + 66.  The matrix part goes through
             step64's linear map c at q-hat (16 roundings, plus 8 u from q-hat's error).  That gives a bound B_k on d/d q-hat and a
             magnitude S_k.  F.normalize's backward (g - q-hat (q-hat . g)) / |c| propagates B with the projection's mass and adds
             8 roundings on the mass of S:
               k < 4: ((B_k + |qh_k| sum_j |qh_j| B_j) + 8 u (S_k + |qh_k| sum_j |qh_j| S_j)) / |c|;  translation (5 + n_atom) u sum |g_xyz|.
    """
    A = len(models) - 1
    base = S64.compose64(models, poses, idft, flip, flip_quat, up)
    dev = models[0]["xyz"].device
    d = lambda t: t.detach().to(dev, F64)
    m64 = [{k: d(v).requires_grad_(True) for k, v in m.items()} for m in models]
    p64 = d(poses).requires_grad_(True) if A else torch.zeros(0, 7, dtype=F64, device=dev)
    i64 = d(idft) if A else torch.zeros(0, 1, dtype=F64, device=dev)
    fq = d(flip_quat) if flip_quat is not None else torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=F64, device=dev)
    fl = flip.to(dev).bool() if flip is not None else None
    cr, ct = d(correction[0]).requires_grad_(True), d(correction[1]).requires_grad_(True)
    out = compose(m64, p64, i64, fl, fq, (cr, ct))
    res = {k: out[k].detach() for k in NAMES}
    ins = [m[k] for m in m64 for k in S64.KEYS] + [cr, ct] + ([p64] if A else [])
    grads = torch.autograd.grad([out[k] for k in NAMES], ins, [d(up[k]) for k in NAMES], allow_unused=True)
    for i, m in enumerate(m64):
        for j, k in enumerate(S64.KEYS):
            g = grads[i * 6 + j]
            res[f"g{i}_{k}"] = g if g is not None else torch.zeros_like(m[k])
    nk = len(m64) * 6
    res["dcorrection"] = torch.cat([grads[nk], grads[nk + 1]])
    if A:
        res["dposes"] = grads[nk + 2]
    for k, v in base.items():
        if k.startswith("b_"):
            res[k] = v.clone()

    nb = int(models[0]["xyz"].shape[0])
    x, r_raw = d(models[0]["xyz"]), d(models[0]["rotation"])
    gx, gq = d(up["xyz"])[:nb], d(up["rotation"])[:nb]
    c = d(correction[0])
    qh = c / c.norm().clamp(min=1e-12)
    R = S64._rot_poly(qh / qh.norm()).reshape(3, 3)
    rn = r_raw.norm(dim=1, keepdim=True).clamp(min=1e-12)
    n = r_raw / rn
    qhe = qh.expand(nb, 4)
    res["b_xyz"][:nb] = U * (24 * x.abs().sum(1, keepdim=True) + 6 * ((R.abs()[None] * x.abs()[:, None, :]).sum(2) + d(correction[1]).abs()))
    res["b_rotation"][:nb] = 16 * U * S64._absmul(qhe, n) + TINY
    res["b_g0_xyz"] = U * (24 * gx.abs().sum(1, keepdim=True) + 6 * (R.abs()[None] * gx.abs()[:, :, None]).sum(1))
    m_gb = S64._absmul(qhe, gq)
    m_out = (m_gb + n.abs() * (n.abs() * m_gb).sum(1, keepdim=True)) / rn
    res["b_g0_rotation"] = 48 * U * m_out + TINY
    # the correction's gradient, closed form and bound
    ga = CO.quat_mul(gq, n * torch.tensor([1.0, -1.0, -1.0, -1.0], dtype=F64, device=dev))
    G = (gx[:, :, None] * x[:, None, :]).sum(0)
    res["dcorrection_closed"] = dcorrection_closed_form(c, G, ga.sum(0), gx.sum(0))
    n_atom = nb // 32 + 66
    s_ga, s_mga = ga.abs().sum(0), (10 * S64._absmul(gq.abs(), n.abs())).sum(0)
    s_G = (gx.abs()[:, :, None] * x.abs()[:, None, :]).sum(0).reshape(9)
    u_ = qh / qh.norm()
    D = torch.autograd.functional.jacobian(S64._rot_poly, u_).T  # [4, 9]
    cabs = (D.abs() + u_.abs()[:, None] * (u_.abs()[:, None] * D.abs()).sum(0, keepdim=True)) / qh.norm()
    cg = (cabs * s_G[None]).sum(1)
    B = U * ((7 + n_atom) * s_ga + s_mga + (30 + n_atom) * cg)
    S = s_ga + cg
    proj = lambda v: v + qh.abs() * (qh.abs() * v).sum()
    bq = (proj(B) + 8 * U * proj(S)) / c.norm()
    bt = (5 + n_atom) * U * gx.abs().sum(0)
    res["b_dcorrection"] = torch.cat([bq, bt]) + TINY
    return res


def cc_blocks(N: int) -> Tuple[int, int]:
    """(blocks, pixels per thread at most) of the colour-correction backward for N = H * W on 16-byte aligned tensors."""
    vec = N % 4 == 0
    items = N // 4 if vec else N
    blocks = max(1, min(-(-items // KCC_THREADS), KCC_MAX_BLOCKS))
    per = -(-items // (blocks * KCC_THREADS)) * (4 if vec else 1)
    return blocks, per


def color64(image, affine, g) -> Dict[str, torch.Tensor]:
    """Closed-form fp64 colour correction of the fp32 image [3, H, W] and affine [3, 4], and its backward for the upstream g.

    Bounds (u = 2^-24):
      out      the kernel forms a0 x0, adds a1 x1 and a2 x2 with two FMAs and then the bias: 4 roundings, each at most u times the
               sum of the magnitudes it has seen, so 4 u (sum_j |a_ij x_j| + |b_i|).  A GEMM in any order with a separate bias add
               (torch's einsum) has at most as many.
      dimage   A^T g the same way without a bias: 3 u sum_i |a_ij g_i|.
      daffine  sum over pixels of g_i [x_j, 1]: each thread adds its pixels (at most `per`, cc_blocks) sequentially, a 5-level warp
               butterfly and 7 sequential adds of the block's warps follow, the blocks are added in double and rounded once:
               (per + 12) u sum |g_i x_j| + u |v|.
    """
    x, A, gg = image.detach().to(F64), affine.detach().to(F64), g.detach().to(F64)
    N = x.shape[1] * x.shape[2]
    xf, gf = x.reshape(3, N), gg.reshape(3, N)
    out = A[:, :3] @ xf + A[:, 3:]
    b_out = 4 * U * ((A[:, :3].abs() @ xf.abs()) + A[:, 3:].abs()) + TINY
    dimage = A[:, :3].T @ gf
    b_dimage = 3 * U * (A[:, :3].abs().T @ gf.abs()) + TINY
    xa = torch.cat([xf, torch.ones(1, N, dtype=F64, device=xf.device)])
    dA = gf @ xa.T
    _, per = cc_blocks(N)
    b_dA = (per + 12) * U * (gf.abs() @ xa.abs().T) + U * dA.abs() + TINY
    shp = x.shape
    return dict(out=out.reshape(shp), b_out=b_out.reshape(shp), dimage=dimage.reshape(shp), b_dimage=b_dimage.reshape(shp), daffine=dA,
                b_daffine=b_dA)


def reg64(affine, affine_sky, weight: float) -> Dict[str, torch.Tensor]:
    """Closed-form regularisation.  value: 12 (or 24) differences from I (1 u each), a butterfly of 5 levels, the division by 12 and
    the product with the weight: 9 u |weight| sum |d| / 12.  Gradients sign(d) * fl(weight / 12): 1 u of |weight| / 12, exact 0 at d = 0."""
    eye = torch.eye(4, dtype=F64)[:3].to(affine.device)
    dA = affine.detach().to(F64) - eye
    dS = affine_sky.detach().to(F64) - eye if affine_sky is not None else torch.zeros_like(dA)
    tot = dA.abs().sum() + dS.abs().sum()
    gw = weight / 12.0
    return dict(value=weight * tot / 12.0, b_value=9 * U * abs(weight) * tot / 12.0 + TINY, g_affine=torch.sign(dA) * gw,
                g_affine_sky=torch.sign(dS) * gw, b_g=U * abs(gw) + TINY)
