"""Torch restatement of the reference's densification and opacity reset, per sub-model, with the normal draws given per parent.

Test-only code (the product never imports oracle/).  It follows the reference line by line so that, on the CPU, it reproduces the
reference's outputs bit for bit when fed the same draws:
  * GaussianModelBkgd.densify_and_prune   lib/models/gaussian_model_bkgd.py:74-114
  * GaussianModelActor.densify_and_prune  lib/models/gaussian_model_actor.py:204-261
  * densify_and_clone / densify_and_split / prune_points / densification_postfix / cat_optimizer / prune_optimizer
                                          lib/models/gaussian_model.py:363-408, 416-520
  * reset_opacity / reset_optimizer       lib/models/gaussian_model.py:344-361, 410-414
  * quaternion_to_matrix                  lib/utils/general_utils.py:125-146

Draws: `draws[n, 18]` per parent, the layout the CUDA kernel uses: [0:3] child 0, [3:6] child 1 of a split parent,
[6 + 3 (2 r + j) : +3] box sample j of row slot r (slot 0: the parent itself or child 0; slot 1: its clone or child 1).
`reference_draws_to_layout` / `layout_to_reference_draws` convert from / to the order in which the reference calls torch.normal.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic")
SCALARS = ("points_total", "points_clone", "points_split", "points_below_min_opacity", "points_big_ws", "points_pruned")
DRAWS = 18


def quaternion_to_matrix(r):
    """general_utils.py:125-146, with the output on r's device."""
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    R = torch.zeros((q.size(0), 3, 3), device=r.device, dtype=r.dtype)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - r * z)
    R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y)
    R[:, 2, 1] = 2 * (y * z + r * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def decisions(t, grad_col, grad_threshold, extent, percent_dense):
    """The gradient and the clone / split masks of the parents (gaussian_model.py:462-464, 497-499; the caller's grads)."""
    grads = t["xyz_gradient_accum"][:, grad_col:grad_col + 1] / t["denom"]
    grads[grads.isnan()] = 0.0
    smax = torch.max(torch.exp(t["scaling"]), dim=1).values
    clone = torch.logical_and(torch.norm(grads, dim=-1) >= grad_threshold, smax <= percent_dense * extent)
    split = torch.logical_and(grads.squeeze(-1) >= grad_threshold, smax > percent_dense * extent)
    return grads, clone, split


def row_parents(clone, split):
    """Parent and slot of every row of [originals not split, clones, child 0 of each split parent, child 1 of each]."""
    idx = torch.arange(clone.shape[0], device=clone.device)
    keep, cl, sp = idx[~split], idx[clone], idx[split]
    parent = torch.cat([keep, cl, sp, sp])
    slot = torch.cat([torch.zeros_like(keep), torch.ones_like(cl), torch.zeros_like(sp), torch.ones_like(sp)])
    section = torch.cat([torch.full_like(keep, 0), torch.full_like(cl, 1), torch.full_like(sp, 2), torch.full_like(sp, 3)])
    return parent, slot, section


def layout_to_reference_draws(draws, clone, split, actor_box):
    """The per-parent layout -> (z_split [2s,3], z_box [rows,2,3] or None) in the order the reference draws them."""
    sp = split.nonzero().squeeze(-1)
    z_split = torch.cat([draws[sp, 0:3], draws[sp, 3:6]])
    if not actor_box:
        return z_split, None
    parent, slot, _ = row_parents(clone, split)
    cols = 6 + 6 * slot[:, None] + torch.arange(6, device=draws.device)[None]
    return z_split, draws[parent[:, None], cols].view(-1, 2, 3)


def reference_draws_to_layout(n, z_split, z_box, clone, split):
    draws = torch.zeros(n, DRAWS, dtype=z_split.dtype, device=z_split.device)
    sp = split.nonzero().squeeze(-1)
    s = sp.numel()
    draws[sp, 0:3] = z_split[:s]
    draws[sp, 3:6] = z_split[s:]
    if z_box is not None:
        parent, slot, _ = row_parents(clone, split)
        cols = 6 + 6 * slot[:, None] + torch.arange(6, device=draws.device)[None]
        draws[parent[:, None], cols] = z_box.reshape(-1, 6)
    return draws


def densify_model(t, kind, draws, *, grad_threshold, grad_col, extent, percent_dense, percent_big_ws, min_opacity, prune_big_points,
                  sphere_center=None, sphere_radius=None, min_xyz=None, max_xyz=None):
    """One sub-model.  t: {name: tensor} for NAMES, "exp_avg" / "exp_avg_sq": {name: tensor or None}, "xyz_gradient_accum", "denom".
    extent / sphere_radius: fp32 tensors [1] as the reference keeps them; grad_threshold / percent_* / min_opacity: Python floats.
    Returns the new tensors (same keys), the scalar dict, the per-parent 4-bit section mask, and each output row's parent and section."""
    n = t["xyz"].shape[0]
    _, clone, split = decisions(t, grad_col, grad_threshold, extent, percent_dense)
    actor = kind == "actor"
    z_split, z_box = layout_to_reference_draws(draws, clone, split, actor and prune_big_points)
    sel = split
    N = 2
    # densify_and_split (gaussian_model.py:469-479); torch.normal(mean, std) = mean + z * std
    get_scaling = torch.exp(t["scaling"])
    stds = get_scaling[sel].repeat(N, 1)
    means = torch.zeros((stds.size(0), 3), device=stds.device)
    samples = means + z_split * stds
    rots = quaternion_to_matrix(t["rotation"][sel]).repeat(N, 1, 1)
    child = {k: t[k][sel].repeat(N, *([1] * (t[k].dim() - 1))) for k in NAMES}
    child["xyz"] = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + t["xyz"][sel].repeat(N, 1)
    child["scaling"] = torch.log(get_scaling[sel].repeat(N, 1) / (0.8 * N))
    rows = {k: torch.cat([t[k][~split], t[k][clone], child[k]]) for k in NAMES}
    zero_new = int(clone.sum()) + N * int(sel.sum())
    moments = {}
    for mk in ("exp_avg", "exp_avg_sq"):
        moments[mk] = {k: (None if t[mk][k] is None else
                           torch.cat([t[mk][k][~split], torch.zeros((zero_new,) + tuple(t[mk][k].shape[1:]), dtype=t[mk][k].dtype,
                                                                    device=t[mk][k].device)])) for k in NAMES}
    # prune (gaussian_model_bkgd.py:90-105 / gaussian_model_actor.py:222-252)
    opacity = torch.sigmoid(rows["opacity"])
    prune_mask = (opacity < min_opacity).squeeze(-1)
    scalars = dict(points_total=n, points_clone=int(clone.sum()), points_split=int(split.sum()), points_below_min_opacity=int(prune_mask.sum()))
    scaling_r = torch.exp(rows["scaling"])
    if prune_big_points:
        big = scaling_r.max(dim=1).values > extent * percent_big_ws
        if not actor:
            dists = torch.linalg.norm(rows["xyz"] - sphere_center, dim=1)
            big[dists > 2 * sphere_radius] = False
            prune_mask = torch.logical_or(prune_mask, big)
        else:
            stds_b = scaling_r[:, None, :].expand(-1, 2, -1)
            samples_b = torch.zeros_like(rows["xyz"])[:, None, :].expand(-1, 2, -1) + z_box * stds_b
            rots_b = quaternion_to_matrix(F.normalize(rows["rotation"]))[:, None, :, :].expand(-1, 2, -1, -1)
            sxyz = torch.matmul(rots_b, samples_b.unsqueeze(-1)).squeeze(-1) + rows["xyz"][:, None, :].expand(-1, 2, -1)
            m = rows["xyz"].shape[0]
            # .view(m, -1) as in the reference, spelt (m, 6) so that an empty model does not fail
            inside = torch.logical_and(torch.all((sxyz >= min_xyz).view(m, 6), dim=-1), torch.all((sxyz <= max_xyz).view(m, 6), dim=-1))
            prune_mask = torch.logical_or(torch.logical_or(prune_mask, big), ~inside)
        scalars["points_big_ws"] = int(big.sum())
    scalars["points_pruned"] = int(prune_mask.sum())
    valid = ~prune_mask
    out = {k: rows[k][valid] for k in NAMES}
    for mk in ("exp_avg", "exp_avg_sq"):
        out[mk] = {k: (None if v is None else v[valid]) for k, v in moments[mk].items()}
    n_new = out["xyz"].shape[0]
    dev = t["xyz"].device
    out["xyz_gradient_accum"] = torch.zeros((n_new, 2), device=dev)
    out["denom"] = torch.zeros((n_new, 1), device=dev)
    out["max_radii2D"] = torch.zeros((n_new,), device=dev)
    parent, _, section = row_parents(clone, split)
    mask = torch.zeros(n, dtype=torch.int64, device=dev)
    mask.index_add_(0, parent[valid], (1 << section[valid]))
    return out, scalars, mask, parent[valid], section[valid]


def reset_opacity(opacity):
    """gaussian_model.py:410-414: inverse_sigmoid(min(sigmoid(o), 0.01)); the caller zeroes the opacity moments."""
    p = torch.min(torch.sigmoid(opacity), torch.ones_like(opacity) * 0.01)
    return torch.log(p / (1 - p))


def margins(t, kind, draws, *, grad_threshold, grad_col, extent, percent_dense, percent_big_ws, min_opacity, prune_big_points,
            sphere_center=None, sphere_radius=None, min_xyz=None, max_xyz=None):
    """Smallest relative margin, in fp64, of every discrete decision a parent's rows depend on: |g| and g against the gradient
    threshold, the max scale against the dense and big thresholds, sigmoid(opacity) against min_opacity, the distance against
    2 r, and every box coordinate against its face.  fp32 code may decide a parent differently only where this is tiny."""
    d = lambda v: torch.as_tensor(v).double().to(t["xyz"].device)
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))
    ext = float(extent.reshape(-1)[0])
    dense_thr, big_thr, g_thr, op_thr = f32(f32(percent_dense) * ext), f32(f32(percent_big_ws) * ext), f32(grad_threshold), f32(min_opacity)
    rel = lambda a, b: (a - b).abs() / torch.maximum(a.abs(), torch.full_like(a, abs(b))).clamp_min(1e-300)
    g = d(t["xyz_gradient_accum"][:, grad_col]) / d(t["denom"][:, 0])
    g = torch.where(torch.isnan(g), torch.zeros_like(g), g)
    s = torch.exp(d(t["scaling"]))
    smax = s.max(dim=1).values
    marg = torch.minimum(rel(g.abs(), g_thr), rel(smax, dense_thr))
    sig = torch.sigmoid(d(t["opacity"][:, 0]))
    marg = torch.minimum(marg, rel(sig, op_thr))
    if not prune_big_points:
        return marg
    _, clone, split = decisions(t, grad_col, grad_threshold, extent, percent_dense)
    child_s = torch.exp(torch.log(s / 1.6))
    marg = torch.minimum(marg, torch.minimum(rel(smax, big_thr), rel(child_s.max(dim=1).values, big_thr)))
    q = d(t["rotation"])
    R = quaternion_to_matrix(q)
    x = d(t["xyz"])
    z = d(draws)
    rows = [(x, s, 0, None)]
    for c in range(2):
        xc = torch.bmm(R, (z[:, 3 * c:3 * c + 3] * s)[..., None])[..., 0] + x
        rows.append((xc, child_s, c, c))
    if kind != "actor":
        c2 = 2 * float(torch.as_tensor(sphere_radius).reshape(-1)[0])
        for xr, _, _, _ in rows:
            marg = torch.minimum(marg, rel(torch.linalg.norm(xr - d(sphere_center), dim=1), c2))
        return marg
    Rn = quaternion_to_matrix(F.normalize(q))
    lo, hi = d(min_xyz).reshape(-1), d(max_xyz).reshape(-1)
    for xr, sr, slot, ch in rows:
        slots = (0, 1) if ch is None else (slot,)
        for sl in slots:
            for j in range(2):
                zz = z[:, 6 + 3 * (2 * sl + j):9 + 3 * (2 * sl + j)]
                y = torch.bmm(Rn, (zz * sr)[..., None])[..., 0] + xr
                for a in range(3):
                    marg = torch.minimum(marg, torch.minimum(rel(y[:, a], float(lo[a])), rel(y[:, a], float(hi[a]))))
    return marg
