"""Float64 restatement of the three feature operations (street_gaussians_b200.features), differentiable with torch autograd.

    normals64(means3D, rotations, scales, camera_center, col=None, flip=None) -> dict(n, col, flip, dot)
        GaussianModel.get_normals on given rows: the column argmin(scales) of quaternion_to_matrix(rotations) (its own normalisation),
        negated where sum(-d n) < 0 or NaN.  `col` / `flip` impose the decisions instead (to follow a float32 run's choices).
    semantics64(bg, actors, labels, mode) -> [P, K]
    finish64(rendered, normal_channels, mode) -> (normals or None, semantic or None)

Every function takes tensors of any float dtype and computes in the dtype given, so the same lines also serve as the fp32 torch
restatement the end-to-end tests compare against.
"""
from __future__ import annotations

import torch

F64 = torch.float64


def quaternion_to_matrix(r):
    """lib/utils/general_utils.py:125-146, restated."""
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, x, y, z = q.unbind(1)
    rows = [1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
            2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
            2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]
    return torch.stack(rows, 1).reshape(-1, 3, 3)


def normals64(means3D, rotations, scales, camera_center, col=None, flip=None):
    R = quaternion_to_matrix(rotations)
    if col is None:
        col = torch.argmin(scales, dim=-1)
    n = R[torch.arange(R.shape[0], device=R.device), :, col]
    d = means3D - camera_center.reshape(1, 3)
    d = d / d.norm(dim=1, keepdim=True)
    dot = torch.sum(-d * n, dim=1, keepdim=True)
    if flip is None:
        flip = ~(dot >= 0).squeeze(1)
    out = torch.where(flip[:, None], -n, n)
    return dict(n=out, col=col, flip=flip, dot=dot.squeeze(1))


def semantics64(bg, actors, labels, mode):
    """StreetGaussianModel.get_semantic: background rows (softmax in 'probabilities'), then per actor a one-column scatter."""
    rows = [bg if mode == "logits" else torch.softmax(bg, dim=1)]
    K = bg.shape[1]
    for s, lab in zip(actors, labels):
        v = s[:, 0] if mode == "logits" else torch.sigmoid(s[:, 0])
        z = torch.zeros((s.shape[0], K), dtype=s.dtype, device=s.device)
        z = z.index_put((torch.arange(s.shape[0], device=s.device), torch.full((s.shape[0],), int(lab), device=s.device)), v)
        rows.append(z)
    return torch.cat(rows, 0)


def finish64(rendered, normal_channels, mode):
    """render_kernel's split and finishing (street_gaussian_renderer.py:245-264)."""
    normals = semantic = None
    if normal_channels:
        normals = torch.nn.functional.normalize(rendered[:normal_channels], dim=0)
    if rendered.shape[0] > normal_channels:
        semantic = rendered[normal_channels:]
        if mode == "probabilities":
            semantic = semantic / (torch.sum(semantic, dim=0, keepdim=True) + 1e-8)
            semantic = torch.log(semantic + 1e-8)
    return normals, semantic


def grads(fn, inputs, upstream, dtype=F64):
    """(outputs, d(sum outputs * upstream) / d inputs) with fn evaluated on `inputs` cast to `dtype`."""
    xs = [x.detach().to(dtype).requires_grad_(True) for x in inputs]
    outs = fn(*xs)
    outs = outs if isinstance(outs, (tuple, list)) else (outs,)
    loss = sum((o * u.to(dtype)).sum() for o, u in zip(outs, upstream) if o is not None)
    gs = torch.autograd.grad(loss, xs, allow_unused=True)
    return [o.detach() if o is not None else None for o in outs], list(gs)
