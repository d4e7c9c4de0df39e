"""Seeded synthetic street scenes for the parity tests and bench.py (SURVEY.md §8d).

Everything is generated on the CPU with an explicit ``torch.Generator`` so the candidate, the compiled reference
and the CPU oracle all see identical bits.  The camera is built the way the reference's ``Camera`` does
(lib/utils/camera_utils.py:52-61: ``world_view_transform = W2C^T``, ``full_proj_transform = W2C^T @ P^T``,
``P`` from lib/utils/graphics_utils.py:51-70 with znear=0.001, zfar=1000).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch


def projection_matrix(znear: float, zfar: float, tanx: float, tany: float) -> torch.Tensor:
    """Same matrix as lib/utils/graphics_utils.py:51-70 (getProjectionMatrix), parameterised by tan(fov/2)."""
    top, right = tany * znear, tanx * znear
    P = torch.zeros(4, 4, dtype=torch.float32)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def projection_matrix_k(znear: float, zfar: float, fx: float, fy: float, cx: float, cy: float, skew: float, width: int,
                        height: int) -> torch.Tensor:
    """Same matrix as lib/utils/graphics_utils.py:72-94 (getProjectionMatrixK): principal point and skew from K, OpenGL depth row."""
    P = torch.zeros(4, 4, dtype=torch.float32)
    P[0, 0] = 2 * fx / width
    P[0, 1] = 2 * skew / width
    P[0, 2] = -1 + 2 * (cx / width)
    P[1, 1] = 2 * fy / height
    P[1, 2] = -1 + 2 * (cy / height)
    P[2, 2] = (zfar + znear) / (zfar - znear)
    P[2, 3] = -1 * 2 * zfar * znear / (zfar - znear)
    P[3, 2] = 1.0
    return P


def make_camera(width: int, height: int, fovx_deg: float = 50.0, w2c: Optional[torch.Tensor] = None,
                sh_degree: int = 3, bg=(0.0, 0.0, 0.0), scale_modifier: float = 1.0, intrinsics=None) -> Dict:
    """intrinsics = (fx, fy, cx, cy, skew) in pixels: the camera of a Waymo frame (lib/datasets/waymo_full_readers.py:100-102,
    lib/utils/camera_utils.py:52-55, 208-209).  The projection comes from K, while tan(fov / 2) comes from the reader's FoVs,
    which pair fx with the height and fy with the width.  So the rasterizer derives its x focal length from fy and its y focal
    length from fx, as the reference does.  fovx_deg is then unused."""
    if intrinsics is None:
        tanx = math.tan(math.radians(fovx_deg) * 0.5)
        tany = tanx * height / width
    else:
        fx, fy, cx, cy, skew = (float(v) for v in intrinsics)
        focal2fov = lambda focal, pixels: 2 * math.atan(pixels / (2 * focal))  # lib/utils/graphics_utils.py:99-100
        tanx = math.tan(focal2fov(fy, width) * 0.5)
        tany = math.tan(focal2fov(fx, height) * 0.5)
    if w2c is None:
        w2c = torch.eye(4, dtype=torch.float32)
    view_t = w2c.t().contiguous()  # world_view_transform
    proj = (projection_matrix(0.001, 1000.0, tanx, tany) if intrinsics is None else
            projection_matrix_k(0.001, 1000.0, fx, fy, cx, cy, skew, width, height))
    proj_t = proj.t().contiguous()
    full = (view_t.unsqueeze(0).bmm(proj_t.unsqueeze(0))).squeeze(0).contiguous()
    campos = view_t.inverse()[3, :3].contiguous()
    return dict(image_height=int(height), image_width=int(width), tanfovx=tanx, tanfovy=tany,
                bg=torch.tensor(bg, dtype=torch.float32), scale_modifier=float(scale_modifier),
                viewmatrix=view_t, projmatrix=full, sh_degree=int(sh_degree), campos=campos,
                prefiltered=False, debug=False)


def random_pose(gen: torch.Generator, max_angle_deg: float = 8.0, max_shift: float = 0.5) -> torch.Tensor:
    """Small random rigid W2C so view/projection transposition bugs cannot hide behind an identity pose."""
    ax = torch.randn(3, generator=gen)
    ax = ax / ax.norm()
    ang = math.radians(max_angle_deg) * float(torch.rand(1, generator=gen))
    K = torch.tensor([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]], dtype=torch.float32)
    R = torch.eye(3) + math.sin(ang) * K + (1 - math.cos(ang)) * (K @ K)
    w2c = torch.eye(4, dtype=torch.float32)
    w2c[:3, :3] = R
    w2c[:3, 3] = (torch.rand(3, generator=gen) * 2 - 1) * max_shift
    return w2c


def _quat_mul(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def _field(gen, n, tanx, tany, zmin=2.0, zmax=80.0, near_frac=0.02, scale_med=0.05):
    z = torch.exp(torch.rand(n, generator=gen) * (math.log(zmax) - math.log(zmin)) + math.log(zmin))
    n_near = int(n * near_frac)
    if n_near:
        z[:n_near] = torch.rand(n_near, generator=gen) * 0.4 - 0.1  # exercises the z<=0.2 near cull
    x = (torch.rand(n, generator=gen) * 2 - 1) * 1.15 * tanx * z
    y = (torch.rand(n, generator=gen) * 2 - 1) * 1.15 * tany * z
    means = torch.stack([x, y, z], -1)
    log_s = torch.randn(n, 3, generator=gen) * 0.7 + math.log(scale_med)
    scales = torch.exp(log_s).clamp(1e-3, 2.0)
    rot = torch.randn(n, 4, generator=gen)
    rot = rot / rot.norm(dim=-1, keepdim=True)
    opac = torch.sigmoid(torch.randn(n, 1, generator=gen) * 2.0)
    return means, scales, rot, opac


def make_scene(P: int, width: int, height: int, sh_degree: int = 3, seed: int = 0, n_vehicles: int = 0,
               per_vehicle: int = 0, semantics: int = 0, pose: bool = False, fovx_deg: float = 50.0,
               bg=(0.0, 0.0, 0.0), scale_med: float = 0.007, with_raw: bool = False, sh_coeffs: Optional[int] = None,
               intrinsics=None, scale_modifier: float = 1.0) -> Dict:
    """P background Gaussians (+ n_vehicles x per_vehicle posed 'vehicle' clusters, composed the way
    lib/models/street_gaussian_model.py:335-363 does: x_world = R_obj x_local + t_obj, q_world = q_obj * q_local).
    with_raw: also return out["raw"] = dict(models=[background, vehicle_0, ...] of RAW parameters (local frame, log scale, logit
    opacity, features_dc / features_rest split; the layout street_gaussians_b200.compose consumes), poses [n_vehicles, 7], idft
    [n_vehicles, 1]) whose composition reproduces the composed arrays above up to fp32 rounding.
    sh_coeffs: coefficients stored per Gaussian (default (sh_degree + 1)^2, as many as the active degree evaluates; more is what a
    model trained towards a higher degree holds before it gets there).  intrinsics, scale_modifier: see make_camera."""
    gen = torch.Generator().manual_seed(seed)
    w2c = random_pose(gen) if pose else None
    cam = make_camera(width, height, fovx_deg, w2c, sh_degree, bg, scale_modifier, intrinsics)
    tanx, tany = cam["tanfovx"], cam["tanfovy"]
    means, scales, rot, opac = _field(gen, P, tanx, tany, scale_med=scale_med)
    raw_local, raw_pose = [], []
    if n_vehicles and per_vehicle:
        ms, ss, rs, os_ = [means], [scales], [rot], [opac]
        for v in range(n_vehicles):
            depth = 8.0 + 32.0 * float(torch.rand(1, generator=gen))
            cx = (float(torch.rand(1, generator=gen)) * 2 - 1) * 0.8 * tanx * depth
            cy = 0.15 * tany * depth
            yaw = float(torch.rand(1, generator=gen)) * 2 * math.pi
            q_obj = torch.tensor([math.cos(yaw / 2), 0.0, math.sin(yaw / 2), 0.0])  # yaw about the camera's y axis
            Rm = torch.tensor([[math.cos(yaw), 0, math.sin(yaw)], [0, 1, 0], [-math.sin(yaw), 0, math.cos(yaw)]],
                              dtype=torch.float32)
            local = (torch.rand(per_vehicle, 3, generator=gen) - 0.5) * torch.tensor([4.5, 1.6, 2.0])
            m = local @ Rm.t() + torch.tensor([cx, cy, depth])
            s = torch.exp(torch.randn(per_vehicle, 3, generator=gen) * 0.5 + math.log(0.03)).clamp(1e-3, 0.5)
            q = torch.randn(per_vehicle, 4, generator=gen)
            raw_local.append((local, q.clone()))
            raw_pose.append(torch.cat([q_obj, torch.tensor([cx, cy, depth])]))
            q = _quat_mul(q_obj.expand_as(q), q / q.norm(dim=-1, keepdim=True))
            q = q / q.norm(dim=-1, keepdim=True)
            o = torch.sigmoid(torch.randn(per_vehicle, 1, generator=gen) * 2.0 + 1.0)
            ms.append(m); ss.append(s); rs.append(q); os_.append(o)
        means, scales, rot, opac = torch.cat(ms), torch.cat(ss), torch.cat(rs), torch.cat(os_)
    n = means.shape[0]
    if w2c is not None:  # express the field in world coordinates so that W2C brings it back in front of the camera
        c2w = torch.linalg.inv(w2c)
        means = means @ c2w[:3, :3].t() + c2w[:3, 3]
    M = (sh_degree + 1) ** 2 if sh_coeffs is None else int(sh_coeffs)
    shs = torch.randn(n, M, 3, generator=gen) * 0.2
    shs[:, 0, :] = torch.randn(n, 3, generator=gen)
    out = dict(cam=cam, means3D=means.float().contiguous(), scales=scales.float().contiguous(),
               rotations=rot.float().contiguous(), opacities=opac.float().contiguous(), shs=shs.float().contiguous())
    if with_raw:
        if w2c is not None:
            raise ValueError("with_raw needs pose=False (the raw actor frames are expressed in the identity-camera world)")
        bounds = [0, P] + [P + (v + 1) * per_vehicle for v in range(len(raw_local))]
        models = []
        for k in range(len(bounds) - 1):
            lo, hi = bounds[k], bounds[k + 1]
            xyz_k, rot_k = (means[lo:hi], rot[lo:hi]) if k == 0 else raw_local[k - 1]
            models.append(dict(xyz=xyz_k.float().contiguous(), rotation=rot_k.float().contiguous(), scaling=torch.log(scales[lo:hi]).float().contiguous(),
                               opacity=torch.logit(opac[lo:hi].double().clamp(1e-7, 1 - 1e-7)).float().contiguous(),
                               features_dc=shs[lo:hi, 0:1].float().contiguous(), features_rest=shs[lo:hi, 1:].float().contiguous()))
        out["raw"] = dict(models=models, poses=torch.stack(raw_pose).float() if raw_pose else torch.zeros(0, 7),
                          idft=torch.ones(len(raw_pose), 1))
    if semantics:
        out["semantics"] = torch.rand(n, semantics, generator=gen).float().contiguous()
    npx = width * height
    out["grad_color"] = (torch.randn(3, height, width, generator=gen) / npx).float()
    out["grad_depth"] = (torch.randn(1, height, width, generator=gen) / npx).float()
    out["grad_alpha"] = (torch.randn(1, height, width, generator=gen) / npx).float()
    if semantics:
        out["grad_semantic"] = (torch.randn(semantics, height, width, generator=gen) / npx).float()
    return out


def smoke_script_scene(num_points: int = 10000, width: int = 1242, height: int = 375, seed: int = 0, semantics: int = 0) -> Dict:
    """Replays script/test_gaussian_rasterization.py:6-52 (its own camera constants, U[0,1) inputs, rotations with w=1
    left un-normalised), but seeded."""
    gen = torch.Generator().manual_seed(seed)
    view = torch.tensor([[0.9598, 0.0081, 0.2806, 0.0], [-0.0123, 0.9998, 0.0134, 0.0], [-0.2804, -0.0163, 0.9597, 0.0],
                         [-2.0954, -0.0935, 4.9320, 1.0]])
    proj = torch.tensor([[1.1205, 0.0312, 0.2806, 0.2806], [-0.0144, 3.8661, 0.0134, 0.0134],
                         [-0.3274, -0.0632, 0.9598, 0.9597], [-2.4464, -0.3614, 4.9225, 4.9320]])
    cam = dict(image_height=height, image_width=width, tanfovx=math.tan(1.416 * 0.5), tanfovy=math.tan(0.506 * 0.5),
               bg=torch.zeros(3), scale_modifier=1.0, viewmatrix=view, projmatrix=proj, sh_degree=0,
               campos=torch.tensor([6.2808e-01, 1.4572e-03, -5.3226e+00]), prefiltered=False, debug=False)
    r = lambda *s: torch.rand(*s, generator=gen)
    rot = r(num_points, 4)
    rot[:, 0] = 1
    out = dict(cam=cam, means3D=r(num_points, 3), shs=r(num_points, 4, 3), opacities=r(num_points, 1), scales=r(num_points, 3),
               rotations=rot)
    if semantics:
        out["semantics"] = r(num_points, semantics)
    npx = width * height
    out["grad_color"] = torch.randn(3, height, width, generator=gen) / npx
    out["grad_depth"] = torch.randn(1, height, width, generator=gen) / npx
    out["grad_alpha"] = torch.randn(1, height, width, generator=gen) / npx
    if semantics:
        out["grad_semantic"] = torch.randn(semantics, height, width, generator=gen) / npx
    return out


# The BASELINE.json configs (BASELINE.md §2 table).
CONFIGS = {
    "A": dict(kind="smoke", num_points=10000, width=256, height=256),
    "A_native": dict(kind="smoke", num_points=10000, width=1242, height=375),
    "B": dict(kind="scene", P=500_000, width=1920, height=1280, sh_degree=3),
    "C": dict(kind="scene", P=1_500_000, width=1920, height=1280, sh_degree=3, n_vehicles=8, per_vehicle=50_000),
    "E": dict(kind="scene", P=8_000_000, width=3840, height=2160, sh_degree=3),
}


def make_config(name: str, seed: int = 0, **over) -> Dict:
    cfg = dict(CONFIGS[name]); cfg.update(over)
    kind = cfg.pop("kind")
    if kind == "smoke":
        return smoke_script_scene(seed=seed, **cfg)
    return make_scene(seed=seed, **cfg)
