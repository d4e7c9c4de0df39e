"""The cameras of the posed / intrinsics tier of the fp64 per-element checks (tests/test_camera64_*.py).

The other per-element scenes render through the identity view of a centred, square-pixel camera: every off-diagonal entry of the
view and projection matrices the kernels read is zero there, and the rasterizer's two focal lengths are the same number.  A
Waymo frame differs in all of these points (lib/datasets/waymo_full_readers.py:100-102, lib/utils/camera_utils.py:52-55, 208-209):
  * the projection comes from K (principal point off centre, skew, OpenGL depth row);
  * tan(fov / 2) comes from FoVs that pair fx with the height and fy with the width, so the rasterizer's x focal length
    W / (2 tanfovx) is the true fy and its y focal length is the true fx (the reference's convention, kept here);
  * the view is a general rigid pose.
  C1  posed: 35 degrees about an oblique axis plus a translation; centred, fx = fy.
  C2  Waymo-like: a 1920 x 1280 front camera's K scaled to the test image (fy / fx = 1.0008, principal point a little off
      centre), swapped FoVs, posed.
  C3  strong: fy = 1.3 fx, cx = 0.3 W, cy = 0.62 H, skew 0.02 fx, posed.  With the swapped FoVs the 1.3 tan(fov / 2) Jacobian
      clamp in x, 0.65 W / fy, lies inside the image right of cx ((W - cx) / fx = 0.7 W / fx > 0.5 W / fx)."""
from __future__ import annotations

import math

import torch

from street_gaussians_b200 import synthetic

CAMERAS = ("C1", "C2", "C3")


def pose(angle_deg=35.0, axis=(1.0, 2.0, 0.5), shift=(0.4, -0.3, 0.6)) -> torch.Tensor:
    """A rigid W2C: rotation by angle_deg about `axis` (Rodrigues), then the translation `shift`."""
    a = torch.tensor(axis, dtype=torch.float64)
    a = a / a.norm()
    K = torch.tensor([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]], dtype=torch.float64)
    ang = math.radians(angle_deg)
    w2c = torch.eye(4, dtype=torch.float64)
    w2c[:3, :3] = torch.eye(3, dtype=torch.float64) + math.sin(ang) * K + (1 - math.cos(ang)) * (K @ K)
    w2c[:3, 3] = torch.tensor(shift, dtype=torch.float64)
    return w2c.float()


# a Waymo front camera at 1920 x 1280 (pixels)
WAYMO_K = dict(fx=2055.6, fy=2057.3, cx=942.7, cy=653.1)


def intrinsics(name, W, H):
    """(fx, fy, cx, cy, skew) of C2 / C3 for a W x H image; None for C1."""
    if name == "C1":
        return None
    if name == "C2":  # scaled by one factor, so that fy / fx and the principal point's offset (in focal lengths) are kept
        s = W / 1920.0
        k = WAYMO_K
        return (k["fx"] * s, k["fy"] * s, W / 2 + (k["cx"] - 960.0) * s, H / 2 + (k["cy"] - 640.0) * s, 0.0)
    if name == "C3":
        fx = 0.8 * W
        return (fx, 1.3 * fx, 0.3 * W, 0.62 * H, 0.02 * fx)
    raise KeyError(name)


def camera(name, W, H, sh_degree=0, scale_modifier=1.0, bg=(0.0, 0.0, 0.0)):
    """Camera dict (synthetic.make_camera) of C1, C2 or C3 for a W x H image."""
    return synthetic.make_camera(W, H, 50.0, pose(), sh_degree, bg, scale_modifier, intrinsics(name, W, H))


def projection(cam):
    """The camera's own projection matrix (fp64, row-vector convention as stored: full = view @ proj)."""
    return torch.linalg.inv(cam["viewmatrix"].double()) @ cam["projmatrix"].double()
