"""CPU half of the posed / intrinsics tier (tests/camera64_case.py): the camera builder against the reference's own
getProjectionMatrixK, Camera and make_rasterizer, each camera's own edge, and the defaults that must not move."""
import math
import os

import numpy as np
import pytest
import torch

import camera64_case as CC
import raster64_case as RC
import refharness as H
from oracle import raster64 as R64
from street_gaussians_b200 import synthetic
from test_raster64_gpu import preprocess_scene

HERE = os.path.dirname(os.path.abspath(__file__))


def test_defaults_unchanged():
    """make_camera / make_scene without intrinsics, sh_coeffs or scale_modifier build what the committed fixtures were made from."""
    z = np.load(os.path.join(HERE, "golden", "sh3_pose.npz"))
    sc = synthetic.make_scene(P=1500, width=160, height=96, sh_degree=3, seed=101, pose=True, scale_med=0.06)
    for k in ("viewmatrix", "projmatrix", "campos"):
        assert np.array_equal(sc["cam"][k].numpy(), z[k]), k
    for k in ("tanfovx", "tanfovy", "scale_modifier", "sh_degree"):
        assert sc["cam"][k] == z[k][()], k
    for k in ("means3D", "shs", "opacities", "scales", "rotations", "grad_color"):
        assert np.array_equal(sc[k].numpy(), z["in_" + k]), k


@pytest.mark.parametrize("name", CC.CAMERAS)
def test_camera_edges(name):
    """Each camera reaches what the identity camera cannot: off-diagonal view and projection entries (the rotation part of the
    EWA covariance, mean2d_bwd's proj[1], proj[4], proj[8], proj[9]); C2 / C3 a principal point off centre and the swapped FoVs
    (the rasterizer's fx is the true fy); C3 skew and focal lengths 30 % apart."""
    W, H_ = 96, 64
    cam = CC.camera(name, W, H_)
    view, full, P = cam["viewmatrix"], cam["projmatrix"], CC.projection(cam)
    for i, j in ((0, 1), (1, 0), (0, 2), (2, 0), (1, 2), (2, 1)):
        assert abs(float(view[i, j])) > 0.05 and abs(float(full[i, j])) > 0.05, (i, j)
    fx_k, fy_k = W / (2 * cam["tanfovx"]), H_ / (2 * cam["tanfovy"])
    K = CC.intrinsics(name, W, H_)
    if K is None:
        assert abs(fx_k / fy_k - 1) < 1e-6
        assert max(abs(float(P[2, 0])), abs(float(P[2, 1])), abs(float(P[1, 0]))) < 1e-5
        return
    fx, fy, cx, cy, skew = K
    assert math.isclose(fx_k, fy, rel_tol=1e-6) and math.isclose(fy_k, fx, rel_tol=1e-6), "swapped FoVs"
    assert abs(float(P[2, 0])) > 1e-3 and abs(float(P[2, 1])) > 1e-3, "principal point off centre"  # stored transposed
    assert abs(float(P[3, 2]) + 0.002) < 1e-6, "OpenGL depth row of getProjectionMatrixK"
    if name == "C2":
        assert 1.0005 < fy / fx < 1.001
    if name == "C3":
        assert abs(float(P[1, 0])) > 1e-3, "skew"
        assert (W - cx) / fx > 0.65 * W / fy, "the x clamp lies inside the image"


def test_strong_camera_clamps_inside_the_image():
    """Under C3 the preprocess scene holds visible Gaussians whose centre is inside the image and yet past the 1.3 tan(fov / 2)
    Jacobian clamp (zero x gradient through the EWA Jacobian): the centred square-pixel cameras cannot produce this."""
    cam = CC.camera("C3", 96, 64, sh_degree=1)
    sc, _, _ = R64.margin_scene(preprocess_scene(1, seed=5, cam=cam, sh_coeffs=16))
    pre = R64.preprocess64(sc)
    px, py = pre["rec"][:, 0], pre["rec"][:, 1]
    inside = (px >= 0) & (px < 96) & (py >= 0) & (py < 64)
    assert int((pre["clamped_x"] & inside & pre["vis"]).sum()) >= 3
    assert int(((pre["clamped_x"] | pre["clamped_y"]) & ~inside & pre["vis"]).sum()) >= 3


def test_pixel_placement_under_each_camera():
    """screen_scene's centres land on the requested pixels and view depths under every camera."""
    for name in CC.CAMERAS:
        cam = CC.camera(name, 97, 61)
        px = torch.tensor([3.25, 50.0, 90.5], dtype=torch.float64)
        py = torch.tensor([5.5, 30.25, 58.0], dtype=torch.float64)
        sc = RC.screen_scene(97, 61, px, py, 3.0, torch.tensor([2.0, 9.0, 40.0], dtype=torch.float64), 0.5, cam=cam, thin=0.1)
        pre = R64.preprocess64(sc)
        assert torch.allclose(pre["rec"][:, 0], px, atol=1e-3) and torch.allclose(pre["rec"][:, 1], py, atol=1e-3), name
        assert torch.allclose(pre["tz"], torch.tensor([2.0, 9.0, 40.0], dtype=torch.float64), rtol=1e-5), name


@pytest.mark.skipif(not H.available() or torch.cuda.is_available(), reason="needs a reference checkout (SGR_REFERENCE_DIR)")
@pytest.mark.parametrize("name", CC.CAMERAS)
def test_camera_builder_matches_reference_camera(name):
    """make_camera(intrinsics=...) against the reference's own Camera (getProjectionMatrixK, world_view_transform,
    full_proj_transform, camera_center) and make_rasterizer's tan(fov / 2), fed the Waymo reader's FoVs."""
    ns = H.load()
    from lib.utils import graphics_utils as gu
    W, H_ = 208, 120
    cam = CC.camera(name, W, H_)
    w2c = CC.pose().double().numpy()
    K = CC.intrinsics(name, W, H_)
    if K is None:
        fovx = math.radians(50.0)
        fovy = 2 * math.atan(math.tan(fovx / 2) * H_ / W)
        Kmat = None
    else:
        fx, fy, cx, cy, skew = K
        Kmat = np.array([[fx, skew, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=np.float64)
        fovy, fovx = gu.focal2fov(fx, H_), gu.focal2fov(fy, W)  # waymo_full_readers.py:100-102
    image = torch.zeros(3, H_, W)
    rc = ns.camera_utils.Camera(id=0, R=w2c[:3, :3].T, T=w2c[:3, 3], FoVx=fovx, FoVy=fovy, K=Kmat, image=image, image_name="c",
                                metadata=dict(frame=0, frame_idx=0, is_val=False, timestamp=0.0, cam=0))
    proj_t = torch.linalg.inv(cam["viewmatrix"]) @ cam["projmatrix"]
    assert torch.allclose(proj_t, rc.projection_matrix.cpu(), rtol=1e-6, atol=1e-7)
    assert torch.allclose(cam["viewmatrix"], rc.world_view_transform.cpu(), rtol=1e-6, atol=1e-7)
    assert torch.allclose(cam["projmatrix"], rc.full_proj_transform.cpu(), rtol=1e-5, atol=1e-6)
    assert torch.allclose(cam["campos"], rc.camera_center.cpu(), rtol=1e-5, atol=1e-6)
    rast = ns.camera_utils.make_rasterizer(rc, active_sh_degree=0, bg_color=torch.zeros(3), scaling_modifier=1.0)
    s = rast.raster_settings
    assert math.isclose(s.tanfovx, cam["tanfovx"], rel_tol=1e-12) and math.isclose(s.tanfovy, cam["tanfovy"], rel_tol=1e-12)
    if Kmat is not None:  # getProjectionMatrixK itself, bit for bit
        P = gu.getProjectionMatrixK(Kmat, H_, W, 0.001, 1000.0)
        assert torch.equal(synthetic.projection_matrix_k(0.001, 1000.0, *K, W, H_), P)
