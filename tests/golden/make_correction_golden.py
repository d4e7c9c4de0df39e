"""Generates tests/golden/callsite/correction_sh{1,3}.npz: what the reference's UNMODIFIED StreetGaussianModel composes with
cfg.model.use_pose_correction (lib/models/camera_pose.py:89-114 through street_gaussian_model.py:311-312, 340-341) from the seeded
raw parameters of tests/compose_case.py, what its ColorCorrection.forward (lib/models/color_correction.py:129-132) makes of a seeded
image and what its regularization_loss (:134-140) gives, with the gradients torch autograd sends back through that code for
seeded upstream gradients.  Run on the build container (CPU, tests/refharness.py):
    python tests/golden/make_correction_golden.py 1 ; python tests/golden/make_correction_golden.py 3
The correction parameters (pose_correction_rots / _trans and affine_trans / affine_trans_sky, per image) are seeded, non-identity
and differ per row; the camera is image CAM_ID, so picking the camera's row is part of what the fixture pins.  The fixture stores
those parameters, the per-frame inputs the reference derived (actor poses, IDFT rows, flip mask and quaternion), the image and
its upstream gradient, and the reference's outputs and gradients; the raw Gaussian parameters are regenerated from the seed.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import compose_case as CC  # noqa: E402
import refharness as H  # noqa: E402

SEED, N_BKGD, ACTORS, CAM_ID, IMG_HW = 7, 600, (250, 150), 5, (24, 40)


def correction_params(seed: int, num_images: int):
    """Seeded per-image corrections: quaternions of norms 0.5-2 around a small rotation, translations ~0.3, affines I + 0.1 noise."""
    g = torch.Generator().manual_seed(seed)
    rots = torch.tensor([1.0, 0.0, 0.0, 0.0]) + 0.2 * torch.randn(num_images, 4, generator=g)
    rots = rots * (0.5 + 1.5 * torch.rand(num_images, 1, generator=g))
    trans = 0.3 * torch.randn(num_images, 3, generator=g)
    eye = torch.eye(4)[:3]
    affine = eye + 0.1 * torch.randn(num_images, 3, 4, generator=g)
    affine_sky = eye + 0.1 * torch.randn(num_images, 3, 4, generator=g)
    return rots, trans, affine, affine_sky


def image_case(seed: int, hw):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(3, *hw, generator=g), torch.randn(3, *hw, generator=g)


def main():
    deg = int(sys.argv[1]) if len(sys.argv) > 1 else 1
    ns = H.load(extra_opts=["model.gaussian.sh_degree", str(deg), "model.use_pose_correction", "True", "model.use_color_correction", "True",
                            "model.pose_correction.mode", "image", "model.color_correction.mode", "image"])
    torch.manual_seed(0)  # the flip mask is torch.rand_like inside parse_camera (street_gaussian_model.py:275-284)
    cam = H.make_camera(ns, frame=3)
    cam.id = CAM_ID
    model = H.make_street_model(ns, n_bkgd=8, n_obj=len(ACTORS), per_obj=8)
    M, C = (model.max_sh_degree + 1) ** 2, int(model.fourier_dim)
    assert model.max_sh_degree == deg and model.use_pose_correction and model.use_color_correction
    raw = CC.make_case(SEED, N_BKGD, ACTORS, M, C)
    subs = [model.background] + [getattr(model, n) for n in model.obj_list]
    for sub, r in zip(subs, raw):
        for k in CC.KEYS:
            setattr(sub, "_" + k, torch.nn.Parameter(r[k].clone()))
    pc, cc = model.pose_correction, model.color_correction
    n_img = pc.pose_correction_rots.shape[0]
    rots, trans, affine, affine_sky = correction_params(SEED + 2, n_img)
    pc.pose_correction_rots = torch.nn.Parameter(rots.clone())
    pc.pose_correction_trans = torch.nn.Parameter(trans.clone())
    cc.affine_trans = torch.nn.Parameter(affine.clone())
    cc.affine_trans_sky = torch.nn.Parameter(affine_sky.clone())
    model.set_visibility(["background"] + model.obj_list)
    model.parse_camera(cam)
    assert model.graph_obj_list == model.obj_list
    model.obj_rots.retain_grad()
    model.obj_trans.retain_grad()
    out = dict(xyz=model.get_xyz, rotation=model.get_rotation, scaling=model.get_scaling, opacity=model.get_opacity, features=model.get_features)
    P = out["xyz"].shape[0]
    up = CC.upstream(SEED + 1, P, M)
    torch.autograd.backward([out[k] for k in up], [up[k] for k in up])
    starts = np.cumsum([0] + [r["xyz"].shape[0] for r in raw])
    poses, dposes, idft = [], [], []
    for a, name in enumerate(model.obj_list):
        lo, hi = starts[a + 1] - N_BKGD, starts[a + 2] - N_BKGD
        rot, tr = model.obj_rots[lo], model.obj_trans[lo]
        poses.append(torch.cat([rot, tr]).detach().numpy())
        dposes.append(torch.cat([model.obj_rots.grad[lo:hi].sum(0), model.obj_trans.grad[lo:hi].sum(0)]).numpy())
        obj = getattr(model, name)
        t = obj.fourier_scale * (model.frame - obj.start_frame) / (obj.end_frame - obj.start_frame)
        idft.append(ns.sh_utils.IDFT(t, obj.fourier_dim)[0].numpy())
    # colour correction of a seeded image, then the regularisation on its own
    image, g_image = image_case(SEED + 3, IMG_HW)
    image.requires_grad_(True)
    corrected = cc(cam, image)
    corrected.backward(g_image)
    reg = cc.regularization_loss(cam)
    ga_img = cc.affine_trans.grad.clone()
    cc.affine_trans.grad = None
    reg.backward()
    f32 = lambda t: t.detach().numpy().astype(np.float32)
    fx = dict(sh_degree=deg, fourier_dim=C, seed=SEED, n_bkgd=N_BKGD, actors=np.array(ACTORS), cam_id=CAM_ID, poses=np.stack(poses).astype(np.float32),
              idft=np.stack(idft).astype(np.float32), flip=model.flip_mask.numpy().astype(np.uint8),
              flip_quat=model.flip_matrix.reshape(4).numpy().astype(np.float32), ref_dposes=np.stack(dposes).astype(np.float32),
              pose_correction_rots=f32(rots), pose_correction_trans=f32(trans), affine_trans=f32(affine), affine_trans_sky=f32(affine_sky),
              ref_g_pose_correction_rots=f32(pc.pose_correction_rots.grad), ref_g_pose_correction_trans=f32(pc.pose_correction_trans.grad),
              image=f32(image), g_image=f32(g_image), ref_corrected=f32(corrected), ref_dimage=f32(image.grad), ref_daffine=f32(ga_img),
              ref_reg=f32(reg), ref_reg_g_affine=f32(cc.affine_trans.grad), ref_reg_g_affine_sky=f32(cc.affine_trans_sky.grad))
    for k, v in out.items():
        fx["ref_" + k] = f32(v)
    for i, sub in enumerate(subs):
        for k in CC.KEYS:
            fx[f"ref_g{i}_{k}"] = f32(getattr(sub, "_" + k).grad)
    os.makedirs(os.path.join(HERE, "callsite"), exist_ok=True)
    path = os.path.join(HERE, "callsite", f"correction_sh{deg}.npz")
    np.savez_compressed(path, **fx)
    print("wrote", path, os.path.getsize(path), "bytes; P =", P, "M =", M, "C =", C, "flipped:", int(model.flip_mask.sum()), "images:", n_img)


if __name__ == "__main__":
    main()
