"""Generates tests/golden/callsite/sky.npz: what the reference's UNMODIFIED SkyCubeMap.forward (lib/models/sky_cubemap.py:77-123)
and the composite line of street_gaussian_renderer.py:111 compute, with the gradients torch autograd sends back through that code to
rgb, acc and the cube map for a seeded upstream gradient.  Run on a CPU-only machine with a reference checkout (tests/refharness.py):
    python tests/golden/make_sky_golden.py
nvdiffrast is not installed, so dr.texture is bound to the restated lookup of tests/sky_oracle.py; everything else is the
reference's own Python.  Three cases on one posed camera with a Waymo-like K (off-centre principal point, fx != fy) that looks at a
cube corner, on an R = 16 cube with texels in [-0.2, 1.2] (the clamp acts both ways):
  train_mask   cfg.mode = 'train' with a sky mask (the mask and rows 0-49), jittered, white background (fill 1)
  train_acc    cfg.mode = 'train' without a sky mask (1 - acc > 1e-3), jittered, black background (fill 0)
  eval_acc     cfg.mode = 'test' (1 - acc > 1e-3), no jitter, white background
The fixture stores each case's inputs, the jitter the reference drew (two torch.rand(H, W) calls), its outputs and gradients.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import refharness as H  # noqa: E402
import sky_oracle as SO  # noqa: E402

SEED, RES, IMG_H, IMG_W = 11, 16, 64, 80
K_NP = np.array([[50.0, 0.0, 41.3], [0.0, 47.0, 29.6], [0.0, 0.0, 1.0]])  # float64: getProjectionMatrixK assigns its entries
CASES = (("train_mask", "train", True, True), ("train_acc", "train", False, False), ("eval_acc", "test", False, True))


def camera_pose():
    """c2w rotation (the reference's Camera R) whose optical axis points at the cube corner (1, -1, 1) with a little roll, and T."""
    z = np.array([1.0, -1.0, 1.1])
    z /= np.linalg.norm(z)
    x = np.cross([0.1, 1.0, 0.0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    return np.stack([x, y, z], 1), np.array([0.7, -1.3, 2.1])


def _patch_to_cuda():
    """sky_cubemap.py:82 calls Tensor.to('cuda', non_blocking=True), which the harness does not redirect."""
    orig = torch.Tensor.to

    def to(self, *a, **k):
        if a and isinstance(a[0], (str, torch.device)) and str(a[0]).startswith("cuda"):
            a = ("cpu",) + a[1:]
        if str(k.get("device", "")).startswith("cuda"):
            k["device"] = "cpu"
        return orig(self, *a, **k)

    torch.Tensor.to = to


def main():
    ns = H.load()
    _patch_to_cuda()
    sys.modules["nvdiffrast.torch"].texture = SO.texture
    from lib.models import sky_cubemap as skm
    cfg = ns.cfg
    cfg.model.sky.resolution = RES
    g = torch.Generator().manual_seed(SEED)
    Rc, Tc = camera_pose()
    cube = -0.2 + 1.4 * torch.rand(6, RES, RES, 3, generator=g)
    fx = dict(res=RES, cube_map=cube.numpy())
    for name, mode, with_mask, white in CASES:
        cfg.mode = mode
        cfg.model.sky.white_background = white
        sky_mask = torch.rand(1, IMG_H, IMG_W, generator=g) < 0.4
        guidance = {"sky_mask": sky_mask.clone()} if with_mask else {}
        cam = ns.camera_utils.Camera(id=0, R=Rc, T=Tc, FoVx=1.3, FoVy=1.1, K=K_NP.astype(np.float64), image=torch.rand(3, IMG_H, IMG_W, generator=g),
                                     image_name="synthetic", metadata=dict(frame=0, cam=0), guidance=guidance)
        model = skm.SkyCubeMap()
        model.sky_cube_map = torch.nn.Parameter(cube.clone())
        rgb = torch.rand(3, IMG_H, IMG_W, generator=g).requires_grad_(True)
        a = torch.rand(1, IMG_H, IMG_W, generator=g)
        a = torch.where(torch.rand(1, IMG_H, IMG_W, generator=g) < 0.3, torch.ones_like(a), a)
        a[0, ::7, ::5] = 0.9995  # 1 - acc < 1e-3: not sky in the acc rule
        acc = a.clone().requires_grad_(True)
        up = torch.randn(3, IMG_H, IMG_W, generator=g)
        draws = []
        orig_rand = torch.rand

        def rand(*args, **kw):
            t = orig_rand(*args, **kw)
            draws.append(t.clone())
            return t

        torch.rand = rand
        try:
            sky = model(cam, acc.detach())                       # street_gaussian_renderer.py:109
        finally:
            torch.rand = orig_rand
        out = rgb + sky * (1 - acc)                              # :111
        out.backward(up)
        assert len(draws) == (2 if mode == "train" else 0)
        f32 = lambda t: t.detach().numpy().astype(np.float32)
        fx["K"] = f32(cam.K)
        fx.update({f"{name}_rgb": f32(rgb), f"{name}_acc": a.numpy(), f"{name}_g": up.numpy(), f"{name}_w2c": f32(cam.world_view_transform.transpose(0, 1)),
                   f"{name}_fill": np.float32(1.0 if white else 0.0), f"{name}_ref_out": f32(out),
                   f"{name}_ref_drgb": f32(rgb.grad), f"{name}_ref_dacc": f32(acc.grad), f"{name}_ref_dcube": f32(model.sky_cube_map.grad)})
        if with_mask:
            fx[f"{name}_sky_mask"] = sky_mask.numpy()
            fx[f"{name}_mask_after"] = guidance["sky_mask"].numpy()  # the reference's in-place rows 0-49
        if draws:
            fx[f"{name}_jx"], fx[f"{name}_jy"] = draws[0].numpy(), draws[1].numpy()
    os.makedirs(os.path.join(HERE, "callsite"), exist_ok=True)
    path = os.path.join(HERE, "callsite", "sky.npz")
    np.savez_compressed(path, **fx)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
