"""Generates tests/golden/callsite/train_losses.npz from the reference's OWN train.py: the object-accumulation block (train.py:114-122)
and the LiDAR depth block (:124-132) are taken out of train.py with `ast` and executed unmodified on seeded CPU tensors, with stubs
for optim_args, gaussians, gaussians_renderer.render_object and scalar_dict.  Stores values and autograd gradients for two seeds of
[1, 70, 93] maps with ~30 % LiDAR density and a mask.  python tests/golden/make_train_loss_golden.py
"""
import ast
import os
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("SGR_REFERENCE_DIR", "/root/reference")  # a checkout of zju3dv/street_gaussians


def case(seed, Hh=70, Ww=93):
    """Rasterizer-like outputs: acc in [0, 1] with exact zeros and ones, depth = acc * z, LiDAR depth = z + noise with outliers on
    ~30 % of the pixels (0 elsewhere), a mask, the objects-only acc (with values the clamp catches) and an object bound."""
    g = torch.Generator().manual_seed(seed)
    shape = (1, Hh, Ww)
    acc = torch.rand(shape, generator=g)
    u = torch.rand(shape, generator=g)
    acc = torch.where(u < 0.03, torch.zeros_like(acc), torch.where(u > 0.97, torch.ones_like(acc), acc))
    z = 2.0 + 58.0 * torch.rand(shape, generator=g)
    depth = acc * z
    noise = 0.3 * torch.randn(shape, generator=g) + torch.where(torch.rand(shape, generator=g) < 0.05, 20.0, 0.0)
    lidar = torch.where(torch.rand(shape, generator=g) < 0.3, (z + noise).clamp_min(0.0), torch.zeros_like(z))
    mask = torch.rand(shape, generator=g) > 0.2
    acc_obj = torch.rand(shape, generator=g) ** 3
    acc_obj[0, 0, :4] = torch.tensor([0.0, 1.0, 5e-7, 1.0 - 5e-7])
    obj_bound = torch.rand(shape, generator=g) > 0.6
    return dict(depth=depth, acc=acc, lidar_depth=lidar, mask=mask, acc_obj=acc_obj, obj_bound=obj_bound)


def _blocks(path):
    """The two `if` statements of the training loop that guard on lambda_reg and lambda_depth_lidar, compiled as they stand."""
    src = open(path).read()
    tree = ast.parse(src)
    found = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.If):
            test = ast.get_source_segment(src, node.test)
            for key in ("lambda_reg", "lambda_depth_lidar"):
                if f"optim_args.{key} > 0" in test and key not in found:
                    found[key] = (node.lineno, node.end_lineno, compile(ast.Module(body=[node], type_ignores=[]), path, "exec"))
    assert set(found) == {"lambda_reg", "lambda_depth_lidar"}, found.keys()
    return found


def main():
    blocks = _blocks(os.path.join(REF, "train.py"))
    out = {}
    for key, (lo, hi, _) in blocks.items():
        out[f"lines_{key}"] = np.array([lo, hi])
    for seed in (0, 1):
        c = case(seed)
        depth = c["depth"].clone().requires_grad_(True)
        acc = c["acc"].clone().requires_grad_(True)
        acc_obj = c["acc_obj"].clone().requires_grad_(True)
        optim_args = types.SimpleNamespace(lambda_reg=1.0, lambda_depth_lidar=1.0, densify_until_iter=0)
        gaussians = types.SimpleNamespace(include_obj=True)
        renderer = types.SimpleNamespace(render_object=lambda cam, gs, parse_camera_again=False: {"rgb": None, "acc": acc_obj})
        env = dict(torch=torch, optim_args=optim_args, gaussians=gaussians, gaussians_renderer=renderer, viewpoint_cam=None, iteration=1,
                   obj_bound=c["obj_bound"], lidar_depth=c["lidar_depth"], mask=c["mask"], depth=depth,
                   render_pkg={"acc": acc, "depth": depth})
        k = f"s{seed}_"
        scalars = {}
        for key in ("lambda_reg", "lambda_depth_lidar"):
            env["scalar_dict"], env["loss"] = scalars, torch.zeros(())
            exec(blocks[key][2], env)
            env["loss"].backward()
        out[k + "obj"] = float(scalars["obj_acc_loss"])
        out[k + "lidar"] = float(scalars["lidar_depth_loss"].detach())  # stored as a tensor at train.py:131
        out[k + "g_acc_obj"] = acc_obj.grad.numpy()
        out[k + "g_depth"] = depth.grad.numpy()
        out[k + "g_acc"] = acc.grad.numpy()
    path = os.path.join(HERE, "callsite", "train_losses.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), {k: v for k, v in out.items() if not hasattr(v, "shape") or v.size == 2})


if __name__ == "__main__":
    main()
