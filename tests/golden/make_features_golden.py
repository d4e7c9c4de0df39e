"""Generates tests/golden/callsite/features.npz: what the reference's UNMODIFIED Python computes for the renderer's feature channels
(street_gaussian_renderer.py:206-264), with the gradients torch autograd sends back through it for seeded upstream gradients.  Run on a
CPU-only machine with a reference checkout (tests/refharness.py):
    python tests/golden/make_features_golden.py
Three parts, each in both semantic modes where it has one:
  sem_<mode>      StreetGaussianModel.get_semantic (street_gaussian_model.py:417-431) of a real model with K = 5 classes, the background
                  and two visible actors of class labels 3 and 1, and the gradients to every model's _semantic
  normals         GaussianModel.get_normals (gaussian_model.py:256-269) of the background, with its gradient to _rotation.  The actors'
                  lines (street_gaussian_model.py:466-477) raise before returning: checked, not stored
  rk_<mode>       render_kernel itself with render.render_normal and data.use_semantic set, the background visible, and the rasterizer's
                  stages replaced by a stand-in that returns a seeded feature image [3 + K, H, W]: the finished maps it returns and the
                  gradient autograd sends to the feature image for seeded gradients on them
Only data goes into the fixture.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import refharness as H  # noqa: E402

K, LABELS, SEED = 5, (3, 1), 23
N_BKGD, PER_OBJ = 400, 120
IMG_W, IMG_H = 40, 24


def stand_in(captured, feature):
    """The rasterizer's three C-ABI stages replaced: the forward returns `feature` as the rendered feature image, the blend backward
    records the gradient that reaches it."""
    from street_gaussians_b200 import rasterizer as R

    def fwd(means3D, sh, colors_precomp, semantics, opacities, scales, rotations, cov3Ds_precomp, settings, band, capacity=None):
        P = means3D.shape[0]
        H_, W_ = int(settings.image_height), int(settings.image_width)
        S = int(semantics.shape[1])
        assert S == feature.shape[0], (S, feature.shape)
        captured["semantics_in"] = semantics.detach().clone()
        st = R._ForwardState()
        st.geom = st.img = st.binning = None
        st.num_instances = 0
        tensors = dict(means3D=means3D, opacities=opacities, sh=sh, colors_precomp=None, scales=scales, rotations=rotations, cov3Ds_precomp=None,
                       semantics=semantics)
        z = lambda c: torch.zeros((c, H_, W_))
        return z(3), torch.ones(P, dtype=torch.int32), z(1), z(1), feature.clone(), st, tensors

    def bwd_blend(settings, band, st, tensors, alpha, gc, gd, ga, gs, grad2d_out=None):
        captured["g_feature"] = gs.detach().clone()
        P = tensors["means3D"].shape[0]
        return torch.zeros((P, 12)), torch.zeros((P, int(tensors["semantics"].shape[1])))

    def bwd_geom(settings, band, st, tensors, radii, grad2d):
        P = tensors["means3D"].shape[0]
        M = tensors["sh"].shape[1]
        z = lambda *s: torch.zeros(s)
        return z(P, 3), z(P, 3), z(P, M, 3), None, z(P, 1), z(P, 3), z(P, 4), None

    saved = (R._forward_impl, R._backward_blend_impl, R._backward_geom_impl)
    R._forward_impl, R._backward_blend_impl, R._backward_geom_impl = fwd, bwd_blend, bwd_geom
    return lambda: setattr(R, "_forward_impl", saved[0]) or setattr(R, "_backward_blend_impl", saved[1]) or setattr(R, "_backward_geom_impl", saved[2])


def main():
    ns = H.load()
    cfg = ns.cfg
    cfg.data.use_semantic = True
    cfg.data.num_classes = K
    g = torch.Generator().manual_seed(SEED)
    f32 = lambda t: t.detach().numpy().astype(np.float32)
    fx = dict(K=np.int32(K), labels=np.array(LABELS, np.int32))

    model = H.make_street_model(ns, n_bkgd=N_BKGD, n_obj=len(LABELS), per_obj=PER_OBJ, seed=SEED)
    cam = H.make_camera(ns, width=IMG_W, height=IMG_H)
    subs = [model.background] + [getattr(model, n) for n in model.obj_list]
    assert model.background._semantic.shape == (N_BKGD, K) and all(getattr(model, n)._semantic.shape == (PER_OBJ, 1) for n in model.obj_list)
    for k, m in enumerate(subs):
        m._semantic = torch.nn.Parameter(torch.randn(m._semantic.shape, generator=g) * 2.0)
        fx[f"semantic_{k}"] = f32(m._semantic)
        if k > 0:
            m.obj_class_label = LABELS[k - 1]

    # ---- get_semantic with actors, both modes
    model.set_visibility(["background"] + model.obj_list)
    model.parse_camera(cam)
    assert list(model.graph_obj_list) == list(model.obj_list)
    for mode in ("logits", "probabilities"):
        for m in subs:
            m.semantic_mode = mode
            m._semantic.grad = None
        out = model.get_semantic
        up = torch.randn(out.shape, generator=g)
        out.backward(up)
        fx[f"sem_{mode}_g"] = up.numpy()
        fx[f"sem_{mode}_out"] = f32(out)
        for k, m in enumerate(subs):
            fx[f"sem_{mode}_grad_{k}"] = f32(m._semantic.grad)

    # ---- get_normals of the background (raw parameters; the composed rows are F.normalize(_rotation) and exp(_scaling))
    bg = model.background
    bg._rotation.grad = None
    normals = bg.get_normals(cam)
    up = torch.randn(normals.shape, generator=g)
    normals.backward(up)
    for k in ("xyz", "rotation", "scaling", "opacity", "features_dc", "features_rest"):
        fx[f"bg_{k}"] = f32(getattr(bg, "_" + k))
    fx.update(camera_center=f32(cam.camera_center), normals_g=up.numpy(), normals_out=f32(normals), normals_grad_rotation=f32(bg._rotation.grad))
    try:  # :473 squeezes the [4] tracking rotation to a row quaternion_to_matrix cannot index; :476 names torch.nn.functinal
        model.get_normals(cam)
    except (IndexError, AttributeError):
        pass
    else:
        raise AssertionError("the reference's actor normals were expected to raise")

    # ---- render_kernel's finishing, background visible
    cfg.render.render_normal = True
    model.set_visibility(["background"])
    model.parse_camera(cam)
    for mode in ("logits", "probabilities"):
        cfg.model.gaussian.semantic_mode = mode
        for m in subs:
            m.semantic_mode = mode
        feature = torch.randn(3 + K, IMG_H, IMG_W, generator=g)
        feature[3:] = torch.rand(K, IMG_H, IMG_W, generator=g) * (2.0 if mode == "probabilities" else 1.0)
        captured = {}
        restore = stand_in(captured, feature)
        try:
            res = ns.renderer.StreetGaussianRenderer().render_kernel(cam, model, white_background=False)
            gn = torch.randn(3, IMG_H, IMG_W, generator=g)
            gs = torch.randn(K, IMG_H, IMG_W, generator=g)
            ((res["normals"] * gn).sum() + (res["semantic"] * gs).sum()).backward()
        finally:
            restore()
        # the call site fed torch.cat([normals, semantics], -1) to the rasterizer
        n_ref = bg.get_normals(cam).detach()
        assert torch.equal(captured["semantics_in"][:, :3], n_ref) and torch.equal(captured["semantics_in"][:, 3:], bg.get_semantic.detach())
        fx.update({f"rk_{mode}_feature": feature.numpy(), f"rk_{mode}_gn": gn.numpy(), f"rk_{mode}_gs": gs.numpy(),
                   f"rk_{mode}_normals": f32(res["normals"]), f"rk_{mode}_semantic": f32(res["semantic"]),
                   f"rk_{mode}_g_feature": f32(captured["g_feature"])})
    path = os.path.join(HERE, "callsite", "features.npz")
    np.savez_compressed(path, **fx)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
