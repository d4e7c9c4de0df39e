"""The reached words of the forward and the backward that reads only their rows (sgr_backward, the autograd path of a single-GPU call
without render layers): the blend backward clears the grad2d rows of the reached Gaussians alone, and the chain rule writes zeros for
the others without reading their rows.  Checked against the two-call backward (sgr_backward_blend, which writes every grad2d row, then
sgr_backward_geom, which reads every row): the reached words cover every non-zero grad2d row; every gradient of an unreached Gaussian
is zero; the reached Gaussians' gradients equal the two-call path's up to the float-atomic noise of the blend backward; a Gaussian
with a non-finite input gives the same NaN / Inf pattern; and a scratch full of NaN, or of another frame's rows, leaves no trace.
Scenes: config C, a saturated and a sparse frame (the saturation split with an empty and a non-empty far slab), a bounded frame that
overflows its capacity, feature channels (S > 0) and a frame with NaN and Inf inputs behind an opaque wall."""
import pytest
import torch

import util
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi
from street_gaussians_b200 import rasterizer as R
from street_gaussians_b200 import synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = ("means3D", "means2D", "sh", "colors", "opacity", "scales", "rotations", "cov3D")


def forward(scene, capacity=None):
    st = util.settings_from(sgb, scene["cam"], DEV)
    dv = lambda k: scene[k].to(DEV) if scene.get(k) is not None else None
    cap = sgb.InstanceCapacity(initial=capacity) if capacity else None
    with torch.no_grad():
        out = R._forward_impl(dv("means3D"), dv("shs"), None, dv("semantics"), dv("opacities"), dv("scales"), dv("rotations"), None, st,
                              None, cap)
    return st, out


def upstream(scene, S, seed=7):
    gen = torch.Generator().manual_seed(seed)
    H, W = scene["cam"]["image_height"], scene["cam"]["image_width"]
    g = lambda c: (torch.randn(c, H, W, generator=gen) / (H * W)).to(DEV)
    return g(3), g(1), g(1), (g(S) if S else None)


def both(st, fwd, ups, scratch=None):
    """(reached [P] bool, grad2d of the two-call path, its 8 gradients + dL_dsemantics, the one-call path's 8 gradients + dL_dsemantics,
    the two-call path's gradients once more: their difference is the float-atomic noise of the blend backward)"""
    color, radii, depth, alpha, sem, fst, tensors = fwd
    P = tensors["means3D"].shape[0]
    gc, gd, ga, gs = ups
    with torch.no_grad():
        g2d, gsem_old = R._backward_blend_impl(st, None, fst, tensors, alpha, gc, gd, ga, gs)
        old = R._backward_geom_impl(st, None, fst, tensors, radii, g2d)
        g2d_again, gsem_again = R._backward_blend_impl(st, None, fst, tensors, alpha, gc, gd, ga, gs)
        again = R._backward_geom_impl(st, None, fst, tensors, radii, g2d_again)
        if scratch is None:
            scratch = torch.full((P, 12), float("nan"), device=DEV)
        new, gsem_new = R._backward_impl(st, None, fst, tensors, radii, alpha, gc, gd, ga, gs, scratch)
    torch.cuda.synchronize()
    reached = R.state_views(st, fst, P)["cval"] != 0
    return reached, g2d, tuple(old) + (gsem_old,), tuple(new) + (gsem_new,), tuple(again) + (gsem_again,)


def check(reached, g2d, old, new, again):
    assert not g2d[~reached].any(), "a grad2d row the reached words miss"
    for name, a, b, a2 in zip(NAMES + ("semantics",), old, new, again):
        if a is None or a.numel() == 0:
            continue
        a, b, a2 = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1), a2.reshape(a2.shape[0], -1)
        assert not b[~reached].any(), (name, "an unreached Gaussian's gradient is not zero")
        assert not a[~reached].any(), (name, "the two-call path gives an unreached Gaussian a gradient")
        fa, fb = torch.isfinite(a), torch.isfinite(b)
        assert torch.equal(fa, fb) and torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a[torch.isinf(a)], b[torch.isinf(b)]), name
        noise = float((a[fa] - a2[fa]).abs().max()) if fa.any() else 0.0
        tol = max(8 * noise, 1e-4 * float(a[fa].abs().max()) if fa.any() else 0.0)
        assert float((a[fa] - b[fa]).abs().max()) <= tol, (name, float((a[fa] - b[fa]).abs().max()), tol)


@pytest.fixture(scope="module")
def config_c():
    return synthetic.make_config("C", seed=0)


def test_config_c(config_c):
    st, fwd = forward(config_c)
    reached, g2d, old, new, again = both(st, fwd, upstream(config_c, 0))
    visible = fwd[1] > 0
    print(f"config C: {int(reached.sum())} reached of {int(visible.sum())} visible Gaussians")
    # the image comes from a small near slab: most visible Gaussians are not reached
    assert reached.any() and int(reached.sum()) < int(visible.sum()) // 4, (int(reached.sum()), int(visible.sum()))
    check(reached, g2d, old, new, again)


@pytest.mark.parametrize("kind", ["saturated", "sparse"])
def test_split_frames(kind):
    if kind == "saturated":  # large opaque splats: every tile saturates in the near slab, the far slab is empty
        scene = synthetic.make_scene(P=60_000, width=800, height=608, sh_degree=3, seed=3, scale_med=0.05)
    else:  # small splats: no tile saturates, every Gaussian with an instance is emitted by the far pass or the near one
        scene = synthetic.make_scene(P=20_000, width=800, height=608, sh_degree=3, seed=4, scale_med=0.002)
    st, fwd = forward(scene)
    status = R.state_views(st, fwd[5], scene["means3D"].shape[0])["status"].cpu()
    far = int(status[_capi.STATUS_FAR_END])
    assert (far == 0) if kind == "saturated" else (far > 0), far
    reached, g2d, old, new, again = both(st, fwd, upstream(scene, 0))
    check(reached, g2d, old, new, again)


def test_bounded_overflow():
    scene = synthetic.make_scene(P=100_000, width=800, height=608, sh_degree=3, seed=5)
    st, fwd = forward(scene)
    R_ = int(fwd[5].num_instances)
    st, fwd = forward(scene, capacity=R_ // 3)
    status = R.state_views(st, fwd[5], scene["means3D"].shape[0])["status"].cpu()
    assert int(status[_capi.STATUS_OVERFLOW]) & 1
    reached, g2d, old, new, again = both(st, fwd, upstream(scene, 0))
    check(reached, g2d, old, new, again)


def test_feature_channels():
    scene = synthetic.make_scene(P=60_000, width=800, height=608, sh_degree=3, seed=6, semantics=3)
    st, fwd = forward(scene)
    reached, g2d, old, new, again = both(st, fwd, upstream(scene, 3))
    check(reached, g2d, old, new, again)


def test_non_finite_inputs_behind_a_wall():
    """Occluded Gaussians with a NaN active SH coefficient, an infinite scale and a NaN rotation: the forward marks them reached, so
    they give the NaN / Inf the two-call path gives; their finite neighbours stay unreached."""
    scene = synthetic.make_scene(P=40_000, width=800, height=608, sh_degree=3, seed=8, scale_med=0.004)
    cam = scene["cam"]
    wall = synthetic.make_scene(P=6_000, width=800, height=608, sh_degree=3, seed=9, scale_med=0.05)
    # the wall: the second scene's splats pulled in front of everything, fully opaque
    view = cam["viewmatrix"]  # (the same camera: make_scene without a pose)
    assert torch.equal(view, wall["cam"]["viewmatrix"])
    m = wall["means3D"].clone()
    m[:, 2] = m[:, 2].clamp(max=1.0) * 0 + 0.6
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        scene[k] = torch.cat([{"means3D": m, "opacities": torch.full_like(wall["opacities"], 0.999)}.get(k, wall[k]), scene[k]]).contiguous()
    st, fwd = forward(scene)
    reached0 = R.state_views(st, fwd[5], scene["means3D"].shape[0])["cval"].cpu() != 0
    visible = (fwd[1] > 0).cpu()
    cand = torch.nonzero(visible & ~reached0).flatten()
    assert cand.numel() >= 3, "no occluded visible Gaussian"
    a, b, c = (int(x) for x in cand[:3])
    scene["shs"][a, 5, 1] = float("nan")
    scene["scales"][b, 0] = float("inf")
    scene["rotations"][c, 2] = float("nan")
    st, fwd = forward(scene)
    reached, g2d, old, new, again = both(st, fwd, upstream(scene, 0))
    radii = fwd[1]
    # (a NaN rotation may cull its Gaussian: a culled one gets zeros on both paths)
    assert all(bool(reached[x]) for x in (a, b, c) if int(radii[x]) > 0) and int(radii[a]) > 0
    assert not torch.isfinite(old[0][a]).all() and not torch.isfinite(new[0][a]).all()
    check(reached, g2d, old, new, again)


def test_no_stale_rows_across_frames():
    """One scratch for two frames whose reached sets differ: the second frame's gradients do not see the first frame's rows."""
    s1 = synthetic.make_scene(P=50_000, width=800, height=608, sh_degree=3, seed=10)
    s2 = synthetic.make_scene(P=50_000, width=800, height=608, sh_degree=3, seed=11)
    scratch = torch.full((50_000, 12), float("nan"), device=DEV)
    st1, f1 = forward(s1)
    r1, _, _, _, _ = both(st1, f1, upstream(s1, 0), scratch)
    assert torch.isfinite(scratch[r1]).all()  # the first frame wrote its rows
    st2, f2 = forward(s2)
    r2, g2d, old, new, again = both(st2, f2, upstream(s2, 0), scratch)
    assert bool((r1 & ~r2).any()) and bool((r2 & ~r1).any())
    check(r2, g2d, old, new, again)


def test_autograd_path_matches_two_call_path():
    """GaussianRasterizer's backward (the one-call path) against the two-call path on the same forward."""
    scene = synthetic.make_scene(P=100_000, width=800, height=608, sh_degree=3, seed=12)
    st = util.settings_from(sgb, scene["cam"], DEV)
    p = {k: scene[k].to(DEV).requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    means2D = torch.zeros_like(p["means3D"], requires_grad=True)
    color, radii, depth, alpha, _ = sgb.GaussianRasterizer(st)(means3D=p["means3D"], means2D=means2D, shs=p["shs"], opacities=p["opacities"],
                                                                scales=p["scales"], rotations=p["rotations"])
    gc, gd, ga, _ = upstream(scene, 0)
    torch.autograd.backward([color, depth, alpha], [gc, gd, ga])
    st2, fwd = forward(scene)
    reached, g2d, old, _, again = both(st2, fwd, (gc, gd, ga, None))
    auto = (p["means3D"].grad, means2D.grad, p["shs"].grad, None, p["opacities"].grad, p["scales"].grad, p["rotations"].grad, None, None)
    check(reached, g2d, old, auto, again)
