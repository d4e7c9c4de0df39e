"""CPU tests of the fp64 restatement (oracle/raster64.py): pinned to the reference's own outputs (tests/golden/*.npz) before any
kernel is compared against it per element, and the margin machinery that makes per-element comparison possible."""
import glob
import os

import numpy as np
import pytest
import torch

import raster64_case as RC
import util
from oracle import raster64 as R64
from test_oracle_cpu import scene_from_npz

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "*.npz")))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_render64_matches_reference_golden(path):
    """render64 meets the reference fixtures at the kernels' bars: radii exact, the flip protocol on every image, 1e-3 per
    gradient tensor.  This pins the conventions (NDC units of mean2D, the |.| column, the halved conic xy entry, the uncapped
    opacity gradient, the scale_modifier quirk) to the reference itself.  The backward reads T_final from the reference's alpha
    image, as the reference's backward does (backward.cu:468): on saturated pixels 1 - sum(w) amplifies the forward's fp32
    rounding by 1 / T_final (up to 1e4), so an fp64 alpha there would measure that amplification, not the conventions."""
    z = np.load(path)
    scene = scene_from_npz(z)
    ref = {k[4:]: z[k] for k in z.files if k.startswith("ref_")}
    res = R64.render64(scene, alpha_img=torch.from_numpy(ref["alpha"]))
    assert (res["radii"].numpy() == ref["radii"]).all()
    mine = {k: v.numpy() for k, v in res.items() if isinstance(v, torch.Tensor)}
    vis = ref["radii"] > 0
    rec = res["pre"]["rec"].numpy()
    maxv = dict(color=float(rec[vis, 8:11].max()) + float(np.abs(z["bg"]).max()), depth=float(rec[vis, 7].max()), alpha=1.0)
    names = ["color", "depth", "alpha"]
    if ref["semantic"].size:
        maxv["semantic"] = float(np.abs(z["in_semantics"]).max())
        names.append("semantic")
    npx = int(z["image_width"]) * int(z["image_height"])
    util.check_forward_flip_protocol(mine, ref, maxv, names=names, max_pixels=max(3, npx // 5000))
    n = 0
    for k, v in ref.items():
        if k.startswith("g_") and k in mine and v.size:
            e = util.rel_err(mine[k].reshape(v.shape), v)
            assert e < 1e-3, (k, e)
            n += 1
    assert n >= 5


def _scene():
    a = RC.filler(96, 64, 300, seed=3, sh_degree=2)
    return RC.cat_scenes(a, RC.stack(96, 64, 40, 24, 40, seed=4, opac=(0.2, 0.4), sigma=30.0, sh_degree=2))


def test_margin_scene_terminates_and_clears_every_decision():
    """After margin_scene no decision lies within delta; it converges, and removes only a small fraction."""
    sc = _scene()
    P = sc["means3D"].shape[0]
    out, removed, keep = R64.margin_scene(sc, delta=1e-5)
    pre = R64.preprocess64(out)
    cam = pre["cam"]
    assert len(R64.margins(pre["rec"], pre["radii"], cam["W"], cam["H"], 1e-5, pre=pre)) == 0
    assert out["means3D"].shape[0] == P - removed == len(keep)
    print(f"margin_scene removed {removed} of {P}")
    assert removed <= 0.05 * P
    # the scene keeps its deep, terminating tile
    bl = R64.blend64(pre["rec"], pre["radii"], cam["W"], cam["H"], cam["bg"])
    assert bl["stopped"].any()


def test_margins_flag_near_threshold_pairs():
    """A Gaussian placed so that one pair's alpha sits exactly on 1/255 is reported; moving it away clears it."""
    W = H = 32
    # o G = 1/255 at the pixel one step right of the centre: o exp(-0.5 a) = 1/255 with the dilated conic a
    sigma2 = 4.0 ** 2 + 0.3
    o = R64.ALPHA_MIN * np.exp(0.5 / sigma2)
    sc = RC.screen_scene(W, H, [10.0], [10.0], [4.0], [5.0], [o])
    pre = R64.preprocess64(sc)
    rec = pre["rec"].clone()
    rec[0, 0], rec[0, 1] = 10.0, 10.0
    rec[0, 2], rec[0, 3], rec[0, 4], rec[0, 5] = 1.0 / sigma2, 0.0, 1.0 / sigma2, o
    assert len(R64.margins(rec, pre["radii"], W, H, 1e-6)) == 1
    rec[0, 5] = o * 1.01
    assert len(R64.margins(rec, pre["radii"], W, H, 1e-6)) == 0


def test_blend64_backward_matches_autograd_of_forward():
    """grad2d of blend64 against torch autograd of blend64's own fp64 forward (same decisions, so the two must agree to fp64
    rounding): pins the recurrences of the backward, the NDC units and the halved conic entry independently of any fixture."""
    sc, _, _ = R64.margin_scene(_scene(), delta=1e-5)
    pre = R64.preprocess64(sc)
    cam = pre["cam"]
    W, H = cam["W"], cam["H"]
    up = dict(color=sc["grad_color"], depth=sc["grad_depth"], alpha=sc["grad_alpha"], semantic=None)
    bl = R64.blend64(pre["rec"], pre["radii"], W, H, cam["bg"], upstream=up)
    rec = pre["rec"].clone().requires_grad_(True)
    # differentiable forward with the same per-pair decisions
    fw = _blend_autograd(rec, bl, W, H, cam["bg"])
    loss = sum((fw[k] * up[k].double()).sum() for k in ("color", "depth", "alpha"))
    (g,) = torch.autograd.grad(loss, rec)
    vis = pre["radii"] > 0
    exp = torch.stack([g[:, 0] * 0.5 * W, g[:, 1] * 0.5 * H, g[:, 2], 0.5 * g[:, 3], g[:, 4], g[:, 5], g[:, 8], g[:, 9], g[:, 10], g[:, 7]], 1)
    got = bl["grad2d"][:, [0, 1, 3, 4, 5, 6, 7, 8, 9, 10]]
    # opacity gradient of the reference: G dL/dalpha, uncapped — autograd of min(0.99, o G) would zero it on capped pairs; the
    # scene has none (asserted), so the two agree
    assert int(bl["n_capped"].sum()) == 0
    err = (got - exp)[vis].abs()
    assert float(err.max()) <= 1e-9 * float(exp[vis].abs().max()), float(err.max())


def _blend_autograd(rec, bl, W, H, bg):
    """fp64 forward of the blend differentiable in the records, replaying blend64's decisions (its tile lists)."""
    HW = W * H
    color = torch.zeros(3, HW, dtype=torch.float64)
    depth = torch.zeros(HW, dtype=torch.float64)
    alpha = torch.zeros(HW, dtype=torch.float64)
    tiles, ids = bl["tiles"], bl["ids"]
    gx = (W + 15) // 16
    for t in torch.unique(tiles).tolist():
        gid = ids[tiles == t]
        xs = torch.arange(16) + (t % gx) * 16
        ys = torch.arange(16) + (t // gx) * 16
        yy, xx = torch.meshgrid(ys, xs, indexing="ij")
        inside = (xx < W) & (yy < H)
        xx, yy = xx[inside], yy[inside]
        r = rec[gid]
        dx = r[:, 0:1] - xx[None].double()
        dy = r[:, 1:2] - yy[None].double()
        power = -0.5 * (r[:, 2:3] * dx * dx + r[:, 4:5] * dy * dy) - r[:, 3:4] * dx * dy
        a = torch.clamp(r[:, 5:6] * torch.exp(torch.clamp(power, max=0)), max=R64.ALPHA_CAP)
        ok = (power <= 0) & (a >= R64.ALPHA_MIN)
        A0 = torch.where(ok, a, torch.zeros_like(a)).detach()
        keep = ok & (torch.cumprod(1 - A0, 0) >= R64.T_STOP)
        A = torch.where(keep, a, torch.zeros_like(a))
        T = torch.cat([torch.ones_like(A[:1]), torch.cumprod(1 - A, 0)[:-1]], 0)
        w = A * T
        p = yy * W + xx
        for ch in range(3):
            color[ch].index_add_(0, p, (w * r[:, 8 + ch:9 + ch]).sum(0))
        depth.index_add_(0, p, (w * r[:, 7:8]).sum(0))
        alpha.index_add_(0, p, w.sum(0))
    Tf = 1 - alpha
    color = color + Tf[None] * bg.reshape(3, 1)
    return dict(color=color.reshape(3, H, W), depth=depth.reshape(1, H, W), alpha=alpha.reshape(1, H, W))


def test_render64_vs_c_oracle_per_element_on_margin_scene():
    """render64 against the plain-C oracle (fp32) per element on a margin scene.  The oracle's alpha image feeds T_final on both
    sides (see test_render64_matches_reference_golden), so what remains is fp32 rounding, bounded per element by
    oracle/raster64.py's chain_bound: the blend's kappa-weighted mass carried through the chain, plus K_CHAIN = 64 roundings (the
    longest path of the fp32 chain rule has 42) of the element's own path terms and of the row's shared intermediates."""
    sc, removed, _ = R64.margin_scene(RC.filler(80, 48, 250, seed=9, sh_degree=3), delta=1e-5)
    orc = util.run_oracle(sc)
    orc.pop("_fw")
    res = R64.render64(sc, alpha_img=torch.from_numpy(orc["alpha"]))
    assert (res["radii"].numpy() == orc["radii"]).all()
    bl = res["blend"]
    for k in ("color", "depth", "alpha"):
        err = np.abs(res[k].numpy() - orc[k])
        bnd = R64.bound(bl["kmass_" + k]).numpy() + 1e-12
        assert (err <= bnd).all(), (k, float((err / bnd).max()))
    worst = {}
    for k in ("g_means2D", "g_opacities", "g_shs", "g_means3D", "g_scales", "g_rotations"):
        a = orc[k].reshape(res[k].shape)
        err = np.abs(res[k].numpy() - a)
        bnd = R64.chain_bound(res, k).numpy() + 1e-30
        if k == "g_means2D":
            err = err[:, :2]; bnd = bnd[:, :2]
        worst[k] = float((err / bnd).max())
        assert (err <= bnd).all(), (k, worst[k])
    print("removed", removed, "max error/bound", worst)
