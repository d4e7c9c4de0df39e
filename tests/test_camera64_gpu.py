"""The fp64 per-element tier under the posed / intrinsics cameras of tests/camera64_case.py (C1 posed, C2 Waymo-like, C3 strong),
a scale_modifier other than 1 and an active SH degree below the stored one.  Same checks and bounds as test_raster64_gpu.py
(check, check_preprocess, check_end_to_end), test_layers_gpu.py (check_layered) and test_sharded64_gpu.py (run_fused); only the
inputs change.  What identity-camera scenes cannot tell apart and these can: the rasterizer's two focal lengths swapped, a
transposed off-diagonal view or projection entry, the backward dropping scale_modifier, SH evaluated at the stored instead of
the active degree, and inactive coefficients leaking into any output."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import camera64_case as CC
import raster64_case as RC
import test_raster64_gpu as T
import util
from oracle import raster64 as R64
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi
from street_gaussians_b200 import rasterizer as R

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ------------------------------------------------------------------------------------------------ blend
@pytest.mark.parametrize("name", ["C2", "C3"])
def test_blend_list_depth_65(name):
    """65 faint splats over one tile (blend_bwd2's batches of 32, blend_bwd's 64) under a posed camera."""
    cam = CC.camera(name, 48, 48)
    K = 65
    for extra in range(16):
        sc = RC.stack(48, 48, 24, 24, K + extra, seed=K, cam=cam)
        sc, _, _ = R64.margin_scene(sc, device=DEV)
        pre = R64.preprocess64(sc, DEV)
        nb = R64.blend64(pre["rec"], pre["radii"], 48, 48, pre["cam"]["bg"])["n_blend"][16:32, 16:32]
        if int(nb.min()) == int(nb.max()) == K:
            break
    bl, _ = T.check(f"{name}_depth65", sc)
    assert int(bl["n_blend"][16:32, 16:32].min()) == int(bl["n_blend"][16:32, 16:32].max()) == K


@pytest.mark.parametrize("name", ["C2", "C3"])
def test_blend_early_termination(name):
    """Tile (0, 0) stops inside the first 256-record batch; tile (3, 0) stops on part of its pixels."""
    W, H = 64, 32
    cam = CC.camera(name, W, H)
    a = RC.stack(W, H, 8, 8, 300, seed=1, opac=(0.25, 0.45), sigma=10.0, cam=cam)
    g = torch.Generator().manual_seed(2)
    b = RC.screen_scene(W, H, 49.0 + torch.rand(40, generator=g, dtype=torch.float64), 8.0 + torch.rand(40, generator=g, dtype=torch.float64),
                        1.2, 1.0 + 0.01 * torch.arange(40, dtype=torch.float64), 0.5 + 0.2 * torch.rand(40, generator=g, dtype=torch.float64),
                        seed=2, cam=cam)
    bl, _ = T.check(f"{name}_termination", RC.cat_scenes(RC.cat_scenes(a, b), RC.filler(W, H, 20, seed=3, cam=cam)))
    assert bool(bl["stopped"][:16, :16].all()) and int(bl["n_list"][0, 0]) > 256
    t2 = bl["stopped"][:16, 48:64]
    assert bool(t2.any()) and not bool(t2.all())


@pytest.mark.parametrize("name", ["C2", "C3"])
def test_blend_large_distant_thin(name):
    """The 1920 x 48 strip of test_raster64_gpu's large_distant_thin case (rectangles over 64 tiles, whole-image splats, centres
    left of and above the image and hundreds of pixels from their tiles, conic condition ~1e4) under a posed camera."""
    W, H = 1920, 48
    cam = CC.camera(name, W, H)
    bgw = (1.0, 1.0, 1.0)
    big = RC.screen_scene(W, H, [300.0, 1200.0, 960.0], [20.0, 30.0, 24.0], [110.13, 90.17, 700.2], [5.0, 6.0, 40.0], [0.3, 0.4, 0.2], seed=5,
                          bg=bgw, cam=cam)
    off = RC.screen_scene(W, H, [-40.0, 100.0, -300.0, 2400.0], [-30.0, -45.0, 20.0, 60.0], [25.1, 20.1, 140.1, 130.2],
                          [3.0, 3.5, 8.0, 9.0], [0.6, 0.5, 0.7, 0.7], seed=6, bg=bgw, cam=cam)
    g = torch.Generator().manual_seed(7)
    n = 40
    thin = RC.screen_scene(W, H, torch.rand(n, generator=g, dtype=torch.float64) * W, torch.rand(n, generator=g, dtype=torch.float64) * H,
                           55.0, 2.0 + torch.rand(n, generator=g, dtype=torch.float64) * 10, 0.6, thin=1e-3, seed=7, bg=bgw, cam=cam)
    far = RC.screen_scene(W, H, [-250.0, -330.0, -410.0, -290.0], [12.0, 30.0, 40.0, -20.0], [150.3, 170.2, 190.1, 160.4],
                          [8.0, 9.0, 10.0, 8.5], [0.6, 0.5, 0.7, 0.6], seed=9, bg=bgw, cam=cam)
    sc = RC.cat_scenes(RC.cat_scenes(RC.cat_scenes(RC.cat_scenes(big, off), far), thin), RC.filler(W, H, 300, seed=8, bg=bgw, cam=cam))
    kept = {}
    bl, k = T.check(f"{name}_large_distant_thin", sc, kept=kept)
    x0, y0, x1, y1 = bl["rect"]
    assert int(((x1 - x0) * (y1 - y0)).max()) > 64
    pre = R64.preprocess64(kept["scene"], DEV)
    vis = pre["vis"]
    px, py = pre["rec"][:, 0], pre["rec"][:, 1]
    assert bool(((px < -200) & vis).any()) and bool(((py < 0) & vis).any())
    assert bool(((pre["clamped_x"] | pre["clamped_y"]) & vis).any())


@pytest.mark.parametrize("name", ["C2", "C3"])
def test_blend_partial_tiles(name):
    """97 x 61: partial tiles in both directions, SH degree 1."""
    cam = CC.camera(name, 97, 61, sh_degree=1)
    T.check(f"{name}_size97x61", RC.filler(97, 61, 98, seed=158, cam=cam))


@pytest.mark.parametrize("name", ["C2", "C3"])
def test_blend_band_and_bounded(name):
    """One cyclic tile-row band and the bounded binning, SH degree 2."""
    cam = CC.camera(name, 96, 80, sh_degree=2)
    sc = RC.cat_scenes(RC.filler(96, 80, 200, seed=11, cam=cam), RC.stack(96, 80, 40, 40, 40, seed=11, cam=cam))
    T.check(f"{name}_band", sc, band=R.TileRowBand(1, 5, 2))
    T.check(f"{name}_bounded", sc, capacity=R.InstanceCapacity(initial=200_000))


# ------------------------------------------------------------------------------------------------ preprocess
# (D, M): the TMA backward (M = 4, 16), the staged one (M = 9), the unstaged one (M = 25), each with inactive coefficients
PRE = [(0, 16), (1, 16), (2, 16), (3, 16), (1, 9), (0, 4), (2, 25), (3, 25)]


def _pre_case(D, M, mod, seed, **kw):
    cam = CC.camera("C3", 96, 64, sh_degree=D, scale_modifier=mod)
    return T.preprocess_scene(D, seed, cam=cam, sh_coeffs=M, **kw)


@pytest.mark.parametrize("i", range(len(PRE)), ids=[f"D{d}_M{m}" for d, m in PRE])
def test_preprocess_per_element(i):
    """Preprocess forward and backward per element under C3 at active degree D with M stored coefficients, scale_modifier
    alternating 0.6 / 1.7.  Gradients of the inactive coefficients must be exactly 0 (chain_bound is 0 there)."""
    D, M = PRE[i]
    mod = (0.6, 1.7)[i % 2]
    pre, k = T.check_preprocess(f"C3_D{D}_M{M}_mod{mod}", _pre_case(D, M, mod, seed=60 + i))
    vis = pre["vis"]
    assert int(k["tensors"]["sh"].shape[1]) == M and k["settings"].sh_degree == D and k["settings"].scale_modifier == mod
    assert bool(((pre["clamped_x"] | pre["clamped_y"]) & vis).sum() >= 3), "Jacobian-clamped Gaussians"
    px, py = pre["rec"][:, 0], pre["rec"][:, 1]
    inside = (px >= 0) & (px < 96) & (py >= 0) & (py < 64)
    assert bool((pre["clamped_x"] & inside & vis).any()), "a clamped centre inside the image"


def test_preprocess_colors_precomp():
    pre, _ = T.check_preprocess("C3_colors_precomp", _pre_case(0, 1, 1.7, seed=70, colors_precomp=True))


GEOM_GRADS = ("g_means3D", "g_means2D", "g_shs", "g_colors_precomp", "g_opacities", "g_scales", "g_rotations", "g_cov3D_precomp")


def _kernel_outputs(scene, grad2d=None):
    """Forward (images, radii, records) and the per-Gaussian chain rule fed `grad2d` (default: this forward's own blend backward).
    Two runs are compared through one grad2d: blend_bwd adds each Gaussian's per-tile sums with float atomics, so a second
    backward of the same frame may differ in the last bits; everything else is deterministic."""
    k = T.run_kernels(scene, backward=grad2d is None)
    g2d = k["grad2d"] if grad2d is None else grad2d
    grads = R._backward_geom_impl(k["settings"], None, k["state"], k["tensors"], k["radii"], g2d)
    torch.cuda.synchronize()
    out = dict(color=k["color"], depth=k["depth"], alpha=k["alpha"], radii=k["radii"], rec=k["rec"], grad2d=g2d)
    out.update({n: g for n, g in zip(GEOM_GRADS, grads) if g is not None})
    return out


def _assert_bit_equal(a, b):
    assert a.keys() == b.keys() and len(a) >= 9
    for key in a:
        assert torch.equal(a[key], b[key]), key


def test_preprocess_cov3d_precomp_ignores_scale_modifier():
    """cov3D_precomp per element under C3 with scale_modifier 1.7, and every output bit-equal to the same call with modifier 1:
    the modifier scales (scales, rotations) only."""
    sc = _pre_case(3, 16, 1.7, seed=71, cov3d=True)
    pre, _ = T.check_preprocess("C3_cov3D_precomp", sc)
    sc, _, _ = R64.margin_scene(sc, device=DEV)
    a = _kernel_outputs(sc)
    _assert_bit_equal(a, _kernel_outputs(dict(sc, cam=dict(sc["cam"], scale_modifier=1.0)), a["grad2d"]))


VARIANT_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import test_camera64_gpu as T
T.test_preprocess_per_element(1)
T.test_inactive_coefficients_never_read(1, 16, float("nan"))
print("OK")
"""


def test_preprocess_without_tma():
    """SGR_NO_TMA=1 (read once per process, so in a fresh interpreter): the staged backward at (D, M) = (1, 16)."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = VARIANT_SCRIPT.format(root=os.path.dirname(here), tests=here)
    p = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, SGR_NO_TMA="1"), capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]


@pytest.mark.parametrize("fill", [float("nan"), float("inf")], ids=["nan", "inf"])
@pytest.mark.parametrize("D,M", [(1, 16), (1, 9), (3, 25), (0, 4)], ids=["tma", "staged", "unstaged", "tma_M4"])
def test_inactive_coefficients_never_read(D, M, fill):
    """Coefficients beyond the active degree seeded with NaN / +Inf: images, radii and every gradient bit-equal to the run with
    zeros there, their own gradients exactly +0, dL/dmeans3D finite.  (The reference never reads them.)"""
    cam = CC.camera("C3", 96, 64, sh_degree=D, scale_modifier=0.6)
    sc, _, _ = R64.margin_scene(T.preprocess_scene(D, 80 + M, cam=cam, sh_coeffs=M), device=DEV)
    n = (D + 1) ** 2
    clean, dirty = dict(sc, shs=sc["shs"].clone()), dict(sc, shs=sc["shs"].clone())
    clean["shs"][:, n:] = 0.0
    dirty["shs"][:, n:] = fill
    a = _kernel_outputs(clean)
    b = _kernel_outputs(dirty, a["grad2d"])
    _assert_bit_equal(a, b)
    g = b["g_shs"]
    assert (g[:, n:] == 0).all() and not torch.signbit(g[:, n:]).any(), "inactive coefficients get +0"
    assert torch.isfinite(b["g_means3D"]).all() and float(b["g_means3D"].abs().max()) > 0
    assert int((b["radii"] > 0).sum()) > 50


# ------------------------------------------------------------------------------------------------ end to end, visibility
def test_end_to_end_autograd_waymo_camera():
    """GaussianRasterizer + autograd against render64 under C2, with semantics and scale_modifier 0.6 (SH degree 3)."""
    cam = CC.camera("C2", 96, 64, sh_degree=3, scale_modifier=0.6)
    T.check_end_to_end("C2_end_to_end", RC.cat_scenes(T.preprocess_scene(3, 31, cam=cam), T.preprocess_scene(3, 32, cam=cam)))


def test_visible_filter_and_mark_visible():
    """visible_filter under C3 (scale_modifier 1.7): radii exact against preprocess64, means2D within check_preprocess's pixel
    bound; markVisible: view depth > 0.2 exactly."""
    cam = CC.camera("C3", 96, 64, sh_degree=1, scale_modifier=1.7)
    sc, _, _ = R64.margin_scene(T.preprocess_scene(1, 90, cam=cam, sh_coeffs=4), device=DEV)
    # points behind the near plane (z_view in (-0.2, 0.15)) for markVisible / the near cull
    g = torch.Generator().manual_seed(91)
    m, rot = RC.to_world(cam, torch.stack([torch.rand(12, generator=g, dtype=torch.float64) * 0.2 - 0.1,
                                           torch.rand(12, generator=g, dtype=torch.float64) * 0.2 - 0.1,
                                           torch.rand(12, generator=g, dtype=torch.float64) * 0.35 - 0.2], 1),
                         torch.tensor([[1.0, 0.0, 0.0, 0.0]], dtype=torch.float64).expand(12, 4))
    sc = dict(sc, means3D=torch.cat([sc["means3D"], m.float()]), rotations=torch.cat([sc["rotations"], rot.float()]),
              scales=torch.cat([sc["scales"], sc["scales"][:12]]), opacities=torch.cat([sc["opacities"], sc["opacities"][:12]]),
              shs=torch.cat([sc["shs"], sc["shs"][:12]]))
    pre = R64.preprocess64(sc, DEV)
    rast = sgb.GaussianRasterizer(util.settings_from(sgb, sc["cam"], DEV))
    radii, m2d = rast.visible_filter(sc["means3D"].to(DEV), sc["scales"].to(DEV), sc["rotations"].to(DEV))
    assert torch.equal(radii, pre["radii"].to(torch.int32))
    vis = pre["vis"]
    e = R64.EPS32 * 64.0
    ref = pre["rec"]
    for c, dim in ((0, "W"), (1, "H")):
        bnd = e * (1 + ref[:, c].abs() + 0.5 * pre["cam"][dim] * pre["ndc_mass"][:, c])
        assert ((m2d[:, c].double() - ref[:, c]).abs()[vis] <= bnd[vis]).all(), c
    assert (m2d[~vis] == 0).all()
    present = rast.markVisible(sc["means3D"].to(DEV))
    assert torch.equal(present, pre["tz"] > 0.2)
    assert int((~present).sum()) >= 6 and int(present.sum()) > 50


# ------------------------------------------------------------------------------------------------ layers, sharded step
def test_layered_gradients_waymo_camera():
    """test_layers_gpu's per-element layered check under C2."""
    import test_layers_gpu as TL
    cam = CC.camera("C2", 96, 64, sh_degree=3)
    a = T.preprocess_scene(3, 51, cam=cam)
    TL.check_layered(RC.cat_scenes(a, T.preprocess_scene(3, 52, cam=cam)), a["means3D"].shape[0])


def test_fused_sharded_step_waymo_camera():
    """test_sharded64_gpu's fused forward + backward on two emulated ranks (case w2_tail, M = 16: the TMA gather) under C2."""
    import test_sharded64_gpu as TS
    TS.run_fused("w2_tail", D=3, compact=True, expect="tma", frames=1, camera=lambda W, H, D: CC.camera("C2", W, H, sh_degree=D))


# ------------------------------------------------------------------------------------------------ error paths
@pytest.mark.parametrize("D,M", [(3, 9), (2, 4)])
def test_sh_degree_above_stored_coefficients_is_rejected(D, M):
    """An active degree that needs more coefficients than stored raises before any kernel is launched."""
    cam = CC.camera("C2", 96, 64, sh_degree=D)
    sc = T.preprocess_scene(D, 95, cam=cam)
    sc["shs"] = sc["shs"][:, :M].contiguous()
    L = _capi.lib()
    torch.cuda.synchronize()
    n0 = L.sgr_launch_count()
    with pytest.raises(_capi.SgrError, match="SH degree"):
        util.run_api(sgb, sc, backward=False)
    assert L.sgr_launch_count() == n0


def test_misaligned_views_are_realigned():
    """rotations and shs as views at a storage offset of one float into a flat buffer (what a slice of a flat parameter buffer
    gives): images, records and the chain rule's gradients bit-equal to the same call on aligned copies; through autograd the
    gradients reach the flat buffers and agree with the aligned call up to the blend's atomic summation order."""
    cam = CC.camera("C2", 96, 64, sh_degree=3)
    sc, _, _ = R64.margin_scene(T.preprocess_scene(3, 96, cam=cam), device=DEV)
    P = sc["means3D"].shape[0]
    flat_r = torch.cat([torch.zeros(1), sc["rotations"].reshape(-1)]).to(DEV)
    flat_s = torch.cat([torch.zeros(1), sc["shs"].reshape(-1)]).to(DEV)
    rot, shs = flat_r[1:].view(P, 4), flat_s[1:].view(P, 16, 3)
    assert rot.data_ptr() % 16 == 4 and shs.data_ptr() % 16 == 4 and rot.is_contiguous() and shs.is_contiguous()
    a = _kernel_outputs(sc)
    _assert_bit_equal(a, _kernel_outputs(dict(sc, rotations=rot, shs=shs), a["grad2d"]))

    ref = util.run_api(sgb, sc)
    st = util.settings_from(sgb, sc["cam"], DEV)
    flat_r.requires_grad_(True)
    flat_s.requires_grad_(True)
    rot, shs = flat_r[1:].view(P, 4), flat_s[1:].view(P, 16, 3)
    leaf = {k: sc[k].to(DEV).clone().requires_grad_(True) for k in ("means3D", "opacities", "scales")}
    m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
    color, radii, depth, alpha, _ = sgb.GaussianRasterizer(st)(means2D=m2d, shs=shs, rotations=rot, **leaf)
    loss = (color * sc["grad_color"].to(DEV)).sum() + (depth * sc["grad_depth"].to(DEV)).sum() + (alpha * sc["grad_alpha"].to(DEV)).sum()
    loss.backward()
    torch.cuda.synchronize()
    for key, v in dict(color=color, radii=radii, depth=depth, alpha=alpha).items():
        assert np.array_equal(v.detach().cpu().numpy(), ref[key]), key
    got = dict(g_means3D=leaf["means3D"].grad, g_means2D=m2d.grad, g_opacities=leaf["opacities"].grad, g_scales=leaf["scales"].grad,
               g_rotations=flat_r.grad[1:].view(P, 4), g_shs=flat_s.grad[1:].view(P, 16, 3))
    for key, v in got.items():
        assert util.rel_err(v.cpu().numpy(), ref[key]) < 1e-5, key
    assert float(flat_r.grad[0]) == 0.0 and float(flat_s.grad[0]) == 0.0
