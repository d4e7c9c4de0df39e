"""The saturation split of the forward (include/sgr.h sgr_set_near_budget, csrc/binning.cu): whatever the near budget B, the images,
radii, per-pixel contributor counts and per-tile list depths equal those of the one-pass binning (B >= R) bit for bit, and grad2d
equals it up to the float-atomic noise of the backward.  Scenes: config C; a sparse scene where no tile saturates; an opaque wall
that saturates every tile inside the near slab; a stack of screen-filling splats swept over every budget, so that some split falls
exactly on the instance that saturates a tile; a frame with partial edge tiles; a bounded frame that overflows its capacity; and
the frames that keep the one-pass binning (render layers, more than 16384 tiles)."""
import pytest
import torch

import util
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi
from street_gaussians_b200 import rasterizer as R
from street_gaussians_b200 import synthetic
from street_gaussians_b200._capi import STATUS_EMITTED, STATUS_INSTANCES, STATUS_NEAR_END, STATUS_OVERFLOW

pytestmark = pytest.mark.gpu
DEV = "cuda"
ALL, AUTO = _capi.NEAR_BUDGET_ALL, _capi.NEAR_BUDGET_AUTO


def render(scene, budget, capacity=None, backward=True):
    """Forward (+ backward blend) of `scene` with near budget `budget`: images, radii, n_contrib, tile_max_contrib, the status words
    and grad2d."""
    cam = scene["cam"]
    st = util.settings_from(sgb, cam, DEV)
    dv = lambda k: scene[k].to(DEV) if scene.get(k) is not None else None
    P = scene["means3D"].shape[0]
    W, H = cam["image_width"], cam["image_height"]
    cap = sgb.InstanceCapacity(initial=capacity) if capacity else None
    with torch.no_grad(), _capi.near_budget(budget):
        color, radii, depth, alpha, _, fst, tensors = R._forward_impl(dv("means3D"), dv("shs"), None, None, dv("opacities"), dv("scales"),
                                                                      dv("rotations"), None, st, None, cap)
    v = R.state_views(st, fst, P)
    out = dict(color=color, depth=depth, alpha=alpha, radii=radii, tile_max=v["tile_max_contrib"].clone(), n_contrib=v["n_contrib"].clone(),
               status=v["status"].cpu())
    if backward:
        gen = torch.Generator().manual_seed(7)
        g = lambda c: (torch.randn(c, H, W, generator=gen) / (H * W)).to(DEV)
        with torch.no_grad():
            out["grad2d"], _ = R._backward_blend_impl(st, None, fst, tensors, alpha, g(3), g(1), g(1), None)
    torch.cuda.synchronize()
    return out


def assert_same(ref, got, noise=None, what=""):
    for k in ("color", "depth", "alpha", "radii", "n_contrib", "tile_max"):
        assert torch.equal(ref[k], got[k]), (what, k)
    if "grad2d" in ref and "grad2d" in got:
        tol = max(4 * noise if noise is not None else 0.0, 1e-5 * float(ref["grad2d"].abs().max()))
        assert float((ref["grad2d"] - got["grad2d"]).abs().max()) <= tol, (what, "grad2d")


def splats(cam, px, py, z, sigma_px, opacity, seed=0):
    """Isotropic Gaussians centred on pixels (px, py) at view depth z with a screen-space sigma of about sigma_px pixels."""
    gen = torch.Generator().manual_seed(seed)
    W, H = cam["image_width"], cam["image_height"]
    px, py, z = px.double(), py.double(), z.double()
    x = ((2 * px + 1) / W - 1) * z * cam["tanfovx"]
    y = ((2 * py + 1) / H - 1) * z * cam["tanfovy"]
    fx = W / (2 * cam["tanfovx"])
    n = px.numel()
    s = (torch.as_tensor(sigma_px, dtype=torch.float64) * z / fx).reshape(-1, 1).expand(n, 3)
    return dict(means3D=torch.stack([x, y, z], 1).float(), scales=s.float().contiguous(), rotations=torch.tensor([[1.0, 0, 0, 0]]).repeat(n, 1),
                opacities=torch.as_tensor(opacity, dtype=torch.float32).reshape(-1, 1).expand(n, 1).contiguous(),
                shs=torch.rand(n, 1, 3, generator=gen))


def scene_of(cam, *parts):
    out = dict(cam=cam)
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        out[k] = torch.cat([p[k] for p in parts]).contiguous()
    return out


def wall_scene(W, H, seed=0, layers=3, background=20000):
    """`layers` opaque walls of overlapping splats (4 px apart, sigma 6 px, opacity 0.99) in front of `background` random splats."""
    cam = synthetic.make_camera(W, H, sh_degree=0)
    gy, gx = torch.meshgrid(torch.arange(0, H, 4), torch.arange(0, W, 4), indexing="ij")
    walls = [splats(cam, gx.flatten(), gy.flatten(), torch.full((gx.numel(),), 2.0 + 0.1 * k), 6.0, 0.99, seed + k) for k in range(layers)]
    gen = torch.Generator().manual_seed(seed + 100)
    n = background
    bg = splats(cam, torch.rand(n, generator=gen) * W, torch.rand(n, generator=gen) * H, 5 + 40 * torch.rand(n, generator=gen),
                1 + 10 * torch.rand(n, generator=gen), 0.3 + 0.6 * torch.rand(n, generator=gen), seed + 200)
    return scene_of(cam, *walls, bg), scene_of(cam, *walls)


@pytest.fixture(scope="module")
def config_c():
    return synthetic.make_config("C", seed=0)


def test_config_C(config_c):
    full = render(config_c, ALL)
    noise = float((render(config_c, ALL)["grad2d"] - full["grad2d"]).abs().max())
    Rn = int(full["status"][STATUS_INSTANCES])
    assert int(full["status"][STATUS_EMITTED]) == Rn
    for b in (AUTO, 0, Rn // 64, Rn // 4, Rn - 1):
        got = render(config_c, b)
        assert_same(full, got, noise, f"B={b}")
        assert int(got["status"][STATUS_INSTANCES]) == Rn
    auto = render(config_c, AUTO, backward=False)
    assert int(auto["status"][STATUS_EMITTED]) < Rn // 2  # most instances lie behind saturated pixels


def test_no_tile_saturates():
    cam = synthetic.make_camera(640, 480, sh_degree=0)
    gen = torch.Generator().manual_seed(5)
    n = 3000
    sc = scene_of(cam, splats(cam, torch.rand(n, generator=gen) * 640, torch.rand(n, generator=gen) * 480, 3 + 30 * torch.rand(n, generator=gen),
                              2 + 6 * torch.rand(n, generator=gen), 0.05))
    full = render(sc, ALL)
    for b in (AUTO, 0, 1, int(full["status"][STATUS_INSTANCES]) // 3):
        got = render(sc, b)
        assert_same(full, got, what=f"B={b}")
        assert int(got["status"][STATUS_EMITTED]) == int(full["status"][STATUS_INSTANCES])  # nothing saturates, so every instance is emitted


def test_every_tile_saturates_in_the_near_slab():
    sc, walls = wall_scene(640, 480)
    R_wall = int(render(walls, ALL, backward=False)["status"][STATUS_INSTANCES])
    full = render(sc, ALL)
    assert int(full["status"][STATUS_INSTANCES]) > R_wall
    got = render(sc, R_wall)
    assert_same(full, got, what="B = the walls' instances")
    st = got["status"]
    assert int(st[STATUS_NEAR_END]) == R_wall and int(st[STATUS_EMITTED]) == R_wall  # the far pass found no unsaturated tile
    for b in (AUTO, 0, R_wall // 2, R_wall + 1):
        assert_same(full, render(sc, b), what=f"B={b}")


def test_every_split_of_a_stack():
    """Ten splats covering the whole 64 x 48 frame at alpha ~0.8, one behind the other: the tiles saturate at the sixth.  Every
    budget from 0 to R is rendered, so the split also falls right behind the instance that saturates each tile."""
    cam = synthetic.make_camera(64, 48, sh_degree=0)
    n = 10
    sc = scene_of(cam, splats(cam, torch.full((n,), 31.5), torch.full((n,), 23.5), 1.0 + torch.arange(n), 400.0, 0.8))
    full = render(sc, ALL)
    Rn = int(full["status"][STATUS_INSTANCES])
    assert Rn == n * 12
    saturated_in_near = 0
    for b in range(Rn + 1):
        got = render(sc, b)
        assert_same(full, got, what=f"B={b}")
        st = got["status"]
        if int(st[STATUS_NEAR_END]) < Rn and int(st[STATUS_EMITTED]) == int(st[STATUS_NEAR_END]):  # every tile saturated inside the near slab
            saturated_in_near += 1
    assert saturated_in_near > 0


def test_partial_edge_tiles():
    sc, _ = wall_scene(1000, 700, seed=3, layers=2)
    full = render(sc, ALL)
    for b in (AUTO, 0, int(full["status"][STATUS_INSTANCES]) // 5):
        got = render(sc, b)
        assert_same(full, got, what=f"B={b}")
        if b != 0:  # (with B = 0 nothing is blended before the far pass, so every instance is emitted)
            assert int(got["status"][STATUS_EMITTED]) < int(full["status"][STATUS_INSTANCES])


def test_bounded_overflow():
    """A bounded frame overflows when the instances it emits exceed the capacity.  It then keeps the Gaussians whose whole instance
    counts fit, as the one-pass binning does, whatever the budget; a capacity between the split's emission and R renders it whole."""
    sc = synthetic.make_config("B", seed=1)
    exact = render(sc, ALL, backward=False)
    Rn = int(exact["status"][STATUS_INSTANCES])
    emitted = {b: int(render(sc, b, backward=False)["status"][STATUS_EMITTED]) for b in (AUTO, 0, Rn // 50)}
    cap = min(emitted.values()) // 2 + 3
    full = render(sc, ALL, capacity=cap)
    assert int(full["status"][STATUS_OVERFLOW]) & 1 and int(full["status"][STATUS_EMITTED]) <= cap
    for b in emitted:
        got = render(sc, b, capacity=cap)
        assert_same(full, got, what=f"B={b}")
        assert int(got["status"][STATUS_INSTANCES]) == Rn and int(got["status"][STATUS_OVERFLOW]) & 1 and int(got["status"][STATUS_EMITTED]) <= int(full["status"][STATUS_EMITTED])
    cap = emitted[AUTO] + 1000
    assert cap < Rn
    got = render(sc, AUTO, capacity=cap, backward=False)
    assert_same(exact, got, what="capacity between E and R")
    assert int(got["status"][STATUS_OVERFLOW]) == 0 and int(got["status"][STATUS_EMITTED]) == emitted[AUTO]


def test_more_tiles_than_bucketing_keeps_one_pass():
    sc = synthetic.make_scene(P=100_000, width=2064, height=2048, sh_degree=0, seed=2, scale_med=0.02)
    full = render(sc, ALL)
    got = render(sc, 0)
    assert_same(full, got, what="2064 x 2048")
    assert int(got["status"][STATUS_EMITTED]) == int(got["status"][STATUS_INSTANCES])


def test_layers_keep_one_pass():
    sc = synthetic.make_config("B", seed=1)
    P = sc["means3D"].shape[0]
    st = util.settings_from(sgb, sc["cam"], DEV)
    dv = {k: sc[k].to(DEV) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    m2d = torch.zeros((P, 3), device=DEV)
    b = P // 3
    with torch.no_grad(), _capi.near_budget(0):
        main = sgb.GaussianRasterizer(st).forward_layers(dv["means3D"], m2d, dv["opacities"], shs=dv["shs"], scales=dv["scales"],
                                                         rotations=dv["rotations"], layers=[R.RenderLayer(b, P, (1.0, 1.0, 1.0))])
        st1 = st._replace(bg=torch.ones(3, device=DEV))
        sep = sgb.GaussianRasterizer(st1)(dv["means3D"][b:], m2d[b:], dv["opacities"][b:], shs=dv["shs"][b:], scales=dv["scales"][b:],
                                          rotations=dv["rotations"][b:])
    (lc, ld, la), = main[5]
    assert torch.equal(lc, sep[0]) and torch.equal(ld, sep[2]) and torch.equal(la, sep[3])
    full = render(sc, ALL, backward=False)
    for k, i in (("color", 0), ("radii", 1), ("depth", 2), ("alpha", 3)):
        assert torch.equal(full[k], main[i]), k
