"""GPU: render layers (GaussianRasterizer.forward_layers, include/sgr.h SgrLayer).  A layer's images equal a separate call on the
sliced tensors bit for bit, the main outputs equal the call without layers, the gradients equal those of the two separate calls,
the main means2D receives the main images' screen-space gradient only, and a bounded-mode layered step captures in a CUDA graph."""
import pytest
import torch

import street_gaussians_b200 as sgb
import util
from oracle import raster64 as R64
from street_gaussians_b200 import _capi, losses, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"
WHITE = (1.0, 1.0, 1.0)


def _composed(W, H, seed, P=3000, n_vehicles=3, per_vehicle=500, requires_grad=False):
    """Background + actors through compose (background rows first, as the composer orders them); returns the raw leaves too."""
    scene = synthetic.make_scene(P=P, width=W, height=H, sh_degree=3, seed=seed, n_vehicles=n_vehicles, per_vehicle=per_vehicle,
                                 with_raw=True, scale_med=0.05)
    raw = scene["raw"]
    models = [{k: v.to(DEV).clone().requires_grad_(requires_grad) for k, v in m.items()} for m in raw["models"]]
    poses = raw["poses"].to(DEV).clone().requires_grad_(requires_grad)
    return scene, models, poses, raw["idft"].to(DEV), P


def _cov6(scales, rot):
    q = rot / rot.norm(dim=1, keepdim=True)
    r, x, y, z = q.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    Mm = R * scales[:, None, :]
    S = Mm @ Mm.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1).contiguous()


def _inputs(variant, xyz, rot, scale, opac, sh, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    kw = dict(means3D=xyz, opacities=opac)
    if variant == "colors_precomp":
        kw["colors_precomp"] = torch.rand(xyz.shape[0], 3, generator=g, device=DEV)
    else:
        kw["shs"] = sh
    if variant == "cov3D_precomp":
        kw["cov3D_precomp"] = _cov6(scale, rot)
    else:
        kw.update(scales=scale, rotations=rot)
    if variant == "semantics":
        kw["semantics"] = torch.rand(xyz.shape[0], 3, generator=g, device=DEV)
    return kw


def _slice(kw, b, e):
    return {k: v[b:e] for k, v in kw.items() if k != "semantics"}


def _separate(st, kw, b, e, bg, capacity=None):
    s = st._replace(bg=torch.tensor(bg, dtype=torch.float32, device=DEV))
    color, radii, depth, alpha, _ = sgb.GaussianRasterizer(s, capacity=capacity)(means2D=None, **_slice(kw, b, e))
    return color, radii, depth, alpha


def _bg_image(bg, H, W):
    return torch.tensor(bg, dtype=torch.float32, device=DEV).reshape(3, 1, 1).expand(3, H, W)


@pytest.mark.parametrize("variant", ["sh", "colors_precomp", "cov3D_precomp", "semantics"])
@pytest.mark.parametrize("W,H", [(320, 208), (301, 197)])
@pytest.mark.parametrize("bounded", [False, True])
def test_layers_equal_separate_calls(W, H, variant, bounded):
    scene, models, poses, idft, nb = _composed(W, H, seed=W + len(variant))
    st = util.settings_from(sgb, scene["cam"], DEV)
    with torch.no_grad():
        xyz, rot, scale, opac, sh = sgb.compose(models, poses, idft)
        kw = _inputs(variant, xyz, rot, scale, opac, sh, seed=W)
        P = xyz.shape[0]
        cap = sgb.InstanceCapacity() if bounded else None
        if bounded:  # one exact frame learns the instance count; the calls below then run sync-free
            sgb.GaussianRasterizer(st, capacity=cap)(means2D=None, **kw)
        rast = sgb.GaussianRasterizer(st, capacity=cap)
        main = rast(means2D=None, **kw)
        specs = [(nb, P, WHITE), (0, nb, WHITE), (nb // 2, nb + 700, (0.2, 0.3, 0.4)), (nb, nb, (0.5, 0.1, 0.9)),
                 (0, P, (0.1, 0.1, 0.1)), (nb // 3, P - 100, (0.0, 0.0, 0.0))]
        out = rast.forward_layers(means2D=None, layers=[sgb.RenderLayer(b, e, bg) for b, e, bg in specs], **kw)
        assert len(out) == 6 and len(out[5]) == len(specs)
        for a, b_ in zip(out[:5], main):
            assert torch.equal(a, b_)
        for (b, e, bg), (c, d, a) in zip(specs, out[5]):
            assert c.shape == (3, H, W) and d.shape == (1, H, W) and a.shape == (1, H, W)
            if b == e:
                assert torch.equal(c, _bg_image(bg, H, W)) and not d.any() and not a.any()
                continue
            sc, sr, sd, sa = _separate(st, kw, b, e, bg, cap)
            assert torch.equal(sr, main[1][b:e])
            assert torch.equal(c, sc) and torch.equal(d, sd) and torch.equal(a, sa), (b, e)
            assert (a > 0).any()
        if bounded:
            rast.synchronize_capacity()


def _train_loss(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(3, H, W, generator=g).to(DEV)
    mask = (torch.rand(1, H, W, generator=g) > 0.1).to(DEV)
    sky = (torch.rand(1, H, W, generator=g) > 0.8).to(DEV)
    obj_bound = (torch.rand(1, H, W, generator=g) > 0.6).to(DEV)
    u_c = (torch.randn(3, H, W, generator=g) / (H * W)).to(DEV)
    u_d = (torch.randn(1, H, W, generator=g) / (H * W)).to(DEV)

    def loss(color, acc, obj_color, obj_depth, obj_acc):
        return losses.photometric_loss(color, gt, mask, 1.0, 0.2) + losses.sky_loss(acc, sky, 0.05) + \
            losses.obj_acc_loss(obj_acc, obj_bound, 0.1) + (u_c * obj_color).sum() + (u_d * obj_depth).sum()
    return loss


@pytest.mark.parametrize("bounded", [False, True])
def test_layer_gradients_equal_two_calls(bounded):
    W, H = 320, 208
    loss_fn = _train_loss(H, W, 5)
    runs = []
    for layered in (True, False):
        scene, models, poses, idft, nb = _composed(W, H, seed=41, requires_grad=True)
        st = util.settings_from(sgb, scene["cam"], DEV)
        cap = None
        if bounded:
            cap = sgb.InstanceCapacity()
            with torch.no_grad():
                xyz, rot, scale, opac, sh = sgb.compose(models, poses, idft)
                sgb.GaussianRasterizer(st, capacity=cap)(means3D=xyz, means2D=None, opacities=opac, shs=sh, scales=scale, rotations=rot)
        xyz, rot, scale, opac, sh = sgb.compose(models, poses, idft)
        P = xyz.shape[0]
        m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
        s2d = torch.zeros(P - nb, 3, device=DEV, requires_grad=True)
        rast = sgb.GaussianRasterizer(st, capacity=cap)
        kw = dict(means3D=xyz, opacities=opac, shs=sh, scales=scale, rotations=rot)
        if layered:
            color, radii, depth, acc, _, ((oc, od, oa),) = rast.forward_layers(means2D=m2d, layers=[sgb.RenderLayer(nb, P, WHITE, s2d)], **kw)
        else:
            color, radii, depth, acc, _ = rast(means2D=m2d, **kw)
            oc, _, od, oa, _ = sgb.GaussianRasterizer(st._replace(bg=torch.ones(3, device=DEV)), capacity=cap)(
                means2D=s2d, **{k: v[nb:] for k, v in kw.items()})
        loss = loss_fn(color, acc, oc, od, oa)
        loss.backward()
        if bounded:
            rast.synchronize_capacity()
        r = dict(color=color.detach(), depth=depth.detach(), acc=acc.detach(), oc=oc.detach(), od=od.detach(), oa=oa.detach(),
                 loss=float(loss), g_poses=poses.grad, g_m2d=m2d.grad, g_s2d=s2d.grad)
        for i, m in enumerate(models):
            for k, v in m.items():
                r[f"g_{i}_{k}"] = v.grad
        runs.append(r)
    a, b = runs
    for k in ("color", "depth", "acc", "oc", "od", "oa"):
        assert torch.equal(a[k], b[k]), k
    assert abs(a["loss"] - b["loss"]) <= 1e-6 * abs(b["loss"])
    for k in a:
        if k.startswith("g_"):
            e = util.rel_err(a[k].cpu().numpy(), b[k].cpu().numpy())
            bar = 1e-5 if k in ("g_m2d", "g_s2d") else 1e-3  # the screen-space sums are the blend's own atomics, not a chain rule
            assert e <= bar, (k, e)
    assert a["g_m2d"].abs().sum() > 0 and a["g_s2d"].abs().sum() > 0


def test_layer_gradient_never_reaches_the_main_means2D():
    W, H = 256, 160
    scene, models, poses, idft, nb = _composed(W, H, seed=7, requires_grad=True)
    st = util.settings_from(sgb, scene["cam"], DEV)
    xyz, rot, scale, opac, sh = sgb.compose(models, poses, idft)
    P = xyz.shape[0]
    m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
    s2d = torch.zeros(P - nb, 3, device=DEV, requires_grad=True)
    out = sgb.GaussianRasterizer(st).forward_layers(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot,
                                                    layers=[sgb.RenderLayer(nb, P, WHITE, s2d), sgb.RenderLayer(0, nb, WHITE)])
    bound = torch.zeros(1, H, W, dtype=torch.bool, device=DEV)
    bound[:, H // 4:, :] = True
    losses.obj_acc_loss(out[5][0][2], bound, 0.1).backward()
    assert m2d.grad is not None and not m2d.grad.any()
    assert s2d.grad.abs().sum() > 0 and poses.grad.abs().sum() > 0
    assert models[0]["xyz"].grad is not None and not models[0]["xyz"].grad.any()  # the background rows lie outside the layer
    assert all(m["xyz"].grad.abs().sum() > 0 and m["opacity"].grad.abs().sum() > 0 for m in models[1:])


def test_layered_bounded_step_captures_in_a_cuda_graph():
    W, H = 256, 160
    base = synthetic.make_scene(P=6000, width=W, height=H, sh_degree=3, seed=3, n_vehicles=2, per_vehicle=800, scale_med=0.05)
    nb = 6000
    st = util.settings_from(sgb, base["cam"], DEV)
    loss_fn = _train_loss(H, W, 9)
    keys = ("means3D", "shs", "opacities", "scales", "rotations")
    white = torch.ones(3, device=DEV)

    def scene(seed):
        g = torch.Generator().manual_seed(seed)
        out = {k: base[k].clone() for k in keys}
        out["means3D"] += 0.02 * torch.randn(out["means3D"].shape, generator=g)
        out["shs"] += 0.1 * torch.randn(out["shs"].shape, generator=g)
        return {k: v.to(DEV) for k, v in out.items()}

    cap = sgb.InstanceCapacity(headroom=1.5)
    rast = sgb.GaussianRasterizer(st, capacity=cap)
    static = {k: v.requires_grad_(True) for k, v in scene(1).items()}
    P = static["means3D"].shape[0]
    m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
    s2d = torch.zeros(P - nb, 3, device=DEV, requires_grad=True)
    leaves = list(static.values()) + [m2d, s2d]

    def step(t, a, b):
        out = rast.forward_layers(means2D=a, layers=[sgb.RenderLayer(nb, P, white, b)], **t)
        (oc, od, oa), = out[5]
        loss_fn(out[0], out[3], oc, od, oa).backward()
        return torch.cat([out[0], out[2], out[3], oc, od, oa])

    with torch.no_grad():  # exact frames learn the instance count; then the capacity is frozen
        for seed in (1, 2, 3):
            sgb.GaussianRasterizer(st, capacity=cap)(means2D=None, **scene(seed))
    cap.freeze()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for x in leaves:
                x.grad = None
            step(static, m2d, s2d)
    torch.cuda.current_stream().wait_stream(s)
    for x in leaves:
        x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        imgs_g = step(static, m2d, s2d)
    for seed in (2, 3):
        new = scene(seed)
        with torch.no_grad():
            for k, v in new.items():
                static[k].copy_(v)
        graph.replay()
        new = {k: v.requires_grad_(True) for k, v in new.items()}
        a, b = torch.zeros_like(m2d, requires_grad=True), torch.zeros_like(s2d, requires_grad=True)
        imgs_e = step(new, a, b)
        torch.cuda.synchronize()
        assert torch.equal(imgs_g, imgs_e)
        for k in keys:
            assert util.rel_err(static[k].grad.cpu().numpy(), new[k].grad.cpu().numpy()) <= 1e-5, k
        for x, y in ((m2d, a), (s2d, b)):
            assert util.rel_err(x.grad.cpu().numpy(), y.grad.cpu().numpy()) <= 1e-5
    cap.freeze(False)
    rast.synchronize_capacity()


def _margin_pair(sc, b):
    """A scene whose full render AND whose render of rows [b, P) both have no near-threshold decision (raster64.margin_scene on each,
    the rows the subset's pass drops removed from the full scene too, until both are clean).  Returns (scene, b)."""
    for _ in range(6):
        sc, _, keep = R64.margin_scene(sc, device=DEV)
        b = int((keep < b).sum())
        P = sc["means3D"].shape[0]
        _, removed, keep_sub = R64.margin_scene(R64.subset(sc, torch.arange(b, P)), device=DEV)
        if removed == 0:
            return sc, b
        keep_all = torch.cat([torch.arange(b), b + keep_sub])
        sc = R64.subset(sc, keep_all)
    raise AssertionError("margin scenes did not converge")


def test_layered_gradients_per_element_vs_float64():
    """The layered call's per-input gradients against render64(full) + render64(layer rows) in float64: the chain rule is applied to
    the summed screen-space sums (exactly what the layered backward evaluates), with the bounds of test_raster64_gpu's end-to-end
    check plus one fp32 rounding of the summed rows.  The main means2D against the full render's, the layer's sink against the layer
    render's; the layer images against the layer render."""
    import raster64_case as RC
    import test_raster64_gpu as T
    sc = RC.cat_scenes(T.preprocess_scene(D=3, seed=51), T.preprocess_scene(D=3, seed=52))
    b0 = T.preprocess_scene(D=3, seed=51)["means3D"].shape[0]
    sc["cam"]["bg"] = torch.tensor([0.1, 0.2, 0.3])
    sc, b = _margin_pair(sc, b0)
    P = sc["means3D"].shape[0]
    assert 0 < b < P
    H, W = sc["cam"]["image_height"], sc["cam"]["image_width"]
    gen = torch.Generator().manual_seed(53)
    lbg = (0.9, 0.7, 0.5)
    up = {k: torch.randn(c, H, W, generator=gen) / (H * W) for k, c in (("color", 3), ("depth", 1), ("alpha", 1))}
    leaf = {k: sc[k].to(DEV).clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
    s2d = torch.zeros(P - b, 3, device=DEV, requires_grad=True)
    st = util.settings_from(sgb, sc["cam"], DEV)
    out = sgb.GaussianRasterizer(st).forward_layers(means2D=m2d, layers=[sgb.RenderLayer(b, P, lbg, s2d)], **leaf)
    (lc, ld, la), = out[5]
    loss = sum((out[i] * sc["grad_" + k].to(DEV)).sum() for i, k in ((0, "color"), (2, "depth"), (3, "alpha"))) + \
        sum((x * up[k].to(DEV)).sum() for x, k in ((lc, "color"), (ld, "depth"), (la, "alpha")))
    loss.backward()

    r = R64.render64(sc, DEV, alpha_img=out[3].detach().cpu())
    sub = R64.subset(sc, torch.arange(b, P))
    sub["cam"] = dict(sc["cam"], bg=torch.tensor(lbg))
    sub.update(grad_color=up["color"], grad_depth=up["depth"], grad_alpha=up["alpha"])
    rs = R64.render64(sub, DEV, alpha_img=la.detach().cpu())
    cond = float(r["pre"]["cond"][r["pre"]["vis"]].max())
    t_rec = R64.EPS32 * 64.0 * (1 + cond) * (1 + max(W, H))
    for key, got in (("color", lc), ("depth", ld), ("alpha", la)):
        bl = rs["blend"]
        err = (got.detach().double() - rs[key]).abs()
        assert (err <= R64.bound(bl["kmass_" + key]) + t_rec * bl["mass_" + key] + 1e-300).all(), key

    def masses(res):
        bl, vis = res["blend"], res["pre"]["vis"].to(torch.float64)[:, None]
        nt = bl["ntiles"].to(torch.float64)[:, None]
        return res["grad2d"], bl["mass_grad2d"] * vis, (bl["kmass_grad2d"] + nt * bl["mass_grad2d"]) * vis

    (g, m, k), (gs, ms, ks) = masses(r), masses(rs)
    g, m, k = g.clone(), m.clone(), k.clone()
    g[b:] += gs
    m[b:] += ms
    k[b:] += ks
    comb = R64.chain64(r["pre"], g, m, k)
    for key, t in (("g_means3D", leaf["means3D"]), ("g_shs", leaf["shs"]), ("g_opacities", leaf["opacities"]),
                   ("g_scales", leaf["scales"]), ("g_rotations", leaf["rotations"])):
        ref = comb[key]
        got = t.grad.double().reshape(ref.shape)
        rowmax = ref.abs().reshape(ref.shape[0], -1).amax(1).reshape((-1,) + (1,) * (ref.dim() - 1))
        bnd = R64.chain_bound(comb, key) + R64.EPS32 * comb["mass_" + key] + t_rec * rowmax + 1e-300
        assert ((got - ref).abs() <= bnd).all(), (key, float(((got - ref).abs() / bnd).max()))
    for got, res in ((m2d.grad, r), (s2d.grad, rs)):
        ref = res["g_means2D"][:, :2]
        bnd = (R64.EPS32 * res["kmass_g_means2D"])[:, :2] + t_rec * ref.abs().amax(1, keepdim=True) + 1e-300
        assert ((got[:, :2].double() - ref).abs() <= bnd).all()
    assert s2d.grad.abs().sum() > 0 and m2d.grad.abs().sum() > 0


def test_layer_edge_cases():
    W, H = 96, 64
    st = util.settings_from(sgb, synthetic.make_camera(W, H), DEV)
    rast = sgb.GaussianRasterizer(st)
    # P == 0: the main outputs keep the rasterizer's zero short-circuit, a layer is colour bg with zero depth and alpha
    z = lambda *s: torch.zeros(*s, device=DEV, requires_grad=True)
    x, o, sh, sc, ro = z(0, 3), z(0, 1), z(0, 16, 3), z(0, 3), z(0, 4)
    out = rast.forward_layers(means3D=x, means2D=None, opacities=o, shs=sh, scales=sc, rotations=ro, layers=[sgb.RenderLayer(0, 0, WHITE)])
    assert not out[0].any() and out[1].numel() == 0
    c, d, a = out[5][0]
    assert torch.equal(c, _bg_image(WHITE, H, W)) and not d.any() and not a.any()
    (c.sum() + out[0].sum()).backward()
    assert x.grad.shape == (0, 3)
    # a range with no visible Gaussian (its rows sit behind the camera), and render_all's shape: no means2D, no grad
    scene = synthetic.make_scene(P=2000, width=W, height=H, sh_degree=3, seed=2, scale_med=0.05)
    kw = {k: scene[k].to(DEV) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    kw["means3D"][1500:, 2] = -5.0
    with torch.no_grad():
        out = rast.forward_layers(means2D=None, layers=[sgb.RenderLayer(1500, 2000, (0.3, 0.6, 0.9)), sgb.RenderLayer(0, 1500, WHITE),
                                                        sgb.RenderLayer(0, 2000, WHITE)], **kw)
    c, d, a = out[5][0]
    assert torch.equal(c, _bg_image((0.3, 0.6, 0.9), H, W)) and not d.any() and not a.any()
    assert not out[1][1500:].any() and out[1][:1500].any()
    for (b, e), (c, d, a) in zip(((0, 1500), (0, 2000)), out[5][1:]):
        sc_, _, sd, sa = _separate(st, kw, b, e, WHITE)
        assert torch.equal(c, sc_) and torch.equal(d, sd) and torch.equal(a, sa)
    # layers are whole-image, single-GPU
    with pytest.raises(_capi.SgrError):
        sgb.GaussianRasterizer(st, band=sgb.TileRowBand(0, 2, 1)).forward_layers(means2D=None, layers=[sgb.RenderLayer(0, 10, WHITE)], **kw)
    with pytest.raises(ValueError):
        rast.forward_layers(means2D=None, layers=[sgb.RenderLayer(0, 2001, WHITE)], **kw)
