"""Render layers in the fused Gaussian-sharded step (sgr_sharded_forward_layers / sgr_sharded_backward_layers), with N ranks emulated on N
streams of one GPU on the scenes of tests/sharded64_case.py, two frames each, then two forwards in a row, the workspace poisoned (0x7f)
everywhere but the barrier pads.  Two layers per rank (tests/sharded_layers_case.py: a background-like head, empty on rank 0, and an
objects-like tail that covers rank 1 whole and ends at the last real row of the last rank), with different backgrounds.

Exact, per rank: main images, radii and status words as the plain fused call; every layer image zero outside the band, the ranks' layer
images summing bit for bit to a single-GPU render of the rank-major concatenation of the layer rows with that bg; the delivered layer bytes
equal to the host restatement; the main dL/dmeans2D bit-equal to the ascending-rank sum of the ranks' main rows (as the plain fused
backward leaves it); each layer sink equal to the ascending-rank
sum of the ranks' partial layer rows read from the sections; with no layer gradient, the launch count equal to the plain fused backward's and
every gradient equal to it up to the rounding of the blend's atomics.  Sensitivity on the kernel's own data: a range shifted by one row, a dropped mask run and the descending rank order each
fail these checks.  Through the module at world 1 against GaussianRasterizer.forward_layers: images bit-equal, gradients of one step
with the objects layer close to the single-GPU layered step's, and the layered
step captured in a CUDA graph replaying the eager images bit for bit."""
import pytest
import torch

import sharded64_case as SC
import sharded_layers_case as LC
import util
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi
from street_gaussians_b200 import rasterizer as R
from street_gaussians_b200 import sharded as SH
from oracle import raster64 as R64
from test_sharded64_gpu import GRAD_NAMES, _local, _ratio, _single, _warm_up_fused_path, band_mask

F64 = torch.float64

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
BGS = [torch.tensor([0.2, 0.5, 0.9]), torch.tensor([1.0, 1.0, 1.0])]  # (moved to the device where used)
REVERSED_DIFFERS = []
_warm = []


def _warm_up_layers():
    """Every kernel of the layered step loaded before ranks spin in emulated barriers (world 1 takes no barrier)."""
    _warm_up_fused_path(DEV)
    if _warm:
        return
    from street_gaussians_b200 import synthetic
    scene = synthetic.make_scene(P=3000, width=160, height=96, sh_degree=3, seed=1, pose=True)
    st = util.settings_from(sgb, scene["cam"], DEV)
    lt = _local(scene, 0, 3000)
    up = [scene[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
    ws = SH.PeerWorkspace.emulate(st, 3000, 1, DEV, layers=2)[0]
    with torch.no_grad():
        out = SH.sharded_forward_raw(st, None, ws, lt, 3000, 500_000, -1, layers=[(0, 1000, BGS[0]), (1000, 3000, BGS[1])])
        sinks = [torch.empty(1000, 3, device=DEV), torch.empty(2000, 3, device=DEV)]
        SH.sharded_backward_raw(st, None, ws, lt, 3000, 500_000, out[2], *up,
                                layers=[(0, 1000, BGS[0], out[4][0][2], up, sinks[0]), (1000, 3000, BGS[1], out[4][1][2], up, sinks[1])])
    torch.cuda.synchronize()
    _warm.append(True)


def _sub_scene(scene, ids):
    sub = dict(scene)
    for k in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp"):
        if scene.get(k) is not None:
            sub[k] = scene[k][ids.to(scene[k].device)]
    return sub


def _layer_reference(scene, st, P_r, ranges, k):
    ids = LC.layer_rows(P_r, ranges, k)
    out = _single(_sub_scene(scene, ids), st._replace(bg=BGS[k].to(DEV)))
    return out[0], out[2], out[3]


def _rows_by_rank(sections, smap, n_total, ascending=True):
    """Ascending (or descending) rank sum of the ranks' partial rows, each rank's row of a Gaussian read from its section at the slot the
    Gaussian was delivered to."""
    acc = torch.zeros((n_total, 12), device=DEV)
    for d in (range(len(smap)) if ascending else reversed(range(len(smap)))):
        sl, gids, _ = smap[d]
        part = torch.zeros_like(acc)
        part[gids.to(DEV)] = sections[d][sl.to(DEV)]
        acc = acc + part
    return acc


def _fp64_layered(tag, scene, rec, radii, alpha, l_alpha, lup, P_r, ranges, kg, l_sinks, world, worst):
    """kg: every rank's gradients (rank-major, GRAD_NAMES).  blend64 of the main frame (its bg and upstream) and of each layer (the
    records of its rows only, its bg, its upstream and alpha); dL/dmeans2D against the main rows, each layer's sink against that layer's
    rows, and every other gradient against chain64 of main + layers, each within the float64 bounds of a cross-rank sum."""
    cam = scene["cam"]
    W, H = int(cam["image_width"]), int(cam["image_height"])
    up = dict(color=scene["grad_color"], depth=scene["grad_depth"], alpha=scene["grad_alpha"])
    bl = R64.blend64(rec.double(), radii, W, H, cam["bg"], upstream=up, alpha_img=alpha)
    g2d, mass, kmass = bl["grad2d"].clone(), bl["mass_grad2d"].clone(), bl["kmass_grad2d"].clone()
    for k in range(2):
        rows = LC.layer_rows(P_r, ranges, k).to(radii.device)
        inside = torch.zeros_like(radii)
        inside[rows] = 1
        lb = R64.blend64(rec.double(), radii * inside, W, H, BGS[k], upstream=dict(color=lup[k][0], depth=lup[k][1], alpha=lup[k][2]),
                         alpha_img=l_alpha[k])
        err = (l_sinks[k].double() - lb["grad2d"][rows, 0:3]).abs()
        _ratio(worst, f"sink{k}", err, SC.sharded_bound(lb, world)[rows, 0:3], tag)
        g2d, mass, kmass = g2d + lb["grad2d"], mass + lb["mass_grad2d"], kmass + lb["kmass_grad2d"]
    pre = R64.preprocess64(scene, DEV, requires_grad=True)
    assert torch.equal(pre["radii"].to(torch.int32), radii), (tag, "radii vs preprocess64")
    vis = radii > 0
    nt = bl["ntiles"].to(F64)[:, None]
    # (the summed rows carry the main and both layers' cross-rank adds plus the two adds of main + layers)
    ch = R64.chain64(pre, g2d, mass, kmass + (nt + world + 2) * mass)
    n = 0
    for key, got in kg.items():
        if got is None:
            continue
        assert bool((got[~vis] == 0).all()), (tag, key, "gradient of a culled Gaussian")
        if key == "g_means2D":
            _ratio(worst, key, (got.double() - bl["grad2d"][:, 0:3]).abs(), SC.sharded_bound(bl, world)[:, 0:3], tag)
        else:
            ref = ch[key]
            _ratio(worst, key, (got.double().reshape(ref.shape) - ref).abs(), R64.chain_bound(ch, key), tag)
        n += 1
    assert n >= 5


def _run(wss, streams, fn):
    out = []
    with torch.no_grad():
        for r, ws in enumerate(wss):
            with torch.cuda.stream(streams[r]):
                out.append(fn(r, ws))
        torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", ["w2_tail", "w3_middle", "w5_empty_rank", "w8_empty_bands"])
def test_fused_layers_exact(name):
    _warm_up_layers()
    cases = [SC.build(name, seed=f, D=3, device=DEV) for f in range(2)]
    world, chunk, W, H = cases[0]["world"], cases[0]["chunk"], cases[0]["W"], cases[0]["H"]
    st = util.settings_from(sgb, cases[0]["scene"]["cam"], DEV)
    wss = SH.PeerWorkspace.emulate(st, chunk, world, DEV, layers=2)
    for ws in wss:
        ws.buf[: ws.off_flags].fill_(0x7f)
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    band = lambda r: SH.cyclic_band(H, r, world)
    worst = {}
    for fi, case in enumerate(cases):
        scene, P_r = case["scene"], case["P_r"]
        tag = f"{name} frame {fi}"
        offs = [sum(P_r[:r]) for r in range(world)]
        P = sum(P_r)
        st = util.settings_from(sgb, scene["cam"], DEV)
        locs = [_local(scene, offs[r], offs[r] + P_r[r]) for r in range(world)]
        up = [scene[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
        g = torch.Generator(device=DEV).manual_seed(300 + fi)
        lup = [[torch.randn(c, H, W, generator=g, device=DEV) for c in (3, 1, 1)] for _ in range(2)]
        ranges = LC.case_ranges(P_r)
        col, rad, dep, alp = _single(scene, st)[:4]
        capacity = int(_single(scene, st)[5].num_instances) + 1000
        gcap = -1 if fi == 0 else chunk * world
        # the plain fused step on the same workspaces: what the layered call must leave unchanged
        st_plain = [torch.zeros(8, dtype=torch.int32).pin_memory() for _ in range(world)]
        plain = _run(wss, streams, lambda r, ws: SH.sharded_forward_raw(st, band(r), ws, locs[r], P_r[r], capacity, gcap, st_plain[r]))
        plain_img = [tuple(t.clone() for t in o[:3]) for o in plain]
        plain_radii = [o[3]["radii"][:P_r[r]].clone() for r, o in enumerate(plain)]
        c0 = _capi.lib().sgr_launch_count()
        plain_g = _run(wss, streams, lambda r, ws: SH.sharded_backward_raw(st, band(r), ws, locs[r], P_r[r], capacity, plain[r][2], *up))
        plain_launches = _capi.lib().sgr_launch_count() - c0
        # ---- layered forward ----
        status = [torch.zeros(8, dtype=torch.int32).pin_memory() for _ in range(world)]
        tables = [[(b, e, BGS[k]) for k, (b, e) in enumerate(ranges[r])] for r in range(world)]
        outs = _run(wss, streams, lambda r, ws: SH.sharded_forward_raw(st, band(r), ws, locs[r], P_r[r], capacity, gcap, status[r],
                                                                       layers=tables[r]))
        for r in range(world):
            assert all(torch.equal(a, b) for a, b in zip(outs[r][:3], plain_img[r])), (tag, r, "main images")
            assert torch.equal(outs[r][3]["radii"][:P_r[r]], plain_radii[r]), (tag, r, "radii")
            assert torch.equal(status[r], st_plain[r]) and int(status[r][4]) == 0 and int(status[r][1]) == 0, (tag, r, status[r], st_plain[r])
        assert torch.equal(sum(o[0] for o in outs), col) and torch.equal(torch.cat([o[3]["radii"][:n] for o, n in zip(outs, P_r)]), rad)
        for k in range(2):
            ref = _layer_reference(scene, st, P_r, ranges, k)
            for i in range(3):
                for r in range(world):
                    outside = ~band_mask(H, r, world)
                    if bool(outside.any()):
                        assert float(outs[r][4][k][i][:, outside].abs().max()) == 0.0, (tag, r, k, i, "outside the band")
                assert torch.equal(sum(o[4][k][i] for o in outs), ref[i]), (tag, k, i, "layer image differs from the single-GPU render")
        rec = torch.cat([o[3]["rec"][:n].clone() for o, n in zip(outs, P_r)])
        masks = SC.masks(rec[:, 0].cpu(), rec[:, 1].cpu(), rad.cpu(), W, H, world)
        smap = LC.mask_slots(masks, P_r, chunk, world, ranges)
        delivered = lambda secs, sm: all(torch.equal(secs[d][sl.to(DEV)].long().cpu(), bits) for d, (sl, _, bits) in enumerate(sm))
        assert delivered([ws.layer_mask for ws in wss], smap), (tag, "delivered layer bytes")
        d = max(range(world), key=lambda k: smap[k][0].numel())
        sl = smap[d][0]
        last = sl // 256 == sl[-1] // 256
        dropped = [ws.layer_mask.clone() for ws in wss]
        dropped[d][sl[last].to(DEV)] = 0x7f
        assert not delivered(dropped, smap), (tag, "a dropped mask run would pass")
        # ---- layered backward, no layer gradient: the plain fused backward ----
        c0 = _capi.lib().sgr_launch_count()
        none_g = _run(wss, streams, lambda r, ws: SH.sharded_backward_raw(
            st, band(r), ws, locs[r], P_r[r], capacity, outs[r][2], *up,
            layers=[(b, e, BGS[k], outs[r][4][k][2], None, None) for k, (b, e) in enumerate(ranges[r])]))
        assert _capi.lib().sgr_launch_count() - c0 == plain_launches, tag
        # (the blend backward adds a Gaussian's pixels with atomics, so two backward runs agree to rounding, and each run exactly with
        # the rows it left in the sections)
        main = _rows_by_rank([ws.grad2d for ws in wss], smap, P)
        for r in range(world):
            assert torch.equal(none_g[r][1], main[offs[r]: offs[r] + P_r[r], 0:3]), (tag, r, "no layer gradient: main dL/dmeans2D")
            for a, b in zip(none_g[r], plain_g[r]):
                assert (a is None and b is None) or b.numel() == 0 or torch.allclose(a, b, rtol=1e-3, atol=1e-4 * float(b.abs().max())), (tag, r)
        # ---- again, with layer gradients (the forward first: the backward above consumed the frame) ----
        outs = _run(wss, streams, lambda r, ws: SH.sharded_forward_raw(st, band(r), ws, locs[r], P_r[r], capacity, gcap, layers=tables[r]))
        sinks = [[torch.full((e - b, 3), float("nan"), device=DEV) for b, e in ranges[r]] for r in range(world)]
        grads = _run(wss, streams, lambda r, ws: SH.sharded_backward_raw(
            st, band(r), ws, locs[r], P_r[r], capacity, outs[r][2], *up,
            layers=[(b, e, BGS[k], outs[r][4][k][2], lup[k], sinks[r][k]) for k, (b, e) in enumerate(ranges[r])]))
        main = _rows_by_rank([ws.grad2d for ws in wss], smap, P)
        for r in range(world):
            assert torch.equal(grads[r][1], main[offs[r]: offs[r] + P_r[r], 0:3]), (tag, r, "main dL/dmeans2D")
        for k in range(2):
            fwd = _rows_by_rank([ws.layer_grad2d[k] for ws in wss], smap, P)
            rev = _rows_by_rank([ws.layer_grad2d[k] for ws in wss], smap, P, ascending=False)
            for r in range(world):
                b, e = ranges[r][k]
                assert torch.equal(sinks[r][k], fwd[offs[r] + b: offs[r] + e, 0:3]), (tag, r, k, "layer sink")
            REVERSED_DIFFERS.append(not torch.equal(fwd[:, 0:3], rev[:, 0:3]))
            # a layer's rows are zero for the Gaussians outside it
            inside = torch.zeros(P, dtype=torch.bool)
            inside[LC.layer_rows(P_r, ranges, k)] = True
            assert float(fwd[~inside.to(DEV)].abs().max()) == 0.0, (tag, k, "rows outside the layer")
        # ---- per element against float64: blend64 of the main frame and of each layer, chain64 on their summed rows ----
        kg = {key: (torch.cat([gr[i] for gr in grads if gr[i] is not None]) if any(gr[i] is not None for gr in grads) else None)
              for i, key in enumerate(GRAD_NAMES)}
        l_alpha = [sum(o[4][k][2] for o in outs) for k in range(2)]
        l_sinks = [torch.cat([sinks[r][k] for r in range(world)]) for k in range(2)]
        _fp64_layered(tag, scene, rec, rad, alp, l_alpha, lup, P_r, ranges, kg, l_sinks, world, worst)
    # forward after forward (no backward): the leading barrier keeps records and masks consistent
    for rep in range(2):
        status = [torch.zeros(8, dtype=torch.int32).pin_memory() for _ in range(world)]
        outs = _run(wss, streams, lambda r, ws: SH.sharded_forward_raw(st, band(r), ws, locs[r], P_r[r], capacity, -1, status[r],
                                                                       layers=tables[r]))
        assert all(int(s[4]) == 0 and int(s[1]) == 0 for s in status), "forward after forward"
        assert torch.equal(sum(o[0] for o in outs), col)
        assert torch.equal(sum(o[4][1][0] for o in outs), _layer_reference(scene, st, P_r, ranges, 1)[0])
    # sensitivity on the kernel's own images: each layer's widest range moved by one row renders another layer
    moved = [list(x) for x in ranges]
    for k in range(2):
        r1 = max(range(world), key=lambda r: ranges[r][k][1] - ranges[r][k][0])
        b, e = ranges[r1][k]
        moved[r1][k] = (b + 1, e + 1) if e < P_r[r1] else (b + 1, e)
    outs = _run(wss, streams, lambda r, ws: SH.sharded_forward_raw(st, band(r), ws, locs[r], P_r[r], capacity, -1,
                                                                   layers=[(b, e, BGS[k]) for k, (b, e) in enumerate(moved[r])]))
    for k in range(2):
        assert not torch.equal(sum(o[4][k][0] for o in outs), _layer_reference(scene, st, P_r, ranges, k)[0]), (name, k, "a shifted range")
    print(name, {k: round(v, 4) for k, v in worst.items()})


def test_gather_order_is_observable():
    """Adding the ranks' layer rows in descending order changes some sink element in the cases above."""
    if not REVERSED_DIFFERS:
        for name in ("w2_tail", "w3_middle", "w5_empty_rank", "w8_empty_bands"):
            test_fused_layers_exact(name)
    assert any(REVERSED_DIFFERS)


def _leaves(sc):
    return {k: sc[k].to(DEV).clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}


def _call(mod, lv, layers):
    return mod.forward_layers(means3D=lv["means3D"], means2D=None, opacities=lv["opacities"], shs=lv["shs"], scales=lv["scales"],
                              rotations=lv["rotations"], layers=layers)


def test_module_world1_matches_single_gpu_layers():
    _warm_up_layers()
    case = SC.build("w2_tail", seed=5, D=3, device=DEV)
    sc = case["scene"]
    st = util.settings_from(sgb, sc["cam"], DEV)
    P = sc["means3D"].shape[0]
    n_bkgd = P // 3
    mod = SH.GaussianShardedRasterizer(st, capacity=sgb.InstanceCapacity(), exchange="p2p")
    lv = _leaves(sc)
    with pytest.raises(_capi.SgrError, match="capacity is known"):
        _call(mod, lv, [sgb.RenderLayer(n_bkgd, P, (1, 1, 1))])
    out = mod(means3D=lv["means3D"], means2D=None, opacities=lv["opacities"], shs=lv["shs"], scales=lv["scales"], rotations=lv["rotations"])
    out[0].sum().backward()
    mod.synchronize_capacity()
    single = sgb.GaussianRasterizer(st)
    results = []
    for m in (mod, single):
        lv = _leaves(sc)
        sink = torch.zeros(P - n_bkgd, 3, device=DEV, requires_grad=True)
        m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
        lv_call = dict(lv)
        o = m.forward_layers(means3D=lv["means3D"], means2D=m2d, opacities=lv["opacities"], shs=lv["shs"], scales=lv["scales"],
                             rotations=lv["rotations"], layers=[sgb.RenderLayer(0, n_bkgd, (0.2, 0.5, 0.9)),
                                                                sgb.RenderLayer(n_bkgd, P, (1, 1, 1), sink)])
        loss = (o[0] * sc["grad_color"].to(DEV)).sum() + (o[5][1][2] * 0.3).sum() + (o[5][1][0] * sc["grad_color"].to(DEV)).sum()
        loss.backward()
        results.append((o, {k: v.grad for k, v in lv.items()}, m2d.grad, sink.grad))
    (om, gm, m2m, skm), (os_, gs, m2s, sks) = results
    assert all(torch.equal(a, b) for a, b in zip(om[:4], os_[:4]))
    for k in range(2):
        assert all(torch.equal(a, b) for a, b in zip(om[5][k], os_[5][k])), k
    # one GPU and world 1 add the same terms; the blend backward's atomics order them differently, and a Gaussian's screen-space sum can
    # cancel to far below its terms, so the comparison is against the largest gradient
    for a, b, k in [(gm[k], gs[k], k) for k in gm] + [(m2m, m2s, "means2D"), (skm, sks, "objects sink")]:
        assert torch.allclose(a, b, rtol=1e-3, atol=1e-3 * float(b.abs().max())), k
    # the layered step captured in a CUDA graph replays bit-equal to eager (the raw calls, world 1)
    lt = _local(sc, 0, P)
    ws = SH.PeerWorkspace.emulate(st, P, 1, DEV, layers=1)[0]
    cap = int(_single(sc, st)[5].num_instances) + 1000
    up = [sc[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
    sk = torch.empty(P - n_bkgd, 3, device=DEV)
    white = BGS[1].to(DEV)  # (nothing crosses from the host inside the capture)

    def step():
        o = SH.sharded_forward_raw(st, None, ws, lt, P, cap, P, layers=[(n_bkgd, P, white)])
        g = SH.sharded_backward_raw(st, None, ws, lt, P, cap, o[2], *up, layers=[(n_bkgd, P, white, o[4][0][2], up, sk)])
        return o[4][0][0], g[0], g[1], sk

    with torch.no_grad():
        eager = [t.clone() for t in step()]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            cap_out = step()
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(eager[0], cap_out[0])  # the layer image; the gradients agree to the rounding of the blend's atomics
    for a, b in zip(eager[1:], cap_out[1:]):
        assert torch.allclose(a, b, rtol=1e-3, atol=1e-3 * float(a.abs().max()))


def _models(sc, n_bkgd):
    """The scene as a background and one actor with the identity pose, in the composer's raw parameters (compose gives the scene back)."""
    raw = dict(xyz=sc["means3D"], rotation=sc["rotations"], scaling=sc["scales"].log(), opacity=torch.logit(sc["opacities"]),
               features_dc=sc["shs"][:, :1], features_rest=sc["shs"][:, 1:])
    cut = lambda lo, hi: {k: v[lo:hi].to(DEV).contiguous().clone().requires_grad_(True) for k, v in raw.items()}
    return [cut(0, n_bkgd), cut(n_bkgd, sc["means3D"].shape[0])]


def test_module_world1_training_step_with_the_objects_layer():
    """compose -> forward_layers with the objects layer -> band_losses.frame_losses(acc_obj=, obj_bound=, rasterizer=) -> backward, at
    world 1 through the peer workspace, against the same step on one GPU (compose, GaussianRasterizer.forward_layers, frame_losses).
    The images and losses are bit-equal; the raw-parameter gradients agree per element within 1e-3 of their row's largest element (the
    blend backward's atomics add the same terms in another order; test_fused_layers_exact checks the layered gradients per element
    against float64)."""
    _warm_up_layers()
    from street_gaussians_b200 import band_losses
    case = SC.build("w3_middle", seed=6, D=3, device=DEV)
    sc = case["scene"]
    st = util.settings_from(sgb, sc["cam"], DEV)
    P = int(sc["means3D"].shape[0])
    n_bkgd = P - P // 4
    H, W = case["H"], case["W"]
    g = torch.Generator(device=DEV).manual_seed(11)
    gt = torch.rand(3, H, W, generator=g, device=DEV)
    mask = torch.rand(1, H, W, generator=g, device=DEV) > 0.2
    bound = torch.rand(1, H, W, generator=g, device=DEV) > 0.5
    poses, idft = torch.tensor([[1.0, 0, 0, 0, 0, 0, 0]], device=DEV), torch.ones(1, 1, device=DEV)
    mod = SH.GaussianShardedRasterizer(st, capacity=sgb.InstanceCapacity(), exchange="p2p")
    results = []
    for sharded in (True, False):
        models = _models(sc, n_bkgd)
        xyz, rot, scale, opac, shs = sgb.compose(models, poses, idft, **(dict(rasterizer=mod) if sharded else {}))
        kw = dict(rasterizer=mod) if sharded else dict(band=sgb.TileRowBand(0, (H + 15) // 16, 1))  # (one GPU: the whole frame's band)
        rast = mod if sharded else sgb.GaussianRasterizer(st)
        call = dict(means3D=xyz, means2D=None, opacities=opac, shs=shs, scales=scale, rotations=rot)
        if sharded:  # a plain step first: the capacity is learnt from it
            out = mod(**call)
            out[0].sum().backward(retain_graph=True)
            mod.synchronize_capacity()
            for m in models:
                for v in m.values():
                    v.grad = None
        color, _, _, alpha, _, ((_, _, acc_obj),) = rast.forward_layers(**call, layers=[sgb.RenderLayer(n_bkgd, P, (1, 1, 1))])
        v = band_losses.frame_losses(color, gt, mask, acc_obj=acc_obj, obj_bound=bound, **kw)
        sum(v.values()).backward()
        results.append((color.detach(), acc_obj.detach(), {k: float(x.detach()) for k, x in v.items()},
                        [{k: t.grad.clone() for k, t in m.items()} for m in models]))
        if sharded:
            mod.synchronize_capacity()
    (c1, a1, v1, g1), (c0, a0, v0, g0) = results
    assert torch.equal(c1, c0) and torch.equal(a1, a0) and v1 == v0, (v1, v0)
    for m in range(2):
        for k in g0[m]:
            a, b = g1[m][k], g0[m][k]
            scale = b.abs().amax(dim=tuple(range(1, b.dim())), keepdim=True) if b.dim() > 1 else b.abs()
            assert bool(((a - b).abs() <= 1e-3 * scale + 1e-6 * float(b.abs().max())).all()), (m, k)
