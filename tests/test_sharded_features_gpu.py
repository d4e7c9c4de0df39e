"""Feature channels in the fused Gaussian-sharded step (sgr_sharded_forward_features / sgr_sharded_backward_features), with N ranks emulated
on N streams of one GPU on the scenes of tests/sharded64_case.py (block run totals 0 .. 256 world, depth ties across ranks, empty bands,
padding at the tail, in the middle and as a whole empty rank), two frames each, then two forwards in a row.

Exact, per rank: status words (no barrier timeout, no overflow), n_sel and the instance count as in tests/test_sharded64_gpu.py, radii, the
delivered semantic rows (every slot of every run holds its Gaussian's S floats: a numpy restatement of the block runs), colour, depth,
alpha and feature images zero outside the band and summing over the ranks to the single-GPU render bit for bit, and the gathered
dL/dsemantics equal to the ranks' partial rows added in ascending rank order.
Per element against float64 (oracle/raster64.py blend64 with the semantics, on the kernel's records and alpha): dL/dsemantics and
g_means2D within the single-GPU bound plus world 2^-24 mass (sharded64_case.sharded_bound), every other parameter gradient within
chain_bound of chain64 on it.
Sensitivity: dropping the last semantic run of a block, shifting a semantic row by one slot, or adding the gathered rows in another rank
order each fail these checks (shown on the kernel's own data).
Through the autograd module at world 1: S <= 32 takes the fused path and S = 33 (forward only) the staged one, both equal to the
single-GPU render; the backward of S = 33 is refused."""
import pytest
import torch

import sharded64_case as SC
import util
from oracle import raster64 as R64
import street_gaussians_b200 as sgb
from street_gaussians_b200 import sharded as SH
from street_gaussians_b200 import synthetic
from test_sharded64_gpu import GRAD_NAMES, _local, _ratio, _single, _warm_up_fused_path, band_mask

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
F64 = torch.float64
_warm = []
REVERSED_DIFFERS = []


def _warm_up_features():
    """Every kernel of the feature form loaded before ranks spin in emulated barriers (world 1 takes no barrier): the scatter and gather
    of the semantic runs and the blend instantiations of every channel bucket."""
    _warm_up_fused_path(DEV)
    if _warm:
        return
    scene = synthetic.make_scene(P=3000, width=160, height=96, sh_degree=3, seed=1, pose=True)
    st = util.settings_from(sgb, scene["cam"], DEV)
    lt = SH._local_tensors(*(scene[k].to(DEV) if scene.get(k) is not None else None for k in ("means3D", "shs", "colors_precomp")), None,
                           *(scene[k].to(DEV) if scene.get(k) is not None else None for k in ("opacities", "scales", "rotations", "cov3D_precomp")))
    up = [scene[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
    with torch.no_grad():
        for S in (3, 8, 16, 32):
            ws = SH.PeerWorkspace.emulate(st, 3000, 1, DEV, S)[0]
            sem = torch.rand(3000, S, device=DEV)
            out = SH.sharded_forward_raw(st, None, ws, lt, 3000, 500_000, -1, semantics=sem)
            SH.sharded_backward_raw(st, None, ws, lt, 3000, 500_000, out[2], *up, torch.randn(S, 96, 160, device=DEV))
    torch.cuda.synchronize()
    _warm.append(True)


def slot_map(masks, P_r, chunk, world):
    """The block runs restated: for every destination d, (slots of d's sem section, global ids) of the Gaussians delivered to d — owner s's
    block b sends the Gaussians of the block that d needs, in ascending order, to slots s chunk + 256 b + 0, 1, ..."""
    out = []
    offs = [sum(P_r[:r]) for r in range(world)]
    for d in range(world):
        slots, gids = [], []
        for s in range(world):
            for b0 in range(0, P_r[s], 256):
                g = torch.arange(offs[s] + b0, offs[s] + min(P_r[s], b0 + 256))
                g = g[((masks[g] >> d) & 1).bool()]
                slots.append(s * chunk + b0 + torch.arange(g.numel()))
                gids.append(g)
        out.append((torch.cat(slots), torch.cat(gids)))
    return out


def _sem_rows_ok(sections, smap, sem):
    """Every delivered slot of every rank's sem section holds its Gaussian's row."""
    return all(torch.equal(sec[sl.to(DEV)], sem[g.to(DEV)]) for sec, (sl, g) in zip(sections, smap))


def _fp64_check(tag, scene, sem, gs, rec, radii, alpha, kg, g_sem, world, worst):
    cam = scene["cam"]
    W, H = int(cam["image_width"]), int(cam["image_height"])
    up = dict(color=scene["grad_color"], depth=scene["grad_depth"], alpha=scene["grad_alpha"], semantic=gs)
    bl = R64.blend64(rec.double(), radii, W, H, cam["bg"], semantics=sem.double(), upstream=up, alpha_img=alpha)
    vis = radii > 0
    err = (g_sem.double() - bl["grad_semantics"]).abs()
    _ratio(worst, "g_semantics", err, SC.sharded_bound(bl, world, "grad_semantics"), tag)
    assert bool((g_sem[~vis] == 0).all()), (tag, "dL/dsemantics of a culled Gaussian")
    pre = R64.preprocess64(scene, DEV, requires_grad=True)
    nt = bl["ntiles"].to(F64)[:, None]
    ch = R64.chain64(pre, bl["grad2d"], bl["mass_grad2d"], bl["kmass_grad2d"] + (nt + world) * bl["mass_grad2d"])
    for key, got in kg.items():
        if got is None:
            continue
        assert bool((got[~vis] == 0).all()), (tag, key, "gradient of a culled Gaussian")
        if key == "g_means2D":
            _ratio(worst, key, (got.double() - bl["grad2d"][:, 0:3]).abs(), SC.sharded_bound(bl, world)[:, 0:3], tag)
        else:
            ref = ch[key]
            _ratio(worst, key, (got.double().reshape(ref.shape) - ref).abs(), R64.chain_bound(ch, key), tag)


CASES = [("w2_tail", 3, 3), ("w3_middle", 17, 1), ("w5_empty_rank", 22, 0), ("w8_empty_bands", 32, 2)]


@pytest.mark.parametrize("name,S,D", CASES, ids=[f"{c[0]}_S{c[1]}" for c in CASES])
def test_fused_features_per_element(name, S, D):
    _warm_up_features()
    cases = [SC.build(name, seed=f, D=D, device=DEV) for f in range(2)]
    world, chunk, W, H = cases[0]["world"], cases[0]["chunk"], cases[0]["W"], cases[0]["H"]
    st = util.settings_from(sgb, cases[0]["scene"]["cam"], DEV)
    wss = SH.PeerWorkspace.emulate(st, chunk, world, DEV, S)
    for ws in wss:
        ws.buf[: ws.off_flags].fill_(0x7f)  # poison everything but the barrier pads, the feature sections included
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    worst = {}
    for fi, case in enumerate(cases):
        scene, P_r = case["scene"], case["P_r"]
        tag = f"{name} S={S} frame {fi}"
        offs = [sum(P_r[:r]) for r in range(world)]
        g = torch.Generator(device=DEV).manual_seed(100 + fi)
        P = sum(P_r)
        sem = torch.rand(P, S, generator=g, device=DEV)
        gs = torch.randn(S, H, W, generator=g, device=DEV)
        st = util.settings_from(sgb, scene["cam"], DEV)
        locs = [_local(scene, offs[r], offs[r] + P_r[r]) for r in range(world)]
        sems = [sem[offs[r]: offs[r] + P_r[r]].clone() for r in range(world)]
        up = [scene[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
        col, rad, dep, alp, sem_img, fst, _ = _single(scene, st, semantics=sem)
        R_band = [int(_single(scene, st, SH.cyclic_band(H, r, world), semantics=sem)[5].num_instances) for r in range(world)]
        capacity = int(fst.num_instances) + 1000
        status = [torch.zeros(8, dtype=torch.int32).pin_memory() for _ in range(world)]
        outs = []
        torch.cuda.synchronize()
        with torch.no_grad():
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    outs.append(SH.sharded_forward_raw(st, SH.cyclic_band(H, r, world), wss[r], locs[r], P_r[r], capacity,
                                                       -1 if fi == 0 else chunk * world, status[r], semantics=sems[r]))
            torch.cuda.synchronize()
        rec = torch.cat([o[3]["rec"][:n].clone() for o, n in zip(outs, P_r)])
        radii = torch.cat([o[3]["radii"][:n].clone() for o, n in zip(outs, P_r)])
        # ---- exact ----
        assert torch.equal(radii, rad), (tag, "radii")
        n_exp, _ = SC.expected_counts(rec[:, 0].cpu(), rec[:, 1].cpu(), radii.cpu(), W, H, world)
        for r in range(world):
            R_r, over, emitted, n_sel, timed_out = (int(v) for v in status[r][:5])
            assert timed_out == 0 and over == 0, (tag, r, timed_out, over)
            assert n_sel == n_exp[r] and R_r == emitted == R_band[r], (tag, r, n_sel, n_exp[r], R_r, emitted, R_band[r])
            outside = ~band_mask(H, r, world)
            for i in (0, 1, 2, 4):
                if bool(outside.any()):
                    assert float(outs[r][i][:, outside].abs().max()) == 0.0, (tag, r, i, "outside the band")
        for i, ref, nm in ((0, col, "color"), (1, dep, "depth"), (2, alp, "alpha"), (4, sem_img, "semantic")):
            assert torch.equal(sum(o[i] for o in outs), ref), f"{tag}: {nm} differs from the single-GPU render"
        masks = SC.masks(rec[:, 0].cpu(), rec[:, 1].cpu(), radii.cpu(), W, H, world)
        smap = slot_map(masks, P_r, chunk, world)
        assert _sem_rows_ok([ws.sem for ws in wss], smap, sem), (tag, "delivered semantic rows")
        # sensitivity of the row check on the kernel's own rows: the last run of a block not delivered (its rows left as they were, here
        # zero), or every row one slot off
        d = max(range(world), key=lambda k: smap[k][0].numel())
        sl, gids = smap[d]
        last = sl // 256 == sl[-1] // 256
        dropped = [ws.sem.clone() for ws in wss]
        dropped[d][sl[last].to(DEV)] = 0.0
        assert not _sem_rows_ok(dropped, smap, sem), (tag, "a dropped run would pass")
        shifted = [(s + 1, g) if k == d else (s, g) for k, (s, g) in enumerate(smap)]
        assert not _sem_rows_ok([ws.sem for ws in wss], shifted, sem), (tag, "a shifted row would pass")
        # ---- backward ----
        with torch.no_grad():
            grads = []
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    grads.append(SH.sharded_backward_raw(st, SH.cyclic_band(H, r, world), wss[r], locs[r], P_r[r], capacity, outs[r][2], *up,
                                                         gs))
            torch.cuda.synchronize()
        g_sem = torch.cat([gr[8] for gr in grads])
        # the gather: partial rows of the ranks that rendered the Gaussian, added from 0 in ascending rank order
        fwd_sum, rev_sum = torch.zeros_like(g_sem), torch.zeros_like(g_sem)
        for r in range(world):
            sl, gids = smap[r]
            part = torch.zeros_like(g_sem)
            part[gids.to(DEV)] = wss[r].gsem[sl.to(DEV)]
            fwd_sum = fwd_sum + part
        for r in reversed(range(world)):
            sl, gids = smap[r]
            part = torch.zeros_like(g_sem)
            part[gids.to(DEV)] = wss[r].gsem[sl.to(DEV)]
            rev_sum = rev_sum + part
        assert torch.equal(g_sem, fwd_sum), (tag, "gathered dL/dsemantics is not the ascending-rank sum of the partial rows")
        REVERSED_DIFFERS.append(not torch.equal(g_sem, rev_sum))
        kg = {k: (torch.cat([gr[i] for gr in grads if gr[i] is not None]) if any(gr[i] is not None for gr in grads) else None)
              for i, k in enumerate(GRAD_NAMES)}
        _fp64_check(tag, scene, sem, gs, rec, radii, alp, kg, g_sem, world, worst)
    # forward after forward (no backward): the leading barrier, images still exact
    with torch.no_grad():
        for rep in range(2):
            status = [torch.zeros(8, dtype=torch.int32).pin_memory() for _ in range(world)]
            outs = []
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    outs.append(SH.sharded_forward_raw(st, SH.cyclic_band(H, r, world), wss[r], locs[r], P_r[r], capacity, -1, status[r],
                                                       semantics=sems[r]))
            torch.cuda.synchronize()
            assert all(int(s[4]) == 0 and int(s[1]) == 0 for s in status), "forward after forward"
            assert torch.equal(sum(o[4] for o in outs), sem_img) and torch.equal(sum(o[0] for o in outs), col)
    print(name, S, {k: round(v, 4) for k, v in worst.items()})


def test_gather_order_is_observable():
    """Adding the partial rows in descending rank order changes some element in the cases above (a wrong order could not pass)."""
    if not REVERSED_DIFFERS:
        for name, S, D in CASES:
            test_fused_features_per_element(name, S, D)
    assert any(REVERSED_DIFFERS)


def _module_frames(S, frames, grad):
    from street_gaussians_b200.sharded import GaussianShardedRasterizer
    case = SC.build("w2_tail", seed=4, D=3, device=DEV)
    sc = case["scene"]
    st = util.settings_from(sgb, sc["cam"], DEV)
    P = sc["means3D"].shape[0]
    sem = torch.rand(P, S, generator=torch.Generator(device=DEV).manual_seed(7), device=DEV)
    ref = _single(sc, st, semantics=sem)
    mod = GaussianShardedRasterizer(st, capacity=sgb.InstanceCapacity(), exchange="p2p")
    paths = []
    for frame in range(frames):
        leaves = {k: sc[k].to(DEV).clone().requires_grad_(grad) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        s_leaf = sem.clone().requires_grad_(grad)
        with torch.set_grad_enabled(grad):
            color, radii, depth, alpha, semantic = mod(means3D=leaves["means3D"], means2D=None, opacities=leaves["opacities"],
                                                       shs=leaves["shs"], scales=leaves["scales"], rotations=leaves["rotations"],
                                                       semantics=s_leaf)
        paths.append(bool(getattr(color.grad_fn, "fused", False)) if grad else mod._ws is not None and mod._ws.S == S)
        assert torch.equal(color.detach(), ref[0]) and torch.equal(semantic.detach(), ref[4]), (S, frame)
        if grad:
            (semantic.sum() + color.sum()).backward()
            assert s_leaf.grad is not None and bool(s_leaf.grad.abs().sum() > 0)
        mod.synchronize_capacity()
    return paths, mod


def test_module_routes_features_to_the_fused_step():
    paths, mod = _module_frames(3, 3, True)
    assert paths == [False, True, True], paths
    assert mod._ws.S == 3


def test_module_routes_33_channels_to_the_staged_step():
    paths, mod = _module_frames(33, 2, False)
    assert paths == [False, False], paths
    with pytest.raises(Exception, match="semantic"):
        _module_frames(33, 1, True)
