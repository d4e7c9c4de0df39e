"""GPU: sharded.rebalance on 2, 3, 5 and 8 ranks emulated by threads on one GPU, exchanging through an in-process transport.  A
with_raw synthetic scene (background + 3 actors, 2 semantic floats per row) is split unevenly across the ranks (empty ranks included),
FusedAdam is stepped three times and the statistics are filled, then every rank calls rebalance().  Checked:
  * the rank-major concatenation of every parameter, both Adam moments and the three statistics is bit-identical before and after;
  * the counts are the even split, and the optimizer's groups and state hold the new tensors (old keys gone, step unchanged);
  * one more FusedAdam step on the new shards equals, bit for bit, the same step on the global arrays the old shards make up;
  * compose, add_densification_stats and densify_and_prune run on the new shards, most of which have sub-models with 0 local rows;
  * the emulated Gaussian-sharded render (project_records -> forward_records -> backward_blend_records on cyclic bands, partial grad2d
    summed in rank order, backward_geom_local) gives bit-identical colour, depth and alpha before and after, and every global row's
    gradients within test_sharded64_gpu's float64 bound, both times."""
import types

import pytest
import torch

import util
from rank_threads import run_ranks
from oracle import raster64 as R64
import street_gaussians_b200 as sgb
from street_gaussians_b200 import sharded as SH
from street_gaussians_b200 import synthetic, training
from test_sharded64_gpu import GRAD_NAMES, check_against_fp64

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
NAMES = training.PARAM_NAMES
STATS = training.STAT_NAMES
WEIGHTS = {2: [3, 1], 3: [1, 0, 5], 5: [6, 1, 1, 0, 2], 8: [9, 0, 1, 1, 2, 0, 1, 3]}


def make_global(seed=3, S=2):
    scene = synthetic.make_scene(P=12_000, width=320, height=208, sh_degree=3, seed=seed, n_vehicles=3, per_vehicle=1500, with_raw=True,
                                 scale_med=0.05)
    raw = scene["raw"]
    poses, idft = raw["poses"].to(DEV), raw["idft"].to(DEV)
    g = torch.Generator().manual_seed(seed)
    models = []
    for r in raw["models"]:
        n = r["xyz"].shape[0]
        m = {"_" + a: v.to(DEV).contiguous() for a, v in r.items()}
        m["_semantic"] = torch.rand(n, S, generator=g).to(DEV)
        models.append(m)
    # keep only the Gaussians no float64 decision lies near a threshold of (the bound of check_against_fp64 assumes that)
    comp = sgb.compose(models, poses, idft)
    full = dict(cam=scene["cam"], means3D=comp[0], rotations=comp[1], scales=comp[2], opacities=comp[3], shs=comp[4])
    _, _, keep = R64.margin_scene(full, device=DEV)
    keep = keep.to(DEV)
    at = 0
    for m in models:
        n = m["_xyz"].shape[0]
        k = keep[(keep >= at) & (keep < at + n)] - at
        for a in list(m):
            m[a] = m[a][k].contiguous()
        at += n
    for m in models:
        n = m["_xyz"].shape[0]
        m["max_radii2D"] = torch.rand(n, generator=g).to(DEV) * 30
        m["denom"] = torch.randint(1, 9, (n, 1), generator=g).float().to(DEV)
        m["xyz_gradient_accum"] = torch.rand(n, 2, generator=g).to(DEV) * m["denom"] * 1e-3
    grads = [[torch.randn(m[a].shape, generator=g).to(DEV) * 1e-2 for a in NAMES] for m in models]
    up = {k: scene[k] for k in ("grad_color", "grad_depth", "grad_alpha")}
    return scene["cam"], poses, idft, models, grads, up


def split(models, world):
    """Per-rank [lo, hi) of every model: the global rows cut by WEIGHTS[world] (rank-major, model-major)."""
    counts = [m["_xyz"].shape[0] for m in models]
    P = sum(counts)
    w = WEIGHTS[world]
    B = [P * sum(w[:r]) // sum(w) for r in range(world + 1)]
    G = [sum(counts[:k]) for k in range(len(models) + 1)]
    return [[(max(B[r], G[k]) - G[k], max(max(B[r], G[k]), min(B[r + 1], G[k + 1])) - G[k]) for k in range(len(models))] for r in range(world)]


def shard_model(k, m, lo, hi):
    o = types.SimpleNamespace(**{a: torch.nn.Parameter(m[a][lo:hi].clone()) for a in NAMES},
                              **{s: m[s][lo:hi].clone() for s in STATS}, percent_dense=0.01, percent_big_ws=0.1)
    if k == 0:
        o.scene_radius, o.sphere_center, o.sphere_radius = torch.tensor([20.0]), torch.zeros(3), torch.tensor([40.0])
    else:
        o.extent, o.min_xyz, o.max_xyz = torch.tensor([3.0]), torch.tensor([-3.0, -1.5, -1.5]), torch.tensor([3.0, 1.5, 1.5])
    return o


def lr(k, a):
    return 1e-3 * (1 + a) / (1 + k)


def make_optimizer(objs):
    return training.FusedAdam([{"params": [getattr(o, a)], "lr": lr(k, ai), "name": a} for k, o in enumerate(objs)
                               for ai, a in enumerate(NAMES)], lr=1e-3, eps=1e-15)


def set_grads(objs, grads, rows):
    for k, o in enumerate(objs):
        lo, hi = rows[k]
        for a, gk in zip(NAMES, grads[k]):
            getattr(o, a).grad = gk[lo:hi].clone()


def rows_of(shards):
    """Per rank, [lo, hi) of every model in the model's global rows, from the shards' counts (rank-major)."""
    nm = len(shards[0])
    at = [0] * nm
    out = []
    for objs in shards:
        rows = []
        for k, o in enumerate(objs):
            n = o._xyz.shape[0]
            rows.append((at[k], at[k] + n))
            at[k] += n
        out.append(rows)
    return out


def snapshot(shards, opts):
    """Per model, the rank-major concatenation of every parameter, both moments and the statistics (as int32 bits)."""
    snap = []
    for k in range(len(shards[0])):
        d = {}
        for a in NAMES:
            ps = [getattr(objs[k], a) for objs in shards]
            d[a] = torch.cat([p.detach() for p in ps])
            for mk in ("exp_avg", "exp_avg_sq"):
                d[a + mk] = torch.cat([opt.state[p][mk] for p, opt in zip(ps, opts)])
        for s in STATS:
            d[s] = torch.cat([getattr(objs[k], s) for objs in shards])
        snap.append({key: v.contiguous().view(torch.int32) for key, v in d.items()})
    return snap


def render(cam, poses, idft, shards, up, st):
    """The Gaussian-sharded step emulated on one GPU: (color, depth, alpha) summed over the ranks' cyclic bands, the kernels' records
    and radii (rank-major, padding dropped), and the ranks' parameter gradients concatenated."""
    world = len(shards)
    H = int(cam["image_height"])
    locs, Ps = [], []
    for objs in shards:
        xyz, rot, scale, opac, sh = sgb.compose(objs, poses, idft)
        locs.append(SH._local_tensors(xyz.detach(), sh.detach(), None, None, opac.detach(), scale.detach(), rot.detach(), None))
        Ps.append(xyz.shape[0])
    chunk = max(Ps)
    P_total = chunk * world
    recs, radii = zip(*(SH.project_records(lt, st, chunk) for lt in locs))
    imgs, g2 = None, None
    upd = [up[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
    for r in range(world):
        band = SH.cyclic_band(H, r, world)
        fs, rec_all, gb, ib = SH.alloc_gathered(st, P_total, 0, DEV)
        rec_all.copy_(torch.cat(recs))
        out = SH.forward_records(st, band, fs, (gb, ib), torch.cat(radii), None)
        imgs = out[:3] if imgs is None else tuple(x + y for x, y in zip(imgs, out[:3]))
        part, _ = SH.backward_blend_records(st, band, fs, P_total, None, out[2], *upd, torch.zeros(0, *out[2].shape[1:], device=DEV))
        g2 = part.clone() if g2 is None else g2 + part
    grads = [SH.backward_geom_local(st, locs[r], recs[r], radii[r], g2[r * chunk:(r + 1) * chunk]) for r in range(world) if Ps[r]]
    kg = {key: torch.cat([g[i] for g in grads]) if grads[0][i] is not None else None for i, key in enumerate(GRAD_NAMES)}
    rec = torch.cat([recs[r][:Ps[r]] for r in range(world)])
    rad = torch.cat([radii[r][:Ps[r]] for r in range(world)])
    return imgs, rec, rad, kg


def check_render(tag, cam, poses, idft, shards, up, st, world):
    with torch.no_grad():
        imgs, rec, rad, kg = render(cam, poses, idft, shards, up, st)
        comp = sgb.compose([{a[1:]: torch.cat([getattr(objs[k], a).detach() for objs in shards]) for a in NAMES[:6]}
                            for k in range(len(shards[0]))], poses, idft)
    scene = dict(cam=cam, means3D=comp[0], rotations=comp[1], scales=comp[2], opacities=comp[3], shs=comp[4], **up)
    check_against_fp64(tag, scene, rec, rad, imgs[2], kg, world, {})
    return imgs


@pytest.mark.parametrize("world", sorted(WEIGHTS))
def test_rebalance_emulated_ranks(world):
    cam, poses, idft, models, grads, up = make_global()
    st = util.settings_from(sgb, cam, DEV)
    cuts = split(models, world)
    shards = [[shard_model(k, m, *cuts[r][k]) for k, m in enumerate(models)] for r in range(world)]
    opts = [make_optimizer(objs) for objs in shards]
    for it in range(3):
        for objs, opt, rows in zip(shards, opts, cuts):
            set_grads(objs, [[g * (1 + it) for g in gk] for gk in grads], rows)
            opt.step()
    before = snapshot(shards, opts)
    imgs0 = check_render("before", cam, poses, idft, shards, up, st, world)
    counts0 = [sum(o._xyz.shape[0] for o in objs) for objs in shards]
    assert max(counts0) - min(counts0) > 1
    old_params = [{id(getattr(o, a)) for o in objs for a in NAMES} for objs in shards]
    # the step the new shards must reproduce: FusedAdam over the global arrays the old shards make up
    glob = [{a: torch.nn.Parameter(torch.cat([getattr(objs[k], a).detach() for objs in shards])) for a in NAMES} for k in range(len(models))]
    gopt = training.FusedAdam([{"params": [glob[k][a]], "lr": lr(k, ai)} for k in range(len(models)) for ai, a in enumerate(NAMES)],
                              lr=1e-3, eps=1e-15)
    for k in range(len(models)):
        for a in NAMES:
            ps = [getattr(objs[k], a) for objs in shards]
            gopt.state[glob[k][a]] = dict(step=3, **{mk: torch.cat([opts[r].state[p][mk] for r, p in enumerate(ps)]) for mk in ("exp_avg", "exp_avg_sq")})
            glob[k][a].grad = grads[k][NAMES.index(a)] * 7
    gopt.step()

    rast = [SH.GaussianShardedRasterizer(st, chunk=max(counts0)) for _ in range(world)]
    P_new = run_ranks(world, lambda r, tr: SH.rebalance(shards[r], opts[r], rasterizer=rast[r], transport=tr))
    base, extra = divmod(sum(counts0), world)
    assert P_new == [base + (r < extra) for r in range(world)]
    assert [sum(o._xyz.shape[0] for o in objs) for objs in shards] == P_new
    assert all(r.chunk == max(P_new) for r in rast)
    after = snapshot(shards, opts)
    for k, (b, a) in enumerate(zip(before, after)):
        for key in b:
            assert torch.equal(b[key], a[key]), (world, k, key)
    for objs, opt, old in zip(shards, opts, old_params):
        held = {id(p) for g in opt.param_groups for p in g["params"]}
        for o in objs:
            for a in NAMES:
                p = getattr(o, a)
                assert id(p) in held and id(p) not in old and isinstance(p, torch.nn.Parameter)
                assert opt.state[p]["step"] == 3 and opt.state[p]["exp_avg"].shape == p.shape
        assert len(opt.state) == len(objs) * len(NAMES)
    assert max(P_new) - min(P_new) <= 1
    # the render is the same: images bit for bit, gradients within the float64 bound
    imgs1 = check_render("after", cam, poses, idft, shards, up, st, world)
    for x, y in zip(imgs0, imgs1):
        assert torch.equal(x, y)
    # one more step on the new shards = the step on the global arrays
    for objs, opt, rows in zip(shards, opts, rows_of(shards)):
        set_grads(objs, [[g * 7 for g in gk] for gk in grads], rows)
        opt.step()
    for k in range(len(models)):
        for a in NAMES:
            ps = [getattr(objs[k], a) for objs in shards]
            assert torch.equal(torch.cat([p.detach() for p in ps]).view(torch.int32), glob[k][a].detach().view(torch.int32)), (k, a)
            for mk in ("exp_avg", "exp_avg_sq"):
                got = torch.cat([opts[r].state[p][mk] for r, p in enumerate(ps)])
                assert torch.equal(got.view(torch.int32), gopt.state[glob[k][a]][mk].view(torch.int32)), (k, a, mk)
    # compose, the statistics and densification accept the new shards, sub-models with 0 local rows included
    assert any(o._xyz.shape[0] == 0 for objs in shards for o in objs)
    for r, (objs, opt) in enumerate(zip(shards, opts)):
        xyz = sgb.compose(objs, poses, idft)[0]
        n = xyz.shape[0]
        radii = torch.randint(0, 4, (n,), device=DEV, dtype=torch.int32)
        training.add_densification_stats(objs, radii, torch.randn(n, 3, device=DEV))
        scal = training.densify_and_prune(objs, 1e-7, 0.005, True, opt, seed=11 + r)
        assert sum(s["points_total"] for s in scal) == n
        assert all(o.xyz_gradient_accum.shape[0] == o._xyz.shape[0] == opt.state[o._xyz]["exp_avg"].shape[0] for o in objs)


def test_rebalance_when_balanced_moves_nothing():
    cam, poses, idft, models, grads, up = make_global(seed=4)
    world = 3
    P = sum(m["_xyz"].shape[0] for m in models)
    base, extra = divmod(P, world)
    B = [r * base + min(r, extra) for r in range(world + 1)]
    G = [0]
    for m in models:
        G.append(G[-1] + m["_xyz"].shape[0])
    cuts = [[(max(B[r], G[k]) - G[k], max(max(B[r], G[k]), min(B[r + 1], G[k + 1])) - G[k]) for k in range(len(models))] for r in range(world)]
    shards = [[shard_model(k, m, *cuts[r][k]) for k, m in enumerate(models)] for r in range(world)]
    ids = [[id(o._xyz) for o in objs] for objs in shards]
    launches = sgb._capi.lib().sgr_launch_count()
    P_new = run_ranks(world, lambda r, tr: SH.rebalance(shards[r], None, transport=tr))
    assert sgb._capi.lib().sgr_launch_count() == launches
    assert P_new == [B[r + 1] - B[r] for r in range(world)]
    assert [[id(o._xyz) for o in objs] for objs in shards] == ids


def test_rebalance_rejects_unequal_adam_steps():
    cam, poses, idft, models, grads, up = make_global(seed=5)
    world = 2
    cuts = split(models, world)
    shards = [[shard_model(k, m, *cuts[r][k]) for k, m in enumerate(models)] for r in range(world)]
    opts = [make_optimizer(objs) for objs in shards]
    for r, (objs, opt) in enumerate(zip(shards, opts)):
        for _ in range(1 + r):
            set_grads(objs, grads, cuts[r])
            opt.step()
    with pytest.raises(ValueError, match="Adam step 1 on rank 0 and Adam step 2 on rank 1"):
        run_ranks(world, lambda r, tr: SH.rebalance(shards[r], opts[r], transport=tr))
