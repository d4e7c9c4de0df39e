"""GPU: checkpoints under Gaussian sharding (sharded.save_checkpoint / save_ply / load_checkpoint over gather_state), with 1, 2, 3, 5 and
8 ranks emulated by threads on one GPU (tests/rank_threads.py).  The scene is a background (SH degree 3, 3 semantic floats) and three
actors: SH degree 1 without semantics, SH degree 3 with semantics, and one of 5 rows (fewer than 8 ranks), split unevenly with empty
ranks.  FusedAdam is stepped three times; the smallest actor's semantics never get a gradient, so they have no Adam state.  Checked:
  * saving at every world size with pieces of a few rows gives the file io.save_checkpoint writes for the concatenated state on one GPU:
    the same keys in the same order, every tensor bit-equal, the same Adam state-dict structure, and the reference's CPU torch.optim.Adam
    (gaussian_model.py:286-303) load_state_dict()s every model's 'optimizer' entry; is_final leaves the training entries out;
  * save_ply writes the bytes io.save_ply writes;
  * loading every (N -> N') pair gives each rank the even split's slice of every parameter, moment and statistic, bit for bit, installed
    in its optimizer by identity;
  * after save at 3 ranks and resume at 2 and 3, the emulated Gaussian-sharded render is bit-identical (gradients within
    test_sharded64_gpu's float64 bound) and one FusedAdam step gives the bytes of the uninterrupted run;
  * unequal Adam steps and mismatched widths raise ValueError on every rank."""
import types

import pytest
import torch

from rank_threads import run_ranks
import test_rebalance_gpu as RB
import util
import street_gaussians_b200 as sgb
from street_gaussians_b200 import io, training
from street_gaussians_b200 import sharded as SH

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
NAMES = training.PARAM_NAMES
STATS = training.STAT_NAMES
WEIGHTS = {1: [1], **RB.WEIGHTS}
MODEL_NAMES = ["background", "obj_000", "obj_001", "obj_002"]
PIECE = 4096  # a few rows per piece: hundreds of pieces per save


def make_models(seed=0):
    g = torch.Generator().manual_seed(seed)
    spec = [(700, 3, 3), (400, 1, 0), (300, 3, 2), (5, 3, 2)]  # rows, SH degree, semantic floats
    models = []
    for n, deg, S in spec:
        r = lambda *s: torch.randn(*s, generator=g).to(DEV)
        m = dict(_xyz=r(n, 3), _features_dc=r(n, 1, 3), _features_rest=r(n, (deg + 1) ** 2 - 1, 3), _opacity=r(n, 1), _scaling=r(n, 3),
                 _rotation=r(n, 4), _semantic=r(n, S), max_radii2D=torch.rand(n, generator=g).to(DEV) * 30,
                 denom=torch.randint(1, 9, (n, 1), generator=g).float().to(DEV))
        m["xyz_gradient_accum"] = torch.rand(n, 2, generator=g).to(DEV) * m["denom"] * 1e-3
        models.append(m)
    grads = [[torch.randn(m[a].shape, generator=g).to(DEV) * 1e-2 for a in NAMES] for m in models]
    return models, grads


def split(models, world):
    """test_rebalance_gpu.split with WEIGHTS[world], world 1 included."""
    counts = [m["_xyz"].shape[0] for m in models]
    P, w = sum(counts), WEIGHTS[world]
    B = [P * sum(w[:r]) // sum(w) for r in range(world + 1)]
    G = [sum(counts[:k]) for k in range(len(models) + 1)]
    return [[(max(B[r], G[k]) - G[k], max(max(B[r], G[k]), min(B[r + 1], G[k + 1])) - G[k]) for k in range(len(models))] for r in range(world)]


def shard(k, m, lo, hi):
    o = RB.shard_model(k, m, lo, hi)
    o.spatial_lr_scale, o.active_sh_degree = 2.5, 3
    return o


def trained_shards(models, grads, world):
    """Shards of the uneven split, each rank's FusedAdam stepped three times; the last actor's semantics get no gradient."""
    cuts = split(models, world)
    shards = [[shard(k, m, *cuts[r][k]) for k, m in enumerate(models)] for r in range(world)]
    opts = [RB.make_optimizer(objs) for objs in shards]
    for it in range(3):
        for objs, opt, rows in zip(shards, opts, cuts):
            RB.set_grads(objs, [[gr * (1 + it) for gr in gk] for gk in grads], rows)
            objs[3]._semantic.grad = None
            opt.step()
    return shards, opts


def global_state(shards, opts):
    """The concatenated models and a FusedAdam over them holding the concatenated state (what one GPU holds)."""
    nm = len(shards[0])
    glob = [types.SimpleNamespace(**{a: torch.nn.Parameter(torch.cat([getattr(objs[k], a).detach() for objs in shards])) for a in NAMES},
                                  **{s: torch.cat([getattr(objs[k], s) for objs in shards]) for s in STATS}, spatial_lr_scale=2.5,
                                  active_sh_degree=3) for k in range(nm)]
    gopt = training.FusedAdam([{"params": [getattr(glob[k], a)], "lr": RB.lr(k, ai), "name": a} for k in range(nm) for ai, a in enumerate(NAMES)],
                              lr=1e-3, eps=1e-15)
    for k in range(nm):
        for a in NAMES:
            ps = [getattr(objs[k], a) for objs in shards]
            if ps[0] in opts[0].state:
                gopt.state[getattr(glob[k], a)] = dict(step=opts[0].state[ps[0]]["step"],
                                                       **{mk: torch.cat([opts[r].state[p][mk] for r, p in enumerate(ps)]) for mk in ("exp_avg", "exp_avg_sq")})
    return glob, gopt


REPLICATED = dict(sky_cubemap={"params": {"sky_cube_map": torch.arange(6 * 4 * 4 * 3, dtype=torch.float32).reshape(6, 4, 4, 3)}},
                  color_correction={"params": {"w": torch.eye(3)}})


def single_gpu_save(path, glob, gopt, is_final=False):
    extras = None
    if not is_final:
        extras = {n: dict(spatial_lr_scale=g.spatial_lr_scale, denom=g.denom, max_radii2D=g.max_radii2D, xyz_gradient_accum=g.xyz_gradient_accum,
                          active_sh_degree=g.active_sh_degree, optimizer=training.adam_state_dict(g, gopt)) for n, g in zip(MODEL_NAMES, glob)}
    io.save_checkpoint(path, {n: {a: getattr(g, a) for a in NAMES} for n, g in zip(MODEL_NAMES, glob)}, 7, extras, **REPLICATED)


def assert_same(a, b, where="sd"):
    assert type(a) is type(b), (where, type(a), type(b))  # an nn.Parameter stays one
    if isinstance(a, dict):
        assert list(a) == list(b), (where, list(a), list(b))
        for k in a:
            assert_same(a[k], b[k], f"{where}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, f"{where}[{i}]")
    elif isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape, (where, a.dtype, b.dtype, a.shape, b.shape)
        assert a.device == b.device and a.requires_grad == b.requires_grad, (where, a.device, b.device, a.requires_grad, b.requires_grad)
        x, y = a.detach().cpu().reshape(-1), b.detach().cpu().reshape(-1)
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), where
    else:
        assert a == b, (where, a, b)


def reference_adam(sd_model):
    """GaussianModel.training_setup's optimizer over CPU copies of the model's tensors (gaussian_model.py:286-303)."""
    keys = ("xyz", "feature_dc", "feature_rest", "opacity", "scaling", "rotation", "semantic")
    ps = [torch.nn.Parameter(sd_model[k].detach().cpu().clone()) for k in keys]
    return torch.optim.Adam([{"params": [p], "lr": 0.1, "name": n} for p, n in zip(ps, training.ADAM_GROUP_NAMES)], lr=0.0, eps=1e-15), ps


@pytest.mark.parametrize("world", sorted(WEIGHTS))
def test_save_matches_single_gpu_files(world, tmp_path):
    models, grads = make_models()
    shards, opts = trained_shards(models, grads, world)
    assert any(o._xyz.shape[0] == 0 for objs in shards for o in objs) or world == 1
    glob, gopt = global_state(shards, opts)
    for is_final in (False, True):
        want, got = tmp_path / f"one_{is_final}.pth", tmp_path / f"sharded_{is_final}.pth"
        single_gpu_save(str(want), glob, gopt, is_final)
        dst = world - 1
        out = run_ranks(world, lambda r, tr: SH.save_checkpoint(str(got), dict(zip(MODEL_NAMES, shards[r])), 7, opts[r], is_final=is_final, dst=dst,
                                                                transport=tr, piece_bytes=PIECE, **REPLICATED))
        assert out == [None] * world
        a, b = torch.load(str(want), weights_only=False), torch.load(str(got), weights_only=False)
        assert_same(a, b)
        if not is_final:
            for n in MODEL_NAMES:
                opt, ps = reference_adam(b[n])
                opt.load_state_dict(b[n]["optimizer"])
                assert torch.equal(opt.state[ps[0]]["exp_avg"], b[n]["optimizer"]["state"][0]["exp_avg"].cpu())
            assert 6 not in b["obj_002"]["optimizer"]["state"] and 6 in b["background"]["optimizer"]["state"]
        else:
            assert "optimizer" not in b["background"] and "denom" not in b["background"]
    # the PLY
    want, got = tmp_path / "one.ply", tmp_path / "sharded.ply"
    io.save_ply(str(want), {n: {a: getattr(g, a) for a in NAMES} for n, g in zip(MODEL_NAMES, glob)})
    run_ranks(world, lambda r, tr: SH.save_ply(str(got), dict(zip(MODEL_NAMES, shards[r])), transport=tr, piece_bytes=PIECE))
    assert want.read_bytes() == got.read_bytes()


def blank_shards(world):
    """Fresh models (one row each, no statistics of the right size) and fresh FusedAdams, as a resuming run builds them."""
    models, _ = make_models(seed=99)
    shards = [[shard(k, m, 0, 1) for k, m in enumerate(models)] for _ in range(world)]
    return shards, [RB.make_optimizer(objs) for objs in shards]


def test_load_every_world_pair(tmp_path):
    models, grads = make_models()
    for N in sorted(WEIGHTS):
        shards, opts = trained_shards(models, grads, N)
        glob, gopt = global_state(shards, opts)
        path = str(tmp_path / f"w{N}.pth")
        run_ranks(N, lambda r, tr: SH.save_checkpoint(path, dict(zip(MODEL_NAMES, shards[r])), 7, opts[r], transport=tr, piece_bytes=PIECE))
        totals = [g._xyz.shape[0] for g in glob]
        for N2 in sorted(WEIGHTS):
            new, nopts = blank_shards(N2)
            rast = [types.SimpleNamespace(chunk=None) for _ in range(N2)]
            for ra in rast:
                ra.repartition = lambda P_local, chunk=None, ra=ra: setattr(ra, "chunk", chunk)
            P = run_ranks(N2, lambda r, tr: SH.load_checkpoint(path, dict(zip(MODEL_NAMES, new[r])), nopts[r], transport=tr, rasterizer=rast[r]))
            sl = SH.even_slices(totals, N2)
            assert P == [sum(hi - lo for lo, hi in row) for row in sl]
            assert all(r.chunk == max(P) for r in rast)
            for r in range(N2):
                held = {id(p) for g in nopts[r].param_groups for p in g["params"]}
                for k, (o, g) in enumerate(zip(new[r], glob)):
                    lo, hi = sl[r][k]
                    for a in NAMES:
                        p, want = getattr(o, a), getattr(g, a)[lo:hi]
                        assert isinstance(p, torch.nn.Parameter) and id(p) in held and p.is_cuda
                        assert_same(p.detach(), want.detach(), (N, N2, r, k, a))
                        st = nopts[r].state.get(p)
                        if getattr(g, a) in gopt.state:
                            gs = gopt.state[getattr(g, a)]
                            assert int(st["step"]) == 3
                            for mk in ("exp_avg", "exp_avg_sq"):
                                assert_same(st[mk], gs[mk][lo:hi], (N, N2, r, k, a, mk))
                        else:
                            assert not st
                    for s in STATS:
                        assert_same(getattr(o, s), getattr(g, s)[lo:hi], (N, N2, r, k, s))
                assert len(nopts[r].state) == sum(1 for g in glob for a in NAMES if getattr(g, a) in gopt.state)


@pytest.mark.parametrize("N2", [2, 3])
def test_resume_renders_and_steps_like_the_uninterrupted_run(N2, tmp_path):
    cam, poses, idft, models, grads, up = RB.make_global()
    st = util.settings_from(sgb, cam, DEV)
    N = 3
    cuts = RB.split(models, N)
    shards = [[RB.shard_model(k, m, *cuts[r][k]) for k, m in enumerate(models)] for r in range(N)]
    opts = [RB.make_optimizer(objs) for objs in shards]
    for it in range(3):
        for objs, opt, rows in zip(shards, opts, cuts):
            RB.set_grads(objs, [[g * (1 + it) for g in gk] for gk in grads], rows)
            opt.step()
    imgs0 = RB.check_render("before", cam, poses, idft, shards, up, st, N)
    names = [f"m{k}" for k in range(len(models))]
    path = str(tmp_path / "ckpt.pth")
    run_ranks(N, lambda r, tr: SH.save_checkpoint(path, dict(zip(names, shards[r])), 3, opts[r], transport=tr, piece_bytes=1 << 16))
    # the uninterrupted run's next step, on the global arrays
    glob, gopt = global_state(shards, opts)
    for k in range(len(models)):
        for a in NAMES:
            getattr(glob[k], a).grad = grads[k][NAMES.index(a)] * 7
    gopt.step()
    # resume at N2 from fresh models
    new = [[RB.shard_model(k, m, 0, 1) for k, m in enumerate(models)] for _ in range(N2)]
    nopts = [RB.make_optimizer(objs) for objs in new]
    run_ranks(N2, lambda r, tr: SH.load_checkpoint(path, dict(zip(names, new[r])), nopts[r], transport=tr))
    imgs1 = RB.check_render("resumed", cam, poses, idft, new, up, st, N2)
    for x, y in zip(imgs0, imgs1):
        assert torch.equal(x, y)
    for objs, opt, rows in zip(new, nopts, RB.rows_of(new)):
        RB.set_grads(objs, [[g * 7 for g in gk] for gk in grads], rows)
        opt.step()
    for k in range(len(models)):
        for a in NAMES:
            ps = [getattr(objs[k], a) for objs in new]
            assert_same(torch.cat([p.detach() for p in ps]), getattr(glob[k], a).detach(), (k, a))
            for mk in ("exp_avg", "exp_avg_sq"):
                assert_same(torch.cat([nopts[r].state[p][mk] for r, p in enumerate(ps)]), gopt.state[getattr(glob[k], a)][mk], (k, a, mk))


def each_rank_raises(world, fn):
    def body(r, tr):
        try:
            fn(r, tr)
        except ValueError as e:
            return e
        return None
    return run_ranks(world, body)


def test_mismatched_ranks_raise_everywhere(tmp_path):
    models, grads = make_models()
    world = 3
    shards, opts = trained_shards(models, grads, world)
    path = str(tmp_path / "x.pth")
    opts[1].step()  # rank 1 one Adam step ahead (its grads are still set)
    errs = each_rank_raises(world, lambda r, tr: SH.save_checkpoint(path, dict(zip(MODEL_NAMES, shards[r])), 1, opts[r], transport=tr))
    assert all(isinstance(e, ValueError) and "Adam step 3 on rank 0 and Adam step 4 on rank 1" in str(e) for e in errs), errs
    shards, opts = trained_shards(models, grads, world)
    shards[2][1]._semantic = torch.nn.Parameter(torch.zeros(shards[2][1]._xyz.shape[0], 5, device=DEV))
    errs = each_rank_raises(world, lambda r, tr: SH.gather_state(shards[r], None, transport=tr))
    assert all(isinstance(e, ValueError) and "on rank 2" in str(e) for e in errs), errs
    assert not (tmp_path / "x.pth").exists()
