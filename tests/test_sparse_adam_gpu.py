"""GPU: training.SparseAdam (sgr_sparse_adam_step) against training.FusedAdam, bit for bit.  Visible rows must carry FusedAdam's
update exactly; invisible rows, tensors without a gradient, tensors of models not passed and non-per-Gaussian tensors must keep
their bits and their step count.  Rows that are never visible are seeded with NaN, so a stray read or write shows."""
import math
import types

import pytest
import torch

import densify_case as DC
from street_gaussians_b200 import training

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = training.PARAM_NAMES
ACTOR_SIZES = (0, 1, 31, 32, 33, 255, 256, 257, 50_000)


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def _width(p):
    return int(math.prod(p.shape[1:]))


def _rows(t):
    return t.detach().reshape(t.shape[0], _width(t))


def _model(n, dc, S, gen):
    m = types.SimpleNamespace()
    for name, tail in zip(NAMES, ((3,), (dc, 3), (15, 3), (1,), (3,), (4,), (S,))):
        setattr(m, name, torch.nn.Parameter(torch.randn((n,) + tail, generator=gen, device=DEV)))
    return m


def _scene(actor_sizes, S, seed=0, n_bkgd=200_000):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return [_model(n_bkgd, 1, S, gen)] + [_model(n, 5, S, gen) for n in actor_sizes], gen


def _segments(models):
    counts = torch.tensor([m._xyz.shape[0] for m in models], device=DEV)
    starts = torch.cumsum(counts, 0) - counts
    seg = torch.repeat_interleave(torch.arange(len(models), device=DEV), counts)
    local = torch.arange(int(counts.sum()), device=DEV) - starts[seg]
    return counts.tolist(), local


def _pattern(name, models, step, gen):
    counts, local = _segments(models)
    P = sum(counts)
    if name == "none":
        return torch.zeros(P, dtype=torch.bool, device=DEV)
    if name == "single":
        v = torch.zeros(P, dtype=torch.bool, device=DEV)
        v[int(torch.randint(0, P, (1,), generator=gen, device=DEV))] = True
        return v
    if name == "tile_first":
        return local % 256 == 0
    if name == "tile_last":
        end = torch.repeat_interleave(torch.tensor(counts, device=DEV), torch.tensor(counts, device=DEV))
        return (local % 256 == 255) | (local == end - 1)
    frac = float(name[len("random"):])
    return torch.rand(P, generator=gen, device=DEV) < frac


def _seed_state(opt, params, gen, step=3):
    for p in params:
        opt.state[p] = {"step": step, "exp_avg": torch.randn(p.shape, generator=gen, device=DEV) * 1e-2,
                        "exp_avg_sq": torch.rand(p.shape, generator=gen, device=DEV) * 1e-4}


def _clone_opt(params, opt, groups_of):
    """FusedAdam over clones of `params`, with the same groups' hyper-parameters and clones of opt's state and gradients."""
    clones, groups = [], []
    for p in params:
        q = torch.nn.Parameter(p.detach().clone())
        q.grad = None if p.grad is None else p.grad.clone()
        g = groups_of[id(p)]
        groups.append({"params": [q], "lr": g["lr"], "betas": g["betas"], "eps": g["eps"]})
        clones.append(q)
    fa = training.FusedAdam(groups)
    for p, q in zip(params, clones):
        st = opt.state[p]
        fa.state[q] = {"step": st["step"], "exp_avg": st["exp_avg"].clone(), "exp_avg_sq": st["exp_avg_sq"].clone()}
    return fa, clones


def _run(models, pattern, gen, steps=3, betas_alt=False):
    """Three masked steps with a changing visibility and per-group lr; after each one, every tensor is compared with FusedAdam
    run on a clone of the state before the step: visible rows bit-equal, invisible rows unchanged."""
    counts, _ = _segments(models)
    params = [getattr(m, n) for m in models for n in NAMES]
    groups = [{"params": [p], "lr": 1e-3 * (1 + i % 5), "betas": (0.8, 0.99) if betas_alt and i % 2 else (0.9, 0.999)}
              for i, p in enumerate(params)]
    opt = training.SparseAdam(groups, eps=1e-15)
    groups_of = {id(g["params"][0]): g for g in opt.param_groups}
    _seed_state(opt, params, gen)
    masks = [_pattern(pattern, models, s, gen) for s in range(steps)]
    full = all(bool(m.all()) for m in masks)
    dense = _clone_opt(params, opt, groups_of) if full else None   # check 3: a FusedAdam run over all steps
    never = ~torch.stack(masks).any(0)
    row_of = {}
    at = 0
    for m, n in zip(models, counts):
        for name in NAMES:
            row_of[id(getattr(m, name))] = slice(at, at + n)
        at += n
    for p in params:   # rows that are never visible hold NaN in the parameter and both moments
        nv = never[row_of[id(p)]]
        for t in (p.data, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"]):
            _rows(t)[nv] = float("nan")
    for s, vis in enumerate(masks):
        radii = torch.where(vis, torch.randint(1, 40, vis.shape, generator=gen, device=DEV), 0).to(torch.int32)
        for i, p in enumerate(params):
            p.grad = torch.randn(p.shape, generator=gen, device=DEV)
            _rows(p.grad)[~vis[row_of[id(p)]]] = float("nan")   # never read
            groups_of[id(p)]["lr"] = 1e-3 * (1 + (i + s) % 5) * (s + 1)
        ref, ref_p = _clone_opt(params, opt, groups_of)
        ref.step()
        before = {id(p): [bits(t).clone() for t in (p, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])] for p in params}
        steps_before = {id(p): opt.state[p]["step"] for p in params}
        if dense is not None:
            for i, (p, q) in enumerate(zip(params, dense[1])):
                q.grad = p.grad.clone()
                dense[0].param_groups[i]["lr"] = groups_of[id(p)]["lr"]
            dense[0].step()
        opt.step(models, radii)
        for p, q in zip(params, ref_p):
            v = vis[row_of[id(p)]]
            got = (p, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])
            exp = (q, ref.state[q]["exp_avg"], ref.state[q]["exp_avg_sq"])
            for j in range(3):
                g, e, b = _rows(bits(got[j])), _rows(bits(exp[j])), _rows(before[id(p)][j])
                assert torch.equal(g[v], e[v]), (pattern, s, tuple(p.shape), j)
                assert torch.equal(g[~v], b[~v]), (pattern, s, tuple(p.shape), j)
                assert torch.isfinite(_rows(got[j])[v]).all()
            assert opt.state[p]["step"] == steps_before[id(p)] + 1 == ref.state[q]["step"]
    if dense is not None:
        for p, q in zip(params, dense[1]):
            assert torch.equal(bits(p), bits(q))
            for key in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(bits(opt.state[p][key]), bits(dense[0].state[q][key]))
    return opt


@pytest.mark.parametrize("S", [0, 3])
@pytest.mark.parametrize("pattern", ["none", "single", "tile_first", "tile_last", "random0.001", "random0.3", "random1.0"])
def test_sparse_adam_matches_fused_adam_on_visible_rows(pattern, S):
    models, gen = _scene(ACTOR_SIZES, S, seed=S)
    _run(models, pattern, gen)


def test_sparse_adam_65_segments_two_beta_buckets():
    models, gen = _scene([(0, 1, 31, 32, 33, 255, 256, 257)[k % 8] for k in range(64)], 3, seed=5, n_bkgd=20_000)
    assert len(models) == 65
    _run(models, "random0.3", gen, betas_alt=True)


def test_sparse_adam_leaves_other_tensors_alone():
    gen = torch.Generator(device=DEV).manual_seed(9)
    a, b, c = _model(1000, 1, 0, gen), _model(300, 5, 3, gen), _model(500, 5, 3, gen)
    pose = torch.nn.Parameter(torch.randn(3, 7, generator=gen, device=DEV))
    held = [getattr(m, n) for m in (a, b) for n in NAMES] + [getattr(c, n) for n in NAMES[:-1]] + [pose]   # c._semantic not held
    opt = training.SparseAdam([{"params": [p], "lr": 1e-2} for p in held], eps=1e-15)
    _seed_state(opt, held, gen, step=4)
    for p in held + [c._semantic]:
        p.grad = torch.randn(p.shape, generator=gen, device=DEV)
    a._scaling.grad = None
    snap = {id(p): [bits(p).clone()] + ([bits(opt.state[p][k]).clone() for k in ("exp_avg", "exp_avg_sq")] if p in opt.state else [])
            for p in held + [c._semantic]}
    radii = (torch.rand(1500, generator=gen, device=DEV) < 0.5).to(torch.int32) * 3
    opt.step([a, c], radii)        # b (an actor absent from the frame) and the pose are not passed
    untouched = [getattr(b, n) for n in NAMES] + [pose, a._scaling]
    for p in untouched:
        assert opt.state[p]["step"] == 4
        assert all(torch.equal(x, y) for x, y in zip(snap[id(p)], [bits(p), bits(opt.state[p]["exp_avg"]), bits(opt.state[p]["exp_avg_sq"])]))
    assert c._semantic not in opt.state and torch.equal(bits(c._semantic), snap[id(c._semantic)][0])
    for p in [a._xyz, a._opacity] + [getattr(c, n) for n in NAMES[:-1]]:
        assert opt.state[p]["step"] == 5
    assert not torch.equal(bits(a._xyz), snap[id(a._xyz)][0])


@pytest.mark.parametrize("bad", ["lr_nan", "lr_inf", "beta_one"])
def test_sparse_adam_bad_group_steps_nothing(bad):
    """A group that sgr_sparse_adam_step would reject, in the last of two (betas, eps) buckets: the call raises before any tensor of
    either bucket is stepped, so no step count advances and no bit changes."""
    models, gen = _scene((31, 300), 0, seed=4, n_bkgd=3000)
    params = [getattr(m, n) for m in models for n in NAMES]
    groups = [{"params": [p], "lr": 1e-3, "betas": (0.8, 0.99) if i % 2 else (0.9, 0.999)} for i, p in enumerate(params)]
    opt = training.SparseAdam(groups, eps=1e-15)
    _seed_state(opt, params, gen)
    for p in params:
        p.grad = torch.randn(p.shape, generator=gen, device=DEV)
    g = opt.param_groups[-2]   # an odd group: the (0.8, 0.99) bucket, which comes second
    if bad == "beta_one":
        g["betas"] = (0.8, 1.0)
    else:
        g["lr"] = float("nan") if bad == "lr_nan" else float("inf")
    snap = {id(p): [bits(t).clone() for t in (p, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])] for p in params}
    radii = torch.ones(3331, dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError, match="lr" if bad != "beta_one" else "betas"):
        opt.step(models, radii)
    torch.cuda.synchronize()
    for p in params:
        assert opt.state[p]["step"] == 3
        assert all(torch.equal(x, bits(t)) for x, t in zip(snap[id(p)], (p, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])))


def test_sparse_adam_through_densify_and_reset_opacity():
    fixture, min_op = DC.load()
    objs_s = [DC.product_model(m, DEV) for m in fixture]
    objs_f = [DC.product_model(m, DEV) for m in fixture]
    opts = []
    for objs, cls in ((objs_s, training.SparseAdam), (objs_f, training.FusedAdam)):
        opt = cls([{"params": [getattr(o, DC.ATTR[a])], "lr": 1e-3 * (1 + i), "name": a} for o in objs for i, a in enumerate(DC.NAMES)], eps=1e-15)
        for o, m in zip(objs, fixture):
            for a in DC.NAMES:
                opt.state[getattr(o, DC.ATTR[a])] = {"step": int(m["in"]["step"][a]), "exp_avg": m["in"]["exp_avg"][a].clone().to(DEV),
                                                     "exp_avg_sq": m["in"]["exp_avg_sq"][a].clone().to(DEV)}
        noise = torch.cat([m["draws"] for m in fixture]).to(DEV).contiguous()
        training.densify_and_prune(objs, [m["grad_threshold"] for m in fixture], min_op, True, opt,
                                   grad_abs=[m["grad_col"] == 1 for m in fixture], noise=noise)
        opts.append(opt)
    sa, fa = opts
    gen = torch.Generator(device=DEV).manual_seed(3)
    counts = [o._xyz.shape[0] for o in objs_s]
    assert counts != [m["in"]["xyz"].shape[0] for m in fixture]
    vis = torch.rand(sum(counts), generator=gen, device=DEV) < 0.4
    radii = vis.to(torch.int32) * 7
    before = {}
    at = 0
    for os_, of, n in zip(objs_s, objs_f, counts):
        for a in DC.NAMES:
            ps, pf = getattr(os_, DC.ATTR[a]), getattr(of, DC.ATTR[a])
            assert torch.equal(bits(ps), bits(pf))
            for key in ("exp_avg", "exp_avg_sq"):
                assert sa.state[ps][key].shape == ps.shape and torch.equal(bits(sa.state[ps][key]), bits(fa.state[pf][key]))
            ps.grad = torch.randn(ps.shape, generator=gen, device=DEV)
            pf.grad = ps.grad.clone()
            before[id(ps)] = (slice(at, at + n), [bits(t).clone() for t in (ps, sa.state[ps]["exp_avg"], sa.state[ps]["exp_avg_sq"])])
        at += n
    sa.step(objs_s, radii)
    fa.step()
    for os_, of in zip(objs_s, objs_f):
        for a in DC.NAMES:
            ps, pf = getattr(os_, DC.ATTR[a]), getattr(of, DC.ATTR[a])
            rows, b = before[id(ps)]
            v = vis[rows]
            for j, (g, e) in enumerate(zip((ps, sa.state[ps]["exp_avg"], sa.state[ps]["exp_avg_sq"]),
                                           (pf, fa.state[pf]["exp_avg"], fa.state[pf]["exp_avg_sq"]))):
                assert torch.equal(_rows(bits(g))[v], _rows(bits(e))[v]), (a, j)
                assert torch.equal(_rows(bits(g))[~v], _rows(b[j])[~v]), (a, j)
            assert sa.state[ps]["step"] == fa.state[pf]["step"]
    training.reset_opacity(objs_s, sa)
    for o in objs_s:
        st = sa.state[o._opacity]
        assert not st["exp_avg"].any() and not st["exp_avg_sq"].any()
        assert (torch.sigmoid(o._opacity.detach()) <= 0.0100001).all()


def test_state_dict_round_trips_fused_sparse_fused():
    models, gen = _scene((31, 300), 0, seed=2, n_bkgd=5000)
    params = [getattr(m, n) for m in models for n in NAMES]
    groups = lambda: [{"params": [p], "lr": 1e-3 * (1 + i % 3)} for i, p in enumerate(params)]
    fa = training.FusedAdam(groups(), eps=1e-15)
    for p in params:
        p.grad = torch.randn(p.shape, generator=gen, device=DEV)
    fa.step()
    sd = fa.state_dict()
    sa = training.SparseAdam(groups(), eps=1e-15)
    sa.load_state_dict(sd)
    snap = {id(p): [bits(fa.state[p][k]).clone() for k in ("exp_avg", "exp_avg_sq")] for p in params}
    for p in params:
        assert sa.state[p]["step"] == 1
        assert all(torch.equal(bits(sa.state[p][k]), s) for k, s in zip(("exp_avg", "exp_avg_sq"), snap[id(p)]))
    radii = (torch.rand(5331, generator=gen, device=DEV) < 0.5).to(torch.int32)
    sa.step(models, radii)
    fb = training.FusedAdam(groups(), eps=1e-15)
    fb.load_state_dict(sa.state_dict())
    for p in params:
        assert fb.state[p]["step"] == sa.state[p]["step"] == 2
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(bits(fb.state[p][k]), bits(sa.state[p][k]))
    fb.step()
    assert all(fb.state[p]["step"] == 3 for p in params)


def test_end_to_end_training_step_leaves_culled_gaussians_alone():
    import street_gaussians_b200 as sgb
    from street_gaussians_b200 import losses, synthetic
    import util
    scene = synthetic.make_scene(P=20_000, width=320, height=208, sh_degree=3, seed=5, n_vehicles=2, per_vehicle=2000, with_raw=True,
                                 scale_med=0.05)
    raw = scene["raw"]
    bg = raw["models"][0]
    bg["xyz"][::3, 2] *= -1.0       # a third of the background behind the camera
    bg["xyz"][1::5, 0] *= 6.0       # a fifth beside it
    objs = []
    for r in raw["models"]:
        o = types.SimpleNamespace(**{"_" + a: torch.nn.Parameter(v.clone().to(DEV)) for a, v in r.items()})
        o._semantic = torch.nn.Parameter(torch.zeros(r["xyz"].shape[0], 0, device=DEV))
        objs.append(o)
    params = [getattr(o, n) for o in objs for n in NAMES]
    opt = training.SparseAdam([{"params": [p], "lr": 1e-3 * (1 + i % 4)} for i, p in enumerate(params)], eps=1e-15)
    gen = torch.Generator(device=DEV).manual_seed(1)
    _seed_state(opt, params, gen)
    rast = sgb.GaussianRasterizer(util.settings_from(sgb, scene["cam"], DEV))
    poses, idft = raw["poses"].to(DEV), raw["idft"].to(DEV)
    gt = torch.rand(3, 208, 320, generator=gen, device=DEV)
    xyz, rot, scale, opac, sh = sgb.compose(objs, poses, idft)
    col, radii, _, _, _ = rast(means3D=xyz, means2D=torch.zeros_like(xyz, requires_grad=True), opacities=opac, shs=sh, scales=scale,
                               rotations=rot)
    losses.photometric_loss(col, gt, None, 1.0, 0.2).backward()
    vis = radii > 0
    n_bg = objs[0]._xyz.shape[0]
    assert vis[:n_bg].any() and (~vis[:n_bg]).any() and vis[n_bg:].any()
    fa, clones = _clone_opt(params, opt, {id(g["params"][0]): g for g in opt.param_groups})
    fa.step()
    before = [bits(p).clone() for p in params]
    opt.step(objs, radii)
    at, moved = 0, False
    for k, o in enumerate(objs):
        n = o._xyz.shape[0]
        v = vis[at:at + n]
        at += n
        for a, name in enumerate(NAMES):
            p = getattr(o, name)
            q, b = clones[k * len(NAMES) + a], before[k * len(NAMES) + a]
            assert torch.equal(_rows(bits(p))[v], _rows(bits(q))[v]), name
            assert torch.equal(_rows(bits(p))[~v], _rows(b)[~v]), name
            moved |= not torch.equal(_rows(bits(q))[~v], _rows(b)[~v])
    assert moved   # the dense step does move culled Gaussians (their momentum); the masked one does not
