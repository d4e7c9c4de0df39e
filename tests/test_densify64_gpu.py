"""GPU: sgr_densify_plan / sgr_densify_apply / sgr_reset_opacity (through street_gaussians_b200.training) element by element against
the fp64 restatement (oracle/densify64.py), on the Philox path the trainer runs (seed=) and on the noise= seam, over the scenes of
tests/densify64_case.py.

Exact: masks, the six counts, every row's parent and section, every copied parameter row, carried moments, zero moments for clones
and children, the optimizer's step counts and state keys, the zeroed statistics.  Within their bounds: child xyz and scaling, the
reset values.  A parent whose fp64 margin is below DELTA may take either decision: the kernel's is forced into the restatement
and everything else is still compared, so no model is skipped."""
import numpy as np
import pytest
import torch

import densify64_case as D
import densify_case as DC
from oracle import densify64 as D64
from street_gaussians_b200 import training

pytestmark = pytest.mark.gpu
DEV = "cuda"
DELTA = 1e-5
MIN_OP = 0.005
SEED = 0x5EED_1234_ABCD


def _run(models, *, seed=None, noise=None, prune_big=True, mode="fused", skip=()):
    objs = [DC.product_model(m, DEV) for m in models]
    groups = [[{"params": [getattr(o, DC.ATTR[a])], "lr": 0.0, "name": a} for a in DC.NAMES] for o in objs]
    opts = [torch.optim.Adam(g, lr=0.0, eps=1e-15) for g in groups] if mode == "adam" else \
        [training.FusedAdam([x for g in groups for x in g], lr=0.0, eps=1e-15)] * len(objs)
    for k, (o, m) in enumerate(zip(objs, models)):
        for a in DC.NAMES:
            if (k, a) in skip or m["in"]["exp_avg"][a] is None:
                continue
            opts[k].state[getattr(o, DC.ATTR[a])] = {"step": torch.tensor(7.0), "exp_avg": m["in"]["exp_avg"][a].clone().to(DEV),
                                                     "exp_avg_sq": m["in"]["exp_avg_sq"][a].clone().to(DEV)}
    opt = opts if mode == "adam" else opts[0]
    scal, masks = training._densify(objs, [m["grad_threshold"] for m in models], MIN_OP, prune_big, opt,
                                    [m["grad_col"] == 1 for m in models], seed, noise, keep_masks=True)
    return objs, opts, scal, masks.cpu().numpy().astype(np.int64)


def _same(got, exp):
    """Bit-equal as fp32, NaN equal to NaN."""
    return np.array_equal(got.astype(np.float32), exp.astype(np.float32), equal_nan=True)


def _within(got, exp, bound):
    got = got.astype(np.float64)
    fin = np.isfinite(exp)
    ok = np.array_equal(np.isnan(got), np.isnan(exp)) and np.array_equal(got[~fin & ~np.isnan(exp)], exp[~fin & ~np.isnan(exp)])
    err = np.abs(got[fin] - exp[fin])
    ratio = float((err / np.maximum(bound[fin], 1e-300)).max()) if err.size else 0.0
    return ok and ratio <= 1.0, ratio


def _check(models, objs, opts, scal, masks, *, seed=None, prune_big=True, skip=(), claims=()):
    """Every model against densify64; returns (forced parents, largest child error / bound)."""
    at, forced_total, worst = 0, 0, 0.0
    for k, (m, o) in enumerate(zip(models, objs)):
        n = m["in"]["xyz"].shape[0]
        kw = DC.oracle_kwargs(m, MIN_OP, prune_big)
        if seed is None:
            draws, db = m["draws"], None
        else:
            draws, db = D64.philox_normals64(seed, np.arange(at, at + n))
        mine = masks[at:at + n]
        at += n
        r0 = D64.densify64(m["in"], m["kind"], draws, draw_bound=db, **kw)
        low = r0["margin"] < DELTA
        diff = mine != r0["natural"]
        assert not (diff & ~low).any(), (k, np.nonzero(diff & ~low)[0][:8], mine[diff & ~low][:8], r0["natural"][diff & ~low][:8])
        fp = np.nonzero(low)[0]
        forced_total += int(diff.sum())
        r = D64.densify64(m["in"], m["kind"], draws, draw_bound=db, decisions=(fp, mine[fp]), **kw)
        for key, v in r0["scalars"].items():  # a parent decided the other way moves each count by at most 2
            assert abs(scal[k][key] - v) <= 2 * int(diff.sum()), (k, key, scal[k][key], v)
            if not diff.any():
                assert scal[k][key] == v, (k, key, scal[k][key], v)
        assert set(scal[k]) == set(r0["scalars"])
        child = r["section"] >= 2
        for a in DC.NAMES:
            got = getattr(o, DC.ATTR[a]).detach().cpu().numpy()
            exp = r["rows"][a]
            assert got.shape == exp.shape, (k, a, got.shape, exp.shape)
            if a in ("xyz", "scaling"):
                assert _same(got[~child], exp[~child]), (k, a)
                ok, ratio = _within(got[child], exp[child], r["bound"][a][child])
                worst = max(worst, ratio)
                assert ok, (k, a, ratio)
            else:
                assert _same(got, exp), (k, a)
            p = getattr(o, DC.ATTR[a])
            st = opts[k].state.get(p)
            if (k, a) in skip or m["in"]["exp_avg"][a] is None:
                assert st is None, (k, a)
                continue
            assert float(st["step"]) == 7.0 and set(st) == {"step", "exp_avg", "exp_avg_sq"}
            for mk in ("exp_avg", "exp_avg_sq"):
                src = m["in"][mk][a].numpy()[r["parent"]]
                src[~r["carries"]] = 0.0
                assert _same(st[mk].cpu().numpy(), src), (k, a, mk)
        for s, w in (("xyz_gradient_accum", (2,)), ("denom", (1,)), ("max_radii2D", ())):
            got = getattr(o, s)
            assert tuple(got.shape) == (r["parent"].size,) + w and not got.any(), (k, s)
    # the old parameters left the optimizers' state: one entry per tensor that had moments
    n_state = sum(len(x.state) for x in {id(x): x for x in opts}.values())
    assert n_state == sum(1 for k, m in enumerate(models) for a in DC.NAMES if (k, a) not in skip and m["in"]["exp_avg"][a] is not None)
    for c in claims:   # designed parents with a known outcome decide it so on the device whatever their margin
        if len(c) == 4 and c[0] not in ("tile",) and c[3] is not None:
            _, k, l, expect = c
            start = sum(mm["in"]["xyz"].shape[0] for mm in models[:k])
            assert masks[start + l] == expect, (c, masks[start + l])
    return forced_total, worst


def _both_paths(build, **kw):
    for seed in (SEED, None):
        models, claims = build()
        noise = None if seed is not None else torch.cat([m["draws"] for m in models]).to(DEV).contiguous()
        res = _run(models, seed=seed, noise=noise, **kw)
        _check(models, *res, seed=seed, claims=claims if kw.get("prune_big", True) else (), prune_big=kw.get("prune_big", True), skip=kw.get("skip", ()))


@pytest.mark.parametrize("case", ["edge_sizes", "many_40", "many_70", "tiles", "box_sensitive"])
def test_densify64_segments_and_tiles(case):
    build = {"edge_sizes": D.edge_sizes, "many_40": lambda: D.many_actors(40, 2), "many_70": lambda: D.many_actors(70, 3),
             "tiles": D.tiles, "box_sensitive": D.box_sensitive}[case]
    _both_paths(build)


@pytest.mark.parametrize("prune_big", [True, False])
@pytest.mark.parametrize("grad_col_bkgd", [0, 1])
def test_densify64_thresholds_and_overflow(prune_big, grad_col_bkgd):
    _both_paths(lambda: D.edges(grad_col_bkgd=grad_col_bkgd), prune_big=prune_big)


@pytest.mark.parametrize("mode", ["fused", "adam"])
@pytest.mark.parametrize("layout", ["M1_S0_fourier5", "missing_moments"])
def test_densify64_optimizer_layouts(mode, layout):
    if layout == "M1_S0_fourier5":
        _both_paths(lambda: D.edges(M=1, S=0, C_act=5), mode=mode)
    else:
        _both_paths(lambda: D.edges(M=4, S=3), mode=mode, skip={(0, "f_rest"), (1, "xyz"), (1, "semantic"), (0, "opacity")})


def test_philox_draws_within_bound_and_seam_matches_seed_path():
    """Child c's xyz is draws [3c, 3c + 3) exactly in the readout scene: the device's Philox normals against philox_normals64.
    Then the device's own draws fed through noise= must give every output bit-equal to seed= (the seam is the production path)."""
    models, _ = D.readout()
    objs, _, scal, masks = _run(models, seed=SEED, prune_big=False)
    P = sum(m["in"]["xyz"].shape[0] for m in models)
    z, zb = D64.philox_normals64(SEED, np.arange(P))
    dev = np.zeros((P, 18), dtype=np.float32)
    at, worst = 0, 0.0
    for m, o, s in zip(models, objs, scal):
        n = m["in"]["xyz"].shape[0]
        assert s["points_split"] == n and (masks[at:at + n] == 12).all()
        xyz = o._xyz.detach().cpu().numpy()
        for c in range(2):
            dev[at:at + n, 3 * c:3 * c + 3] = xyz[c * n:(c + 1) * n]
        at += n
    err = np.abs(dev[:, :6].astype(np.float64) - z[:, :6])
    ratio = err / zb[:, :6]
    worst = float(ratio.max())
    print(f"\nPhilox draws on the device vs philox_normals64: {P * 6} draws, max |err| {err.max():.3e}, "
          f"max err/bound {worst:.3f} (bound assumes __sincosf within 2^-19)")
    assert worst <= 1.0
    # the seam: a scene of the same composed size that reads only draws [0, 6) (no box test), random poses and scales
    g = torch.Generator().manual_seed(21)
    for m in models:
        t = m["in"]
        n = t["xyz"].shape[0]
        t["xyz"] = torch.randn(n, 3, generator=g)
        t["rotation"] = torch.randn(n, 4, generator=g)
        t["scaling"] = torch.randn(n, 3, generator=g) * 0.5
        t["opacity"] = torch.randn(n, 1, generator=g) * 4
        t["xyz_gradient_accum"] = torch.rand(n, 2, generator=g) * 2e-3
    a = _run(models, seed=SEED, prune_big=False)
    b = _run(models, noise=torch.from_numpy(dev).to(DEV), prune_big=False)
    assert a[2] == b[2] and np.array_equal(a[3], b[3])
    for oa, ob in zip(a[0], b[0]):
        for name in list(DC.ATTR.values()) + ["xyz_gradient_accum", "denom", "max_radii2D"]:
            assert torch.equal(getattr(oa, name), getattr(ob, name)), name
    for pa, pb in zip((p for g_ in a[1][0].param_groups for p in g_["params"]), (p for g_ in b[1][0].param_groups for p in g_["params"])):
        for mk in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(a[1][0].state[pa][mk], b[1][0].state[pb][mk])


def test_reset_opacity64_three_launches():
    """1 background + 70 actors (three launches of 32 segments), raw opacity from -200 to 200 with both sides of the 0.01 cap and
    the whole region where sigmoid is subnormal in fp32; against the reference's own expression in torch on the same device
    (bit-equal) and against reset_opacity64 (within its bound outside that region)."""
    rs = np.random.RandomState(4)
    logit = float(np.log(0.01 / 0.99))
    vals = np.concatenate([np.linspace(-200, 200, 40001), np.linspace(-110, -80, 30001), logit + np.arange(-64, 65) * 4.8e-7,
                           [-100.0, 100.0, 0.0, -0.0, -88.72284, -87.33655, -103.97208]]).astype(np.float32)
    rs.shuffle(vals)
    sizes = [0 if rs.rand() < 0.15 else int(rs.randint(1, 3000)) for _ in range(71)]
    sizes[0] = 0
    sizes[5] = sizes[40] = 0
    tot = sum(sizes)
    vals = np.resize(vals, tot)
    objs, at = [], 0
    for k, n in enumerate(sizes):
        o = {"_opacity": torch.nn.Parameter(torch.from_numpy(vals[at:at + n].copy()).reshape(n, 1).to(DEV)),
             "_xyz": torch.nn.Parameter(torch.zeros(n, 3, device=DEV))}
        objs.append(o)
        at += n
    opt = training.FusedAdam([{"params": [o["_opacity"], o["_xyz"]], "lr": 0.0} for o in objs], lr=0.0)
    for o in objs:
        for name in ("_opacity", "_xyz"):
            p = o[name]
            opt.state[p] = {"step": torch.tensor(3.0), "exp_avg": torch.rand_like(p) + 1, "exp_avg_sq": torch.rand_like(p) + 1}
    before_xyz = {id(o["_xyz"]): opt.state[o["_xyz"]]["exp_avg"].clone() for o in objs}
    src = torch.from_numpy(vals).to(DEV)
    training.reset_opacity(objs, opt)
    got = torch.cat([o["_opacity"].detach().reshape(-1) for o in objs])
    sig = torch.sigmoid(src)
    ref = torch.log(torch.min(sig, torch.ones_like(sig) * 0.01) / (1 - torch.min(sig, torch.ones_like(sig) * 0.01)))
    assert torch.equal(got, ref), int((got != ref).sum())
    r, bound, region = D64.reset_opacity64(vals)
    g64 = got.cpu().numpy().astype(np.float64)
    ok, ratio = _within(g64[~region], r[~region], bound[~region])
    assert ok, ratio
    assert region.sum() > 1000 and np.isneginf(g64[vals <= -104]).all()
    for o in objs:
        st = opt.state[o["_opacity"]]
        assert not st["exp_avg"].any() and not st["exp_avg_sq"].any() and float(st["step"]) == 3.0
        assert torch.equal(opt.state[o["_xyz"]]["exp_avg"], before_xyz[id(o["_xyz"])])
