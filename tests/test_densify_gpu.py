"""GPU: sgr_densify_plan / sgr_densify_apply / sgr_reset_opacity (through street_gaussians_b200.training) against the reference's own
densify_and_prune (tests/golden/callsite/densify.npz) and against the torch oracle (oracle/densify_oracle.py) with fp64 margins."""
import types

import numpy as np
import pytest
import torch

import densify_case as DC
from oracle import densify_oracle as DO
from street_gaussians_b200 import training

pytestmark = pytest.mark.gpu
DEV = "cuda"
ULP = 2.0 ** -24


def _ulp(x):
    return (torch.nextafter(x.abs(), torch.full_like(x, float("inf"))) - x.abs())


def _attach_state(opt, p, m, v, step):
    opt.state[p] = {"step": torch.tensor(float(step)), "exp_avg": m.clone().to(DEV).contiguous(), "exp_avg_sq": v.clone().to(DEV).contiguous()}


def _optimizers(objs, models, mode, skip=()):
    """Per-model torch.optim.Adam (the reference's layout) or one FusedAdam whose groups repeat the names of every model."""
    groups = [[{"params": [getattr(o, DC.ATTR[a])], "lr": 0.0, "name": a} for a in DC.NAMES] for o in objs]
    opts = [torch.optim.Adam(g, lr=0.0, eps=1e-15) for g in groups] if mode == "adam" else \
        [training.FusedAdam([x for g in groups for x in g], lr=0.0, eps=1e-15)]
    for k, (o, m) in enumerate(zip(objs, models)):
        opt = opts[k] if mode == "adam" else opts[0]
        for a in DC.NAMES:
            if (k, a) in skip:
                continue
            _attach_state(opt, getattr(o, DC.ATTR[a]), m["in"]["exp_avg"][a], m["in"]["exp_avg_sq"][a], m["in"]["step"][a])
    return opts if mode == "adam" else opts[0]


def _child_xyz_bound(t, draws, parent, section):
    """|R| |z s| + |xyz| per element, times 16 roundings: the error budget of R (z (*) s) + x in fp32 against the reference's.  An
    entry of R carries an absolute rounding error of a few 2^-24 however small it is (R is built from a unit quaternion), so |R|
    is taken as its bound 1: |R| |z s| -> sum_k |z_k s_k|."""
    p = parent.to(DEV)
    c = (section.to(DEV) - 2).clamp(min=0)
    s = torch.exp(t["scaling"].to(DEV).double())[p]
    z = torch.stack([draws.to(DEV).double()[p, 3 * c + j] for j in range(3)], dim=1)
    mag = (z * s).abs().sum(dim=1, keepdim=True) + t["xyz"].to(DEV).double()[p].abs()
    return 16 * ULP * mag


def _compare_model(k, out_p, out_m, ref, parent, section, t, draws, step_expect=None, opt_state=None):
    child = section >= 2
    for a in DC.NAMES:
        got, exp = out_p[a].detach(), ref[a].to(DEV)
        assert got.shape == exp.shape, (k, a)
        if got.numel() == 0:
            continue
        if a == "xyz":
            rows = ~child.to(DEV)
            assert torch.equal(got[rows], exp[rows]), (k, a)
            if child.any():
                bound = _child_xyz_bound(t, draws, parent[child], section[child])
                err = (got[child.to(DEV)].double() - exp[child.to(DEV)].double()).abs()
                assert (err <= bound).all(), (k, float((err / bound).max()))
        elif a == "scaling":
            rows = ~child.to(DEV)
            assert torch.equal(got[rows], exp[rows]), (k, a)
            if child.any():
                e = exp[child.to(DEV)]
                err = (got[child.to(DEV)] - e).abs()
                assert (err <= 2 * _ulp(e) + 2 * ULP * 2).all(), (k, float(err.max()))
        else:
            assert torch.equal(got, exp), (k, a)
        if out_m is not None and out_m[a] is not None:
            for j, mk in enumerate(("exp_avg", "exp_avg_sq")):
                assert torch.equal(out_m[a][j], ref[mk][a].to(DEV)), (k, a, mk)
                assert not out_m[a][j][(section != 0).to(DEV)].any()


def _run_fixture(mode):
    models, min_op = DC.load()
    objs = [DC.product_model(m, DEV) for m in models]
    opt = _optimizers(objs, models, mode)
    noise = torch.cat([m["draws"] for m in models]).to(DEV).contiguous()
    scal = training.densify_and_prune(objs, [m["grad_threshold"] for m in models], min_op, True, opt,
                                      grad_abs=[m["grad_col"] == 1 for m in models], noise=noise)
    opts = opt if isinstance(opt, list) else [opt] * len(models)
    for k, (o, m) in enumerate(zip(objs, models)):
        for key, v in m["scalars"].items():
            assert scal[k][key] == v, (k, key)
        _, _, _, parent, section = DO.densify_model(m["in"], m["kind"], m["draws"], **DC.oracle_kwargs(m, min_op))
        params = {a: getattr(o, DC.ATTR[a]) for a in DC.NAMES}
        mom = {}
        for a, p in params.items():
            assert any(p is q for g in opts[k].param_groups for q in g["params"]), (k, a)
            st = opts[k].state[p]
            assert float(st["step"]) == m["out"]["step"][a]
            mom[a] = (st["exp_avg"], st["exp_avg_sq"])
        _compare_model(k, params, mom, m["out"], parent, section, m["in"], m["draws"])
        for s in ("xyz_gradient_accum", "denom", "max_radii2D"):
            got = getattr(o, s)
            assert got.shape == m["out"][s].shape and not got.any()
    # the old parameters left the optimizers' state
    n_state = sum(len(x.state) for x in set(opts))
    assert n_state == 7 * len(models)


@pytest.mark.parametrize("mode", ["adam", "fused_shared"])
def test_densify_matches_reference_fixture(mode):
    _run_fixture(mode)


# ---- synthetic scenes against the oracle on the GPU ----
def _synthetic(n_bkgd, n_act, per_act, M=16, S=0, C=5, seed=0, state=True):
    g = torch.Generator().manual_seed(seed)
    models, metas = [], []
    for k in range(1 + n_act):
        n = n_bkgd if k == 0 else per_act
        bk = k == 0
        rn = lambda *s: torch.randn(*s, generator=g)
        t = dict(xyz=rn(n, 3) * (torch.tensor([8.0, 3.0, 10.0]) if bk else torch.tensor([1.2, 0.5, 0.4])) + (torch.tensor([0.0, 0.0, 20.0]) if bk else 0),
                 f_dc=rn(n, 1 if bk else C, 3), f_rest=rn(n, M - 1, 3) * 0.2, opacity=rn(n, 1) * 3.0,
                 scaling=math_log(0.1 if bk else 0.03) + rn(n, 3) * 0.6, rotation=rn(n, 4), semantic=torch.rand(n, S, generator=g))
        denom = torch.randint(0, 6, (n, 1), generator=g).float()
        t["xyz_gradient_accum"] = denom * torch.rand(n, 2, generator=g) * (1.6e-3 if bk else 4e-4)
        t["denom"], t["max_radii2D"] = denom, torch.rand(n, generator=g) * 20
        for mk in ("exp_avg", "exp_avg_sq"):
            t[mk] = {a: (rn(*t[a].shape).abs() * 1e-3 if state else None) for a in DC.NAMES}
        t["step"] = {a: 7.0 for a in DC.NAMES}
        meta = dict(kind="background" if bk else "actor", grad_col=1 if bk else 0, grad_threshold=6e-4 if bk else 2e-4,
                    extent=torch.tensor([20.0 if bk else 3.375]), percent_dense=0.01, percent_big_ws=0.1, in_=t,
                    draws=torch.randn(n, 18, generator=g))
        if bk:
            meta.update(sphere_center=torch.tensor([0.0, 0.0, 20.0]), sphere_radius=torch.tensor([12.0]))
        else:
            meta.update(min_xyz=torch.tensor([-2.25, -1.0, -0.8]), max_xyz=torch.tensor([2.25, 1.0, 0.8]))
        meta["in"] = t
        models.append(meta)
    return models


def math_log(x):
    return float(np.log(x))


def _run_vs_oracle(models, min_op=0.005, prune_big=True, objs_skip_state=(), seed=None, use_noise=True):
    objs = [DC.product_model(m, DEV) for m in models]
    skip = set(objs_skip_state)
    opt = training.FusedAdam([{"params": [getattr(o, DC.ATTR[a])], "lr": 0.0, "name": a} for o in objs for a in DC.NAMES], lr=0.0)
    for k, (o, m) in enumerate(zip(objs, models)):
        for a in DC.NAMES:
            if (k, a) not in skip and m["in"]["exp_avg"][a] is not None:
                _attach_state(opt, getattr(o, DC.ATTR[a]), m["in"]["exp_avg"][a], m["in"]["exp_avg_sq"][a], 7)
    noise = torch.cat([m["draws"] for m in models]).to(DEV).contiguous() if use_noise else None
    scal, masks = training._densify(objs, [m["grad_threshold"] for m in models], min_op, prune_big, opt,
                                    [m["grad_col"] == 1 for m in models], seed, noise, keep_masks=True)
    at = 0
    forced = []
    for k, (o, m) in enumerate(zip(objs, models)):
        t = {a: v.to(DEV) if torch.is_tensor(v) else v for a, v in m["in"].items()}
        t["exp_avg"] = {a: (None if (k, a) in skip or v is None else v.to(DEV)) for a, v in m["in"]["exp_avg"].items()}
        t["exp_avg_sq"] = {a: (None if (k, a) in skip or v is None else v.to(DEV)) for a, v in m["in"]["exp_avg_sq"].items()}
        kw = DC.oracle_kwargs(m, min_op, prune_big)
        kw = {a: (v.to(DEV) if torch.is_tensor(v) else v) for a, v in kw.items()}
        n = t["xyz"].shape[0]
        draws = m["draws"].to(DEV)
        ref, rscal, rmask, parent, section = DO.densify_model(t, m["kind"], draws, **kw)
        mine = masks[at:at + n].to(torch.int64)
        at += n
        diff = mine != rmask
        params = {a: getattr(o, DC.ATTR[a]) for a in DC.NAMES}
        mom = {a: ((opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"]) if p in opt.state else None) for a, p in params.items()}
        for a, p in params.items():
            if t["exp_avg"][a] is None:
                assert p not in opt.state
        rr = _with_moments(ref)
        nd = int(diff.sum())
        forced.append(nd)
        if nd:
            # allowed only where a decision lies within a relative 1e-5 of its threshold (fp64); only those parents' rows are
            # left out, the rest of the model is compared row for row
            marg = DO.margins(t, m["kind"], draws, **kw)
            assert (marg[diff] < 1e-5).all(), (k, nd, float(marg[diff].max()))
            mparent, msection = _rows_of(mine)
            keep_k = ~torch.isin(mparent, diff.nonzero().squeeze(-1))
            keep_o = ~torch.isin(parent, diff.nonzero().squeeze(-1))
            assert torch.equal(mparent[keep_k], parent[keep_o]) and torch.equal(msection[keep_k], section[keep_o])
            params = {a: p.detach()[keep_k] for a, p in params.items()}
            mom = {a: (None if v is None else tuple(x[keep_k] for x in v)) for a, v in mom.items()}
            rr = {a: (v[keep_o] if torch.is_tensor(v) and v.dim() and v.shape[0] == keep_o.shape[0] else v) for a, v in rr.items()}
            for mk in ("exp_avg", "exp_avg_sq"):
                rr[mk] = {a: (v[keep_o] if v.numel() else v) for a, v in rr[mk].items()}
            parent, section = parent[keep_o], section[keep_o]
        for key, v in rscal.items():  # a parent decided the other way moves each count by at most 2
            assert abs(scal[k][key] - v) <= 2 * nd, (k, key, scal[k][key], v)
        _compare_model(k, params, mom, rr, parent.cpu(), section.cpu(), t, draws)
    if any(forced):
        print(f"\nnear-threshold parents settled by the kernel's decision, per model: {forced}")
    return objs, opt, scal


def _rows_of(mask):
    """Parent and section of every output row the 4-bit masks describe, in the apply kernel's order (section, then parent)."""
    parent = torch.cat([((mask >> s) & 1).nonzero().squeeze(-1) for s in range(4)])
    section = torch.cat([torch.full((int(((mask >> s) & 1).sum()),), s, dtype=torch.int64, device=mask.device) for s in range(4)])
    return parent, section


def _with_moments(r):
    out = dict(r)
    out["exp_avg"] = {a: (v if v is not None else torch.zeros(0)) for a, v in r["exp_avg"].items()}
    out["exp_avg_sq"] = {a: (v if v is not None else torch.zeros(0)) for a, v in r["exp_avg_sq"].items()}
    return out


@pytest.mark.parametrize("S", [0, 3])
def test_densify_vs_oracle_200k_plus_8x50k(S):
    _run_vs_oracle(_synthetic(200_000, 8, 50_000, M=16, S=S, seed=S))


def test_densify_vs_oracle_config_c_size():
    _run_vs_oracle(_synthetic(1_500_000, 8, 50_000, M=16, S=0, seed=4))


@pytest.mark.parametrize("case", ["empty_segment", "nothing_selected", "everything_pruned", "all_split", "denom_zero", "no_prune_big",
                                  "M1", "no_state"])
def test_densify_edge_cases(case):
    models = _synthetic(3000, 3, 700, M=1 if case == "M1" else 4, S=2, seed=11)
    kw = {}
    if case == "empty_segment":
        models = _synthetic(3000, 3, 700, M=4, S=2, seed=12)
        m = models[2]
        for a in list(m["in"]):
            v = m["in"][a]
            if torch.is_tensor(v):
                m["in"][a] = v[:0]
            elif isinstance(v, dict):
                m["in"][a] = {b: (None if x is None else x[:0]) if torch.is_tensor(x) or x is None else x for b, x in v.items()}
        m["draws"] = m["draws"][:0]
    elif case == "nothing_selected":
        for m in models:
            m["grad_threshold"] = 1e9
    elif case == "everything_pruned":
        kw["min_op"] = 1.0
    elif case == "all_split":
        for m in models:
            m["grad_threshold"] = 1e-30
            m["in"]["scaling"] = m["in"]["scaling"].abs() + 1.0
            m["in"]["xyz_gradient_accum"] = m["in"]["xyz_gradient_accum"] + 1.0
            m["in"]["denom"] = m["in"]["denom"] + 1.0
    elif case == "denom_zero":
        for m in models:
            m["in"]["denom"].zero_()
            m["in"]["xyz_gradient_accum"].zero_()
    elif case == "no_prune_big":
        kw["prune_big"] = False
    elif case == "no_state":
        kw["objs_skip_state"] = [(0, "f_rest"), (2, "xyz"), (1, "semantic")]
    objs, opt, scal = _run_vs_oracle(models, **kw)
    if case == "everything_pruned":
        assert all(o._xyz.shape[0] == 0 for o in objs)
    if case == "all_split":
        assert all(s["points_split"] == s["points_total"] for s in scal)
    if case == "nothing_selected":
        assert all(s["points_clone"] == 0 and s["points_split"] == 0 for s in scal)


def test_philox_draws_deterministic_and_normal():
    def run(seed):
        models = _synthetic(60_000, 2, 10_000, M=4, S=0, seed=3)
        for m in models:   # every parent splits, nothing is pruned
            m["grad_threshold"] = 1e-30
            m["in"]["scaling"] = m["in"]["scaling"].clamp(max=-1.0) + 0.0
            m["percent_dense"] = 1e-6
            m["in"]["xyz_gradient_accum"] = m["in"]["xyz_gradient_accum"] + 1.0
            m["in"]["denom"] = m["in"]["denom"] + 1.0
        objs = [DC.product_model(m, DEV) for m in models]
        scal = training.densify_and_prune(objs, [m["grad_threshold"] for m in models], 0.0, False, None, seed=seed)
        return models, objs, scal

    m1, a, s1 = run(1234)
    _, b, _ = run(1234)
    _, c, _ = run(99)
    for x, y, w in zip(a, b, c):
        for n in DC.ATTR.values():
            assert torch.equal(getattr(x, n), getattr(y, n))
        assert not torch.equal(x._xyz, w._xyz)
    zs = []
    for m, o, s in zip(m1, a, s1):
        assert s["points_split"] == s["points_total"]
        n = s["points_total"]
        t = m["in"]
        R = DO.quaternion_to_matrix(t["rotation"].to(DEV).double())
        sc = torch.exp(t["scaling"].to(DEV).double())
        x = t["xyz"].to(DEV).double()
        for c in range(2):
            xc = o._xyz.detach()[c * n:(c + 1) * n].double()
            zs.append((torch.bmm(R.transpose(1, 2), (xc - x)[..., None])[..., 0] / sc).reshape(-1))
    z = torch.cat(zs)
    assert z.numel() >= 100_000 * 3
    assert abs(float(z.mean())) < 0.01 and abs(float(z.var()) - 1.0) < 0.01


def test_training_loop_with_densification():
    import street_gaussians_b200 as sgb
    from street_gaussians_b200 import losses, synthetic
    import util
    scene = synthetic.make_scene(P=20_000, width=320, height=208, sh_degree=3, seed=5, n_vehicles=2, per_vehicle=2000, with_raw=True,
                                 scale_med=0.05)
    raw = scene["raw"]
    objs = []
    for k, r in enumerate(raw["models"]):
        o = types.SimpleNamespace(**{"_" + a: torch.nn.Parameter(v.clone().to(DEV)) for a, v in r.items()})
        n = r["xyz"].shape[0]
        o._semantic = torch.nn.Parameter(torch.zeros(n, 0, device=DEV))
        o.max_radii2D, o.xyz_gradient_accum, o.denom = torch.zeros(n, device=DEV), torch.zeros(n, 2, device=DEV), torch.zeros(n, 1, device=DEV)
        o.percent_dense, o.percent_big_ws = 0.01, 0.1
        if k == 0:
            o.scene_radius, o.sphere_center, o.sphere_radius = torch.tensor([20.0], device=DEV), torch.zeros(3, device=DEV), torch.tensor([40.0], device=DEV)
        else:
            o.extent, o.min_xyz, o.max_xyz = torch.tensor([3.0], device=DEV), torch.tensor([-3.0, -1.5, -1.5], device=DEV), torch.tensor([3.0, 1.5, 1.5], device=DEV)
        objs.append(o)
    opt = training.FusedAdam([{"params": [getattr(o, "_" + a)], "lr": 1e-3, "name": a} for o in objs
                              for a in ("xyz", "features_dc", "features_rest", "opacity", "scaling", "rotation")], lr=1e-3, eps=1e-15)
    st = util.settings_from(sgb, scene["cam"], DEV)
    rast = sgb.GaussianRasterizer(st)
    poses, idft = raw["poses"].to(DEV), raw["idft"].to(DEV)
    gt = torch.rand(3, 208, 320, device=DEV)

    def step():
        xyz, rot, scale, opac, sh = sgb.compose(objs, poses, idft)
        m2d = torch.zeros_like(xyz, requires_grad=True)
        col, radii, _, _, _ = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot)
        loss = losses.photometric_loss(col, gt, None, 1.0, 0.2)
        opt.zero_grad()
        loss.backward()
        training.add_densification_stats(objs, radii, m2d.grad)
        return xyz.shape[0], radii

    P0, _ = step()
    sc = training.densify_and_prune(objs, [1e-7] * len(objs), 0.005, False, opt, seed=7)
    assert sum(s["points_clone"] + s["points_split"] for s in sc) > 0
    P1 = sum(o._xyz.shape[0] for o in objs)
    assert P1 != P0 and all(o.xyz_gradient_accum.shape[0] == o._xyz.shape[0] for o in objs)
    P2, radii = step()
    assert P2 == P1 and int((radii > 0).sum()) > 0
    for o in objs:
        assert o._xyz.grad is not None and o._xyz.grad.shape == o._xyz.shape
    assert objs[0]._xyz.grad.abs().sum() > 0
    before = [o._xyz.detach().clone() for o in objs]
    opt.step()
    assert any(not torch.equal(b, o._xyz) for b, o in zip(before, objs))


def test_reset_opacity_vs_oracle():
    models, _ = DC.load()
    objs = [DC.product_model(m, DEV) for m in models]
    opt = _optimizers(objs, models, "fused_shared")
    before = {id(p): (s["exp_avg"].clone(), s["exp_avg_sq"].clone()) for p, s in opt.state.items()}
    training.reset_opacity(objs, opt)
    for o, m in zip(objs, models):
        exp = DO.reset_opacity(m["in"]["opacity"].to(DEV))
        err = (o._opacity.detach() - exp).abs()
        assert (err <= 4 * _ulp(exp)).all(), float(err.max())
        for a in DC.NAMES:
            p = getattr(o, DC.ATTR[a])
            s = opt.state[p]
            if a == "opacity":
                assert not s["exp_avg"].any() and not s["exp_avg_sq"].any()
            else:
                assert torch.equal(s["exp_avg"], before[id(p)][0]) and torch.equal(s["exp_avg_sq"], before[id(p)][1])
