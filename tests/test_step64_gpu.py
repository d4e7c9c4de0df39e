"""The fp64 per-element tier for the kernels of a training step other than the rasterizer: the composer (compose_fwd / compose_bwd /
compose_pose_finalize), the image loss (ssim_stats / ssim_grad), Adam (adam_kernel) and the densification statistics
(densify_stats_kernel), each output element against oracle/step64.py's fp64 value within its derived bound.  Each scene is built
around an edge the kernels branch on (segment tables longer than one launch, warp and block boundaries, both SH copy paths, more
than one Adam launch, flat SSIM regions, empty masks) and asserts that edge.  REPORT collects the largest error / bound per check."""
import ctypes as C
import math

import pytest
import torch

import compose_case as CC
import street_gaussians_b200 as sgb
from oracle import step64 as S64
from street_gaussians_b200 import _capi, losses, training
from street_gaussians_b200._capi import ptr, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPORT = {}
U = S64.U
NAMES = ("xyz", "rotation", "scaling", "opacity", "features")


def within(worst, key, got, val, bnd):
    err = (got.detach().to(torch.float64) - val).abs()
    bad = ~(err <= bnd)
    assert not bool(bad.any()), (key, int(bad.sum()), torch.nonzero(bad)[:6].tolist(), err[bad][:6].tolist(), bnd[bad][:6].tolist())
    r = float((err / (bnd + 1e-300)).max()) if err.numel() else 0.0
    worst[key] = max(worst.get(key, 0.0), r)


def report(name, worst):
    REPORT[name] = {k: round(v, 4) for k, v in worst.items()}
    print(name, REPORT[name])


# ----------------------------------------------------------------------------------------------- composer
def compose_scene(seed, n_bkgd, actors, M, Cf, flip="mixed", qnorm=None, raw_scale=None, trans=1.0):
    models = CC.make_case(seed, n_bkgd, actors, M, Cf)
    g = torch.Generator().manual_seed(seed + 100)
    A = len(actors)
    poses = torch.randn(A, 7, generator=g)
    poses[:, 4:] *= trans
    if qnorm is not None:
        poses[:, :4] *= torch.tensor(qnorm)[torch.arange(A) % len(qnorm)][:, None] / poses[:, :4].norm(dim=1, keepdim=True)
    if raw_scale is not None:
        for m in models:
            n = m["rotation"].shape[0]
            m["rotation"] = m["rotation"] * torch.logspace(math.log10(raw_scale), 0, max(n, 1))[:n, None]
    idft = torch.randn(A, Cf, generator=g)
    na = sum(actors)
    fl = None
    if flip == "mixed":
        fl = torch.rand(na, generator=g) < 0.5
    elif flip == "all":
        fl = torch.ones(na, dtype=torch.bool)
    return models, poses, idft, fl, torch.tensor([0.0, 0.0, 1.0, 0.0])


def check_compose(name, models, poses, idft, flip, fq, seed=0):
    M = models[0]["features_rest"].shape[1] + 1
    P = sum(m["xyz"].shape[0] for m in models)
    A = len(models) - 1
    up = CC.upstream(seed + 7, P, M)
    dm = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in models]
    dp = poses.to(DEV).requires_grad_(True) if A else None
    out = sgb.compose(dm, dp, idft.to(DEV) if A else None, flip.to(DEV) if flip is not None else None,
                      fq.to(DEV) if flip is not None else None)
    torch.autograd.backward(list(out), [up[k].to(DEV) for k in NAMES])
    torch.cuda.synchronize()
    r = S64.compose64([{k: v.to(DEV) for k, v in m.items()} for m in models], poses.to(DEV), idft.to(DEV), flip, fq.to(DEV),
                      {k: v.to(DEV) for k, v in up.items()})
    worst = {}
    for k, t in zip(NAMES, out):
        within(worst, k, t, r[k], r["b_" + k])
    assert torch.equal(out[4][:, 1:].double(), r["features"][:, 1:]), "features_rest is a copy"
    for i, m in enumerate(dm):
        for k in CC.KEYS:
            within(worst, f"g_{k}", m[k].grad.reshape(r[f"g{i}_{k}"].shape), r[f"g{i}_{k}"], r[f"b_g{i}_{k}"])
        assert torch.equal(m["features_rest"].grad.double(), r[f"g{i}_features_rest"]), "features_rest gradient is a copy"
    if A:
        within(worst, "dposes", dp.grad, r["dposes"], r["b_dposes"])
    report(name, worst)
    return r, out, dp


SIZES = [0, 1, 31, 32, 33, 255, 256, 257]
SEG_CASES = [  # (segments, M, fourier_dim, flip)
    (1, 16, 1, "none"), (32, 4, 5, "mixed"), (33, 9, 8, "all"), (41, 1, 5, "mixed"), (64, 16, 1, "none"), (65, 4, 8, "mixed")]


@pytest.mark.parametrize("nseg,M,Cf,flip", SEG_CASES, ids=[f"seg{c[0]}_M{c[1]}_C{c[2]}_{c[3]}" for c in SEG_CASES])
def test_compose_segment_tables(nseg, M, Cf, flip):
    """Tables of 1 to 65 segments (launch groups of SGR_MAX_SEGMENTS_PER_LAUNCH = 32: the groups after the first start with an actor,
    and their pose / IDFT / pose-sum rows are offset by the group's first segment), actor sizes 0 (first, middle, last), 1, 31, 32, 33,
    255, 256, 257 after a 1001-Gaussian background, so segment boundaries fall inside warps and at block edges; M = 1, 4, 9, 16 runs
    the warp-cooperative and the per-thread SH copies (R3 = 0, 9, 24, 45)."""
    A = nseg - 1
    actors = [SIZES[(k * 3 + nseg) % len(SIZES)] for k in range(A)]
    if A >= 3:
        actors[0] = actors[A // 2] = 0
        if nseg != 33:  # (at 33 the last actor is the only segment of the second launch group)
            actors[-1] = 0
    models, poses, idft, fl, fq = compose_scene(nseg, 1001, actors, M, Cf, "none" if flip == "none" else flip)
    r, out, dp = check_compose(f"compose_seg{nseg}_M{M}_C{Cf}_{flip}", models, poses, idft, fl, fq, seed=nseg)
    assert len(models) == nseg and out[4].shape[1] == M
    if A >= 3:
        assert {0, 1, 31, 32, 33, 255, 256, 257} <= set(actors)
        for a in (0, A // 2, A - 1):  # empty actors: no pose gradient
            assert actors[a] or float(dp.grad[a].abs().sum()) == 0.0
    if nseg > 32:
        assert sum(actors[31:]) > 0, "a later launch group holds Gaussians"


def test_compose_small_actor_next_to_large():
    """A 3-Gaussian actor next to a 50 000-Gaussian one: its pose gradient is checked against its own bound, which is far below
    what a per-tensor tolerance scaled by the large actor would allow."""
    models, poses, idft, fl, fq = compose_scene(7, 2000, [3, 50000], 16, 5)
    r, _, _ = check_compose("compose_small_large", models, poses, idft, fl, fq, seed=7)
    assert float(r["b_dposes"][0].max()) < 1e-3 * float(r["dposes"][1].abs().max())


def test_compose_pose_and_raw_quaternion_extremes():
    """Non-unit actor quaternions (|q| = 0.3 and 7), raw Gaussian quaternions with norms down to 1e-6 (the rotation gradient grows
    as 1 / |raw|), translations around 1e3."""
    models, poses, idft, fl, fq = compose_scene(9, 700, [300, 257, 64], 9, 5, qnorm=[0.3, 7.0, 1.0], raw_scale=1e-6, trans=1e3)
    check_compose("compose_extremes", models, poses, idft, fl, fq, seed=9)
    rn = torch.cat([m["rotation"] for m in models]).norm(dim=1)
    assert float(rn.min()) < 2e-6 and float(poses[:, 4:].abs().max()) > 500


def test_compose_config_c_shape():
    """Config C's shape once: a 1.5 M background and 8 actors of 50 000, M = 16, fourier_dim 5."""
    models, poses, idft, fl, fq = compose_scene(13, 1_500_000, [50_000] * 8, 16, 5)
    check_compose("compose_config_c", models, poses, idft, fl, fq, seed=13)


def _segments(models, M):
    segs = (_capi.SgrSegment * len(models))()
    start = 0
    for k, m in enumerate(models):
        s = segs[k]
        n = int(m["xyz"].shape[0])
        s.start, s.count, s.fourier_dim, s.posed = start, n, int(m["features_dc"].shape[1]), int(k > 0)
        s.xyz, s.rotation, s.scaling, s.opacity, s.features_dc, s.features_rest = (
            m[k2].data_ptr() if m[k2].numel() else None for k2 in CC.KEYS)
        start += n
    return segs, start


@pytest.mark.parametrize("actors", [[40, 0, 7] + [5] * 30 + [0, 3], [0, 0, 0]], ids=["36_segments", "all_empty"])
def test_compose_backward_c_abi_unposed_rows_are_zero(actors):
    """sgr_compose_backward called the way composer.py calls it, with the background's pose row left zero: the rows of unposed
    segments are exactly 0 (include/sgr.h), every other row finite, in every launch group; also with every segment empty (P = 0)."""
    M = 4
    models = [{k: v.to(DEV) for k, v in m.items()} for m in CC.make_case(3, 0 if not sum(actors) else 100, actors, M, 5)]
    nseg = len(models)
    segs, P = _segments(models, M)
    g = torch.Generator().manual_seed(4)
    pose_tab = torch.zeros(nseg, 8)
    pose_tab[1:, :7] = torch.randn(nseg - 1, 7, generator=g)
    idft_tab = torch.zeros(nseg, _capi.MAX_FOURIER)
    idft_tab[1:, :5] = torch.randn(nseg - 1, 5, generator=g)
    pose_tab, idft_tab = pose_tab.to(DEV), idft_tab.to(DEV)
    up = {k: v.to(DEV) for k, v in CC.upstream(5, P, M).items()}
    grads = [torch.empty_like(m[k]) for m in models for k in CC.KEYS]
    gtab = (_capi.SgrSegmentGrads * nseg)()
    for k in range(nseg):
        gk = gtab[k]
        gk.xyz, gk.rotation, gk.scaling, gk.opacity, gk.features_dc, gk.features_rest = (
            t.data_ptr() if t.numel() else None for t in grads[6 * k: 6 * k + 6])
    dposes = torch.full((nseg, 8), float("nan"), device=DEV)
    scratch = torch.empty(nseg, 16, device=DEV)
    L = _capi.lib()
    p = lambda t: ptr(t) if t.numel() else None
    rc = L.sgr_compose_backward(segs, gtab, nseg, M, ptr(pose_tab), ptr(idft_tab), None, None, p(up["xyz"]), p(up["rotation"]),
                                p(up["scaling"]), p(up["opacity"]), p(up["features"]), ptr(dposes), ptr(scratch), stream(torch.device(DEV)))
    _capi.check(rc, "sgr_compose_backward")
    d = dposes.cpu()
    assert torch.equal(d[0], torch.zeros(8)), d[0]
    assert bool(torch.isfinite(d).all())
    assert torch.equal(d[:, 7], torch.zeros(nseg))
    for a, n in enumerate(actors):
        if n == 0:
            assert torch.equal(d[a + 1], torch.zeros(8)), (a, d[a + 1])
    if P == 0:
        assert torch.equal(d, torch.zeros(nseg, 8))
    else:
        assert nseg > 32 and bool((d[33:, :7] != 0).any()), "the second launch group carries pose gradients"


# ----------------------------------------------------------------------------------------------- image loss
def loss_scene(C, H, W, seed, mask="random", kind="random"):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(C, H, W, generator=g) * 1.4 - 0.2  # values outside [0, 1]
    img = gt + 0.1 * torch.randn(C, H, W, generator=g)
    if kind == "regions" and H >= 32 and W >= 32:
        img[:, :H // 4, :W // 4] = gt[:, :H // 4, :W // 4]                     # x = y exactly
        img[:, H // 4:H // 2, :W // 4] = 0.37                                  # constant x, nearly flat y
        gt[:, H // 4:H // 2, :W // 4] = 0.37 + 1e-4 * torch.rand(C, H // 2 - H // 4, W // 4, generator=g)
        img[:, H // 2:, W // 2:] = 0.6                                         # x = y = constant
        gt[:, H // 2:, W // 2:] = 0.6
    elif kind == "same":
        img = gt.clone()
    elif kind == "zeros":
        img, gt = torch.zeros(C, H, W), torch.zeros(C, H, W)
    m = None
    if mask == "random":
        m = torch.rand(1, H, W, generator=g) > 0.3
    elif mask == "islands":  # single on-pixels on tile edges (rows / columns 15, 16, 31, 32 and the image border) in an empty mask
        m = torch.zeros(1, H, W, dtype=torch.bool)
        for yy in [0, 15, 16, 31, 32, H - 1]:
            for xx in [0, 15, 16, 31, 32, W - 1]:
                if yy < H and xx < W and (yy + xx) % 2 == 1:
                    m[0, yy, xx] = True
        m[0, 5, 5] = True
    elif mask == "ones":
        m = torch.ones(1, H, W, dtype=torch.bool)
    elif mask == "empty":
        m = torch.zeros(1, H, W, dtype=torch.bool)
    return img, gt, m


def capi_image_loss(img, gt, mask, w_l1, w_ssim):
    L = _capi.lib()
    Cn, H, W = img.shape
    x, y = img.to(DEV).contiguous(), gt.to(DEV).contiguous()
    m = mask.reshape(-1).to(DEV, torch.uint8).contiguous() if mask is not None else None
    grad = torch.empty_like(x)
    scalars = torch.empty(4, device=DEV)
    nb = int(L.sgr_image_loss_scratch_bytes(Cn, H, W))
    scratch = torch.empty(nb, device=DEV, dtype=torch.uint8)
    rc = L.sgr_image_loss(Cn, H, W, ptr(x), ptr(y), ptr(m), float(w_l1), float(w_ssim), ptr(grad), ptr(scalars), ptr(scratch), nb,
                          stream(torch.device(DEV)))
    _capi.check(rc, "sgr_image_loss")
    return grad, scalars.cpu()


def scalar_within(worst, key, got, val, bnd):
    if math.isnan(val):
        assert math.isnan(got), (key, got)
        return
    err = abs(got - val)
    assert err <= bnd, (key, got, val, err, bnd)
    worst[key] = max(worst.get(key, 0.0), err / (bnd + 1e-300))


LOSS_CASES = [  # (C, H, W, mask, kind)
    (3, 1280, 1920, "random", "regions"), (3, 1279, 1921, "none", "regions"), (1, 37, 16, "islands", "random"),
    (4, 16, 5, "ones", "random"), (3, 10, 10, "empty", "random"), (1, 1, 1, "none", "random"), (3, 48, 64, "none", "same"),
    (3, 48, 64, "random", "zeros"), (4, 40, 33, "islands", "regions")]


@pytest.mark.parametrize("C,H,W,mask,kind", LOSS_CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}_{c[3]}_{c[4]}" for c in LOSS_CASES])
def test_image_loss(C, H, W, mask, kind):
    """sgr_image_loss (scalars and dL/dimage of the photometric weights) and losses.l1_loss / ssim / photometric_loss with an upstream
    gradient of 2.5, per element, against image_loss64; the bound's linearisation premise holds on every pixel."""
    img, gt, m = loss_scene(C, H, W, C * 1000 + H + W, mask, kind)
    worst = {}
    lam = 0.2
    wl, ws = (1.0 - lam) * 1.0, -lam
    r = S64.image_loss64(img.to(DEV), gt.to(DEV), m.to(DEV) if m is not None else None, wl, ws)
    assert float(r["premise"].max()) < 1e-2, float(r["premise"].max())
    grad, sc = capi_image_loss(img, gt, m, wl, ws)
    within(worst, "grad", grad, r["grad"], r["b_grad"])
    scalar_within(worst, "value", float(sc[0]), r["value"], r["b_value"])
    scalar_within(worst, "l1", float(sc[1]), r["l1"], r["b_l1"])
    scalar_within(worst, "ssim", float(sc[2]), r["ssim"], r["b_ssim"])
    assert float(sc[3]) == r["count"]
    md = m.to(DEV) if m is not None else None
    for fn, w1, w2, extra in ((losses.l1_loss, 1.0, 0.0, 0.0), (lambda a, b, mm: losses.ssim(a, b, mask=mm), 0.0, 1.0, 0.0),
                              (lambda a, b, mm: losses.photometric_loss(a, b, mm, 1.0, lam), wl, ws, lam)):
        rr = S64.image_loss64(img.to(DEV), gt.to(DEV), md, w1, w2)
        x = img.to(DEV).requires_grad_(True)
        v = fn(x, gt.to(DEV), md)
        (2.5 * v).backward()
        tag = f"w{w1:g}_{w2:g}"
        scalar_within(worst, "value_" + tag, float(v), rr["value"] + extra, rr["b_value"] + U * abs(rr["value"] + extra))
        within(worst, "grad_" + tag, x.grad, 2.5 * rr["grad"], 2.5 * rr["b_grad"] + U * (2.5 * rr["grad"]).abs())
    if mask == "empty":
        assert math.isnan(float(sc[1])) and float(sc[3]) == 0.0 and bool((grad == 0).all())
        assert abs(float(sc[2]) - 1.0) <= r["b_ssim"] and abs(float(losses.ssim(img.to(DEV), gt.to(DEV), mask=md)) - 1.0) <= r["b_ssim"]
    if mask == "ones":
        g0, s0 = capi_image_loss(img, gt, None, wl, ws)
        assert torch.equal(g0, grad) and torch.equal(s0, sc), "an all-ones mask is bit-equal to no mask"
    if kind == "regions" and H >= 32:
        assert bool((img[:, H // 4:H // 2, :W // 4] == 0.37).all()) and bool((gt[:, H // 2:, W // 2:] == 0.6).all()), "flat regions"
        assert bool((img[:, :H // 4, :W // 4] == gt[:, :H // 4, :W // 4]).all()), "x = y exactly"
    if mask == "islands":
        assert int(m.sum()) >= 5 and bool(m[0, 15:17].any() | m[0, :, 15:17].any())
    report(f"loss_{C}x{H}x{W}_{mask}_{kind}", worst)


# ----------------------------------------------------------------------------------------------- Adam
NUMELS = [0, 1, 8191, 8192, 8193]


def adam_grad(shape, g, scale_exp):
    n = int(torch.Size(shape).numel())
    mag = torch.logspace(-19, 3, max(n, 1))[torch.randperm(max(n, 1), generator=g)][:n]
    sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    v = (mag * sign).reshape(shape)
    if n:
        v.reshape(-1)[: max(1, n // 10)] = 0.0  # exact zeros: m and v decay
    return v * (10.0 ** scale_exp)


@pytest.mark.parametrize("ntens", [1, 47, 48, 49, 54, 96, 97])
def test_fused_adam(ntens):
    """FusedAdam over ntens tensors (launches of kAdamTensors = 48): numel 0, 1, 8191, 8192, 8193 and one of 2^20 + 3, per-tensor
    step counts 1, 2, 1000, 30000 in the same launch, a parameter without a gradient just before the 48-tensor boundary, zero,
    tiny (1e-19) and large (1e3) gradients with sign flips, and an lr change between steps.  Every step starts from the kernel's
    own fp32 state; after the steps, step and the moments also match torch.optim.Adam's."""
    g = torch.Generator().manual_seed(ntens)
    shapes = [(NUMELS[k % len(NUMELS)],) for k in range(ntens)]
    if ntens >= 49:
        shapes[ntens // 2] = (2 ** 20 + 3,)
    base = [torch.randn(s, generator=g) for s in shapes]
    lrs = [1e-3 * (1 + k % 5) for k in range(ntens)]
    pa = [torch.nn.Parameter(b.clone().to(DEV)) for b in base]
    pb = [torch.nn.Parameter(b.clone().to(DEV)) for b in base]
    oa = training.FusedAdam([dict(params=[p], lr=lr) for p, lr in zip(pa, lrs)], lr=0.0, eps=1e-15)
    ob = torch.optim.Adam([dict(params=[p], lr=lr) for p, lr in zip(pb, lrs)], lr=0.0, eps=1e-15)
    pre = [0, 1, 999, 29999]
    for k in range(ntens):  # per-tensor step counts: 1, 2, 1000, 30000 on the first step
        s0 = pre[k % 4]
        if s0:
            m0 = torch.randn(shapes[k], generator=g) * 1e-2
            v0 = torch.rand(shapes[k], generator=g) * 1e-3
            oa.state[pa[k]] = dict(step=s0, exp_avg=m0.to(DEV), exp_avg_sq=v0.to(DEV))
            ob.state[pb[k]] = dict(step=torch.tensor(float(s0)), exp_avg=m0.clone().to(DEV), exp_avg_sq=v0.clone().to(DEV))
    skip = 46 if ntens >= 48 else None
    worst = {}
    steps_seen = set()
    for it in range(3):
        for k, (a, b) in enumerate(zip(pa, pb)):
            gr = adam_grad(shapes[k], g, it - 1).to(DEV)
            a.grad, b.grad = gr.clone(), gr.clone()
        if skip is not None:
            pa[skip].grad = pb[skip].grad = None
        if it == 1:
            for grp_a, grp_b in zip(oa.param_groups[::3], ob.param_groups[::3]):
                grp_a["lr"] = grp_b["lr"] = 7e-5
        snap = []
        for k, p in enumerate(pa):
            st = oa.state.get(p, {})
            z = torch.zeros_like(p)
            snap.append((p.detach().clone(), st.get("exp_avg", z).clone(), st.get("exp_avg_sq", z).clone(), int(st.get("step", 0)) + 1,
                         oa.param_groups[k]["lr"]))
        oa.step()
        ob.step()
        torch.cuda.synchronize()
        for k, p in enumerate(pa):
            p0, m0, v0, step, lr = snap[k]
            if k == skip:
                assert torch.equal(p.detach(), p0)
                continue
            steps_seen.add(step)
            r = S64.adam64(p0, p.grad, m0, v0, lr, step)
            st = oa.state[p]
            assert int(st["step"]) == step
            within(worst, "p", p.detach(), r["p"], r["b_p"])
            within(worst, "m", st["exp_avg"], r["m"], r["b_m"])
            within(worst, "v", st["exp_avg_sq"], r["v"], r["b_v"])
        oa.zero_grad(set_to_none=True)
        ob.zero_grad(set_to_none=True)
    assert {1, 2, 1000, 30000} <= steps_seen or ntens < 4
    for k, (a, b) in enumerate(zip(pa, pb)):
        if k == skip:
            assert a not in oa.state or int(oa.state[a]["step"]) == int(ob.state[b]["step"])
            continue
        assert int(oa.state[a]["step"]) == int(ob.state[b]["step"])
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.allclose(oa.state[a][key], ob.state[b][key], rtol=1e-5, atol=1e-37), (k, key)
        assert torch.allclose(a.detach(), b.detach(), rtol=1e-5, atol=1e-6), k
    report(f"adam_{ntens}", worst)


def test_sgr_adam_step_direct():
    """sgr_adam_step with a hand-built table of 97 tensors whose steps differ within each launch (1, 2, 1000, 30000, ...)."""
    g = torch.Generator().manual_seed(1)
    n = 97
    shapes = [NUMELS[k % len(NUMELS)] if k != 50 else 2 ** 20 + 3 for k in range(n)]
    ps = [torch.randn(s, generator=g).to(DEV) for s in shapes]
    gs = [adam_grad((s,), g, 0).to(DEV) for s in shapes]
    ms = [(torch.randn(s, generator=g) * 1e-2).to(DEV) for s in shapes]
    vs = [(torch.rand(s, generator=g) * 1e-3).to(DEV) for s in shapes]
    steps = [[1, 2, 1000, 30000, 7][k % 5] for k in range(n)]
    lrs = [float(torch.tensor(1e-3 * (1 + k % 3)).float()) for k in range(n)]
    snap = [(p.clone(), m.clone(), v.clone()) for p, m, v in zip(ps, ms, vs)]
    tab = (_capi.SgrAdamTensor * n)()
    for k in range(n):
        t = tab[k]
        t.param, t.grad, t.exp_avg, t.exp_avg_sq = ps[k].data_ptr(), gs[k].data_ptr(), ms[k].data_ptr(), vs[k].data_ptr()
        t.numel, t.lr, t.step = shapes[k], lrs[k], steps[k]
    rc = _capi.lib().sgr_adam_step(tab, n, 0.9, 0.999, 1e-15, stream(torch.device(DEV)))
    _capi.check(rc, "sgr_adam_step")
    torch.cuda.synchronize()
    worst = {}
    for k in range(n):
        r = S64.adam64(snap[k][0], gs[k], snap[k][1], snap[k][2], lrs[k], steps[k])
        within(worst, "p", ps[k], r["p"], r["b_p"])
        within(worst, "m", ms[k], r["m"], r["b_m"])
        within(worst, "v", vs[k], r["v"], r["b_v"])
    report("adam_direct", worst)


# ----------------------------------------------------------------------------------------------- densification statistics
STAT_CASES = [[777], [100, 0, 37] + [33] * 29, [0] + [300] * 31 + [5], [17, 0, 256, 1] * 16 + [0]]


@pytest.mark.parametrize("counts", STAT_CASES, ids=[f"seg{len(c)}" for c in STAT_CASES])
def test_densify_stats(counts):
    """1, 32, 33 and 65 segments (launch groups of 32) with empty segments and boundaries inside 256-thread blocks, radii <= 0, three
    calls accumulating; max_radii2D and denom exact, xyz_gradient_accum within stats64's bound, each call from the kernel's state."""
    g = torch.Generator().manual_seed(len(counts))
    P = sum(counts)
    models = [dict(max_radii2D=(torch.rand(n, generator=g) * 30).to(DEV), xyz_gradient_accum=torch.rand(n, 2, generator=g).to(DEV),
                   denom=torch.randint(0, 20, (n, 1), generator=g).float().to(DEV)) for n in counts]
    worst = {}
    for call in range(3):
        radii = torch.randint(-3, 41, (P,), generator=g, dtype=torch.int32)
        grad = torch.randn(P, 3, generator=g) * (10.0 ** (call - 1))
        snap = [{k: v.clone() for k, v in m.items()} for m in models]
        training.add_densification_stats(models, radii.to(DEV), grad.to(DEV))
        torch.cuda.synchronize()
        start = 0
        for m, s, n in zip(models, snap, counts):
            r = S64.stats64(s["max_radii2D"], s["xyz_gradient_accum"], s["denom"], radii[start:start + n].to(DEV), grad[start:start + n].to(DEV))
            assert torch.equal(m["max_radii2D"].double(), r["max_radii2D"]) and torch.equal(m["denom"].double(), r["denom"])
            within(worst, "xyz_gradient_accum", m["xyz_gradient_accum"], r["xyz_gradient_accum"], r["b_xyz_gradient_accum"])
            start += n
        assert bool((radii <= 0).any()) and bool((radii > 0).any())
    if len(counts) > 32:
        assert sum(counts[32:]) > 0
    report(f"stats_seg{len(counts)}", worst)
