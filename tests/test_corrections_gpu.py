"""GPU: the background pose correction in the composer (sgr_compose_forward_corrected / sgr_compose_backward_corrected through
compose(pose_correction=...)) and the colour correction (sgr_color_correct_* / sgr_color_correction_reg through
street_gaussians_b200.corrections) against the reference's own outputs (tests/golden/callsite/correction_sh*.npz), per element
against the fp64 restatements of tests/correction_oracle.py, bit for bit where the correction is the identity, and end to end at
config C against the reference's torch lines."""
import math

import numpy as np
import pytest
import torch

import compose_case as CC
import correction_oracle as CR
import street_gaussians_b200 as sgb
import util
from street_gaussians_b200 import losses, synthetic
from test_compose_cpu import rel
from test_corrections_cpu import FIX, IDS, load

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = CR.NAMES


def to_dev(models):
    return [{k: v.detach().to(DEV).requires_grad_(True) for k, v in m.items()} for m in models]


def within(got, val, bnd, what):
    got, val, bnd = (torch.as_tensor(t).to(DEV, torch.float64) for t in (got, val, bnd))
    err = (got - val).abs()
    bad = ~(err <= bnd)
    assert not bool(bad.any()), (what, int(bad.sum()), float(err[bad].max()), float(bnd[bad].min()))
    return float((err / (bnd + 1e-300)).max())


@pytest.mark.parametrize("path", FIX, ids=IDS)
def test_corrections_vs_reference_fixture(path):
    z, M, models, poses, idft, flip, fq, rots, trans = load(path)
    cid = int(z["cam_id"])
    dm = to_dev(models)
    dp = poses.detach().to(DEV).requires_grad_(True)
    dr, dt = rots.detach().to(DEV).requires_grad_(True), trans.detach().to(DEV).requires_grad_(True)
    out = sgb.compose(dm, dp, idft.to(DEV), flip.to(DEV), fq.to(DEV), pose_correction=(dr[cid], dt[cid]))
    for k, t in zip(NAMES, out):
        assert rel(t.detach().cpu().numpy(), z["ref_" + k]) < 2e-6, k
    up = CC.upstream(int(z["seed"]) + 1, out[0].shape[0], M)
    torch.autograd.backward(list(out), [up[k].to(DEV) for k in NAMES])
    for i, m in enumerate(dm):
        for k in CC.KEYS:
            assert rel(m[k].grad.cpu().numpy(), z[f"ref_g{i}_{k}"]) < 3e-5, (i, k)
    assert rel(dp.grad.cpu().numpy(), z["ref_dposes"]) < 3e-5
    assert rel(dr.grad.cpu().numpy(), z["ref_g_pose_correction_rots"]) < 3e-5
    assert rel(dt.grad.cpu().numpy(), z["ref_g_pose_correction_trans"]) < 3e-5
    A = torch.from_numpy(z["affine_trans"]).to(DEV).requires_grad_(True)
    S = torch.from_numpy(z["affine_trans_sky"]).to(DEV).requires_grad_(True)
    img = torch.from_numpy(z["image"]).to(DEV).requires_grad_(True)
    o = sgb.color_correct(img, A[cid])
    assert rel(o.detach().cpu().numpy(), z["ref_corrected"]) < 1e-6
    o.backward(torch.from_numpy(z["g_image"]).to(DEV))
    assert rel(img.grad.cpu().numpy(), z["ref_dimage"]) < 1e-6
    assert rel(A.grad.cpu().numpy(), z["ref_daffine"]) < 2e-5
    A.grad = None
    r = sgb.color_correction_reg_loss(A[cid], S[cid])
    assert abs(float(r.detach()) - float(z["ref_reg"])) <= 1e-6 * abs(float(z["ref_reg"]))
    r.backward()
    assert np.array_equal(A.grad.cpu().numpy(), z["ref_reg_g_affine"]) and np.array_equal(S.grad.cpu().numpy(), z["ref_reg_g_affine_sky"])


def _quat(kind, g):
    base = {"unit": torch.tensor([0.96, 0.1, -0.2, 0.15]), "tiny": 1e-3 * torch.tensor([0.9, 0.2, -0.3, 0.25]),
            "large": 1e3 * torch.tensor([0.8, -0.3, 0.4, 0.3]), "near180": torch.tensor([1e-4, 0.6, -0.48, 0.64])}[kind]
    return base if kind == "near180" else base / (base.norm() if kind == "unit" else 1.0)


def _run_case(nb, actors, use_flip, M, C, qkind, seed):
    g = torch.Generator().manual_seed(seed)
    models = CC.make_case(seed, nb, list(actors), M, C)
    A = len(actors)
    poses = torch.randn(A, 7, generator=g) if A else torch.zeros(0, 7)
    idft = torch.randn(A, C, generator=g) if A else torch.zeros(0, C)
    flip = (torch.rand(sum(actors), generator=g) < 0.5) if use_flip and A else None
    fq = torch.tensor([0.0, 0.0, 1.0, 0.0])
    corr = (_quat(qkind, g), 0.5 * torch.randn(3, generator=g))
    P = nb + sum(actors)
    up = CC.upstream(seed + 1, P, M)
    dev_models = [{k: v.to(DEV) for k, v in m.items()} for m in models]
    r = CR.compose64(dev_models, poses.to(DEV), idft.to(DEV), flip.to(DEV) if flip is not None else None, fq.to(DEV),
                     {k: v.to(DEV) for k, v in up.items()}, (corr[0].to(DEV), corr[1].to(DEV)))
    dm = to_dev(models)
    dp = poses.to(DEV).requires_grad_(True) if A else None
    cr, ct = corr[0].to(DEV).requires_grad_(True), corr[1].to(DEV).requires_grad_(True)
    out = sgb.compose(dm, dp, idft.to(DEV) if A else None, flip.to(DEV) if flip is not None else None, fq.to(DEV) if flip is not None else None,
                      pose_correction=(cr, ct))
    torch.autograd.backward(list(out), [up[k].to(DEV) for k in NAMES])
    worst = 0.0
    for k, t in zip(NAMES, out):
        worst = max(worst, within(t.detach(), r[k], r["b_" + k], k))
    for i, m in enumerate(dm):
        for k in CC.KEYS:
            if m[k].numel():
                worst = max(worst, within(m[k].grad, r[f"g{i}_{k}"], r[f"b_g{i}_{k}"], (i, k)))
    within(torch.cat([cr.grad, ct.grad]), r["dcorrection"], r["b_dcorrection"], "dcorrection")
    if A:
        live = [a for a, n in enumerate(actors) if n > 0]
        within(dp.grad[live], r["dposes"][live], r["b_dposes"][live], "dposes")
    return worst


CASES = [  # (background, actors, flip, M, fourier_dim, correction quaternion)
    (0, (300,), False, 16, 5, "unit"), (1, (), False, 1, 1, "unit"), (255, (1,), True, 4, 1, "tiny"), (256, (8,) * 8, True, 9, 3, "large"),
    (257, tuple(range(1, 41)), True, 16, 8, "near180"), (1001, (37, 0, 501), True, 16, 2, "unit"), (4097, (64, 33), False, 4, 7, "large"),
    (513, (), False, 9, 4, "near180"), (300, (29,) * 8, True, 1, 6, "tiny"),
]


@pytest.mark.parametrize("case", CASES, ids=[f"bg{c[0]}-a{len(c[1])}-M{c[3]}-C{c[4]}-{c[5]}" for c in CASES])
def test_pose_correction_per_element_vs_float64(case):
    _run_case(*case, seed=11 + CASES.index(case))


def test_pose_correction_config_c_background_per_element():
    worst = _run_case(1_500_000, (50_000,) * 8, True, 16, 5, "unit", seed=3)
    assert worst > 1e-4, worst


def test_zero_correction_quaternion_gives_nan_like_the_reference():
    models = CC.make_case(2, 300, [40], 4, 2)
    dm = to_dev(models)
    poses, idft = torch.randn(1, 7, device=DEV), torch.randn(1, 2, device=DEV)
    cr, ct = torch.zeros(4, device=DEV, requires_grad=True), torch.zeros(3, device=DEV, requires_grad=True)
    out = sgb.compose(dm, poses, idft, pose_correction=(cr, ct))
    om = [{k: v.detach().cpu().requires_grad_(True) for k, v in m.items()} for m in models]
    ocr, oct_ = torch.zeros(4, requires_grad=True), torch.zeros(3, requires_grad=True)
    ref = CR.compose(om, poses.cpu(), idft.cpu(), None, torch.tensor([1.0, 0, 0, 0]), (ocr, oct_))
    for k, t in zip(NAMES, out):
        a, b = t.detach().cpu(), ref[k].detach()
        assert torch.equal(torch.isnan(a), torch.isnan(b)), k
        assert torch.allclose(a[~torch.isnan(a)], b[~torch.isnan(b)], rtol=2e-6, atol=1e-6), k
    assert bool(torch.isnan(out[0][:300]).all()) and not bool(torch.isnan(out[0][300:]).any())
    up = CC.upstream(4, 340, 4)
    torch.autograd.backward(list(out), [up[k].to(DEV) for k in NAMES])
    torch.autograd.backward([ref[k] for k in NAMES], [up[k] for k in NAMES])
    assert torch.equal(torch.isnan(cr.grad.cpu()), torch.isnan(ocr.grad)) and bool(torch.isnan(cr.grad).all())
    assert torch.equal(torch.isnan(dm[0]["xyz"].grad.cpu()), torch.isnan(om[0]["xyz"].grad))
    assert rel(dm[1]["xyz"].grad.cpu().numpy(), om[1]["xyz"].grad.numpy()) < 3e-5


@pytest.mark.parametrize("actors,flip", [((), False), ((37, 0, 501), True), (tuple([20] * 40), True)])
def test_identity_correction_is_bit_equal_to_no_correction(actors, flip):
    models = CC.make_case(8, 1001, list(actors), 16, 3)
    A = len(actors)
    g = torch.Generator().manual_seed(1)
    poses = torch.randn(A, 7, generator=g).to(DEV) if A else None
    idft = torch.randn(A, 3, generator=g).to(DEV) if A else None
    fm = (torch.rand(sum(actors), generator=g) < 0.5).to(DEV) if flip else None
    fq = torch.tensor([0.0, 0.0, 1.0, 0.0], device=DEV) if flip else None
    up = CC.upstream(2, 1001 + sum(actors), 16)
    res = []
    for corr in (None, (torch.tensor([1.0, 0, 0, 0], device=DEV, requires_grad=True), torch.zeros(3, device=DEV, requires_grad=True))):
        dm = to_dev(models)
        dp = poses.clone().requires_grad_(True) if A else None
        out = sgb.compose(dm, dp, idft, fm, fq, pose_correction=corr)
        torch.autograd.backward(list(out), [up[k].to(DEV) for k in NAMES])
        res.append(([t.detach() for t in out], [m[k].grad for m in dm for k in CC.KEYS], dp.grad if A else None))
    (o0, g0, p0), (o1, g1, p1) = res
    assert all(torch.equal(a, b) for a, b in zip(o0, o1))
    assert all(torch.equal(a, b) for a, b in zip(g0, g1))
    assert p0 is None or rel(p0.cpu().numpy(), p1.cpu().numpy()) < 1e-6  # float atomics: the order of the actor sums may differ


IMAGES = [(1, 1), (1, 37), (1, 1920), (1279, 1921), (1280, 1920)]


@pytest.mark.parametrize("H,W", IMAGES, ids=[f"{h}x{w}" for h, w in IMAGES])
def test_color_correct_per_element_vs_float64(H, W):
    g = torch.Generator(device=DEV).manual_seed(H + W)
    img, gout = torch.rand(3, H, W, generator=g, device=DEV), torch.randn(3, H, W, generator=g, device=DEV)
    A = torch.eye(4, device=DEV)[:3] + 0.3 * torch.randn(3, 4, generator=g, device=DEV)
    r = CR.color64(img, A, gout)
    i, a = img.clone().requires_grad_(True), A.clone().requires_grad_(True)
    o = sgb.color_correct(i, a)
    o.backward(gout)
    within(o.detach(), r["out"], r["b_out"], "out")
    within(i.grad, r["dimage"], r["b_dimage"], "dimage")
    within(a.grad, r["daffine"], r["b_daffine"], "daffine")
    # a second backward gives the same dL/dA bit for bit
    first = a.grad.clone()
    a.grad = None
    sgb.color_correct(i, a).backward(gout)
    assert torch.equal(first, a.grad)
    # an identity affine returns the image and the upstream gradient bit for bit
    e = torch.eye(4, device=DEV)[:3].requires_grad_(True)
    i.grad = None
    o = sgb.color_correct(i, e)
    assert torch.equal(o.detach(), img)
    o.backward(gout)
    assert torch.equal(i.grad, gout)


def test_color_correct_nonfinite_pixels_propagate_like_torch():
    g = torch.Generator(device=DEV).manual_seed(5)
    img = torch.rand(3, 33, 47, generator=g, device=DEV)
    img[0, 3, 4], img[1, 10, 10], img[2, 20, 1], img[0, 30, 46] = math.inf, -math.inf, math.nan, math.nan
    A = torch.eye(4, device=DEV)[:3] + 0.2 * torch.randn(3, 4, generator=g, device=DEV)
    gout = torch.randn(3, 33, 47, generator=g, device=DEV)
    i1, a1 = img.clone().requires_grad_(True), A.clone().requires_grad_(True)
    o1 = sgb.color_correct(i1, a1)
    o1.backward(gout)
    i2, a2 = img.clone().requires_grad_(True), A.clone().requires_grad_(True)
    o2 = CR.color(i2, a2)
    o2.backward(gout)
    for x, y in ((o1, o2), (i1.grad, i2.grad), (a1.grad, a2.grad)):
        x, y = x.detach(), y.detach()
        assert torch.equal(torch.isnan(x), torch.isnan(y)) and torch.equal(torch.isinf(x), torch.isinf(y))
        fin = torch.isfinite(y)
        assert torch.equal(x[~fin & ~torch.isnan(y)], y[~fin & ~torch.isnan(y)])
        assert torch.allclose(x[fin], y[fin], rtol=1e-5, atol=1e-6)


def test_color_correction_reg_vs_float64():
    g = torch.Generator(device=DEV).manual_seed(6)
    A = torch.eye(4, device=DEV)[:3] + 0.1 * torch.randn(3, 4, generator=g, device=DEV)
    S = torch.eye(4, device=DEV)[:3] + 0.1 * torch.randn(3, 4, generator=g, device=DEV)
    A[1, 1] = 1.0
    for sky in (S, None):
        r = CR.reg64(A, sky, 0.3)
        a = A.clone().requires_grad_(True)
        s = sky.clone().requires_grad_(True) if sky is not None else None
        v = sgb.color_correction_reg_loss(a, s, weight=0.3)
        v.backward()
        within(v.detach(), r["value"], r["b_value"], "value")
        within(a.grad, r["g_affine"], r["b_g"], "g_affine")
        assert float(a.grad[1, 1]) == 0.0
        if sky is not None:
            within(s.grad, r["g_affine_sky"], r["b_g"], "g_affine_sky")


def _config_c():
    cfg = dict(synthetic.CONFIGS["C"])
    cfg.pop("kind")
    sc = synthetic.make_scene(seed=0, with_raw=True, **cfg)
    cam = sc["cam"]
    st = sgb.GaussianRasterizationSettings(image_height=cam["image_height"], image_width=cam["image_width"], tanfovx=cam["tanfovx"],
                                           tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=DEV), scale_modifier=cam["scale_modifier"],
                                           viewmatrix=cam["viewmatrix"].to(DEV), projmatrix=cam["projmatrix"].to(DEV), sh_degree=cam["sh_degree"],
                                           campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    return sc["raw"], st, cam["image_height"], cam["image_width"]


def test_corrected_step_end_to_end_config_c_vs_reference_torch_lines():
    raw, st, H, W = _config_c()
    g = torch.Generator(device=DEV).manual_seed(2)
    gt = torch.rand(3, H, W, generator=g, device=DEV)
    rots = torch.tensor([[1.0, 0, 0, 0], [0.999, 0.01, -0.02, 0.015]], device=DEV) * torch.tensor([[1.0], [1.3]], device=DEV)
    trans = torch.tensor([[0.0, 0, 0], [0.05, -0.02, 0.03]], device=DEV)
    affine = torch.eye(4, device=DEV)[:3].repeat(2, 1, 1) + 0.05 * torch.randn(2, 3, 4, generator=g, device=DEV)
    rast = sgb.GaussianRasterizer(st)

    def step(impl):
        models = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in raw["models"]]
        poses = raw["poses"].to(DEV).requires_grad_(True)
        r, t, a = rots.clone().requires_grad_(True), trans.clone().requires_grad_(True), affine.clone().requires_grad_(True)
        if impl == "sgr":
            xyz, rot, scale, opac, sh = sgb.compose(models, poses, raw["idft"].to(DEV), pose_correction=(r[1], t[1]))
        else:
            o = CR.compose(models, poses, raw["idft"].to(DEV), None, None, (r[1], t[1]))
            xyz, rot, scale, opac, sh = (o[k] for k in NAMES)
        m2d = torch.zeros_like(xyz, requires_grad=True)
        col = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot)[0]
        col = sgb.color_correct(col, a[1]) if impl == "sgr" else CR.color(col, a[1])
        loss = losses.photometric_loss(col, gt, None, 1.0, 0.2)
        loss.backward()
        return col.detach(), [v.grad for m in models for v in m.values()] + [poses.grad, r.grad, t.grad, a.grad]

    ca, ga = step("sgr")
    cb, gb = step("torch")
    # 1e-4 per pixel, except pixels explained by at most two flips of the rasterizer's per-pair thresholds: the fp32 composer and
    # torch's lines round positions differently, which is enough to move a pair across alpha = 1/255 somewhere in 2.46 M pixels
    offenders = util.check_forward_flip_protocol(dict(color=ca.cpu().numpy()), dict(color=cb.cpu().numpy()), dict(color=float(cb.abs().max())))
    assert len(offenders) < 100, len(offenders)
    for k, (x, y) in enumerate(zip(ga, gb)):
        assert rel(x.cpu().numpy(), y.cpu().numpy()) < 1e-3, k
    assert float(ga[-3][1].abs().sum()) > 0 and float(ga[-3][0].abs().sum()) == 0.0


def test_corrected_step_captures_in_a_cuda_graph():
    models = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in CC.make_case(4, 20000, [3000, 0, 500], 16, 5)]
    poses = torch.randn(3, 7, device=DEV, requires_grad=True)
    idft = torch.randn(3, 5, device=DEV)
    cr = torch.tensor([0.9, 0.1, -0.1, 0.2], device=DEV, requires_grad=True)
    ct = torch.tensor([0.1, 0.2, -0.3], device=DEV, requires_grad=True)
    aff = (torch.eye(4, device=DEV)[:3] + 0.1).requires_grad_(True)
    img = torch.rand(3, 96, 128, device=DEV, requires_grad=True)
    leaves = [v for m in models for v in m.values()] + [poses, cr, ct, aff, img]
    P = 23500
    up = {k: v.to(DEV) for k, v in CC.upstream(3, P, 16).items()}
    gimg = torch.randn(3, 96, 128, device=DEV)

    def step():
        out = sgb.compose(models, poses, idft, pose_correction=(cr, ct))
        o = sgb.color_correct(img, aff)
        torch.autograd.backward(list(out) + [o], [up[k] for k in NAMES] + [gimg])
        return torch.cat([t.reshape(-1) for t in out] + [o.reshape(-1)])

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for x in leaves:
                x.grad = None
            eager = step()
    torch.cuda.current_stream().wait_stream(s)
    eager_grads = [x.grad.clone() for x in leaves]
    for x in leaves:
        x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    for x in leaves:
        x.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager)
    for x, e in zip(leaves, eager_grads):
        assert torch.allclose(x.grad, e, rtol=1e-5, atol=1e-6)
    assert torch.equal(aff.grad, eager_grads[-2])
