"""CPU: pin the fp64 restatements of oracle/step64.py (composer, image loss, Adam, densification statistics) to the reference's own
outputs and to fp64 torch, and check that their bounds are neither vacuous nor too tight: the fp32 torch oracles, standing in for the
kernels, fall inside the bounds on every element, and somewhere the largest error / bound ratio exceeds 1e-3."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_loss_golden import case as loss_case  # noqa: E402
import compose_case as CC  # noqa: E402
from oracle import compose_oracle as CO  # noqa: E402
from oracle import loss_oracle as LO  # noqa: E402
from oracle import step64 as S64  # noqa: E402
from test_compose_cpu import FIX as COMPOSE_FIX, load_case, rel  # noqa: E402
from test_losses_cpu import FIX as LOSS_FIX  # noqa: E402

F64 = torch.float64
NAMES = ("xyz", "rotation", "scaling", "opacity", "features")


def ratio(got, val, bnd):
    """max |got - val| / bound, asserting every element lies inside its bound."""
    err = (torch.as_tensor(got).to(F64) - torch.as_tensor(val).to(F64)).abs()
    bnd = torch.as_tensor(bnd).to(F64)
    bad = err > bnd
    assert not bool(bad.any()), (int(bad.sum()), float(err[bad][:4].max()), float(bnd[bad][:4].min()))
    return float((err / (bnd + 1e-300)).max())


def compose_inputs(path):
    z, M, models, poses, idft, flip, fq = load_case(path, requires_grad=False)
    up = CC.upstream(int(z["seed"]) + 1, sum(m["xyz"].shape[0] for m in models), M)
    return z, M, models, poses, idft, flip.bool(), fq, up


@pytest.mark.parametrize("path", COMPOSE_FIX, ids=[os.path.basename(p) for p in COMPOSE_FIX])
def test_compose64_matches_reference_model(path):
    z, M, models, poses, idft, flip, fq, up = compose_inputs(path)
    r = S64.compose64(models, poses, idft, flip, fq, up)
    for k in NAMES:
        assert rel(r[k].numpy(), z["ref_" + k]) < 1e-6, k
    for i in range(len(models)):
        for k in CC.KEYS:
            assert rel(r[f"g{i}_{k}"].numpy(), z[f"ref_g{i}_{k}"]) < 2e-5, (i, k)
    assert rel(r["dposes"].numpy(), z["ref_dposes"]) < 2e-5


@pytest.mark.parametrize("path", COMPOSE_FIX, ids=[os.path.basename(p) for p in COMPOSE_FIX])
def test_compose64_bounds_hold_fp32_oracle(path):
    """compose_oracle in fp32 with fp32 autograd is inside every bound; features_rest is bit-equal."""
    z, M, models, poses, idft, flip, fq, up = compose_inputs(path)
    r = S64.compose64(models, poses, idft, flip, fq, up)
    mm = [{k: v.clone().requires_grad_(True) for k, v in m.items()} for m in models]
    pp = poses.clone().requires_grad_(True)
    o = CO.compose(mm, pp, idft, flip, fq)
    worst = {}
    for k in NAMES:
        worst[k] = ratio(o[k].detach(), r[k], r["b_" + k])
    assert torch.equal(o["features"][:, 1:].detach().double(), r["features"][:, 1:])
    torch.autograd.backward([o[k] for k in NAMES], [up[k] for k in NAMES])
    for i, m in enumerate(mm):
        for k in CC.KEYS:
            worst[f"g{i}_{k}"] = ratio(m[k].grad, r[f"g{i}_{k}"], r[f"b_g{i}_{k}"])
        assert torch.equal(m["features_rest"].grad.double(), r[f"g{i}_features_rest"])
    worst["dposes"] = ratio(pp.grad, r["dposes"], r["b_dposes"])
    print(os.path.basename(path), {k: round(v, 4) for k, v in worst.items()})
    assert max(worst.values()) > 1e-3


def test_compose64_small_raw_quaternions_and_large_translations():
    """The rotation bound scales with 1 / |raw|; xyz with |t|: the fp32 oracle stays inside at |raw| = 1e-6 and |t| = 1e3."""
    g = torch.Generator().manual_seed(5)
    models = CC.make_case(21, 300, [200, 100], 4, 3)
    for m in models:
        m["rotation"] = m["rotation"] * torch.logspace(-6, 1, m["rotation"].shape[0])[:, None]
    poses = torch.randn(2, 7, generator=g)
    poses[:, 4:] *= 1e3
    poses[0, :4] *= 0.3 / poses[0, :4].norm()
    poses[1, :4] *= 7.0 / poses[1, :4].norm()
    idft = torch.randn(2, 3, generator=g)
    up = CC.upstream(8, 600, 4)
    r = S64.compose64(models, poses, idft, None, None, up)
    mm = [{k: v.clone().requires_grad_(True) for k, v in m.items()} for m in models]
    pp = poses.clone().requires_grad_(True)
    o = CO.compose(mm, pp, idft, None, torch.tensor([1.0, 0, 0, 0]))
    for k in NAMES:
        ratio(o[k].detach(), r[k], r["b_" + k])
    torch.autograd.backward([o[k] for k in NAMES], [up[k] for k in NAMES])
    for i, m in enumerate(mm):
        for k in CC.KEYS:
            ratio(m[k].grad, r[f"g{i}_{k}"], r[f"b_g{i}_{k}"])
    ratio(pp.grad, r["dposes"], r["b_dposes"])


# ----------------------------------------------------------------------------------------------- image loss
def loss64_autograd(img, gt, mask, w_l1, w_ssim):
    """The fp64 forward with the kernel's window, differentiated by autograd."""
    x = img.to(F64).requires_grad_(True)
    y = gt.to(F64)
    C = x.shape[0]
    win = S64.window_2d()[None, None].expand(C, 1, 11, 11).contiguous()
    if mask is not None:
        xm, ym = torch.where(mask, x, 0.0), torch.where(mask, y, 0.0)
    else:
        xm, ym = x, y
    conv = lambda t: F.conv2d(t[None], win, padding=5, groups=C)[0]
    mu1, mu2 = conv(xm), conv(ym)
    s1, s2, s12 = conv(xm * xm) - mu1 ** 2, conv(ym * ym) - mu2 ** 2, conv(xm * ym) - mu1 * mu2
    C1, C2 = S64.C1_32, S64.C2_32
    ss = (((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 ** 2 + mu2 ** 2 + C1) * (s1 + s2 + C2))).mean()
    l1 = LO.l1_loss(x, y, mask)
    loss = w_l1 * l1 + w_ssim * ss
    (g,) = torch.autograd.grad(loss, x)
    return float(l1), float(ss), g


def test_image_loss64_matches_reference_functions():
    z = np.load(LOSS_FIX)
    for seed in (0, 1):
        img, gt, mask = loss_case(seed)
        for tag, m in (("nomask", None), ("mask", mask)):
            k = f"s{seed}_{tag}_"
            a = S64.image_loss64(img, gt, m, 1.0, 0.0)
            assert abs(a["value"] - float(z[k + "l1"])) < 1e-7 and rel(a["grad"].numpy(), z[k + "g_l1"]) < 1e-6
            b = S64.image_loss64(img, gt, m, 0.0, 1.0)
            assert abs(b["value"] - float(z[k + "ssim"])) < 1e-6 and rel(b["grad"].numpy(), z[k + "g_ssim"]) < 1e-5
            assert float(b["premise"].max()) < 1e-2


@pytest.mark.parametrize("C,H,W", [(3, 70, 93), (1, 16, 5), (4, 10, 10), (3, 1, 1)])
def test_image_loss64_closed_form_matches_fp64_autograd(C, H, W):
    g = torch.Generator().manual_seed(C * H + W)
    gt = torch.rand(C, H, W, generator=g)
    img = gt + 0.2 * torch.randn(C, H, W, generator=g)
    img[:, : H // 2, : W // 2] = gt[:, : H // 2, : W // 2]  # x = y exactly: sign(0) = 0
    mask = torch.rand(1, H, W, generator=g) > 0.3
    for m in (None, mask):
        for wl, ws in ((0.8, -0.2), (1.0, 0.0), (0.0, 1.0)):
            a = S64.image_loss64(img, gt, m, wl, ws)
            l1, ss, ga = loss64_autograd(img, gt, m, wl, ws)
            assert abs(a["ssim"] - ss) < 1e-12 and (abs(a["l1"] - l1) < 1e-12 or (math.isnan(l1) and math.isnan(a["l1"])))
            assert float((a["grad"] - ga).abs().max()) <= 1e-12 * max(1e-30, float(ga.abs().max())), (wl, ws)


def test_window_matches_make_window_and_reference():
    """window_1d is make_window's arithmetic and the reference's fp32 1D window bit for bit; its exact outer product is within 2^-23
    (relative, per weight) of the reference's fp32 2D window g.mm(g.t()).float() (loss_utils.py:84-89).  (A sequential fp32 sum,
    which make_window once used, is one ulp low and puts the outer product 2^-22 away.)"""
    w = S64.window_1d()
    g = np.array([np.float32(math.exp(-float((k - 5) ** 2) / 4.5)) for k in range(11)], np.float32)
    s = np.float32(math.fsum(float(v) for v in g))
    assert np.array_equal(w, (g / s).astype(np.float32))
    g_ref = torch.tensor([math.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)])
    assert np.array_equal(w, (g_ref / g_ref.sum()).numpy())
    assert np.array_equal(w, w[::-1])  # symmetric: the convolution is its own adjoint
    ref = LO._window(1, torch.float32, "cpu")[0, 0].double()
    mine = S64.window_2d()
    assert float(((mine - ref).abs() / ref).max()) <= 2.0 ** -23


def test_image_loss64_bounds_hold_fp32_oracle():
    """loss_oracle in fp32 (the reference's window, conv2d, autograd) is inside every bound, including flat and constant regions
    where sig = E[x^2] - mu^2 cancels."""
    worst = []
    for seed in (0, 1):
        img, gt, mask = loss_case(seed)
        img[:, 10:30, 20:50] = 0.25
        gt[:, 10:30, 20:50] = 0.25 + 1e-3 * torch.rand(3, 20, 30, generator=torch.Generator().manual_seed(seed))
        for m in (None, mask):
            r = S64.image_loss64(img, gt, m, 0.8, -0.2)
            assert float(r["premise"].max()) < 1e-2
            x = img.clone().requires_grad_(True)
            v = 0.8 * LO.l1_loss(x, gt, m) - 0.2 * LO.ssim(x, gt, m)
            v.backward()
            worst.append(ratio(x.grad, r["grad"], r["b_grad"]))
            worst.append(ratio(torch.tensor(float(v)), torch.tensor(r["value"]), torch.tensor(r["b_value"])))
    print("image_loss64 worst", [round(w, 4) for w in worst])
    assert max(worst) > 1e-3


# ----------------------------------------------------------------------------------------------- Adam
def _torch_adam(p, g, m, v, lr, step, dtype):
    q = torch.nn.Parameter(p.clone().to(dtype))
    opt = torch.optim.Adam([q], lr=lr, eps=1e-15)
    opt.state[q] = dict(step=torch.tensor(float(step - 1)), exp_avg=m.clone().to(dtype), exp_avg_sq=v.clone().to(dtype))
    q.grad = g.clone().to(dtype)
    opt.step()
    st = opt.state[q]
    return q.detach(), st["exp_avg"], st["exp_avg_sq"]


def adam_state(n, seed):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=g)
    grad = torch.randn(n, generator=g) * torch.logspace(-19, 3, n)[torch.randperm(n, generator=g)]
    grad[:7] = 0.0
    m = torch.randn(n, generator=g) * 1e-2
    v = torch.rand(n, generator=g) * 1e-3
    v[:3] = 0.0
    m[:3] = 0.0
    return p, grad, m, v


@pytest.mark.parametrize("step", [1, 2, 1000, 30000])
def test_adam64_matches_torch_adam_fp64(step):
    p, g, m, v = adam_state(4097, step)
    r = S64.adam64(p, g, m, v, 1.6e-4, step)
    tp, tm, tv = _torch_adam(p, g, m, v, 1.6e-4, step, F64)
    for a, b in ((r["p"], tp), (r["m"], tm), (r["v"], tv)):
        assert float((a - b).abs().max()) <= 1e-14 * float(b.abs().max() + 1e-300)


def test_adam64_bounds_hold_fp32_torch_adam():
    worst = {}
    for step in (1, 2, 1000, 30000):
        p, g, m, v = adam_state(8193, step + 1)
        r = S64.adam64(p, g, m, v, 5e-3, step)
        tp, tm, tv = _torch_adam(p, g, m, v, 5e-3, step, torch.float32)
        for k, t in (("p", tp), ("m", tm), ("v", tv)):
            worst[(step, k)] = ratio(t, r[k], r["b_" + k])
    print("adam64 worst", {str(k): round(w, 4) for k, w in worst.items()})
    assert max(worst.values()) > 1e-3


def test_stats64_matches_reference_semantics():
    g = torch.Generator().manual_seed(2)
    n = 500
    radii = torch.randint(-2, 30, (n,), generator=g, dtype=torch.int32)
    g2 = torch.randn(n, 3, generator=g)
    mr, ga, dn = torch.rand(n, generator=g) * 20, torch.rand(n, 2, generator=g), torch.randint(0, 9, (n, 1), generator=g).float()
    r = S64.stats64(mr, ga, dn, radii, g2)
    vis = radii > 0
    m2, a2, d2 = mr.clone(), ga.clone(), dn.clone()
    m2[vis] = torch.max(m2[vis], radii[vis].float())
    a2[vis, 0:1] += torch.norm(g2[vis, :2], dim=-1, keepdim=True)
    a2[vis, 1:2] += torch.norm(g2[vis, 2:], dim=-1, keepdim=True)
    d2[vis] += 1
    assert torch.equal(r["max_radii2D"], m2.double()) and torch.equal(r["denom"], d2.double())
    assert ratio(a2, r["xyz_gradient_accum"], r["b_xyz_gradient_accum"]) > 1e-3
