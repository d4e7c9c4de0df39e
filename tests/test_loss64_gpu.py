"""The fp64 tier of the sky, object-accumulation and LiDAR depth losses: acc_loss_kernel<SkyForm / ObjForm> and the five LiDAR
kernels against oracle/step64.py's acc_loss64 / lidar64 on the cases of tests/loss64_case.py, each of which asserts its edge.

  LiDAR     the selected set is exactly the restatement's (ties at the lowest flat indices, across tiles and blocks); dL/ddepth and
            dL/dacc, after autograd's x g_out, are bit-equal to the fp32 restatement; the value is within (u + (k + 2) 2^-53) |v| +
            2^-149 of the fp64 mean; n and k (scalars[2..3], read by a direct C call) are exact.
  sky, obj  every gradient element and the value within acc_loss64's bound; NaN in acc gives a NaN value and a zero gradient there.
REPORT collects the largest error / bound per check."""
import ctypes as C

import numpy as np
import pytest
import torch

import loss64_case as LC
from oracle import step64 as S64
from street_gaussians_b200 import _capi, losses
from street_gaussians_b200._capi import ptr, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPORT = {}
LIDAR_CASES = LC.lidar_cases()
ACC_CASES = LC.acc_cases()


def _np(t):
    return t.detach().cpu().reshape(-1).numpy()


def lidar_direct(c, with_grads):
    """sgr_lidar_depth_loss called through ctypes: all four scalars {weight * mean, mean, n, k}."""
    L = _capi.lib()
    d, a, l = (c[k].to(DEV).contiguous() for k in ("depth", "acc", "lidar"))
    m = c["mask"].reshape(-1).to(DEV, torch.uint8).contiguous() if c["mask"] is not None else None
    N = d.numel()
    gd = torch.empty_like(d) if with_grads else None
    ga = torch.empty_like(a) if with_grads else None
    scalars = torch.empty(4, device=DEV)
    nbytes = int(L.sgr_lidar_depth_loss_scratch_bytes(N))
    scratch = torch.empty(nbytes, device=DEV, dtype=torch.uint8)
    rc = L.sgr_lidar_depth_loss(N, ptr(d), ptr(a), ptr(l), ptr(m), C.c_double(c["keep"]), C.c_float(c["weight"]), ptr(gd), ptr(ga),
                                ptr(scalars), ptr(scratch), nbytes, stream(torch.device(DEV)))
    _capi.check(rc, "sgr_lidar_depth_loss")
    torch.cuda.synchronize()
    return scalars.cpu().numpy()


def check_value(key, got, val, bnd):
    if not np.isfinite(val):
        assert (np.isnan(got) and np.isnan(val)) or got == val, (key, got, val)
        return 0.0
    err = abs(got - val)
    assert err <= bnd, (key, got, val, bnd)
    return err / bnd if bnd > 0 else 0.0


@pytest.mark.parametrize("case", LIDAR_CASES, ids=[c["name"] for c in LIDAR_CASES])
def test_lidar_depth_loss_vs_lidar64(case):
    r = S64.lidar64(case["depth"], case["acc"], case["lidar"], case["mask"], case["weight"], case["keep"])
    case["edge"](case, r)
    need = case["need"]
    d = case["depth"].to(DEV).requires_grad_("depth" in need)
    a = case["acc"].to(DEV).requires_grad_("acc" in need)
    v = losses.lidar_depth_loss(d, a, case["lidar"].to(DEV), case["mask"].to(DEV) if case["mask"] is not None else None,
                                weight=case["weight"], keep=case["keep"])
    if need:
        (case["g_out"] * v).backward()
    torch.cuda.synchronize()
    worst = {"value": check_value("value", float(v.detach()), r["value"], r["b_value"])}
    g_out = np.float32(case["g_out"])
    sel_signed = r["sel"] & (r["gd"] != 0)
    for leaf, name, want in ((d, "depth", r["gd"]), (a, "acc", r["ga"])):
        if name not in need:
            assert leaf.grad is None
            continue
        got = _np(leaf.grad)
        want = want * g_out
        if name == "depth":  # the selection, read off dL/ddepth (pixels whose sign(df) is 0 carry no gradient in either)
            picked = got != 0
            assert np.array_equal(picked, sel_signed), (int((picked & ~sel_signed).sum()), int((~picked & sel_signed).sum()))
        bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
        assert not bad.any(), (name, int(bad.sum()), np.nonzero(bad)[0][:6].tolist(), got[bad][:6].tolist(), want[bad][:6].tolist())
    for with_grads in ((True, False) if need else (False,)):
        s = lidar_direct(case, with_grads)
        assert s[2] == r["n"] and s[3] == r["k"], (s, r["n"], r["k"])
        worst["value"] = max(worst["value"], check_value("scalars[0]", float(s[0]), r["value"], r["b_value"]))
        if r["k"]:
            mean = r["value"] / float(np.float32(case["weight"]))
            check_value("scalars[1]", float(s[1]), mean, r["b_value"] / abs(float(np.float32(case["weight"]))))
    REPORT[f"lidar_{case['name']}"] = {k: round(x, 4) for k, x in worst.items()}
    print(case["name"], REPORT[f"lidar_{case['name']}"], "k", r["k"], "ties", r["ties"], "take", r["take"])


def within(worst, key, got, val, bnd):
    err = (got.detach().to(torch.float64).cpu() - val.cpu()).abs()
    bad = ~(err <= bnd.cpu())
    assert not bool(bad.any()), (key, int(bad.sum()), torch.nonzero(bad)[:6].tolist(), err[bad][:6].tolist(), bnd.cpu()[bad][:6].tolist())
    worst[key] = max(worst.get(key, 0.0), float((err / (bnd.cpu() + 1e-300)).max()))


@pytest.mark.parametrize("kind", ["sky", "obj"])
@pytest.mark.parametrize("case", ACC_CASES, ids=[c["name"] for c in ACC_CASES])
def test_acc_loss_vs_acc_loss64(kind, case):
    r = S64.acc_loss64(kind, case["acc"], case["flag"], case["weight"])
    case["edge"](case, r)
    fn = losses.sky_loss if kind == "sky" else losses.obj_acc_loss
    a = case["acc"].to(DEV).requires_grad_(True)
    v = fn(a, case["flag"].to(DEV), case["weight"])
    (case["g_out"] * v).backward()
    torch.cuda.synchronize()
    g_out = float(np.float32(case["g_out"]))
    worst = {"value": check_value("value", float(v.detach()), r["value"], r["b_value"])}
    # autograd's x g_out is one more fp32 rounding
    within(worst, "grad", a.grad.reshape(-1), r["grad"] * g_out, r["b_grad"] * abs(g_out) + S64.U * (r["grad"] * g_out).abs())
    got = a.grad.reshape(-1).cpu()
    assert not bool((got[~r["inside"].cpu()] != 0).any())
    nan = torch.isnan(case["acc"].reshape(-1))
    if bool(nan.any()):
        assert np.isnan(float(v.detach())) and bool((got[nan] == 0).all())
    REPORT[f"{kind}_{case['name']}"] = {k: round(x, 4) for k, x in worst.items()}
    print(kind, case["name"], REPORT[f"{kind}_{case['name']}"])
