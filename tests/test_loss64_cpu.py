"""CPU: pin the restatements acc_loss64 and lidar64 (oracle/step64.py) of the sky, object-accumulation and LiDAR depth losses to the
reference's own train.py lines (tests/golden/callsite/train_losses.npz) and to fp64 autograd of the torch restatements; check that the
LiDAR keys are bit-equal to torch's fp32 err, that the selection is torch.topk's wherever the k-th key is not tied, that the fp32
torch oracles fall inside every acc_loss64 bound without the bound being vacuous, what torch does with a NaN accumulation, and that
every case of tests/loss64_case.py sits on the edge it was built for."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_train_loss_golden import case as train_case  # noqa: E402
import loss64_case as LC  # noqa: E402
import train_loss_oracle as TO  # noqa: E402
from oracle import loss_oracle as LO  # noqa: E402
from oracle import step64 as S64  # noqa: E402
from test_step64_cpu import ratio  # noqa: E402
from test_train_losses_cpu import TRAIN_FIX  # noqa: E402

F64 = torch.float64
TORCH_FORM = {"sky": LO.sky_loss, "obj": TO.obj_acc_loss}
LIDAR_CASES = LC.lidar_cases()
ACC_CASES = LC.acc_cases()


def torch_err(depth, acc, lidar):
    """The reference's expression (train.py:127-129) in fp32 on the CPU, over every pixel."""
    return torch.abs(depth / (acc + 1e-10) - lidar)


def torch_acc_loss(kind, acc, flag, weight, dtype=torch.float32):
    a = acc.to(dtype).clone().requires_grad_(True)
    v = TORCH_FORM[kind](a, flag, weight)
    v.backward()
    return float(v.detach()), a.grad.reshape(-1)


# ----------------------------------------------------------------------------------------------- sky / object losses
@pytest.mark.parametrize("seed", [0, 1])
def test_acc_loss64_matches_reference_fixture(seed):
    """The reference's own object-accumulation lines: value within 2e-6 and every fp32 gradient element inside acc_loss64's bound."""
    z = np.load(TRAIN_FIX)
    c = train_case(seed)
    r = S64.acc_loss64("obj", c["acc_obj"], c["obj_bound"], 1.0)
    ref = float(z[f"s{seed}_obj"])
    assert abs(r["value"] - ref) <= 2e-6 * abs(ref)
    ratio(torch.from_numpy(z[f"s{seed}_g_acc_obj"]).reshape(-1), r["grad"], r["b_grad"])


@pytest.mark.parametrize("kind", ["sky", "obj"])
def test_acc_loss64_matches_fp64_autograd(kind):
    """Off the clamp (where the fp64 and fp32 clamp edges differ), acc_loss64 is fp64 autograd of the torch restatement."""
    g = torch.Generator().manual_seed(3)
    acc = (torch.rand(1, 60, 70, generator=g) * 0.99998 + 1e-5)
    flag = torch.rand(1, 60, 70, generator=g) > 0.5
    r = S64.acc_loss64(kind, acc, flag, 0.3)
    v, gr = torch_acc_loss(kind, acc, flag, 0.3, F64)
    assert abs(r["value"] - v) <= 1e-13 * abs(v)
    assert torch.allclose(r["grad"], gr, rtol=1e-12, atol=0.0)


@pytest.mark.parametrize("kind", ["sky", "obj"])
@pytest.mark.parametrize("case", ACC_CASES, ids=[c["name"] for c in ACC_CASES])
def test_acc_loss64_bounds_hold_fp32_torch(kind, case):
    """The fp32 torch restatement, standing in for the kernel, is inside every bound; the clamp edges pass or stop the gradient
    exactly as acc_loss64's `inside` says; a NaN gives a NaN value in both."""
    r = S64.acc_loss64(kind, case["acc"], case["flag"], case["weight"])
    case["edge"](case, r)
    v, gr = torch_acc_loss(kind, case["acc"], case["flag"], case["weight"])
    ins = r["inside"]
    assert not bool((gr[~ins] != 0).any())
    rg = ratio(gr, r["grad"], r["b_grad"])
    if np.isnan(r["value"]):
        assert np.isnan(v)
    else:
        assert abs(v - r["value"]) <= r["b_value"], (v, r["value"], r["b_value"])
    print(case["name"], kind, round(rg, 4))


def test_acc_loss64_bounds_are_not_vacuous():
    worst = 0.0
    for kind in ("sky", "obj"):
        for case in ACC_CASES[:2]:
            r = S64.acc_loss64(kind, case["acc"], case["flag"], case["weight"])
            worst = max(worst, ratio(torch_acc_loss(kind, case["acc"], case["flag"], case["weight"])[1], r["grad"], r["b_grad"]))
    assert worst > 1e-3, worst


@pytest.mark.parametrize("kind", ["sky", "obj"])
def test_torch_propagates_nan_through_the_clamp(kind):
    """torch.clamp keeps NaN: the reference's value is NaN and the NaN pixel's gradient is 0 (the other pixels keep theirs)."""
    acc = torch.tensor([[[0.3, float("nan"), 0.7]]])
    flag = torch.tensor([[[True, False, True]]])
    v, gr = torch_acc_loss(kind, acc, flag, 1.0)
    assert np.isnan(v) and gr[1] == 0 and bool((gr[[0, 2]] != 0).all())
    r = S64.acc_loss64(kind, acc, flag, 1.0)
    assert np.isnan(r["value"]) and r["grad"][1] == 0 and torch.allclose(r["grad"][[0, 2]], gr[[0, 2]].double(), rtol=1e-6)


# ----------------------------------------------------------------------------------------------- LiDAR
def fixture_case(seed):
    c = train_case(seed)
    return dict(depth=c["depth"], acc=c["acc"], lidar=c["lidar_depth"], mask=c["mask"])


def lidar_of(c, **kw):
    return S64.lidar64(c["depth"], c["acc"], c["lidar"], c["mask"], kw.get("weight", c.get("weight", 1.0)), kw.get("keep", c.get("keep", 0.95)))


@pytest.mark.parametrize("seed", [0, 1])
def test_lidar64_matches_reference_fixture(seed):
    """The reference's own LiDAR lines: value within 2e-6, dL/ddepth and dL/dacc bit-equal (the keys are untied there)."""
    z = np.load(TRAIN_FIX)
    c = fixture_case(seed)
    r = lidar_of(c, weight=1.0, keep=0.95)
    assert r["ties"] == 1
    ref = float(z[f"s{seed}_lidar"])
    assert abs(r["value"] - ref) <= 2e-6 * abs(ref)
    assert np.array_equal(r["gd"], z[f"s{seed}_g_depth"].reshape(-1)) and np.array_equal(r["ga"], z[f"s{seed}_g_acc"].reshape(-1))


@pytest.mark.parametrize("seed", [0, 1])
def test_lidar64_matches_fp64_autograd(seed):
    c = fixture_case(seed)
    r = lidar_of(c, weight=0.7, keep=0.95)
    d, a = c["depth"].double().requires_grad_(True), c["acc"].double().requires_grad_(True)
    v = TO.lidar_depth_loss(d, a, c["lidar"].double(), c["mask"], weight=float(np.float32(0.7)))
    v.backward()
    assert abs(r["value"] - float(v)) <= 1e-6 * abs(float(v))
    assert np.allclose(r["gd"], d.grad.reshape(-1).numpy(), rtol=1e-6, atol=0.0)
    assert np.allclose(r["ga"], a.grad.reshape(-1).numpy(), rtol=1e-6, atol=1e-30)


def _lidar_case_ids():
    return [c["name"] for c in LIDAR_CASES]


@pytest.mark.parametrize("case", LIDAR_CASES, ids=_lidar_case_ids())
def test_lidar_keys_are_torch_err_bit_for_bit(case):
    """lidar64's keys are the bits of torch's fp32 err on every valid pixel; NaN only as NaN."""
    r = lidar_of(case)
    err = torch_err(case["depth"], case["acc"], case["lidar"]).reshape(-1).numpy()
    v = r["valid"]
    nan = np.isnan(err)
    assert np.array_equal(nan[v], r["key"][v] == S64.NAN_KEY)
    assert np.array_equal(err[v & ~nan].view(np.uint32), r["key"][v & ~nan].astype(np.uint32))


@pytest.mark.parametrize("case", LIDAR_CASES, ids=_lidar_case_ids())
def test_lidar_cases_sit_on_their_edge(case):
    r = lidar_of(case)
    case["edge"](case, r)
    assert int(r["sel"].sum()) == r["k"] and not (r["sel"] & ~r["valid"]).any()
    if r["k"]:
        ks = r["key"][r["sel"]]
        assert ks.max() == r["t"] and (r["key"][r["valid"] & ~r["sel"]] >= r["t"]).all()


@pytest.mark.parametrize("case", [c for c in LIDAR_CASES if not c["name"].startswith("radix_nan")], ids=lambda c: c["name"])
def test_lidar64_selection_is_torch_topk_off_ties(case):
    """torch.topk(largest=False) selects the same pixels, apart from which of the pixels tied at the k-th key it takes."""
    r = lidar_of(case)
    if r["k"] == 0:
        return
    valid = torch.from_numpy(r["valid"])
    err = torch_err(case["depth"], case["acc"], case["lidar"]).reshape(-1)
    flat = torch.nonzero(valid).reshape(-1)
    _, i = torch.topk(err[valid], r["k"], largest=False)
    top = np.zeros(r["key"].size, bool)
    top[flat[i].numpy()] = True
    off = ~(r["valid"] & (r["key"] == r["t"]))
    assert np.array_equal(top[off], r["sel"][off])
    if r["ties"] == 1:
        assert np.array_equal(top, r["sel"])
    assert int(top.sum()) == r["k"]


@pytest.mark.parametrize("case", [c for c in LIDAR_CASES if c["depth"].numel() <= 300_000], ids=lambda c: c["name"])
def test_lidar64_gradients_are_torch_fp32_off_ties(case):
    """fp32 autograd of the torch restatement gives the same gradients bit for bit wherever the k-th key is not tied (torch.topk's
    own pick among ties is unspecified); mean and weight are applied by torch in a different order, so gk is compared, not assumed."""
    r = lidar_of(case)
    if r["k"] == 0 or r["ties"] > 1:
        return
    d, a = case["depth"].clone().requires_grad_(True), case["acc"].clone().requires_grad_(True)
    TO.lidar_depth_loss(d, a, case["lidar"], case["mask"], weight=1.0, keep=case["keep"]).backward()
    r1 = lidar_of(case, weight=1.0)
    assert np.array_equal(r1["gd"], d.grad.reshape(-1).numpy(), equal_nan=True)
    assert np.array_equal(r1["ga"], a.grad.reshape(-1).numpy(), equal_nan=True)
