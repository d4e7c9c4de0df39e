"""GPU: the sky cube map composite (sgr_sky_composite_forward / _backward through street_gaussians_b200.sky_composite) against the
reference's own outputs (tests/golden/callsite/sky.npz), element by element against the float64 restatement of tests/sky_oracle.py
at 1920x1280 with R = 1024 on cameras that straddle a face edge and a cube corner, with the reference's jitter, on a frame without
sky, without host synchronisation and under CUDA-graph capture, and inside one training step against the torch restatement."""
import math

import numpy as np
import pytest
import torch

import sky_oracle as SO
import street_gaussians_b200 as sgb
from street_gaussians_b200 import losses, synthetic
from street_gaussians_b200.training import FusedAdam
from test_compose_cpu import rel
from test_sky_cpu import CASES, load

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64


def outside(got, val, bnd):
    err = (got.to(F64) - val).abs()
    return ~(err <= bnd), err


def check(got, val, bnd, what, r=None):
    bad, err = outside(got, val, bnd)
    if bool(bad.any()):
        where = bad.nonzero()[:10].tolist()
        info = ""
        if r is not None and got.dim() == 3 and got.shape[1:] == r["x"].shape:
            info = [(int(r["face"][p[1], p[2]]), float(r["x"][p[1], p[2]]), float(r["y"][p[1], p[2]])) for p in where]
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside their bound, worst {float((err / bnd)[bad].max()):.3g}x, at {where} {info}")
    return float((err / bnd).max())


def _run(rgb, acc, cube, K, w2c, g, sky_mask=None, perturb=False, white=True):
    r_, a_, c_ = (t.clone().requires_grad_(True) for t in (rgb, acc, cube))
    out = sgb.sky_composite(r_, a_, c_, K, w2c, sky_mask=sky_mask, perturb=perturb, white_background=white)
    out.backward(g)
    return out.detach(), r_.grad, a_.grad, c_.grad


@pytest.mark.parametrize("case", CASES)
def test_sky_vs_reference_fixture(case, monkeypatch):
    z, a = load(case)
    d = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in a.items()}
    perturb = a["jx"] is not None
    if perturb:  # hand the kernel the two draws the reference made
        draws = [d["jx"], d["jy"]]
        monkeypatch.setattr(torch, "rand", lambda *s, **k: draws.pop(0).clone())
    out, drgb, dacc, dcube = _run(d["rgb"], d["acc"], d["cube"], d["K"], d["w2c"], d["g"], d["sky_mask"], perturb, d["fill"] == 1.0)
    monkeypatch.undo()
    ref = lambda k: z[f"{case}_{k}"]
    assert float(np.abs(out.cpu().numpy() - ref("ref_out")).max()) < 1e-4
    assert torch.equal(drgb.cpu(), torch.from_numpy(ref("ref_drgb")))
    assert rel(dacc.cpu().numpy(), ref("ref_dacc")) < 1e-3
    assert rel(dcube.cpu().numpy(), ref("ref_dcube")) < 1e-3


def _look_at(target, roll=0.0):
    """w2c [4, 4] of a camera at (3, -2, 5) looking along `target` (a world direction), rolled by `roll` radians."""
    z = torch.tensor(target, dtype=F64)
    z = z / z.norm()
    x = torch.linalg.cross(torch.tensor([math.sin(roll), math.cos(roll), 0.0], dtype=F64), z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    Rc = torch.stack([x, y, z], 1)  # camera-to-world rotation
    w2c = torch.eye(4, dtype=F64)
    w2c[:3, :3] = Rc.T
    w2c[:3, 3] = -Rc.T @ torch.tensor([3.0, -2.0, 5.0], dtype=F64)
    return w2c.float()


H, W, RES = 1280, 1920, 1024
K_WAYMO = torch.tensor([[2055.6, 0.0, 939.7], [0.0, 2051.3, 641.1], [0.0, 0.0, 1.0]])
VIEWS = {"edge": ([1.0, -0.15, 1.0], 0.1), "corner": ([1.0, -1.0, 1.0], 0.2)}


def _frame(seed, R=RES):
    g = torch.Generator(device=DEV).manual_seed(seed)
    cube = -0.2 + 1.4 * torch.rand(6, R, R, 3, generator=g, device=DEV)
    rgb = torch.rand(3, H, W, generator=g, device=DEV)
    acc = torch.rand(1, H, W, generator=g, device=DEV)
    acc = torch.where(torch.rand(1, H, W, generator=g, device=DEV) < 0.4, torch.zeros_like(acc), acc)
    acc[:, 600:900, 700:1300] = 1.0
    up = torch.randn(3, H, W, generator=g, device=DEV)
    mask = torch.rand(1, H, W, generator=g, device=DEV) < 0.5
    return cube, rgb, acc, up, mask


@pytest.mark.parametrize("view", list(VIEWS))
@pytest.mark.parametrize("masked", [False, True], ids=["acc", "sky_mask"])
def test_sky_per_element_vs_float64(view, masked):
    cube, rgb, acc, up, mask = _frame(3 + masked)
    w2c = _look_at(*VIEWS[view]).to(DEV)
    K = K_WAYMO.to(DEV)
    sky_mask = mask if masked else None
    white = not masked
    out, drgb, dacc, dcube = _run(rgb, acc, cube, K, w2c, up, sky_mask, False, white)
    r = SO.sky64(rgb, acc, cube, K, w2c, up, sky_mask, None, None, 1.0 if white else 0.0)
    sampled = SO.sky_mask_of(acc, sky_mask)
    faces = set(torch.unique(r["face"][sampled]).tolist())
    assert len(faces) >= (3 if view == "corner" else 2), faces
    check(out, r["out"], r["b_out"], "rgb_out", r)
    check(dacc, r["dacc"], r["b_dacc"], "dacc", r)
    assert torch.equal(drgb, up)
    check(dcube, r["dcube"], r["b_dcube"], "dcube")
    assert int((dcube != 0).sum()) > 1000


def test_perturb_draws_the_reference_jitter_from_the_seeded_generator():
    cube, rgb, acc, up, mask = _frame(5, R=256)
    w2c, K = _look_at(*VIEWS["corner"]).to(DEV), K_WAYMO.to(DEV)
    torch.manual_seed(1234)
    out, _, dacc, dcube = _run(rgb, acc, cube, K, w2c, up, mask, True, True)
    torch.manual_seed(1234)
    jx = torch.rand(H, W, device=DEV)  # graphics_utils.py:195-196
    jy = torch.rand(H, W, device=DEV)
    r = SO.sky64(rgb, acc, cube, K, w2c, up, mask, jx, jy, 1.0)
    check(out, r["out"], r["b_out"], "rgb_out (perturbed)", r)
    check(dacc, r["dacc"], r["b_dacc"], "dacc (perturbed)", r)
    check(dcube, r["dcube"], r["b_dcube"], "dcube (perturbed)")
    r0 = SO.sky64(rgb, acc, cube, K, w2c, up, mask, None, None, 1.0)
    assert float((r0["out"] - out.to(F64)).abs().max()) > 1e-3  # the jitter moved the samples


@pytest.mark.parametrize("white", [True, False])
def test_frame_without_sky(white):
    cube, rgb, _, up, _ = _frame(6, R=64)
    acc = torch.full((1, H, W), 0.9995, device=DEV)
    acc[:, :, ::3] = 1.0
    w2c, K = _look_at(*VIEWS["corner"]).to(DEV), K_WAYMO.to(DEV)
    out, _, dacc, dcube = _run(rgb, acc, cube, K, w2c, up, None, False, white)
    fill = 1.0 if white else 0.0
    assert torch.equal(out, rgb + fill * (1 - acc))
    assert torch.equal(dcube, torch.zeros_like(dcube))
    assert torch.allclose(dacc, -(fill * up).sum(0, keepdim=True), rtol=1e-6, atol=1e-6)


def test_callers_mask_is_not_written():
    cube, rgb, acc, up, mask = _frame(7, R=64)
    before = mask.clone()
    w2c, K = _look_at(*VIEWS["edge"]).to(DEV), K_WAYMO.to(DEV)
    _run(rgb, acc, cube, K, w2c, up, mask, True, True)
    assert torch.equal(mask, before) and not bool(mask[:, :50].all())


def test_no_host_sync_and_graph_capture_replays_eager():
    cube, rgb, acc, up, mask = _frame(8, R=128)
    w2c, K = _look_at(*VIEWS["corner"]).to(DEV), K_WAYMO.to(DEV)
    r_, a_, c_ = (t.clone().requires_grad_(True) for t in (rgb, acc, cube))

    def step():
        out = sgb.sky_composite(r_, a_, c_, K, w2c, sky_mask=mask, perturb=False)
        out.backward(up)
        return out.detach()

    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sgb.sky_composite(r_, a_, c_, K, w2c, sky_mask=mask, perturb=True).backward(up)
        sgb.sky_composite(r_, a_, c_, K, w2c).backward(up)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for x in (r_, a_, c_):
                x.grad = None
            eager = step()
    torch.cuda.current_stream().wait_stream(s)
    eager_grads = [x.grad.clone() for x in (r_, a_, c_)]
    for x in (r_, a_, c_):
        x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    for x in (r_, a_, c_):
        x.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager)
    assert torch.equal(r_.grad, eager_grads[0]) and torch.equal(a_.grad, eager_grads[1])
    # float atomics: the order of the texel sums may differ, so the replay's dL/dcube is held to the oracle's bound like the eager one
    r = SO.sky64(rgb, acc, cube, K, w2c, up, mask, None, None, 1.0)
    check(eager_grads[2], r["dcube"], r["b_dcube"], "dcube (eager)")
    check(c_.grad, r["dcube"], r["b_dcube"], "dcube (replay)")


def test_training_step_with_sky_matches_torch_restatement():
    """compose -> GaussianRasterizer -> sky -> color_correct -> photometric + sky loss -> backward -> FusedAdam over the Gaussians and
    the cube map, with sky_composite and with the fp32 torch restatement of the sky."""
    Hs, Ws, R = 320, 480, 128
    sc = synthetic.make_scene(P=20000, width=Ws, height=Hs, sh_degree=3, seed=4, n_vehicles=2, per_vehicle=2000, with_raw=True, scale_med=0.05)
    raw, cam = sc["raw"], sc["cam"]
    st = sgb.GaussianRasterizationSettings(image_height=Hs, image_width=Ws, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=DEV),
                                           scale_modifier=1.0, viewmatrix=cam["viewmatrix"].to(DEV), projmatrix=cam["projmatrix"].to(DEV),
                                           sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    fx, fy = Ws / (2 * cam["tanfovx"]), Hs / (2 * cam["tanfovy"])
    K = torch.tensor([[fx, 0, Ws / 2], [0, fy, Hs / 2], [0, 0, 1.0]], device=DEV)
    w2c = cam["viewmatrix"].to(DEV).T.contiguous()
    g = torch.Generator(device=DEV).manual_seed(9)
    gt = torch.rand(3, Hs, Ws, generator=g, device=DEV)
    sky_mask = torch.rand(1, Hs, Ws, generator=g, device=DEV) < 0.3
    loss_mask = sky_mask.clone()
    loss_mask[:, :50] = True  # the reference's sky loss sees the rows 0-49 SkyCubeMap.forward set in place
    cube0 = 0.999 * torch.ones(6, R, R, 3, device=DEV) + 0.2 * torch.rand(6, R, R, 3, generator=g, device=DEV) - 0.1
    affine = (torch.eye(4, device=DEV)[:3] + 0.05 * torch.randn(3, 4, generator=g, device=DEV))
    rast = sgb.GaussianRasterizer(st)

    def step(impl):
        models = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in raw["models"]]
        cube = torch.nn.Parameter(cube0.clone())
        xyz, rot, scale, opac, sh = sgb.compose(models, raw["poses"].to(DEV), raw["idft"].to(DEV))
        m2d = torch.zeros_like(xyz, requires_grad=True)
        res = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot)
        rgb, acc = res[0], res[3]
        seen = {}
        if impl == "sgr":
            out = sgb.sky_composite(rgb, acc, cube, K, w2c, sky_mask=sky_mask)
        else:
            out = SO.composite(rgb, acc, cube, K, w2c, sky_mask, None, None, 1.0)
        out.register_hook(lambda gr: seen.setdefault("g", gr.detach().clone()))
        col = sgb.color_correct(out, affine)
        loss = losses.photometric_loss(col, gt, None, 1.0, 0.2) + losses.sky_loss(acc, loss_mask, 1.0)
        loss.backward()
        grads = [v.grad.clone() for m in models for v in m.values()]
        params = [v for m in models for v in m.values()]
        opt = FusedAdam([{"params": params, "lr": 1e-3}, {"params": [cube], "lr": 0.01, "eps": 1e-15}], eps=1e-15)
        opt.step()
        return dict(out=out.detach(), rgb=rgb.detach(), acc=acc.detach(), g=seen["g"], grads=grads, dcube=cube.grad.clone(), cube=cube.detach().clone())

    a, b = step("sgr"), step("torch")
    assert torch.equal(a["rgb"], b["rgb"]) and torch.equal(a["acc"], b["acc"])
    assert float((a["out"] - b["out"]).abs().max()) < 1e-4
    for k, (x, y) in enumerate(zip(a["grads"], b["grads"])):
        assert rel(x.cpu().numpy(), y.cpu().numpy()) < 1e-3, k
    r = SO.sky64(a["rgb"], a["acc"], cube0, K, w2c, a["g"], sky_mask, None, None, 1.0)
    check(a["dcube"], r["dcube"], r["b_dcube"], "dcube in the step")
    # Adam's first step with eps = 1e-15 moves a texel by lr against the sign of its gradient (to the fp32 rounding of the bias
    # corrections, ~1e-4 relative): wherever the oracle's gradient is farther from zero than its bound, the update is the oracle's
    sure = r["dcube"].abs() > r["b_dcube"]
    step_ = (a["cube"] - cube0).to(F64)
    assert int(sure.sum()) > 1000
    assert bool((torch.sign(step_[sure]) == -torch.sign(r["dcube"][sure])).all())
    assert float((step_[sure].abs() - 0.01).abs().max()) < 1e-5
