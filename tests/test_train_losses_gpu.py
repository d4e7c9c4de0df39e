"""GPU: sgr_lidar_depth_loss / sgr_obj_acc_loss through losses.lidar_depth_loss / losses.obj_acc_loss, against the reference's own
train.py lines (tests/golden/callsite/train_losses.npz), the torch restatement run on the GPU (tests/train_loss_oracle.py), under
CUDA-graph capture, and end to end through the rasterizer's backward."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_train_loss_golden import case  # noqa: E402
import street_gaussians_b200 as sgb  # noqa: E402
import train_loss_oracle as TO  # noqa: E402
import util  # noqa: E402
from oracle import loss_oracle as LO  # noqa: E402
from street_gaussians_b200 import _capi, losses, synthetic  # noqa: E402
from test_losses_cpu import rel  # noqa: E402
from test_train_losses_cpu import TRAIN_FIX  # noqa: E402

pytestmark = pytest.mark.gpu


def _lidar_both(depth0, acc0, lidar, mask, weight=1.0, keep=0.95, g_out=1.0):
    """(value, dL/ddepth, dL/dacc) of the fused call and of the torch restatement, with upstream gradient g_out."""
    res = []
    for fn in (losses.lidar_depth_loss, TO.lidar_depth_loss):
        d, a = depth0.clone().requires_grad_(True), acc0.clone().requires_grad_(True)
        v = fn(d, a, lidar, mask, weight=weight, keep=keep)
        (g_out * v).backward()
        res.append((float(v.detach()), d.grad, a.grad))
    return res


def _err(depth, acc, lidar):
    return (depth / (acc + 1e-10) - lidar).abs()


def test_lidar_and_obj_loss_vs_reference_fixture():
    z = np.load(TRAIN_FIX)
    for seed in (0, 1):
        c = {k: v.cuda() for k, v in case(seed).items()}
        k = f"s{seed}_"
        d, a = c["depth"].clone().requires_grad_(True), c["acc"].clone().requires_grad_(True)
        v = losses.lidar_depth_loss(d, a, c["lidar_depth"], c["mask"])
        v.backward()
        v = v.detach()
        ref = float(z[k + "lidar"])
        assert abs(float(v) - ref) <= 2e-6 * abs(ref), (k, float(v), ref)
        assert rel(d.grad.cpu().numpy(), z[k + "g_depth"]) <= 1e-5 and rel(a.grad.cpu().numpy(), z[k + "g_acc"]) <= 1e-5, k
        a = c["acc_obj"].clone().requires_grad_(True)
        v = losses.obj_acc_loss(a, c["obj_bound"])
        v.backward()
        v = v.detach()
        ref = float(z[k + "obj"])
        assert abs(float(v) - ref) <= 2e-6 * abs(ref), (k, float(v), ref)
        assert rel(a.grad.cpu().numpy(), z[k + "g_acc_obj"]) <= 1e-5, k


def _lidar_inputs(H, W, density, seed):
    g = torch.Generator().manual_seed(seed)
    acc = torch.rand(1, H, W, generator=g)
    acc[torch.rand(1, H, W, generator=g) < 0.02] = 0.0
    z = 2.0 + 78.0 * torch.rand(1, H, W, generator=g)
    depth = acc * z * (1.0 + 0.01 * torch.randn(1, H, W, generator=g))
    lidar = torch.where(torch.rand(1, H, W, generator=g) < density, z + 0.5 * torch.randn(1, H, W, generator=g), torch.zeros_like(z))
    lidar[torch.rand(1, H, W, generator=g) < 0.03] += 30.0  # outliers the trimming removes
    mask = torch.rand(1, H, W, generator=g) > 0.25
    return depth.cuda(), acc.cuda(), lidar.clamp_min(0.0).cuda(), mask.cuda()


@pytest.mark.parametrize("H,W", [(1280, 1920), (37, 16), (16, 5)])
@pytest.mark.parametrize("density", [0.05, 1.0])
def test_lidar_depth_loss_vs_oracle(H, W, density):
    depth, acc, lidar, mask = _lidar_inputs(H, W, density, seed=H * 7 + W + int(density * 100))
    for m in (None, mask):
        (va, gda, gaa), (vb, gdb, gab) = _lidar_both(depth, acc, lidar, m, weight=0.1, g_out=2.5)
        assert abs(va - vb) <= 2e-6 * abs(vb), (va, vb)
        # pixels whose error equals the k-th smallest may be picked differently by torch.topk; compare the others
        valid = (lidar > 0) & m if m is not None else lidar > 0
        err = _err(depth, acc, lidar)
        k = int(0.95 * int(valid.sum()))
        t = torch.sort(err[valid]).values[k - 1]
        off = ~(valid & (err == t))
        assert rel(gda[off].cpu().numpy(), gdb[off].cpu().numpy()) <= 1e-5 and rel(gaa[off].cpu().numpy(), gab[off].cpu().numpy()) <= 1e-5
        assert int((gda != 0).sum()) == int((gdb != 0).sum())


def test_lidar_depth_loss_ties_take_the_lowest_indices():
    """Quantised errors: hundreds of pixels share the k-th smallest value."""
    H, W = 300, 401
    g = torch.Generator().manual_seed(11)
    depth = torch.randint(5, 60, (1, H, W), generator=g).float()  # acc = 1: e == depth exactly
    acc = torch.ones(1, H, W)
    q = torch.randint(-12, 13, (1, H, W), generator=g).float() * 0.25  # |e - lidar| in multiples of 1/4
    lidar = torch.where(torch.rand(1, H, W, generator=g) < 0.4, depth + q, torch.zeros_like(depth))
    mask = torch.rand(1, H, W, generator=g) > 0.1
    depth, acc, lidar, mask = depth.cuda(), acc.cuda(), lidar.cuda(), mask.cuda()
    (va, gda, gaa), (vb, gdb, gab) = _lidar_both(depth, acc, lidar, mask)
    assert abs(va - vb) <= 2e-6 * abs(vb)
    valid = (lidar > 0) & mask
    err = _err(depth, acc, lidar)
    e_valid = err[valid]
    k = int(0.95 * e_valid.numel())
    t = torch.sort(e_valid).values[k - 1]
    tie = valid & (err == t)
    lt = int((e_valid < t).sum())
    assert t > 0 and int(tie.sum()) > 100 and int(tie.sum()) > k - lt
    off = ~tie
    assert rel(gda[off].cpu().numpy(), gdb[off].cpu().numpy()) <= 1e-6
    assert rel(gaa[off].cpu().numpy(), gab[off].cpu().numpy()) <= 1e-6
    picked = tie & (gda != 0)
    assert int(picked.sum()) == k - lt
    tie_idx = torch.nonzero(tie.reshape(-1)).reshape(-1)
    assert torch.equal(torch.nonzero(picked.reshape(-1)).reshape(-1), tie_idx[: k - lt])


def test_lidar_depth_loss_edge_cases():
    H, W = 40, 50
    depth, acc, lidar, mask = _lidar_inputs(H, W, 0.5, seed=5)
    for n in (0, 1):  # k = int(0.95 n) = 0: NaN value and all-zero gradients, as the reference
        ld = torch.zeros_like(lidar)
        if n:
            ld[0, 3, 7] = 12.0
        (va, gda, gaa), (vb, _, _) = _lidar_both(depth, acc, ld, None)
        assert np.isnan(va) and np.isnan(vb)
        assert int((gda != 0).sum()) == 0 and int((gaa != 0).sum()) == 0
    # keep = 1.0: every valid pixel, outliers included
    (va, gda, gaa), (vb, gdb, gab) = _lidar_both(depth, acc, lidar, mask, keep=1.0)
    assert abs(va - vb) <= 2e-6 * abs(vb) and rel(gda.cpu().numpy(), gdb.cpu().numpy()) <= 1e-5
    assert rel(gaa.cpu().numpy(), gab.cpu().numpy()) <= 1e-5
    # all errors equal: value = that error, the lowest-index k valid pixels carry the gradient
    dq = torch.randint(1, 50, (1, H, W), generator=torch.Generator().manual_seed(6)).float().cuda()  # acc = 1: e == depth exactly
    aq = torch.ones_like(acc)
    ld = torch.where(lidar > 0, dq + 2.0, torch.zeros_like(dq))
    (va, gda, _), (vb, _, _) = _lidar_both(dq, aq, ld, None)
    assert va == 2.0 and vb == 2.0
    valid = (ld > 0).reshape(-1)
    k = int(0.95 * int(valid.sum()))
    assert torch.equal(torch.nonzero(gda.reshape(-1) != 0).reshape(-1), torch.nonzero(valid).reshape(-1)[:k])
    # acc = 0 pixels: e = depth / 1e-10; keep = 1 makes them count
    a0 = acc.clone()
    a0[0, ::3, ::4] = 0.0
    (va, gda, gaa), (vb, gdb, gab) = _lidar_both(depth, a0, lidar, mask, keep=1.0)
    assert abs(va - vb) <= 2e-6 * abs(vb) and rel(gda.cpu().numpy(), gdb.cpu().numpy()) <= 1e-5
    assert rel(gaa.cpu().numpy(), gab.cpu().numpy()) <= 1e-5


def test_lidar_depth_loss_rejects_bad_arguments():
    depth, acc, lidar, mask = _lidar_inputs(8, 8, 0.5, seed=1)
    for keep in (0.0, 1.5, float("nan")):
        with pytest.raises(_capi.SgrError, match="keep"):
            losses.lidar_depth_loss(depth, acc, lidar, mask, keep=keep)
    with pytest.raises(ValueError):
        losses.lidar_depth_loss(depth, acc[..., :4], lidar, mask)


@pytest.mark.parametrize("H,W", [(1280, 1920), (37, 16), (16, 5)])
def test_obj_acc_loss_vs_oracle(H, W):
    g = torch.Generator().manual_seed(H + 3 * W)
    acc0 = (torch.rand(1, H, W, generator=g) ** 2).cuda()
    acc0[0, 0, :4] = torch.tensor([0.0, 1.0, 5e-7, 1.0 - 5e-7])[: min(4, W)].cuda()  # values the clamp catches: zero gradient there
    bound = (torch.rand(1, H, W, generator=g) > 0.5).cuda()
    x = acc0.clone().requires_grad_(True)
    a = losses.obj_acc_loss(x, bound, 0.1)
    (3.0 * a).backward()
    y = acc0.clone().requires_grad_(True)
    b = TO.obj_acc_loss(y, bound, 0.1)
    (3.0 * b).backward()
    assert abs(float(a) - float(b)) <= 1e-6 * abs(float(b)) and rel(x.grad.cpu().numpy(), y.grad.cpu().numpy()) <= 1e-5
    assert int((x.grad[0, 0, :min(4, W)] != 0).sum()) == 0


def test_fused_losses_capture_in_a_cuda_graph():
    """The four fused losses, forward and backward, captured once and replayed on new inputs: gradients bit-equal to an eager call."""
    H, W = 192, 256

    def inputs(seed):
        g = torch.Generator().manual_seed(seed)
        depth, acc, lidar, mask = _lidar_inputs(H, W, 0.3, seed)
        return dict(image=torch.rand(3, H, W, generator=g).cuda(), gt=torch.rand(3, H, W, generator=g).cuda(), mask=mask,
                    sky=(torch.rand(1, H, W, generator=g) > 0.7).cuda(), acc=acc, depth=depth, lidar=lidar,
                    acc_obj=torch.rand(1, H, W, generator=g).cuda(), obj_bound=(torch.rand(1, H, W, generator=g) > 0.5).cuda())

    def step(t):
        vals = [losses.photometric_loss(t["image"], t["gt"], t["mask"], 1.0, 0.2), losses.sky_loss(t["acc"], t["sky"], 0.05),
                losses.obj_acc_loss(t["acc_obj"], t["obj_bound"], 0.1), losses.lidar_depth_loss(t["depth"], t["acc"], t["lidar"], t["mask"], 0.1)]
        sum(vals).backward()
        return torch.stack(vals)

    leaves = ("image", "acc", "depth", "acc_obj")
    static = inputs(1)
    for k in leaves:
        static[k].requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for k in leaves:
                static[k].grad = None
            step(static)
    torch.cuda.current_stream().wait_stream(s)
    for k in leaves:
        static[k].grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        vals_g = step(static)
    for seed in (2, 3):
        new = inputs(seed)
        with torch.no_grad():
            for k, v in new.items():
                static[k].copy_(v)
        graph.replay()
        for k in leaves:
            new[k].requires_grad_(True)
        vals_e = step(new)
        torch.cuda.synchronize()
        assert torch.allclose(vals_g, vals_e, rtol=1e-6, atol=0.0), (vals_g, vals_e)
        for k in leaves:
            assert torch.equal(static[k].grad, new[k].grad), k


def test_end_to_end_default_loss_through_the_rasterizer():
    """The default training loss (L1 + SSIM, sky, object accumulation, LiDAR depth) of a rendered scene, backpropagated through the
    rasterizer once from the fused losses and once from the torch restatements: identical images, Gaussian gradients within 1e-3."""
    scene = synthetic.make_scene(P=20_000, width=320, height=208, sh_degree=3, seed=17, pose=True, scale_med=0.05)
    cam = scene["cam"]
    H, W = cam["image_height"], cam["image_width"]
    g = torch.Generator().manual_seed(17)
    gt = torch.rand(3, H, W, generator=g).cuda()
    mask = (torch.rand(1, H, W, generator=g) > 0.1).cuda()
    sky = (torch.rand(1, H, W, generator=g) > 0.8).cuda()
    obj_bound = torch.zeros(1, H, W, dtype=torch.bool)
    obj_bound[:, H // 4: H // 2, W // 3: 2 * W // 3] = True
    obj_bound = obj_bound.cuda()
    lidar_pick = torch.rand(1, H, W, generator=g) < 0.3
    noise = 1.0 + 0.05 * torch.randn(1, H, W, generator=g)
    n_obj = scene["means3D"].shape[0] // 5
    runs = []
    for fused in (True, False):
        st = util.settings_from(sgb, cam, "cuda")
        rast = sgb.GaussianRasterizer(st)
        leaf = {k: scene[k].cuda().clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        means2D = torch.zeros_like(leaf["means3D"], requires_grad=True)
        color, radii, depth, acc, _ = rast(means3D=leaf["means3D"], means2D=means2D, opacities=leaf["opacities"], shs=leaf["shs"],
                                           scales=leaf["scales"], rotations=leaf["rotations"])
        sl = slice(0, n_obj)  # the first fifth of the Gaussians plays the objects-only render (render_object)
        _, _, _, acc_obj, _ = rast(means3D=leaf["means3D"][sl], means2D=means2D[sl], opacities=leaf["opacities"][sl], shs=leaf["shs"][sl],
                                   scales=leaf["scales"][sl], rotations=leaf["rotations"][sl])
        with torch.no_grad():
            e = depth / (acc + 1e-10)
            lidar = torch.where(lidar_pick.cuda() & (acc > 0.3), e * noise.cuda(), torch.zeros_like(e))
        assert int((lidar > 0).sum()) > 1000
        if fused:
            loss = losses.photometric_loss(color, gt, mask, 1.0, 0.2) + 1.0 * losses.sky_loss(acc, sky) + \
                   losses.obj_acc_loss(acc_obj, obj_bound, 0.1) + losses.lidar_depth_loss(depth, acc, lidar, mask, 0.1)
        else:
            loss = LO.photometric_loss(color, gt, mask, 1.0, 0.2) + 1.0 * LO.sky_loss(acc, sky) + \
                   TO.obj_acc_loss(acc_obj, obj_bound, 0.1) + TO.lidar_depth_loss(depth, acc, lidar, mask, 0.1)
        loss.backward()
        runs.append(dict(loss=float(loss), color=color.detach(), depth=depth.detach(), acc=acc.detach(), acc_obj=acc_obj.detach(),
                         **{"g_" + k: v.grad for k, v in leaf.items()}, g_means2D=means2D.grad))
    a, b = runs
    for k in ("color", "depth", "acc", "acc_obj"):
        assert torch.equal(a[k], b[k]), k
    assert abs(a["loss"] - b["loss"]) <= 2e-6 * abs(b["loss"])
    for k in a:
        if k.startswith("g_"):
            assert util.rel_err(a[k].cpu().numpy(), b[k].cpu().numpy()) <= 1e-3, (k, util.rel_err(a[k].cpu().numpy(), b[k].cpu().numpy()))
