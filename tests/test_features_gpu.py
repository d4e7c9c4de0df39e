"""GPU: the feature operations (gaussian_normals, compose_semantics, finish_features) against the reference's own outputs and gradients
(tests/golden/callsite/features.npz), element by element against the float64 restatement of tests/feature_oracle.py at several sizes,
at their edges (tied scales, a dot product of exactly 0 and near it, a Gaussian at the camera centre, a zero normal, a zero
probability sum), chained through compose down to the raw parameters, poses and pose correction, end to end through the rasterizer
against the reference's torch lines, under CUDA-graph capture, without host synchronisation and bit for bit on repeated backwards."""
import pytest
import torch

import feature_oracle as FO
import street_gaussians_b200 as sgb
from street_gaussians_b200 import synthetic
from test_compose_cpu import rel
from test_features_cpu import MODES, fixture, semantic_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
RAW = ("xyz", "rotation", "scaling", "opacity", "features_dc", "features_rest")


def within(got, ref, bound, what):
    err = (got.to(F64) - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        idx = bad.nonzero()[:8].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside their bound, worst {float((err / bound)[bad].max()):.3g}x at {idx}")


def rowscale(t):
    return t.abs().amax(dim=tuple(range(1, t.dim())), keepdim=True) if t.dim() > 1 else t.abs()


# ---- against the reference ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", MODES)
def test_semantics_vs_reference_fixture(mode):
    z = fixture()
    bg, actors, labels = semantic_inputs(z)
    models = [dict(semantic=t.to(DEV).requires_grad_(True)) for t in [bg] + actors]
    out = sgb.compose_semantics(models, labels, mode)
    out.backward(z[f"sem_{mode}_g"].to(DEV))
    assert rel(out.detach().cpu().numpy(), z[f"sem_{mode}_out"].numpy()) < 2e-6
    for k, m in enumerate(models):
        assert rel(m["semantic"].grad.cpu().numpy(), z[f"sem_{mode}_grad_{k}"].numpy()) < 3e-5, k


def test_normals_vs_reference_fixture():
    z = fixture()
    bg = {k: z[f"bg_{k}"].to(DEV).requires_grad_(True) for k in RAW}
    xyz, rot, scale, _, _ = sgb.compose([bg])
    n = sgb.gaussian_normals(xyz, rot, scale, z["camera_center"].to(DEV))
    n.backward(z["normals_g"].to(DEV))
    assert rel(n.detach().cpu().numpy(), z["normals_out"].numpy()) < 2e-6
    assert rel(bg["rotation"].grad.cpu().numpy(), z["normals_grad_rotation"].numpy()) < 3e-5
    assert all(bg[k].grad is None or not bool(bg[k].grad.any()) for k in RAW if k != "rotation")


@pytest.mark.parametrize("mode", MODES)
def test_finishing_vs_render_kernel_fixture(mode):
    z = fixture()
    x = z[f"rk_{mode}_feature"].to(DEV).requires_grad_(True)
    n, s = sgb.finish_features(x, 3, mode)
    ((n * z[f"rk_{mode}_gn"].to(DEV)).sum() + (s * z[f"rk_{mode}_gs"].to(DEV)).sum()).backward()
    assert rel(n.detach().cpu().numpy(), z[f"rk_{mode}_normals"].numpy()) < 2e-6
    assert rel(s.detach().cpu().numpy(), z[f"rk_{mode}_semantic"].numpy()) < 2e-6
    assert rel(x.grad.cpu().numpy(), z[f"rk_{mode}_g_feature"].numpy()) < 3e-5


# ---- normals against float64 ----------------------------------------------------------------------------------------------------

def _normal_rows(P, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    means = torch.randn(P, 3, generator=g, device=DEV) * 10
    rot = torch.randn(P, 4, generator=g, device=DEV)
    scales = torch.exp(torch.randn(P, 3, generator=g, device=DEV))
    centre = torch.randn(3, generator=g, device=DEV)
    up = torch.randn(P, 3, generator=g, device=DEV)
    return means, rot, scales, centre, up


def _run_normals(means, rot, scales, centre, up):
    r = rot.clone().requires_grad_(True)
    n = sgb.gaussian_normals(means, r, scales, centre)
    n.backward(up)
    return n.detach(), r.grad


def _decisions_of(n, rot):
    """The column and the sign a float32 normal took: the candidate +-R[:, c] nearest to it."""
    R = FO.quaternion_to_matrix(rot.to(F64))
    cand = torch.stack([R[:, :, c] for c in range(3)] + [-R[:, :, c] for c in range(3)], 1)  # [P, 6, 3]
    k = (cand - n.to(F64)[:, None]).abs().amax(-1).argmin(1)
    return k % 3, k >= 3


def check_normals(means, rot, scales, centre, up, n, grot, strict=True):
    col, flip = _decisions_of(n, rot)
    o = FO.normals64(means.to(F64), rot.to(F64), scales.to(F64), centre.to(F64))
    if strict:  # where the float64 decision is clear, the kernel took it
        s = scales.to(F64).sort(1).values
        clear = ((s[:, 1] - s[:, 0]) > 1e-6 * s[:, 1]) & (o["dot"].abs() > 1e-5)
        assert bool((col[clear] == o["col"][clear]).all()) and bool((flip[clear] == o["flip"][clear]).all())
    (ref,), (g,) = FO.grads(lambda r: FO.normals64(means.to(F64), r, scales.to(F64), centre.to(F64), col, flip)["n"], [rot], [up])
    within(n, ref, 1e-6 * torch.ones_like(ref), "normals")  # unit-length entries through ~10 fp32 roundings
    scale = (up.to(F64).norm(dim=1, keepdim=True) / rot.to(F64).norm(dim=1, keepdim=True))
    within(grot, g, 4e-6 * scale + 1e-6 * g.abs(), "dL/drotations")


@pytest.mark.parametrize("P", [1, 1000, 200003])
def test_normals_per_element_vs_float64(P):
    means, rot, scales, centre, up = _normal_rows(P, P)
    n, grot = _run_normals(means, rot, scales, centre, up)
    check_normals(means, rot, scales, centre, up, n, grot)


def test_tied_scales_take_the_lowest_index():
    P = 12
    means, rot, _, centre, up = _normal_rows(P, 5)
    s = torch.tensor([[1.0, 1.0, 2.0], [2.0, 1.0, 1.0], [1.0, 2.0, 1.0], [0.5, 0.5, 0.5]] * 3, device=DEV)
    n, grot = _run_normals(means, rot, s, centre, up)
    col, _ = _decisions_of(n, rot)
    assert col.tolist() == [0, 1, 0, 0] * 3
    check_normals(means, rot, s, centre, up, n, grot, strict=False)


def test_zero_dot_keeps_n_and_camera_centre_takes_minus_n():
    rot = torch.tensor([[1.0, 0.0, 0.0, 0.0]] * 3, device=DEV)
    scales = torch.tensor([[0.1, 1.0, 1.0]] * 3, device=DEV)  # column 0: n = (1, 0, 0)
    centre = torch.tensor([1.0, 2.0, -1.0], device=DEV)
    means = centre + torch.tensor([[0.0, 3.0, 4.0], [0.0, 0.0, 0.0], [-2.0, 0.0, 0.0]], device=DEV)
    up = torch.randn(3, 3, device=DEV)
    n, grot = _run_normals(means, rot, scales, centre, up)
    assert n.tolist() == [[1.0, 0.0, 0.0], [-1.0, -0.0, -0.0], [1.0, 0.0, 0.0]]
    ref = FO.normals64(means, rot, scales, centre)["n"]  # torch's own lines in float32 take the same decisions
    assert torch.equal(n, ref)
    check_normals(means, rot, scales, centre, up, n, grot, strict=False)


def test_backward_follows_forward_sign_near_zero_dot():
    P = 4096
    g = torch.Generator(device=DEV).manual_seed(17)
    rot = torch.randn(P, 4, generator=g, device=DEV)
    scales = torch.exp(torch.randn(P, 3, generator=g, device=DEV))
    centre = torch.randn(3, generator=g, device=DEV)
    # put each Gaussian on the plane through the camera centre perpendicular to its normal, then nudge it by ~1e-7 either way
    n0 = FO.normals64(torch.zeros(P, 3, device=DEV), rot, scales, torch.ones(3, device=DEV))
    R = FO.quaternion_to_matrix(rot)
    nn = R[torch.arange(P, device=DEV), :, n0["col"]]
    a = torch.randn(P, 3, generator=g, device=DEV)
    t = torch.linalg.cross(nn, a)
    t = t / t.norm(dim=1, keepdim=True)
    eps = (torch.rand(P, 1, generator=g, device=DEV) - 0.5) * 4e-7
    means = centre + 5 * t + eps * nn
    up = torch.randn(P, 3, generator=g, device=DEV)
    n, grot = _run_normals(means, rot, scales, centre, up)
    o = FO.normals64(means.to(F64), rot.to(F64), scales.to(F64), centre.to(F64))
    assert float(o["dot"].abs().max()) < 1e-5
    _, flip = _decisions_of(n, rot)
    assert 0 < int(flip.sum()) < P  # both signs occur
    check_normals(means, rot, scales, centre, up, n, grot, strict=False)  # every row's gradient takes its forward sign


# ---- semantics against float64 --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", [1, 8, 29])
@pytest.mark.parametrize("mode", MODES)
def test_semantics_per_element_vs_float64(K, mode):
    g = torch.Generator(device=DEV).manual_seed(K)
    counts = [700, 0, 33, 1] + [5 + 3 * a for a in range(36)]  # more actors than one launch takes, one without rows
    labels = [(7 * a + 3) % K for a in range(len(counts))]
    bg = torch.randn(50001, K, generator=g, device=DEV) * 3
    actors = [torch.randn(c, 1, generator=g, device=DEV) * 3 for c in counts]
    models = [dict(semantic=t.clone().requires_grad_(True)) for t in [bg] + actors]
    out = sgb.compose_semantics(models, labels, mode)
    up = torch.randn(out.shape, generator=g, device=DEV)
    out.backward(up)
    (ref,), gs = FO.grads(lambda b, *a: FO.semantics64(b, a, labels, mode), [bg] + actors, [up])
    within(out.detach(), ref, 2e-6 * ref.abs() + 1e-7 * rowscale(ref), "semantics")
    # logits: exact copies and gathers; probabilities: y (g - sum g y) and g (1 - y) y, whose fp32 sums err by a few ulp of max |g|
    gmax = float(up.abs().max())
    weight = [ref[:bg.shape[0]]] + [torch.full_like(gr, 0.25) for gr in gs[1:]]
    for k, (m, gr, w) in enumerate(zip(models, gs, weight)):
        bound = 1e-6 * gr.abs() + (1e-5 * gmax * w if mode == "probabilities" else 0.0) + 1e-30
        within(m["semantic"].grad, gr, bound, f"dL/d_semantic of model {k}")
    if mode == "logits":
        assert torch.equal(out[:bg.shape[0]].detach(), bg) and torch.equal(models[0]["semantic"].grad, up[:bg.shape[0]])


# ---- finishing against float64 --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("H,W", [(1, 1), (37, 53), (1280, 1920)])
@pytest.mark.parametrize("nc,K", [(3, 0), (3, 8), (0, 1), (3, 29)])
@pytest.mark.parametrize("mode", MODES)
def test_finishing_per_element_vs_float64(H, W, nc, K, mode):
    g = torch.Generator(device=DEV).manual_seed(H + K)
    x = torch.cat([torch.randn(nc, H, W, generator=g, device=DEV), torch.rand(K, H, W, generator=g, device=DEV)])
    if H * W > 2:
        x[:nc, 0, 0] = 0.0        # a pixel whose normal is exactly 0
        x[nc:, 0, 1] = 0.0        # a pixel whose probabilities sum to 0
    gn = torch.randn(nc, H, W, generator=g, device=DEV)
    gsem = torch.randn(K, H, W, generator=g, device=DEV)
    xx = x.clone().requires_grad_(True)
    n, s = sgb.finish_features(xx, nc, mode)
    assert (n is None) == (nc == 0) and (s is None) == (K == 0)
    loss = (n * gn).sum() if n is not None else 0
    loss = loss + ((s * gsem).sum() if s is not None else 0)
    loss.backward()
    (rn, rs), (rg,) = FO.grads(lambda v: FO.finish64(v, nc, mode), [x], [gn, gsem])
    if nc:
        within(n.detach(), rn, 4e-7 * (rn.abs() + 1e-30) + 1e-7, "normals")
    if K:
        within(s.detach(), rs, 1e-6 * rs.abs() + 1e-6, "semantic")
        if mode == "logits":
            assert torch.equal(s.detach(), x[nc:])
    # fp32 cancels in g - y (g . y) and in h - sum h p: each channel is held to a few ulp of its terms' size, per pixel
    x64 = x.to(F64)
    bound = [2e-5 * rg.abs()]
    if nc:
        d = x64[:nc].norm(dim=0).clamp_min(1e-12)
        bound[0][:nc] += 4e-6 * gn.to(F64).norm(dim=0) / d
    if K and mode == "probabilities":
        t = x64[nc:].sum(0) + 1e-8
        h = gsem.to(F64).abs() / (x64[nc:] / t + 1e-8)
        bound[0][nc:] += 2e-6 * K * h.amax(0) / t
    within(xx.grad, rg, bound[0], "dL/drendered")


# ---- chained through compose, and end to end ------------------------------------------------------------------------------------

def _scene(P=60000, Hs=256, Ws=384, seed=4):
    sc = synthetic.make_scene(P=P, width=Ws, height=Hs, sh_degree=3, seed=seed, n_vehicles=3, per_vehicle=3000, with_raw=True, scale_med=0.05)
    raw, cam = sc["raw"], sc["cam"]
    n_act = len(raw["models"]) - 1
    g = torch.Generator().manual_seed(seed)
    flip = torch.rand(sum(int(m["xyz"].shape[0]) for m in raw["models"][1:]), generator=g) < 0.5
    flip_quat = torch.tensor([0.0, 0.0, 1.0, 0.0])
    corr = (torch.nn.functional.normalize(torch.tensor([1.0, 0.02, -0.03, 0.01]), dim=0), torch.tensor([0.05, -0.02, 0.1]))
    return raw, cam, n_act, flip, flip_quat, corr


def _models(raw, K, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for k, m in enumerate(raw["models"]):
        d = {key: v.clone().to(DEV).requires_grad_(True) for key, v in m.items()}
        d["semantic"] = (torch.randn(int(m["xyz"].shape[0]), K if k == 0 else 1, generator=g) * 2).to(DEV).requires_grad_(True)
        out.append(d)
    return out


def test_normals_gradients_chain_through_compose_to_raw_poses_and_correction():
    raw, cam, n_act, flip, flip_quat, corr = _scene()
    models = _models(raw, 4, 1)
    poses = raw["poses"].to(DEV).requires_grad_(True)
    cr, ct = (t.to(DEV).requires_grad_(True) for t in corr)
    centre = cam["campos"].to(DEV)

    def run(impl):
        for m in models:
            for v in m.values():
                v.grad = None
        poses.grad = cr.grad = ct.grad = None
        xyz, rot, scale, _, _ = sgb.compose(models, poses, raw["idft"].to(DEV), flip.to(DEV), flip_quat.to(DEV), pose_correction=(cr, ct))
        up = torch.randn(xyz.shape, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
        if impl == "sgr":
            n = sgb.gaussian_normals(xyz, rot, scale, centre)
            n.backward(up)
            return n.detach(), rot.detach(), xyz.detach(), scale.detach(), up
        r = rot.detach()
        col, fl = _decisions_of(n_sgr, r)
        (_,), (g64,) = FO.grads(lambda q: FO.normals64(xyz.detach().to(F64), q, scale.detach().to(F64), centre.to(F64), col, fl)["n"], [r], [up])
        rot.backward(g64.float())
        return None

    n_sgr, rot, xyz, scale, up = run("sgr")
    collect = lambda: [m["rotation"].grad.clone() for m in models] + [poses.grad.clone(), cr.grad.clone(), ct.grad.clone()]
    ours = collect()
    check_normals(xyz, rot, scale, centre, up, n_sgr, _grot_of(xyz, rot, scale, centre, up))
    run("oracle")
    theirs = collect()
    for k, (a, b) in enumerate(zip(ours, theirs)):  # the raw rotations of every model, the poses and the correction
        assert rel(a.cpu().numpy(), b.cpu().numpy()) < 3e-5, k
    assert all(bool(a.abs().max() > 0) for a in ours[:-1])
    assert not bool(ours[-1].any()) and not bool(theirs[-1].any())  # the correction's translation moves no normal


def _grot_of(xyz, rot, scale, centre, up):
    r = rot.clone().requires_grad_(True)
    sgb.gaussian_normals(xyz, r, scale, centre).backward(up)
    return r.grad


@pytest.mark.parametrize("mode", MODES)
def test_end_to_end_against_reference_torch_lines(mode):
    """compose -> gaussian_normals + compose_semantics -> GaussianRasterizer (S = 3 + K) -> finish_features -> loss -> backward, against
    the same pipeline with the reference's torch lines for the feature steps (the actors' normals with torch.nn.functional spelt right)."""
    K = 19
    Hs, Ws = 256, 384
    raw, cam, n_act, flip, flip_quat, corr = _scene(Hs=Hs, Ws=Ws)
    labels = [(5 * a + 2) % K for a in range(n_act)]
    st = sgb.GaussianRasterizationSettings(image_height=Hs, image_width=Ws, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=DEV),
                                           scale_modifier=1.0, viewmatrix=cam["viewmatrix"].to(DEV), projmatrix=cam["projmatrix"].to(DEV),
                                           sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    rast = sgb.GaussianRasterizer(st)
    centre = cam["campos"].to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(8)
    gt_n = torch.randn(3, Hs, Ws, generator=gen, device=DEV)
    gt_s = torch.randn(K, Hs, Ws, generator=gen, device=DEV)

    def step(impl):
        models = _models(raw, K, 2)
        poses = raw["poses"].to(DEV).requires_grad_(True)
        xyz, rot, scale, opac, sh = sgb.compose(models, poses, raw["idft"].to(DEV), flip.to(DEV), flip_quat.to(DEV),
                                                pose_correction=tuple(t.to(DEV) for t in corr))
        if impl == "sgr":
            normals = sgb.gaussian_normals(xyz, rot, scale, centre)
            sem = sgb.compose_semantics(models, labels, mode)
        else:
            normals = FO.normals64(xyz, rot, scale, centre)["n"]
            sem = FO.semantics64(models[0]["semantic"], [m["semantic"] for m in models[1:]], labels, mode)
        feat = torch.cat([normals, sem], -1)
        m2d = torch.zeros_like(xyz, requires_grad=True)
        res = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot, semantics=feat)
        rendered = res[4]
        if impl == "sgr":
            n_img, s_img = sgb.finish_features(rendered, 3, mode)
        else:
            n_img, s_img = FO.finish64(rendered, 3, mode)
        loss = (n_img * gt_n).mean() + (s_img * gt_s).mean() + res[0].mean()
        loss.backward()
        grads = [v.grad.clone() for m in models for v in m.values() if v.grad is not None] + [poses.grad.clone()]
        return dict(n=n_img.detach(), s=s_img.detach(), rendered=rendered.detach(), grads=grads)

    a, b = step("sgr"), step("torch")
    assert a["rendered"].shape == (3 + K, Hs, Ws)
    assert float((a["rendered"] - b["rendered"]).abs().max()) < 1e-4
    assert float((a["n"] - b["n"]).abs().max()) < 1e-4 * max(1.0, float(b["n"].abs().max()))
    fin = torch.isfinite(b["s"])
    assert bool(fin.all())
    assert float((a["s"] - b["s"]).abs().max()) < 1e-4 * max(1.0, float(b["s"].abs().max()))
    assert len(a["grads"]) == len(b["grads"])
    for k, (x, y) in enumerate(zip(a["grads"], b["grads"])):
        assert rel(x.cpu().numpy(), y.cpu().numpy()) < 1e-3, k


# ---- graphs, host synchronisation and determinism -------------------------------------------------------------------------------

def _capture_matches_eager(step, leaves):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for x in leaves:
                x.grad = None
            eager = step()
    torch.cuda.current_stream().wait_stream(s)
    eager_grads = [x.grad.clone() for x in leaves]
    for _ in range(2):  # repeated backwards agree bit for bit
        for x in leaves:
            x.grad = None
        again = step()
        assert torch.equal(again, eager) and all(torch.equal(x.grad, e) for x, e in zip(leaves, eager_grads))
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
        assert torch.equal(x.grad, e)


def test_normals_capture_sync_free_and_deterministic():
    means, rot, scales, centre, up = _normal_rows(100003, 9)
    r = rot.clone().requires_grad_(True)

    def step():
        n = sgb.gaussian_normals(means, r, scales, centre)
        n.backward(up)
        return n.detach()

    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _capture_matches_eager(step, [r])


@pytest.mark.parametrize("mode", MODES)
def test_semantics_capture_sync_free_and_deterministic(mode):
    g = torch.Generator(device=DEV).manual_seed(11)
    leaves = [torch.randn(20000, 8, generator=g, device=DEV).requires_grad_(True)] + [torch.randn(c, 1, generator=g, device=DEV).requires_grad_(True)
                                                                                       for c in (300, 7, 1200)]
    up = torch.randn(20000 + 1507, 8, generator=g, device=DEV)

    def step():
        out = sgb.compose_semantics([dict(semantic=t) for t in leaves], [1, 7, 0], mode)
        out.backward(up)
        return out.detach()

    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _capture_matches_eager(step, leaves)


@pytest.mark.parametrize("mode", MODES)
def test_finishing_capture_sync_free_and_deterministic(mode):
    g = torch.Generator(device=DEV).manual_seed(12)
    x = torch.rand(3 + 8, 320, 480, generator=g, device=DEV).requires_grad_(True)
    gn, gs = torch.randn(3, 320, 480, generator=g, device=DEV), torch.randn(8, 320, 480, generator=g, device=DEV)

    def step():
        n, s = sgb.finish_features(x, 3, mode)
        ((n * gn).sum() + (s * gs).sum()).backward()
        return torch.cat([n.detach(), s.detach()])

    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _capture_matches_eager(step, [x])
