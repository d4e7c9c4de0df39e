"""GPU: the tracked actor poses (sgr_actor_pose_forward / _backward through street_gaussians_b200.ActorPose) against the reference's
own outputs (tests/golden/callsite/actor_pose.npz) and per element against the float64 restatement of tests/actor_pose_oracle.py,
on the fixture's cases and on random track tables with 0, 1, 8, 40 and 257 actors; bit-identical repeated backward, no host
synchronisation, CUDA-graph capture with compose, NaN / inf offsets, and a composed training step against the torch lines."""
import numpy as np
import pytest
import torch

import actor_pose_case as AC
import actor_pose_oracle as AO
import street_gaussians_b200 as sgb
import util
from oracle import compose_oracle as CO
from street_gaussians_b200 import losses, synthetic
from street_gaussians_b200.training import FusedAdam
from test_actor_pose_cpu import NAMES, NAN_GRAD_CASES, close, fixture, rel

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64


def make_pose(meta, opt_track=True, fourier_dim=5, fourier_scale=1.0):
    return sgb.ActorPose(meta["obj_tracklets"], meta["tracklet_timestamps"], meta["camera_timestamps"], meta["obj_meta"], opt_track=opt_track,
                         fourier_dim=fourier_dim, fourier_scale=fourier_scale, device=DEV)


def set_params(pose, ot, orr):
    with torch.no_grad():
        pose.opt_trans.copy_(torch.as_tensor(ot))
        pose.opt_rots.copy_(torch.as_tensor(orr))


def run(pose, vis, case, w=None, frame=None):
    for p in pose.parameters():
        p.grad = None
    ego = torch.as_tensor(AC.ego_pose(case["ego"]) if isinstance(case["ego"], str) else case["ego"]).to(DEV)
    poses, idft = pose(vis, timestamp=float(case["t"]), cam=case["cam"], is_val=case["is_val"], ego_pose=ego, frame=frame)
    if w is not None and pose.opt_track and len(vis):
        (poses * w).sum().backward()
    return poses.detach(), idft, ego


def check(got, val, bnd, what):
    err = (got.to(F64) - val).abs()
    bad = ~(err <= bnd)
    if bool(bad.any()):
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside their bound, worst {float((err / bnd)[bad].max()):.3g}x at "
                             f"{bad.nonzero()[:8].tolist()}")


@pytest.mark.parametrize("name", NAMES)
def test_vs_reference_fixture_and_float64(name):
    z, meta, T = fixture()
    case = AC.BY_NAME[name]
    pose = make_pose(meta, case["opt_track"], int(z["fourier_dim"]), float(z["fourier_scale"]))
    if case["opt_track"]:
        set_params(pose, z[f"params_{case['params']}_trans"], z[f"params_{case['params']}_rots"])
    vis = [int(v) for v in z[f"{name}_visible"]]
    w = torch.from_numpy(z[f"{name}_w"]).to(DEV)
    poses, idft, ego = run(pose, vis, case, w, frame=case["frame"])
    assert close(poses.cpu().numpy(), z[f"{name}_poses"], 1e-6)
    assert close(idft.cpu().numpy(), z[f"{name}_idft"], 1e-6)
    in_t, in_r = pose.input_trans, pose.input_rots
    if case["opt_track"]:
        assert rel(pose.opt_trans.grad.cpu().numpy(), z[f"{name}_dtrans"]) < 2e-5
        if name in NAN_GRAD_CASES:  # the reference's NaN; the kernel gives the small-angle branch's finite gradient
            assert torch.isfinite(pose.opt_rots.grad).all()
        else:
            assert rel(pose.opt_rots.grad.cpu().numpy(), z[f"{name}_drots"]) < 2e-5
    r = AO.bounds(T, vis, float(case["t"]), case["cam"], case["is_val"], ego, in_t, in_r, pose.opt_trans if case["opt_track"] else None,
                  pose.opt_rots if case["opt_track"] else None, w)
    check(poses, r["poses"], r["b_poses"], f"{name} poses")
    if case["opt_track"]:
        check(pose.opt_trans.grad, r["dtrans"], r["b_dtrans"], f"{name} dtrans")
        check(pose.opt_rots.grad, r["drots"], r["b_drots"], f"{name} drots")


def random_table(n_tracks, seed, F=24, K=None, at=10):
    """n_tracks tracks of 2-14 entries, each spanning frames `at` and `at` + 1 (where the camera looks, so every actor is visible, as
    parse_camera's actors are), on random free columns of a [F, K] table; non-uniform timestamps near 1.6e9 s; two cameras."""
    g = np.random.default_rng(seed)
    K = K or max(n_tracks, 1)
    ts = 1.6e9 + np.concatenate([[0.0], np.cumsum(g.uniform(0.08, 0.12, F - 1))])
    tr = np.zeros((F, K, 8), np.float32)
    tr[..., 0] = -1
    tr[..., 4] = 1
    free = [list(g.permutation(K)) for _ in range(F)]
    obj_meta = {}
    for k in range(n_tracks):
        tid = 1000 + 3 * k
        s, e = at - int(g.integers(0, 7)), at + 1 + int(g.integers(0, 7))
        frames = [f for f in range(s, e + 1) if free[f]]
        assert at in frames and at + 1 in frames, "table too small"
        for f in frames:
            q = g.standard_normal(4)
            q /= np.linalg.norm(q)
            tr[f, free[f].pop()] = [tid, *(g.standard_normal(3) * 20), *q]
        obj_meta[tid] = dict(start_frame=frames[0], end_frame=frames[-1], start_timestamp=float(ts[frames[0]]), end_timestamp=float(ts[frames[-1]]))
    cams = {0: dict(train_timestamps=list(ts[::2])), 1: dict(train_timestamps=list(ts[1::3]))}
    meta = dict(obj_tracklets=tr, tracklet_timestamps=ts, camera_timestamps=cams, obj_meta=obj_meta)
    ot = (0.2 * g.standard_normal((F, K, 3))).astype(np.float32)
    orr = (g.standard_normal((F, K, 1))).astype(np.float32)
    return meta, ot, orr, ts


@pytest.mark.parametrize("n", [0, 1, 8, 40, 257])
@pytest.mark.parametrize("is_val", [False, True], ids=["train", "val"])
def test_random_tables_vs_torch_lines_and_float64(n, is_val):
    meta, ot, orr, ts = random_table(max(n, 1), seed=n + 7 * is_val)
    pose = make_pose(meta)
    set_params(pose, ot, orr)
    T = AO.Table(meta["obj_tracklets"], ts, meta["camera_timestamps"], meta["obj_meta"])
    vis = list(meta["obj_meta"])[:n]
    g = np.random.default_rng(n)
    ego = np.eye(4, dtype=np.float32)
    ego[:3, :3] = AC._rot(g.standard_normal(3), 2.0)
    ego[:3, 3] = g.standard_normal(3) * 10
    case = dict(t=float(ts[10] + g.uniform(0.0, ts[11] - ts[10])), cam=1, is_val=is_val, ego=ego)
    w = torch.randn(n, 7, generator=torch.Generator().manual_seed(n)).to(DEV)
    poses, idft, egot = run(pose, vis, case, w, frame=5)
    assert poses.shape == (n, 7) and idft.shape == (n, 5)
    ot_, orr_ = pose.opt_trans.detach().clone().requires_grad_(True), pose.opt_rots.detach().clone().requires_grad_(True)
    ref = AO.poses(T, vis, case["t"], 1, is_val, egot, pose.input_trans, pose.input_rots, ot_, orr_, finite=True)
    if n:
        # rotations to 1e-6; translations to 1e-6 of the tracklet coordinates they interpolate (the validation path cancels terms)
        scale = max(1.0, float(pose.input_trans.abs().max()))
        assert close(poses[:, :4].cpu().numpy(), ref[:, :4].detach().cpu().numpy(), 1e-6)
        assert float((poses[:, 4:] - ref[:, 4:]).abs().max()) <= 1e-6 * scale
        (ref * w).sum().backward()
        assert rel(pose.opt_trans.grad.cpu().numpy(), ot_.grad.cpu().numpy()) < 2e-5
        assert rel(pose.opt_rots.grad.cpu().numpy(), orr_.grad.cpu().numpy()) < 2e-5
        r = AO.bounds(T, vis, case["t"], 1, is_val, egot, pose.input_trans, pose.input_rots, pose.opt_trans, pose.opt_rots, w)
        check(poses, r["poses"], r["b_poses"], "poses")
        check(pose.opt_trans.grad, r["dtrans"], r["b_dtrans"], "dtrans")
        check(pose.opt_rots.grad, r["drots"], r["b_drots"], "drots")
        # at most 4 rows per actor (8 on the validation path) receive gradient
        assert int((pose.opt_rots.grad != 0).sum()) <= (8 if is_val else 4) * n


def test_repeated_backward_is_bit_identical_and_sync_free():
    meta, ot, orr, ts = random_table(40, seed=3, K=48)  # theta2's row (frame_ind1, column_ind2) is often another actor's
    pose = make_pose(meta)
    set_params(pose, ot, orr)
    vis = list(meta["obj_meta"])
    case = dict(t=float(ts[10] + 0.01), cam=0, is_val=True, ego=torch.from_numpy(AC.ego_pose("b2")).to(DEV))
    w = torch.randn(40, 7, device=DEV)
    run(pose, vis, case, w)
    first = (pose.opt_trans.grad.clone(), pose.opt_rots.grad.clone())
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    again = []
    try:
        for _ in range(3):
            run(pose, vis, case, w, frame=3)
            again.append((pose.opt_trans.grad, pose.opt_rots.grad))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for gt_, gr_ in again:
        assert torch.equal(gt_, first[0]) and torch.equal(gr_, first[1])


def test_graph_capture_of_tracks_and_compose_replays_eager():
    sc = synthetic.make_scene(P=2000, width=64, height=48, sh_degree=1, seed=2, n_vehicles=3, per_vehicle=100, with_raw=True)
    models = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in sc["raw"]["models"]]
    meta, ot, orr, ts = random_table(3, seed=5)
    pose = make_pose(meta, fourier_dim=1)
    set_params(pose, ot, orr)
    vis = list(meta["obj_meta"])
    ego = torch.from_numpy(AC.ego_pose("b1")).to(DEV)
    g = torch.randn(2300, 3, device=DEV)

    def step():
        poses, idft = pose(vis, timestamp=float(ts[10] + 0.02), cam=0, is_val=False, ego_pose=ego, frame=10)
        xyz = sgb.compose(models, poses, idft)[0]
        gt_, gr_ = torch.autograd.grad((xyz * g).sum(), [pose.opt_trans, pose.opt_rots])
        return xyz.detach(), gt_, gr_

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            eager = step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured[0], eager[0])
    # dL/dposes comes from compose's backward, whose per-actor sums may take another order; the offsets' gradient follows it
    for x, y in zip(captured[1:], eager[1:]):
        assert rel(x.cpu().numpy(), y.cpu().numpy()) < 1e-5
    assert bool((captured[2] != 0).any())


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")], ids=["nan", "inf", "-inf"])
def test_non_finite_offsets_propagate_like_torch(bad):
    """A non-finite translation offset and a non-finite yaw offset on rows the camera actually reads: which pose elements and which
    gradient elements come out NaN / inf is torch's (the clamps of the slerp propagate NaN as torch.clamp does)."""
    z, meta, T = fixture()
    case = AC.BY_NAME["train_mid"]
    vis = [0, 2, 3]
    ot, orr = (x.copy() for x in AC.params()["seeded"])
    info = []
    AO.poses(T, [0], float(case["t"]), 0, False, torch.eye(4), torch.zeros(AC.F, AC.K, 3), torch.zeros(AC.F, AC.K, 4),
             torch.from_numpy(ot), torch.from_numpy(orr), info=info)
    first, _, theta2 = next(r[1:] for r in info if isinstance(r, tuple) and r[0] == "rows")
    assert first == (13, 1) and theta2 == (13, 0)  # track 0: entry (13, 1) first, theta2 read at (13, 0)
    ot[13, 1, 0] = bad    # trans1 of track 0
    orr[13, 1, 0] = bad   # theta1 of track 0 (and theta2 of track 2, whose first entry is (13, 0) and second on column 1)
    pose = make_pose(meta)
    set_params(pose, ot, orr)
    w = torch.from_numpy(z["train_mid_w"]).to(DEV)
    poses, _, ego = run(pose, vis, case, w)
    ot_ = torch.from_numpy(ot).to(DEV).requires_grad_(True)
    orr_ = torch.from_numpy(orr).to(DEV).requires_grad_(True)
    ref = AO.poses(T, vis, float(case["t"]), 0, False, ego, pose.input_trans, pose.input_rots, ot_, orr_, finite=True)
    (ref * w).sum().backward()
    for what, got, want in (("poses", poses, ref.detach()), ("dtrans", pose.opt_trans.grad, ot_.grad), ("drots", pose.opt_rots.grad, orr_.grad)):
        assert torch.equal(torch.isnan(got), torch.isnan(want)), what
        assert torch.equal(torch.isinf(got), torch.isinf(want)) and torch.equal(got[torch.isinf(got)], want[torch.isinf(want)]), what
        fin = torch.isfinite(want)
        assert close(got[fin].cpu().numpy(), want[fin].cpu().numpy(), 2e-5 if what != "poses" else 1e-6), what
    assert bool(torch.isnan(poses[0, :4]).all()) and bool(torch.isnan(pose.opt_rots.grad[13, 1]).all())
    assert not bool(torch.isfinite(poses[0, 4:]).all()) and bool(torch.isfinite(poses[2]).all())


def test_composed_step_matches_torch_lines():
    """tracks -> compose -> rasterize -> photometric_loss -> backward -> FusedAdam at config C's shape (1.5M + 8 x 50k, 1920 x 1280),
    with the fused poses and compose, and with the torch lines of both (tests/actor_pose_oracle.py, oracle/compose_oracle.py)."""
    sc = synthetic.make_config("C", seed=0, with_raw=True)
    raw, cam = sc["raw"], sc["cam"]
    H, W = cam["image_height"], cam["image_width"]
    # tracks that carry each vehicle's rotation, mostly in front of the background field (it starts 2 m out and saturates the
    # frame: vehicles behind it get no gradient), two entries per track around frame 4, small learned offsets
    F, K, n = 8, 8, raw["poses"].shape[0]
    ts = 1.6e9 + np.arange(F) * 0.1 + np.array([0, 0.01, -0.02, 0.0, 0.015, 0.0, -0.01, 0.0])
    tr = np.zeros((F, K, 8), np.float32)
    tr[..., 0] = -1
    for k in range(n):
        for f in range(F):
            q, t = raw["poses"][k, :4].numpy(), np.array([-1.0 + 0.3 * k, 0.1, 1.6 + 0.05 * k])
            tr[f, k] = [k, *(t + 0.05 * (f - 4) * np.array([1.0, 0.0, 0.3])), *q]
    ts_ = ts.astype(np.float64)
    obj_meta = {k: dict(start_frame=0, end_frame=F - 1, start_timestamp=float(ts_[0]), end_timestamp=float(ts_[-1])) for k in range(n)}
    meta = dict(obj_tracklets=tr, tracklet_timestamps=ts_, camera_timestamps={0: dict(train_timestamps=list(ts_))}, obj_meta=obj_meta)
    g = np.random.default_rng(0)
    ot0 = (0.02 * g.standard_normal((F, K, 3))).astype(np.float32)
    orr0 = (0.05 * g.standard_normal((F, K, 1))).astype(np.float32)
    T = AO.Table(tr, ts_, meta["camera_timestamps"], obj_meta)
    t_cam = float(ts_[4] + 0.03)
    ego = torch.eye(4, device=DEV)
    st = sgb.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=DEV),
                                           scale_modifier=1.0, viewmatrix=cam["viewmatrix"].to(DEV), projmatrix=cam["projmatrix"].to(DEV),
                                           sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    rast = sgb.GaussianRasterizer(st)
    gt = torch.rand(3, H, W, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
    vis = list(range(n))

    def step(impl):
        models = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in raw["models"]]
        if impl == "sgr":
            pose = make_pose(meta, fourier_dim=1)
            set_params(pose, ot0, orr0)
            ot, orr = pose.opt_trans, pose.opt_rots
            poses, idft = pose(vis, timestamp=t_cam, cam=0, is_val=False, ego_pose=ego, frame=4)
            xyz, rot, scale, opac, sh = sgb.compose(models, poses, idft)
        else:
            ot = torch.nn.Parameter(torch.from_numpy(ot0).to(DEV))
            orr = torch.nn.Parameter(torch.from_numpy(orr0).to(DEV))
            it = torch.from_numpy(tr).to(DEV)
            poses = AO.poses(T, vis, t_cam, 0, False, ego, it[..., 1:4], it[..., 4:8], ot, orr, finite=True)
            idft = AO.idft_rows(T, vis, 4, 1, 1.0).to(DEV)
            o = CO.compose(models, poses, idft, None, None)
            xyz, rot, scale, opac, sh = o["xyz"], o["rotation"], o["scaling"], o["opacity"], o["features"]
        m2d = torch.zeros_like(xyz, requires_grad=True)
        img = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot)[0]
        losses.photometric_loss(img, gt, None, 1.0, 0.2).backward()
        grads = [v.grad.clone() for m in models for v in m.values()] + [ot.grad.clone(), orr.grad.clone()]
        FusedAdam([{"params": [ot], "lr": 1e-3}, {"params": [orr], "lr": 1e-3}], eps=1e-15).step()
        return img.detach(), grads, (ot.detach().clone(), orr.detach().clone())

    a, b = step("sgr"), step("torch")
    # 1e-4 per pixel, except pixels explained by at most two flips of the rasterizer's per-pair thresholds: the two arms' poses and
    # composed positions differ in the last bits, enough to move a pair across alpha = 1/255 somewhere in 2.46 M pixels
    offenders = util.check_forward_flip_protocol(dict(color=a[0].cpu().numpy()), dict(color=b[0].cpu().numpy()), dict(color=float(b[0].abs().max())))
    assert len(offenders) < 100, len(offenders)
    for k, (x, y) in enumerate(zip(a[1], b[1])):
        assert rel(x.cpu().numpy(), y.cpu().numpy()) < 1e-3, k
    assert bool((a[1][-2] != 0).any()), "no gradient reached opt_trans"
    assert bool((a[1][-1] != 0).any()), f"no gradient reached opt_rots; |d opt_trans| = {float(a[1][-2].abs().sum())}"
    # FusedAdam's first step moves every row with a gradient by lr against its sign, as torch.optim.Adam(eps=1e-15) does
    for p_a, p0, gr in zip(a[2], (ot0, orr0), a[1][-2:]):
        step_ = p_a.cpu().double() - torch.from_numpy(p0).double()
        sure = gr.cpu().abs() > 1e-6 * float(gr.abs().max())
        assert bool((torch.sign(step_[sure]) == -torch.sign(gr.cpu()[sure].double())).all())


def test_reference_checkpoint_loads_and_fused_adam_steps_like_torch_adam(tmp_path):
    """The parameters carry the reference's names, so a checkpoint's actor_pose['params'] (train.py:218-223 saves
    ActorPose.save_state_dict) loads through io.load_checkpoint; FusedAdam(eps=1e-15) moves them as torch.optim.Adam does
    (actor_pose.py:66)."""
    from street_gaussians_b200 import io
    _, meta, _ = fixture()
    pose = make_pose(meta)
    assert set(pose.state_dict()) == {"opt_trans", "opt_rots"}
    ot, orr = AC.params()["seeded"]
    torch.save({"actor_pose": {"params": {"opt_trans": torch.from_numpy(ot), "opt_rots": torch.from_numpy(orr)}}, "iter": 7}, tmp_path / "ckpt.pth")
    ck = io.load_checkpoint(str(tmp_path / "ckpt.pth"))
    pose.load_state_dict(ck["actor_pose"]["params"])
    assert torch.equal(pose.opt_trans.cpu(), torch.from_numpy(ot)) and torch.equal(pose.opt_rots.cpu(), torch.from_numpy(orr))
    case = AC.BY_NAME["val"]
    w = torch.randn(3, 7, device=DEV)
    twin = [torch.nn.Parameter(p.detach().clone()) for p in (pose.opt_trans, pose.opt_rots)]
    fused = FusedAdam([{"params": [pose.opt_trans], "lr": 1e-3}, {"params": [pose.opt_rots], "lr": 2e-3}], eps=1e-15)
    ref = torch.optim.Adam([{"params": [twin[0]], "lr": 1e-3}, {"params": [twin[1]], "lr": 2e-3}], lr=0, eps=1e-15)
    for _ in range(3):
        run(pose, [0, 1, 2], case, w)
        twin[0].grad, twin[1].grad = pose.opt_trans.grad.clone(), pose.opt_rots.grad.clone()
        fused.step()
        ref.step()
    assert float((pose.opt_trans - twin[0]).abs().max()) < 1e-6 and float((pose.opt_rots - twin[1]).abs().max()) < 1e-6
    assert float((pose.opt_rots.detach().cpu() - torch.from_numpy(orr)).abs().max()) > 1e-3
