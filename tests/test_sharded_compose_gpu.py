"""GPU: the composer under Gaussian sharding (composer.compose(..., rasterizer=) with the peer-memory reduction, include/sgr.h
sgr_compose_backward_rows / sgr_compose_pose_reduce_peers / sgr_compose_pose_finalize), with 1, 2, 3, 5 and 8 ranks emulated by threads
(tests/rank_threads.py) on streams of one GPU through PeerWorkspace.emulate.

Scenes are config-C-like: a background, 8 tracked actors (fourier_dim 5, SH degree 3), a flip mask, the background pose correction, and
the actor poses from ActorPose with opt_track (learned opt_trans / opt_rots).  Rank r holds the global rows [B_r, B_(r+1)) of the
model-major composed array (the split GaussianShardedRasterizer documents); splits are uneven (so the background and some actors have 0
rows on some ranks, a whole rank may hold none) and the even split sharded.rebalance_plan gives after rebalancing.

Checked, per rank: the composed rows bit-identical to the matching rows of the single-GPU compose, and every raw gradient row too; dL/dposes,
dL/dcorrection, opt_trans.grad and opt_rots.grad bit-identical on every rank, and dL/dposes / dL/dcorrection within the single-GPU call's
float64 bound (tests/correction_oracle.py compose64) widened by world more fp32 additions of every term, stated as sharded64_case states
it: the single-GPU bound's atomics count n_atom gains `world` (one add per rank), i.e. the bound scales by (5 + n_atom + world) / (5 + n_atom);
opt_trans.grad / opt_rots.grad equal ActorPose's backward of those dL/dposes bit for bit.  One FusedAdam step then leaves every replicated
parameter bit-identical on every rank.
Sensitivity, on the ranks' own accumulator rows: dropping a rank, adding the ranks in another order on one rank, or skipping the finalize
each fail those checks."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import compose_case as CC
import correction_oracle as CR
import street_gaussians_b200 as sgb
from rank_threads import run_ranks
from street_gaussians_b200 import _capi
from street_gaussians_b200 import sharded as SH
from street_gaussians_b200.training import FusedAdam

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
NAMES = ("xyz", "rotation", "scaling", "opacity", "features")
M, FOURIER, ACTORS = 16, 5, (900, 37, 1500, 256, 0, 5, 1200, 333)
N_BG = 6000
_warm = []


def _settings():
    z = torch.zeros(3, device=DEV)
    return sgb.GaussianRasterizationSettings(32, 32, 0.5, 0.5, z, 1.0, torch.eye(4, device=DEV), torch.eye(4, device=DEV), 0, z, False, False)


def _tracks(n_act, F=12):
    """n_act tracks on every frame of F, moving and turning slowly: the ActorPose inputs."""
    ts = 1.6e9 + 0.1 * np.arange(F)
    tr = np.zeros((F, n_act, 8), np.float32)
    meta = {}
    for a in range(n_act):
        for f in range(F):
            yaw = 0.3 * a + 0.05 * f
            tr[f, a] = [a, -5.0 + 2.0 * a + 0.9 * f, 0.2 * a, 12.0 + a - 0.1 * f, np.cos(yaw / 2), 0.0, 0.0, np.sin(yaw / 2)]
        meta[a] = dict(start_frame=0, end_frame=F - 1, start_timestamp=float(ts[0]), end_timestamp=float(ts[-1]))
    return tr, ts, meta


def _actor_pose(tracks, seed):
    pose = sgb.ActorPose(*tracks[:2], None, tracks[2], opt_track=True, fourier_dim=FOURIER, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    with torch.no_grad():
        pose.opt_trans.copy_(0.1 * torch.randn(pose.opt_trans.shape, generator=g, device=DEV))
        pose.opt_rots.copy_(0.2 * torch.randn(pose.opt_rots.shape, generator=g, device=DEV))
    return pose


def _scene(seed):
    models = CC.make_case(seed, N_BG, list(ACTORS), M, FOURIER)
    g = torch.Generator().manual_seed(seed + 1)
    flip = torch.rand(sum(ACTORS), generator=g) < 0.5
    q = torch.tensor([1.0, 0.0, 0.0, 0.0]) + 0.1 * torch.randn(4, generator=g)
    corr = (q, 0.3 * torch.randn(3, generator=g))
    P = N_BG + sum(ACTORS)
    up = CC.upstream(seed + 2, P, M)
    return dict(models=[{k: v.to(DEV) for k, v in m.items()} for m in models], flip=flip.to(DEV), fq=torch.tensor([0.0, 0.0, 1.0, 0.0], device=DEV),
                corr=tuple(t.to(DEV) for t in corr), up={k: v.to(DEV) for k, v in up.items()}, P=P, tracks=_tracks(len(ACTORS)), seed=seed)


def _counts(sc, B):
    """counts[r][m]: rows of sub-model m that rank r holds when it owns the global rows [B[r], B[r+1])."""
    sizes = [int(m["xyz"].shape[0]) for m in sc["models"]]
    starts = np.concatenate([[0], np.cumsum(sizes)])
    return [[max(0, min(B[r + 1], starts[m + 1]) - max(B[r], starts[m])) for m in range(len(sizes))] for r in range(len(B) - 1)]


def _local(sc, B, r):
    """Rank r's rows of every sub-model (fresh leaves), its rows of the flip mask and its slice of the upstream gradients."""
    sizes = [int(m["xyz"].shape[0]) for m in sc["models"]]
    starts = np.concatenate([[0], np.cumsum(sizes)])
    loc, flip = [], []
    for m, mod in enumerate(sc["models"]):
        lo, hi = max(B[r], starts[m]) - starts[m], max(max(B[r], starts[m]), min(B[r + 1], starts[m + 1])) - starts[m]
        loc.append({k: v[lo:hi].detach().clone().requires_grad_(True) for k, v in mod.items()})
        if m > 0:
            a0 = starts[m] - N_BG
            flip.append(sc["flip"][a0 + lo:a0 + hi])
    return loc, torch.cat(flip), {k: v[B[r]:B[r + 1]] for k, v in sc["up"].items()}


def _step(sc, models, flip, up, **kw):
    """compose -> backward -> one FusedAdam step of the replicated parameters.  Returns what the checks read."""
    pose = _actor_pose(sc["tracks"], sc["seed"])
    poses, idft = pose(list(range(len(ACTORS))), timestamp=1.6e9 + 0.55, frame=5)
    poses.retain_grad()
    cr, ct = (t.clone().requires_grad_(True) for t in sc["corr"])
    out = sgb.compose(models, poses, idft, flip, sc["fq"], pose_correction=(cr, ct), **kw)
    torch.autograd.backward(list(out), [up[k] for k in NAMES])
    res = dict(out=[o.detach() for o in out], dposes=poses.grad.clone(), dcorr=torch.cat([cr.grad, ct.grad]),
               g_trans=pose.opt_trans.grad.clone(), g_rots=pose.opt_rots.grad.clone(),
               raw=[{k: m[k].grad for k in CC.KEYS} for m in models], poses=poses.detach(), idft=idft)
    # ActorPose's backward of these dposes, called on its own: the opt gradients must be its bits
    pose.zero_grad()
    p2, _ = pose(list(range(len(ACTORS))), timestamp=1.6e9 + 0.55, frame=5)
    res["g_trans_of_dposes"], res["g_rots_of_dposes"] = torch.autograd.grad(p2, [pose.opt_trans, pose.opt_rots], res["dposes"])
    pose.opt_trans.grad, pose.opt_rots.grad = res["g_trans"].clone(), res["g_rots"].clone()
    params = [pose.opt_trans, pose.opt_rots, cr, ct]
    FusedAdam(params, lr=1e-3).step()
    res["stepped"] = [p.detach().clone() for p in params]
    return res


def _warm_up():
    """Every kernel of the sharded composer loaded before ranks spin in emulated barriers (see test_sharded64_gpu._warm_up_fused_path): the
    path at world 1 (no barrier) and the barrier kernel itself on a pair of workspaces before anything spins."""
    if _warm:
        return
    from test_sharded64_gpu import _warm_up_fused_path
    _warm_up_fused_path(DEV)
    sc = _scene(99)
    ws = SH.PeerWorkspace.emulate(_settings(), 8, 1, DEV)[0]
    loc, flip, up = _local(sc, [0, sc["P"]], 0)
    _step(sc, loc, flip, up, rasterizer=_stand_in(ws))
    _step(sc, loc, flip, up)
    torch.cuda.synchronize()
    _warm.append(True)


def _stand_in(ws):
    """What compose(rasterizer=) reads of a GaussianShardedRasterizer(exchange="p2p"), around an emulated workspace."""
    return types.SimpleNamespace(exchange="p2p", group=None, pose_workspace=lambda: ws)


def _run_sharded(sc, B):
    world = len(B) - 1
    wss = SH.PeerWorkspace.emulate(_settings(), 8, world, DEV)
    for ws in wss:
        ws.buf[ws.off_pose: ws.off_flags].fill_(0x7f)  # poisoned: the section needs no content on entry
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    torch.cuda.synchronize()

    def rank(r, _tr):
        with torch.cuda.stream(streams[r]):
            loc, flip, up = _local(sc, B, r)
            return _step(sc, loc, flip, up, rasterizer=_stand_in(wss[r]))

    res = run_ranks(world, rank)
    torch.cuda.synchronize()
    return res


def _single(sc):
    models = [{k: v.detach().clone().requires_grad_(True) for k, v in m.items()} for m in sc["models"]]
    return _step(sc, models, sc["flip"], sc["up"])


def _bound64(sc, single, world):
    """float64 values and bounds of dL/dposes and dL/dcorrection: the single-GPU bound with world more fp32 additions of every term."""
    r = CR.compose64(sc["models"], single["poses"], single["idft"], sc["flip"], sc["fq"], sc["up"], sc["corr"])
    n_act = torch.tensor(ACTORS, dtype=torch.float64, device=DEV)[:, None] // 32 + 66
    n_bg = N_BG // 32 + 66
    return (r["dposes"], r["b_dposes"] * (5 + n_act + world) / (5 + n_act), r["dcorrection"], r["b_dcorrection"] * (5 + n_bg + world) / (5 + n_bg))


def _within(got, ref, bound):
    return bool(((got.double() - ref).abs() <= bound).all())


def _splits(P, world):
    """(tag, B): an uneven split with the rows weighted 1 : 2 : ... : world and, with world > 1, the same split with rank (world - 1) // 2
    holding nothing (its rows go to the next rank)."""
    w = [r + 1 for r in range(world)]
    uneven = [P * sum(w[:r]) // sum(w) for r in range(world + 1)]
    out = [("uneven", uneven)]
    if world > 1:
        k = (world - 1) // 2
        e = list(uneven)
        e[k + 1] = e[k]
        out.append(("empty_rank", e))
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_sharded_compose_is_the_frame_on_every_rank(world):
    _warm_up()
    sc = _scene(7 + world)
    single = _single(sc)
    dposes64, b_dposes, dcorr64, b_dcorr = _bound64(sc, single, world)
    live = [a for a, n in enumerate(ACTORS) if n > 0]
    assert _within(single["dposes"][live], dposes64[live], b_dposes[live]) and _within(single["dcorr"], dcorr64, b_dcorr)
    for tag, B in _splits(sc["P"], world):
        counts = _counts(sc, B)
        plan = SH.rebalance_plan(counts)
        Bn = [0]
        for row in plan.counts:
            Bn.append(Bn[-1] + sum(row))
        for tag2, BB in ((tag, B), (tag + "+rebalanced", Bn)):
            cnt = _counts(sc, BB)
            if world > 1 and tag2 == "uneven":
                assert any(c == 0 for row in cnt for c in row), (tag2, cnt)  # some sub-model has no rows on some rank
            res = _run_sharded(sc, BB)
            for r, rr in enumerate(res):
                lo, hi = BB[r], BB[r + 1]
                for k, a, b in zip(NAMES, rr["out"], single["out"]):
                    assert torch.equal(a, b[lo:hi]), (world, tag2, r, k)
                for m, (lm, sm) in enumerate(zip(rr["raw"], _raw_rows(sc, single, BB, r))):
                    for k in CC.KEYS:
                        assert torch.equal(lm[k], sm[k]), (world, tag2, r, m, k)
                for key in ("dposes", "dcorr", "g_trans", "g_rots"):
                    assert torch.equal(rr[key], res[0][key]), (world, tag2, r, key)
                assert torch.equal(rr["g_trans"], rr["g_trans_of_dposes"]) and torch.equal(rr["g_rots"], rr["g_rots_of_dposes"])
                for a, b in zip(rr["stepped"], res[0]["stepped"]):
                    assert torch.equal(a, b), (world, tag2, r, "after FusedAdam")
            assert _within(res[0]["dposes"][live], dposes64[live], b_dposes[live]), (world, tag2, "dposes")
            assert _within(res[0]["dcorr"], dcorr64, b_dcorr), (world, tag2, "dcorrection")
            dead = [a for a, n in enumerate(ACTORS) if n == 0]
            assert float(res[0]["dposes"][dead].abs().sum()) == 0.0


def _raw_rows(sc, single, B, r):
    sizes = [int(m["xyz"].shape[0]) for m in sc["models"]]
    starts = np.concatenate([[0], np.cumsum(sizes)])
    out = []
    for m in range(len(sizes)):
        lo = max(B[r], starts[m]) - starts[m]
        hi = max(lo, min(B[r + 1], starts[m + 1]) - starts[m])
        out.append({k: single["raw"][m][k][lo:hi] for k in CC.KEYS})
    return out


def _rows_and_finalize(sc, poses, idft, B):
    """Every rank's accumulator rows by sgr_compose_backward_rows, and a finalize of any sum of them (sgr_compose_pose_finalize)."""
    L = _capi.lib()
    nseg = len(sc["models"])
    pose_tab = torch.zeros((nseg, 8), device=DEV)
    pose_tab[1:, :7] = poses
    idft_tab = torch.zeros((nseg, _capi.MAX_FOURIER), device=DEV)
    idft_tab[1:, :FOURIER] = idft
    corr = torch.zeros(8, device=DEV)
    corr[:4], corr[4:7] = sc["corr"]
    fq = sc["fq"]
    rows, keep = [], []
    for r in range(len(B) - 1):
        loc, flip, up = _local(sc, B, r)
        segs = (_capi.SgrSegment * nseg)()
        grads = (_capi.SgrSegmentGrads * nseg)()
        start = 0
        flip_full = torch.zeros(B[r + 1] - B[r], dtype=torch.uint8, device=DEV)
        flip_full[int(loc[0]["xyz"].shape[0]):] = flip.to(torch.uint8)
        for k, m in enumerate(loc):
            n = int(m["xyz"].shape[0])
            s = segs[k]
            s.start, s.count, s.fourier_dim, s.posed = start, n, int(m["features_dc"].shape[1]), int(k > 0)
            gt = [torch.empty_like(m[key]) for key in CC.KEYS]
            keep += [m, gt]
            s.xyz, s.rotation, s.scaling, s.opacity, s.features_dc, s.features_rest = (m[key].data_ptr() if n else None for key in CC.KEYS)
            g = grads[k]
            g.xyz, g.rotation, g.scaling, g.opacity, g.features_dc, g.features_rest = (t.data_ptr() if n else None for t in gt)
            start += n
        acc = torch.empty((int(L.sgr_compose_pose_rows(nseg, 1)), 16), device=DEV)
        _capi.call("sgr_compose_backward_rows", DEV, segs, grads, nseg, M, _capi.ptr(pose_tab), _capi.ptr(idft_tab), _capi.ptr(flip_full),
                   _capi.ptr(fq), _capi.ptr(corr), *(_capi.ptr(up[k].contiguous()) for k in NAMES), _capi.ptr(acc), acc.numel() * 4)
        rows.append(acc)
        keep.append(segs)

    def finalize(acc):
        dposes, dcorr = torch.empty((nseg, 8), device=DEV), torch.empty(8, device=DEV)
        _capi.call("sgr_compose_pose_finalize", DEV, keep[-1], nseg, _capi.ptr(pose_tab), _capi.ptr(corr), _capi.ptr(acc.contiguous()),
                   acc.numel() * 4, _capi.ptr(dposes), _capi.ptr(dcorr))
        return dposes[1:, :7], torch.cat([dcorr[:4], dcorr[4:7]])

    return rows, finalize


@pytest.mark.parametrize("world", [3, 8])
def test_mutations_of_the_reduction_fail_the_checks(world):
    """On the ranks' own accumulator rows: the rank-order sum finalized is within the bound, like the p2p path; a dropped rank and a missing finalize
    leave the float64 bound, and one rank adding in another order no longer agrees bit for bit with the others (seen on at least one
    row of one split)."""
    _warm_up()
    sc = _scene(40 + world)
    single = _single(sc)
    dposes64, b_dposes, dcorr64, b_dcorr = _bound64(sc, single, world)
    live = [a for a, n in enumerate(ACTORS) if n > 0]
    B = _splits(sc["P"], world)[0][1]
    res = _run_sharded(sc, B)
    rows, finalize = _rows_and_finalize(sc, single["poses"], single["idft"], B)
    total = torch.zeros_like(rows[0])
    for a in rows:
        total = total + a
    dp, dc = finalize(total)
    # (the rows come from a second backward, whose float atomics may order the sums differently from the p2p run's: not bit for bit)
    assert _within(dp[live], dposes64[live], b_dposes[live]) and _within(dc, dcorr64, b_dcorr)
    assert _within(res[0]["dposes"][live], dposes64[live], b_dposes[live]) and _within(res[0]["dcorr"], dcorr64, b_dcorr)
    # a dropped rank: the one with the most background rows
    heavy = max(range(world), key=lambda r: _counts(sc, B)[r][0])
    dropped = torch.zeros_like(total)
    for r, a in enumerate(rows):
        if r != heavy:
            dropped = dropped + a
    dp2, dc2 = finalize(dropped)
    assert not (_within(dp2[live], dposes64[live], b_dposes[live]) and _within(dc2, dcorr64, b_dcorr))
    # no finalize: the summed rows' rotation and translation sums taken as the gradient
    raw_rows = torch.cat([total[1:len(ACTORS) + 1, 9:13], total[1:len(ACTORS) + 1, 13:16]], 1)
    assert not _within(raw_rows[live], dposes64[live], b_dposes[live])
    # another rank order on one rank: its bytes differ from the others' on some row
    rev = torch.zeros_like(total)
    for a in reversed(rows):
        rev = rev + a
    dp3, dc3 = finalize(rev)
    differs = not (torch.equal(dp3, dp) and torch.equal(dc3, dc))
    if not differs:  # the few-row sums may round alike: shuffle by a rotation of the order
        rot = torch.zeros_like(total)
        for a in rows[1:] + rows[:1]:
            rot = rot + a
        differs = not torch.equal(finalize(rot)[0], dp)
    assert differs, "every order gave the same bytes: the order check would not see a mutation"


def test_compose_reduction_options():
    """None for both keeps the single-GPU call; group= takes the all-reduce (here without a process group: the identity) and gives the
    single-GPU values; a rasterizer with another group is refused; exchange="nccl" uses the rasterizer's group."""
    from street_gaussians_b200 import composer
    sc = _scene(3)
    single = _single(sc)
    calls = []
    real = composer._reduction
    assert real(None, None) is None
    r = types.SimpleNamespace(exchange="nccl", group="g")
    assert real(None, r) == ("nccl", "g")
    with pytest.raises(ValueError, match="differs"):
        real("h", r)
    import street_gaussians_b200.band_losses as BL
    orig = BL.all_reduce_sum
    BL.all_reduce_sum = lambda t, group=None: calls.append(group) or t
    try:
        models = [{k: v.detach().clone().requires_grad_(True) for k, v in m.items()} for m in sc["models"]]
        res = _step(sc, models, sc["flip"], sc["up"], group="world")
    finally:
        BL.all_reduce_sum = orig
    assert calls == ["world"]
    for a, b in zip(res["out"], single["out"]):
        assert torch.equal(a, b)
    dposes64, b_dposes, dcorr64, b_dcorr = _bound64(sc, single, 1)
    live = [a for a, n in enumerate(ACTORS) if n > 0]
    assert _within(res["dposes"][live], dposes64[live], b_dposes[live]) and _within(res["dcorr"], dcorr64, b_dcorr)
    with pytest.raises(_capi.SgrError, match="forward"):
        SH.GaussianShardedRasterizer(_settings(), exchange="p2p").pose_workspace()
