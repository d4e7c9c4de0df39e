"""torchrun check of the Gaussian-sharded multi-GPU mode against the single-GPU rasterizer on the same seeded scene.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 \
        tools/check_gaussian_sharded.py

Every rank renders the WHOLE scene with GaussianRasterizer (the checker) and its own share with
GaussianShardedRasterizer (NCCL all-gather of records / reduce-scatter of grad2d; with the argument p2p the peer-memory exchange,
whose bounded passes run the fused step, feature channels (S = 3 + 4) included; that case has run at world 1 only, not on several
H100s).  Own image rows must be bit-identical,
foreign rows zero, and the gradients of the rank's own Gaussians equal up to float summation order.  That order differs
between ANY two runs (float atomics), so the run-to-run difference of the single-GPU rasterizer is measured beside it
and printed as `floor`; the bound asserted is GRAD_TOL = 5e-4 of max|ref| per tensor — half the 1e-3 parity bar the
single-GPU path is held to against the reference.

Three further legs run each rank's band stages against the single-GPU calls on the gathered frame: the training losses (band_losses.py),
the sky composite and colour correction with band= / group= (their parameter gradients all-reduced), and the feature maps' finishing
(finish_features(band=)) on an S = 3 + 4 render (normals and semantics).  None of these legs has been run on several H100s yet; the
single-GPU emulations of tests/test_band_losses_gpu.py, tests/test_band_image_gpu.py and tests/test_band_features_gpu.py cover their
kernels.

With the argument `rebalance` only the rebalance leg runs (run_rebalance): sharded.rebalance over NCCL on an uneven split, against the
global arrays each rank restates.  It has run at world 1 only, not on several H100s; tests/test_rebalance_gpu.py emulates 2 to 8 ranks.

With the argument `checkpoint` only the checkpoint leg runs (run_checkpoint): sharded.save_checkpoint at world N over torch.distributed,
sharded.load_checkpoint at the same world N into fresh models, and the next training step against the uninterrupted one.  It has run at
world 1 only, not on several H100s; tests/test_sharded_checkpoint_gpu.py emulates 1 to 8 ranks on one GPU.

With the argument `compose` (NCCL all_reduce of the accumulator rows) or `compose-p2p` (the rasterizer's peer workspace) only the composer
leg runs (run_compose): compose(..., group= / rasterizer=) on each rank's rows of a config-C-like scene, before and after the rebalanced
split.  It has run at world 1 only, not on several H100s; tests/test_sharded_compose_gpu.py emulates 2 to 8 ranks on one GPU.

With the argument `layers` only the render-layer leg runs (run_layers): GaussianShardedRasterizer.forward_layers with the objects-only and
background-only layers through the fused peer-memory step, against GaussianRasterizer.forward_layers on the whole scene.  It has run at
world 1 only, not on several H100s; tests/test_sharded_layers_gpu.py emulates 2 to 8 ranks on one GPU.

With the argument `losses-p2p` only the loss leg runs, through the p2p rasterizer: frame_losses / the losses.py wrappers with rasterizer=,
so the halo and the sums go over its peer workspace (sgr_band_halo_exchange_peers / sgr_band_peer_sum).  Each rank's values must be the
same bytes on every rank and the whole frame's, and its gradient rows bit-equal to the single-GPU losses'.  It has run at world 1 only,
not on several H100s; tests/test_band_losses_p2p_gpu.py emulates 2 to 8 ranks on one GPU.

With the argument `image-p2p` only the sky and colour-correction leg runs, through the p2p rasterizer: sky_composite / color_correct with
rasterizer=, so the cube map's touched blocks and the colour correction's sums go over its peer memory (sgr_sky_grad_peer_sum /
sgr_band_peer_sum).  Rows as in the NCCL leg; both parameter gradients must also be the same bytes on every rank.  It has not been run
on several H100s; tests/test_sky_p2p_gpu.py emulates 2 to 8 ranks on one GPU.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import street_gaussians_b200 as sgb  # noqa: E402
from street_gaussians_b200 import synthetic  # noqa: E402
from street_gaussians_b200.sharded import GaussianShardedRasterizer, band_of_rows  # noqa: E402
import util  # noqa: E402

KEYS = ("means3D", "shs", "opacities", "scales", "rotations")
GRAD_TOL = 5e-4
POSE_TOL = 1e-4  # composer pose / correction gradients: sums of ~5e5 fp32 terms, added in another order than the single-GPU atomics


def run_case(rank, world, dev, S, P, W, H, bounded, exchange="nccl"):
    scene = synthetic.make_scene(P=P, width=W, height=H, sh_degree=3, seed=77, pose=True, semantics=S)
    st = util.settings_from(sgb, scene["cam"], dev)
    chunk = (P + world - 1) // world
    lo, hi = min(P, rank * chunk), min(P, (rank + 1) * chunk)
    rows = band_of_rows(H, rank, world).to(dev)
    m = rows.view(1, H, 1).float()
    up = {k: scene[k].to(dev) for k in ("grad_color", "grad_depth", "grad_alpha")}
    up_sem = scene["grad_semantic"].to(dev) if S else None

    # checker: whole scene on this GPU, upstream gradients of ALL bands (the job-wide loss)
    full = {k: scene[k].to(dev).requires_grad_(True) for k in KEYS}
    sem_full = scene["semantics"].to(dev).requires_grad_(True) if S else None
    m2d_full = torch.zeros(P, 3, device=dev, requires_grad=True)
    ref = sgb.GaussianRasterizer(st)(means3D=full["means3D"], means2D=m2d_full, opacities=full["opacities"], shs=full["shs"],
                                     scales=full["scales"], rotations=full["rotations"], semantics=sem_full)
    outs, grads = [ref[0], ref[2], ref[3]], [up["grad_color"], up["grad_depth"], up["grad_alpha"]]
    if S:
        outs.append(ref[4]); grads.append(up_sem)
    torch.autograd.backward(outs, grads)
    first = {k: full[k].grad.clone() for k in KEYS}
    for k in KEYS:
        full[k].grad = None
    m2d_full.grad = None
    if S:
        sem_full.grad = None
    ref = sgb.GaussianRasterizer(st)(means3D=full["means3D"], means2D=m2d_full, opacities=full["opacities"], shs=full["shs"],
                                     scales=full["scales"], rotations=full["rotations"], semantics=sem_full)
    outs = [ref[0], ref[2], ref[3]] + ([ref[4]] if S else [])
    torch.autograd.backward(outs, grads)
    floor = max(util.rel_err(first[k].double().cpu().numpy(), full[k].grad.double().cpu().numpy()) for k in KEYS)

    cap = sgb.InstanceCapacity() if bounded else None
    rast = GaussianShardedRasterizer(st, capacity=cap, exchange=exchange)
    worst = 0.0
    # bounded variant: pass 1 is exact (learns the instance capacity); with exchange='p2p' pass 2 is the first FUSED frame
    # (sgr_sharded_forward / sgr_sharded_backward, depth order compacted into all slots), passes 3-4 run with the learnt Gaussian capacity
    for rep in range(4 if bounded else 1):
        loc = {k: scene[k][lo:hi].to(dev).requires_grad_(True) for k in KEYS}
        sem_loc = scene["semantics"][lo:hi].to(dev).requires_grad_(True) if S else None
        m2d = torch.zeros(hi - lo, 3, device=dev, requires_grad=True)
        got = rast(means3D=loc["means3D"], means2D=m2d, opacities=loc["opacities"], shs=loc["shs"], scales=loc["scales"],
                   rotations=loc["rotations"], semantics=sem_loc)
        outs, grads = [got[0], got[2], got[3]], [up["grad_color"] * m, up["grad_depth"] * m, up["grad_alpha"] * m]
        if S:
            outs.append(got[4]); grads.append(up_sem * m)
        torch.autograd.backward(outs, grads)
        rast.synchronize_capacity()
        assert torch.equal(got[1], ref[1][lo:hi]), "radii"
        for a, b, name in ((got[0], ref[0], "color"), (got[2], ref[2], "depth"), (got[3], ref[3], "alpha"), (got[4], ref[4], "semantic")):
            if a.numel() == 0:
                continue
            assert torch.equal(a[:, rows], b.detach()[:, rows]), f"{name}: own rows differ"
            assert float(a.detach()[:, ~rows].abs().max()) == 0.0 if (~rows).any() else True, f"{name}: foreign rows not zero"
        for k in KEYS:
            e = util.rel_err(loc[k].grad.double().cpu().numpy(), full[k].grad[lo:hi].double().cpu().numpy())
            worst = max(worst, e)
            assert e < GRAD_TOL, (k, e)
        e = util.rel_err(m2d.grad.double().cpu().numpy(), m2d_full.grad[lo:hi].double().cpu().numpy())
        assert e < GRAD_TOL, ("means2D", e)
        if S:
            e = util.rel_err(sem_loc.grad.double().cpu().numpy(), sem_full.grad[lo:hi].double().cpu().numpy())
            assert e < GRAD_TOL, ("semantics", e)
    if bounded:  # forward-only frames back to back (eval loop): the leading barrier of the fused path / the staged path's extra barrier
        with torch.no_grad():
            for _ in range(3):
                got = rast(means3D=loc["means3D"], means2D=None, opacities=loc["opacities"], shs=loc["shs"], scales=loc["scales"],
                           rotations=loc["rotations"], semantics=sem_loc)
                assert torch.equal(got[0][:, rows], ref[0].detach()[:, rows]), "no_grad forward: own rows differ"
        rast.synchronize_capacity()
    return worst, floor


def run_losses(rank, world, dev, W=1280, H=720, exchange="nccl"):
    """Loss leg: each rank's band losses (band_losses.py) on its banded render against the single-GPU losses of the gathered frame.
    exchange="p2p": the losses take rasterizer= of the p2p rasterizer that rendered the rows (halo and sums over its peer workspace), and
    the values must also be the same bytes on every rank."""
    from street_gaussians_b200 import band_losses, losses
    scene = synthetic.make_scene(P=60_001, width=W, height=H, sh_degree=3, seed=78, pose=True)
    st = util.settings_from(sgb, scene["cam"], dev)
    rast = GaussianShardedRasterizer(st, exchange=exchange)
    P = scene["means3D"].shape[0]
    chunk = (P + world - 1) // world
    lo, hi = min(P, rank * chunk), min(P, (rank + 1) * chunk)
    with torch.no_grad():
        got = rast(means3D=scene["means3D"][lo:hi].to(dev), means2D=None, opacities=scene["opacities"][lo:hi].to(dev),
                   shs=scene["shs"][lo:hi].to(dev), scales=scene["scales"][lo:hi].to(dev), rotations=scene["rotations"][lo:hi].to(dev))
    color, depth, acc = got[0], got[2], got[3]
    full = [t.clone() for t in (color, depth, acc)]
    for t in full:
        if world > 1:
            dist.all_reduce(t)
    g = torch.Generator(device=dev).manual_seed(5)  # the data inputs are the same whole frames on every rank
    gt = torch.rand(3, H, W, device=dev, generator=g)
    mask = torch.rand(1, H, W, device=dev, generator=g) > 0.1
    sky = torch.rand(1, H, W, device=dev, generator=g) > 0.5
    lidar = full[1] * (1 + 0.05 * torch.randn(1, H, W, device=dev, generator=g)) * (torch.rand(1, H, W, device=dev, generator=g) > 0.5)
    rows = band_of_rows(H, rank, world).to(dev)
    band = rast.band if rast.band is not None else sgb.TileRowBand(0, (H + 15) // 16, 1)

    def grads(fn, *xs):
        xs = [x.detach().clone().requires_grad_(True) for x in xs]
        v = fn(*xs)
        v.backward()
        return v.detach(), [x.grad for x in xs]

    obj = torch.rand(1, H, W, device=dev, generator=g) > 0.7
    frame = lambda x, a, **kw: sum(band_losses.frame_losses(x, gt, mask, acc=a, sky_mask=sky, acc_obj=a, obj_bound=obj, **kw).values())
    checks = (("photometric", lambda x, **kw: losses.photometric_loss(x, gt, mask, **kw), (0,)),
              ("sky", lambda a, **kw: losses.sky_loss(a, sky, **kw), (2,)),
              ("lidar", lambda d, a, **kw: losses.lidar_depth_loss(d, a, lidar, mask, **kw), (1, 2)),
              ("frame", lambda x, a, **kw: frame(x, a, **kw) if kw else (losses.photometric_loss(x, gt, mask) + losses.sky_loss(a, sky) +
                                                                         losses.obj_acc_loss(a, obj)), (0, 2)))
    how = dict(rasterizer=rast) if exchange == "p2p" else dict(band=band, group=None)
    for name, fn, which in checks:
        if name == "frame" and exchange != "p2p":
            continue
        v_ref, g_ref = grads(fn, *(full[i] for i in which))
        v, g_band = grads(lambda *xs: fn(*xs, **how), *((color, depth, acc)[i] for i in which))
        if exchange == "p2p" and world > 1:
            alls = [torch.empty_like(v.reshape(1)) for _ in range(world)]
            dist.all_gather(alls, v.reshape(1))
            assert all(torch.equal(t, v.reshape(1)) for t in alls), f"{name}: values differ across ranks"
        a, b = float(v), float(v_ref)
        assert (a != a and b != b) or abs(a - b) <= 4e-6 * abs(b), (name, a, b)
        for x, y in zip(g_band, g_ref):
            assert torch.equal(x[:, rows].contiguous().view(torch.int32), y[:, rows].contiguous().view(torch.int32)), f"{name}: gradient rows differ"
            assert not bool(x[:, ~rows].any()), f"{name}: foreign gradient rows not zero"


def run_image_stages(rank, world, dev, W=1280, H=720, R=256, exchange="nccl"):
    """Sky and colour-correction leg: sky_composite and color_correct with band= / group= on each rank's banded render against the
    whole-frame calls on the gathered frame.  Output and image-gradient rows bit-equal, foreign rows zero; the all-reduced cube gradient
    equal to the whole-frame one up to the order of its float atomics (1e-5 of max|ref|), and the all-reduced affine gradient within one
    fp32 ulp of its fp64 sum.  exchange="p2p": the two stages take rasterizer= of the p2p rasterizer that rendered the rows (the cube's
    touched blocks and the affine sums over its peer memory), and both parameter gradients must also be the same bytes on every rank; at
    world 1 those calls are the whole-frame ones, so the affine gradient is theirs bit for bit."""
    from street_gaussians_b200 import corrections
    scene = synthetic.make_scene(P=60_001, width=W, height=H, sh_degree=3, seed=79, pose=True)
    st = util.settings_from(sgb, scene["cam"], dev)
    rast = GaussianShardedRasterizer(st, exchange=exchange)
    P = scene["means3D"].shape[0]
    chunk = (P + world - 1) // world
    lo, hi = min(P, rank * chunk), min(P, (rank + 1) * chunk)
    with torch.no_grad():
        got = rast(means3D=scene["means3D"][lo:hi].to(dev), means2D=None, opacities=scene["opacities"][lo:hi].to(dev),
                   shs=scene["shs"][lo:hi].to(dev), scales=scene["scales"][lo:hi].to(dev), rotations=scene["rotations"][lo:hi].to(dev))
    color, acc = got[0], got[3]
    full = [t.clone() for t in (color, acc)]
    for t in full:
        if world > 1:
            dist.all_reduce(t)
    g = torch.Generator(device=dev).manual_seed(6)  # the same whole-frame inputs on every rank
    cube = torch.rand(6, R, R, 3, device=dev, generator=g)
    affine = torch.eye(4, device=dev)[:3] + 0.05 * torch.randn(3, 4, device=dev, generator=g)
    sky_mask = torch.rand(1, H, W, device=dev, generator=g) > 0.5
    up = torch.randn(3, H, W, device=dev, generator=g)
    f = W / (2 * float(st.tanfovx))
    K = torch.tensor([[f, 0.0, W / 2], [0.0, f, H / 2], [0.0, 0.0, 1.0]], device=dev)
    w2c = st.viewmatrix.T.contiguous()
    rows = band_of_rows(H, rank, world).to(dev)
    band = rast.band if rast.band is not None else sgb.TileRowBand(0, (H + 15) // 16, 1)

    def step(rgb, a, b):
        xs = [t.detach().clone().requires_grad_(True) for t in (rgb, a, cube, affine)]
        kw = dict(rasterizer=rast) if b is not None and exchange == "p2p" else dict(band=b)
        out = sgb.sky_composite(xs[0], xs[1], xs[2], K, w2c, sky_mask=sky_mask, **kw)
        col = corrections.color_correct(out, xs[3], **kw)
        col.backward(torch.where(rows.view(1, -1, 1), up, torch.zeros_like(up)) if b is not None else up)
        return [col.detach()] + [x.grad for x in xs]

    ref = step(full[0], full[1], None)
    got = step(color, acc, band)
    bits = lambda x: x.contiguous().view(torch.int32)
    for name, x, y in (("rgb_out", got[0], ref[0]), ("dL/drgb", got[1], ref[1]), ("dL/dacc", got[2], ref[2])):
        assert torch.equal(bits(x[:, rows]), bits(y[:, rows])), f"{name}: band rows differ"
        assert not bool(x[:, ~rows].any()), f"{name}: foreign rows not zero"
    assert float((got[3] - ref[3]).abs().max()) <= 1e-5 * float(ref[3].abs().max()), "dL/dcube"
    x64 = torch.cat([sgb.sky_composite(*full, cube, K, w2c, sky_mask=sky_mask).detach().reshape(3, -1), torch.ones(1, H * W, device=dev)]).double()
    exact = (up.reshape(3, -1).double() @ x64.T).cpu().numpy()
    if exchange == "p2p" and world == 1:  # rasterizer= at world 1 takes the whole-frame calls: the reference's own fp32 sums
        assert torch.equal(bits(got[4]), bits(ref[4])), "dL/daffine"
    else:
        assert (np.abs(got[4].cpu().double().numpy() - exact) <= np.spacing(np.abs(exact).astype(np.float32))).all(), "dL/daffine"
    if exchange == "p2p" and world > 1:
        for name, x in (("dL/dcube", got[3]), ("dL/daffine", got[4])):
            first = x.clone()
            dist.broadcast(first, 0)
            assert torch.equal(bits(x), bits(first)), f"{name}: bytes differ from rank 0's"


def run_features(rank, world, dev, W=1280, H=720, K=4):
    """Feature leg: the sharded rasterizer with feature channels (3 normal channels, then K semantic ones) and finish_features(band=) on
    each rank's banded feature image, in both semantic modes, against finish_features on the gathered frame.  Output and dL/drendered rows
    bit-equal, foreign rows zero (the finishing is per pixel: no collective)."""
    from street_gaussians_b200 import features
    scene = synthetic.make_scene(P=60_001, width=W, height=H, sh_degree=3, seed=80, pose=True, semantics=3 + K)
    st = util.settings_from(sgb, scene["cam"], dev)
    rast = GaussianShardedRasterizer(st)
    P = scene["means3D"].shape[0]
    chunk = (P + world - 1) // world
    lo, hi = min(P, rank * chunk), min(P, (rank + 1) * chunk)
    sem = scene["semantics"].abs()  # accumulated probabilities are non-negative
    with torch.no_grad():
        got = rast(means3D=scene["means3D"][lo:hi].to(dev), means2D=None, opacities=scene["opacities"][lo:hi].to(dev),
                   shs=scene["shs"][lo:hi].to(dev), scales=scene["scales"][lo:hi].to(dev), rotations=scene["rotations"][lo:hi].to(dev),
                   semantics=sem[lo:hi].to(dev))
    feat = got[4]
    full = feat.clone()
    if world > 1:
        dist.all_reduce(full)
    g = torch.Generator(device=dev).manual_seed(7)
    gn, gs = torch.randn(3, H, W, device=dev, generator=g), torch.randn(K, H, W, device=dev, generator=g)
    rows = band_of_rows(H, rank, world).to(dev)
    band = rast.band if rast.band is not None else sgb.TileRowBand(0, (H + 15) // 16, 1)
    bits = lambda x: x.contiguous().view(torch.int32)

    def step(x, mode, b):
        x = x.detach().clone().requires_grad_(True)
        n, s = features.finish_features(x, 3, mode, band=b)
        torch.autograd.backward([n, s], [gn, gs])
        return n.detach(), s.detach(), x.grad

    for mode in ("logits", "probabilities"):
        ref, out = step(full, mode, None), step(feat, mode, band)
        for name, x, y in zip(("normals", "semantic", "dL/drendered"), out, ref):
            assert torch.equal(bits(x[:, rows]), bits(y[:, rows])), f"{mode} {name}: band rows differ"
            assert not bool(x[:, ~rows].any()), f"{mode} {name}: foreign rows not zero"


def run_rebalance(rank, world, dev, W=640, H=400):
    """Rebalance leg (argument `rebalance`): every rank builds the same with_raw scene, owns an uneven share of it (rank r weighted r + 1,
    the last rank three times more), steps FusedAdam three times on it and calls sharded.rebalance (NCCL all_gather and batch_isend_irecv).
    Each rank restates the global arrays and their Adam steps on its own GPU (the update is elementwise), so afterwards its new rows of
    every parameter, both moments and the statistics must be the even split's slice of them, bit for bit; one more step too.  The
    Gaussian-sharded render before and after has the single-GPU render's own rows bit for bit; densify_and_prune runs on the result."""
    import types
    from street_gaussians_b200 import sharded, training
    names, stats = training.PARAM_NAMES, training.STAT_NAMES
    scene = synthetic.make_scene(P=200_000, width=W, height=H, sh_degree=3, seed=81, n_vehicles=4, per_vehicle=20_000, with_raw=True,
                                 scale_med=0.02)
    raw = scene["raw"]
    poses, idft = raw["poses"].to(dev), raw["idft"].to(dev)
    g = torch.Generator().manual_seed(9)
    glob = []
    for r in raw["models"]:
        n = r["xyz"].shape[0]
        m = {"_" + a: v.to(dev).contiguous() for a, v in r.items()}
        m["_semantic"] = torch.rand(n, 2, generator=g).to(dev)
        m["max_radii2D"], m["xyz_gradient_accum"], m["denom"] = (torch.rand(n, generator=g).to(dev), torch.rand(n, 2, generator=g).to(dev),
                                                                 torch.rand(n, 1, generator=g).to(dev) + 1)
        glob.append(m)
    counts = [m["_xyz"].shape[0] for m in glob]
    P = sum(counts)
    w = [r + 1 for r in range(world)]
    w[-1] *= 3
    B = [P * sum(w[:r]) // sum(w) for r in range(world + 1)]
    G = [sum(counts[:k]) for k in range(len(glob) + 1)]
    rows = lambda Bs: [(max(Bs[rank], G[k]) - G[k], max(max(Bs[rank], G[k]), min(Bs[rank + 1], G[k + 1])) - G[k]) for k in range(len(glob))]
    grads = [[torch.randn(m[a].shape, generator=g).to(dev) * 1e-2 for a in names] for m in glob]

    def model(k, m, lo, hi):
        o = types.SimpleNamespace(**{a: torch.nn.Parameter(m[a][lo:hi].clone()) for a in names}, **{s: m[s][lo:hi].clone() for s in stats},
                                  percent_dense=0.01, percent_big_ws=0.1)
        if k == 0:
            o.scene_radius, o.sphere_center, o.sphere_radius = torch.tensor([20.0]), torch.zeros(3), torch.tensor([40.0])
        else:
            o.extent, o.min_xyz, o.max_xyz = torch.tensor([3.0]), torch.tensor([-3.0, -1.5, -1.5]), torch.tensor([3.0, 1.5, 1.5])
        return o

    def adam(objs):
        return training.FusedAdam([{"params": [getattr(o, a)], "lr": 1e-3 * (1 + i)} for o in objs for i, a in enumerate(names)], eps=1e-15)

    def step(objs, opt, rr, scale):
        for k, o in enumerate(objs):
            for a, gk in zip(names, grads[k]):
                getattr(o, a).grad = gk[rr[k][0]:rr[k][1]] * scale
        opt.step()

    full = [model(k, m, 0, counts[k]) for k, m in enumerate(glob)]
    mine = [model(k, m, *rows(B)[k]) for k, m in enumerate(glob)]
    fopt, opt = adam(full), adam(mine)
    for it in range(3):
        step(full, fopt, [(0, n) for n in counts], 1 + it)
        step(mine, opt, rows(B), 1 + it)
    st = util.settings_from(sgb, scene["cam"], dev)
    img_rows = band_of_rows(H, rank, world).to(dev)
    with torch.no_grad():
        xyz, rot, scale, opac, sh = sgb.compose(full, poses, idft)
        ref = sgb.GaussianRasterizer(st)(means3D=xyz, means2D=None, opacities=opac, shs=sh, scales=scale, rotations=rot)
    rast = GaussianShardedRasterizer(st)

    def render_own_rows(tag):
        with torch.no_grad():
            xyz, rot, scale, opac, sh = sgb.compose(mine, poses, idft)
            got = rast(means3D=xyz, means2D=None, opacities=opac, shs=sh, scales=scale, rotations=rot)
        for a, b, name in ((got[0], ref[0], "color"), (got[2], ref[2], "depth"), (got[3], ref[3], "alpha")):
            assert torch.equal(a[:, img_rows], b[:, img_rows]), f"rebalance {tag}: {name} own rows differ"

    render_own_rows("before")
    P_new = sharded.rebalance(mine, opt, rasterizer=rast)
    base, extra = divmod(P, world)
    Bn = [r * base + min(r, extra) for r in range(world + 1)]
    assert P_new == Bn[rank + 1] - Bn[rank] and rast.chunk == base + (extra > 0), (P_new, rast.chunk)
    bits = lambda t: t.detach().contiguous().view(torch.int32)
    for k, (o, f) in enumerate(zip(mine, full)):
        lo, hi = rows(Bn)[k]
        for a in names:
            p, q = getattr(o, a), getattr(f, a)
            assert torch.equal(bits(p), bits(q[lo:hi])), (k, a)
            assert any(p is x for grp in opt.param_groups for x in grp["params"]) and opt.state[p]["step"] == 3
            for mk in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(bits(opt.state[p][mk]), bits(fopt.state[q][mk][lo:hi])), (k, a, mk)
        for s in stats:
            assert torch.equal(bits(getattr(o, s)), bits(getattr(f, s)[lo:hi])), (k, s)
    step(full, fopt, [(0, n) for n in counts], 7)
    step(mine, opt, rows(Bn), 7)
    for k, (o, f) in enumerate(zip(mine, full)):
        lo, hi = rows(Bn)[k]
        for a in names:
            assert torch.equal(bits(getattr(o, a)), bits(getattr(f, a)[lo:hi])), ("step after rebalance", k, a)
    with torch.no_grad():  # the render of the stepped arrays, before the comparison render
        xyz, rot, scale, opac, sh = sgb.compose(full, poses, idft)
        ref = sgb.GaussianRasterizer(st)(means3D=xyz, means2D=None, opacities=opac, shs=sh, scales=scale, rotations=rot)
    render_own_rows("after")
    training.densify_and_prune(mine, 1e-7, 0.005, True, opt, seed=rank)
    return P_new


def run_checkpoint(rank, world, dev, W=640, H=400):
    """Checkpoint leg (argument `checkpoint`): every rank owns the even split of a with_raw scene and steps FusedAdam three times on it;
    sharded.save_checkpoint gathers the rows to rank 0 over torch.distributed (ProcessGroupTransport: the all_gather of the table, then one
    batch_isend_irecv per piece of at most 1 MiB) and writes the file; every rank then resumes into fresh models and a fresh FusedAdam with
    sharded.load_checkpoint.  The resumed rows, moments and statistics must be the uninterrupted run's bit for bit, and one training step
    (compose -> GaussianShardedRasterizer -> loss -> backward -> FusedAdam) on both must give bit-equal own image rows and parameter
    gradients within GRAD_TOL of each other (their float atomics add in any order, so the steps' bytes may differ)."""
    import tempfile
    import types
    from street_gaussians_b200 import sharded, training
    names, stats = training.PARAM_NAMES, training.STAT_NAMES
    scene = synthetic.make_scene(P=200_000, width=W, height=H, sh_degree=3, seed=83, n_vehicles=4, per_vehicle=20_000, with_raw=True,
                                 scale_med=0.02)
    raw = scene["raw"]
    poses, idft = raw["poses"].to(dev), raw["idft"].to(dev)
    g = torch.Generator().manual_seed(10)
    glob = []
    for r in raw["models"]:
        n = r["xyz"].shape[0]
        m = {"_" + a: v.to(dev).contiguous() for a, v in r.items()}
        m["_semantic"] = torch.rand(n, 2, generator=g).to(dev)
        m["max_radii2D"], m["xyz_gradient_accum"], m["denom"] = (torch.rand(n, generator=g).to(dev), torch.rand(n, 2, generator=g).to(dev),
                                                                 torch.rand(n, 1, generator=g).to(dev) + 1)
        glob.append(m)
    rows = sharded.even_slices([m["_xyz"].shape[0] for m in glob], world)[rank]
    grads = [[torch.randn(m[a].shape, generator=g).to(dev) * 1e-2 for a in names] for m in glob]

    def model(m, lo, hi):
        return types.SimpleNamespace(**{a: torch.nn.Parameter(m[a][lo:hi].clone()) for a in names}, **{s: m[s][lo:hi].clone() for s in stats},
                                     spatial_lr_scale=1.0, active_sh_degree=3)

    def adam(objs):
        return training.FusedAdam([{"params": [getattr(o, a)], "lr": 1e-3 * (1 + i), "name": a} for o in objs for i, a in enumerate(names)],
                                  eps=1e-15)

    mine = [model(m, lo, hi) for m, (lo, hi) in zip(glob, rows)]
    opt = adam(mine)
    for it in range(3):
        for k, o in enumerate(mine):
            for a, gk in zip(names, grads[k]):
                getattr(o, a).grad = gk[rows[k][0]:rows[k][1]] * (1 + it)
        opt.step()
    st = util.settings_from(sgb, scene["cam"], dev)
    gw = torch.Generator(device=dev).manual_seed(4)
    wc = torch.randn((3, H, W), generator=gw, device=dev)
    img_rows = band_of_rows(H, rank, world).to(dev)
    path = [os.path.join(tempfile.mkdtemp(prefix="sgr_ckpt_"), "iteration_3.pth")] if rank == 0 else [None]
    if world > 1:
        dist.broadcast_object_list(path, src=0)
    path = path[0]
    named = lambda objs: {f"m{k}": o for k, o in enumerate(objs)}
    sharded.save_checkpoint(path, named(mine), 3, opt, piece_bytes=1 << 20)
    if world > 1:
        dist.barrier()
    new = [model(m, 0, 1) for m in glob]
    nopt = adam(new)
    rast = GaussianShardedRasterizer(st)
    P = sharded.load_checkpoint(path, named(new), nopt, rasterizer=rast)
    assert P == sum(hi - lo for lo, hi in rows) and rast.chunk == max(sum(hi - lo for lo, hi in r) for r in sharded.even_slices(
        [m["_xyz"].shape[0] for m in glob], world)), (P, rast.chunk)
    bits = lambda t: t.detach().contiguous().view(torch.int32)
    for k, (o, q) in enumerate(zip(new, mine)):
        for a in names:
            p, pq = getattr(o, a), getattr(q, a)
            assert torch.equal(bits(p), bits(pq)), ("resumed", k, a)
            assert any(p is x for grp in nopt.param_groups for x in grp["params"]) and int(nopt.state[p]["step"]) == 3
            for mk in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(bits(nopt.state[p][mk]), bits(opt.state[pq][mk])), ("resumed", k, a, mk)
        for s in stats:
            assert torch.equal(bits(getattr(o, s)), bits(getattr(q, s))), ("resumed", k, s)

    def train_step(objs, o, r):
        o.zero_grad(set_to_none=True)
        xyz, rot, scale, opac, sh = sgb.compose(objs, poses, idft)
        color = r(means3D=xyz, means2D=None, opacities=opac, shs=sh, scales=scale, rotations=rot)[0]
        (color * wc).sum().backward()
        gr = [None if getattr(x, a).grad is None else getattr(x, a).grad.clone() for x in objs for a in names[:6]]
        o.step()
        return color.detach(), gr

    c0, g0 = train_step(mine, opt, GaussianShardedRasterizer(st))
    c1, g1 = train_step(new, nopt, rast)
    assert torch.equal(c0[:, img_rows], c1[:, img_rows]), "resumed step: own image rows differ"
    worst = 0.0
    for a, b in zip(g0, g1):
        assert (a is None) == (b is None), "resumed step: a gradient is missing"
        if a is not None and a.numel():
            err = float((a - b).abs().max()) / max(float(a.abs().max()), 1e-30)
            worst = max(worst, err)
    assert worst <= GRAD_TOL, ("resumed step: gradients", worst)
    if rank == 0:
        os.remove(path)
        os.rmdir(os.path.dirname(path))
    return P, worst


def run_compose(rank, world, dev, exchange, n_bg=400_000, actors=(20_000, 0, 7_000, 35_000, 1_000, 12_000, 3, 50_000)):
    """compose(..., rasterizer=) on this rank's rows of a config-C-like scene (background, 8 tracked actors, flip mask, pose correction)
    against compose() of the whole scene: own composed rows and raw gradient rows bit-equal, dL/dposes and dL/dcorrection the same bytes on
    every rank and within POSE_TOL of max|ref| of the single-GPU call (whose float atomics order its sums differently)."""
    import compose_case as CC
    from street_gaussians_b200.sharded import rebalance_plan
    names = ("xyz", "rotation", "scaling", "opacity", "features")
    models = [{k: v.to(dev) for k, v in m.items()} for m in CC.make_case(5, n_bg, list(actors), 16, 5)]
    g = torch.Generator().manual_seed(6)
    poses, idft = torch.randn(len(actors), 7, generator=g).to(dev), torch.randn(len(actors), 5, generator=g).to(dev)
    flip, fq = (torch.rand(sum(actors), generator=g) < 0.5).to(dev), torch.tensor([0.0, 0.0, 1.0, 0.0], device=dev)
    corr = ((torch.tensor([1.0, 0, 0, 0]) + 0.1 * torch.randn(4, generator=g)).to(dev), torch.randn(3, generator=g).to(dev))
    P = n_bg + sum(actors)
    up = {k: v.to(dev) for k, v in CC.upstream(7, P, 16).items()}
    starts = np.concatenate([[0], np.cumsum([int(m["xyz"].shape[0]) for m in models])])

    def run(mods, fl, upr, **kw):
        mods = [{k: v.detach().clone().requires_grad_(True) for k, v in m.items()} for m in mods]
        dp, cr, ct = poses.clone().requires_grad_(True), corr[0].clone().requires_grad_(True), corr[1].clone().requires_grad_(True)
        out = sgb.compose(mods, dp, idft, fl, fq, pose_correction=(cr, ct), **kw)
        torch.autograd.backward(list(out), [upr[k] for k in names])
        return [o.detach() for o in out], [{k: m[k].grad for k in m} for m in mods], dp.grad, torch.cat([cr.grad, ct.grad])

    ref_out, ref_raw, ref_dp, ref_dc = run(models, flip, up)
    uneven = [P * r * (r + 1) // (world * (world + 1)) for r in range(world + 1)]
    counts = [[max(0, min(uneven[r + 1], starts[m + 1]) - max(uneven[r], starts[m])) for m in range(len(models))] for r in range(world)]
    even = [0]
    for row in rebalance_plan(counts).counts:
        even.append(even[-1] + sum(row))
    for tag, B in (("uneven", uneven), ("rebalanced", even)):
        lo, hi = B[rank], B[rank + 1]
        mine, fl = [], []
        for m, mod in enumerate(models):
            a, b = max(lo, starts[m]) - starts[m], max(lo, min(hi, starts[m + 1])) - starts[m]
            a, b = min(a, b), b
            mine.append({k: v[a:b] for k, v in mod.items()})
            if m:
                fl.append(flip[starts[m] - n_bg + a: starts[m] - n_bg + b])
        st = util.settings_from(sgb, synthetic.make_scene(P=8, width=64, height=48, sh_degree=0, seed=1)["cam"], dev)
        rast = GaussianShardedRasterizer(st, exchange=exchange)
        if exchange == "p2p":  # COLLECTIVE: the workspace a forward of the rasterizer would have set up
            rast.repartition(hi - lo)
            rast.workspace(dev)
        out, raw, dp, dc = run(mine, torch.cat(fl), {k: v[lo:hi] for k, v in up.items()}, rasterizer=rast)
        for k, a, b in zip(names, out, ref_out):
            assert torch.equal(a, b[lo:hi]), (tag, k)
        for m, (a, b) in enumerate(zip(raw, ref_raw)):
            s0, s1 = max(lo, starts[m]) - starts[m], max(lo, min(hi, starts[m + 1])) - starts[m]
            for k in a:
                assert torch.equal(a[k], b[k][min(s0, s1):s1]), (tag, m, k)
        both = torch.cat([dp.reshape(-1), dc])
        if world > 1:
            alls = [torch.empty_like(both) for _ in range(world)]
            dist.all_gather(alls, both)
            assert all(torch.equal(a, both) for a in alls), (tag, "pose gradients differ across ranks")
        for a, b in ((dp, ref_dp), (dc, ref_dc)):
            assert float((a - b).abs().max()) <= POSE_TOL * float(b.abs().max()), (tag, float((a - b).abs().max()), float(b.abs().max()))
    return P


def run_layers(rank, world, dev, P=300_000, W=1280, H=720):
    """The objects-only and background-only layers through the fused peer-memory step (forward_layers, exchange='p2p'), against
    GaussianRasterizer.forward_layers on the whole scene: own rows of every image bit-equal, foreign rows zero, the gradients of the own
    Gaussians and of each layer's means2D sink within GRAD_TOL.  The objects layer gets an alpha gradient on every rank (the
    object-accumulation loss), the background layer none."""
    scene = synthetic.make_scene(P=P, width=W, height=H, sh_degree=3, seed=78, pose=True)
    st = util.settings_from(sgb, scene["cam"], dev)
    n_bkgd = P - P // 5
    chunk = (P + world - 1) // world
    lo, hi = min(P, rank * chunk), min(P, (rank + 1) * chunk)
    rows = band_of_rows(H, rank, world).to(dev)
    m = rows.view(1, H, 1).float()
    up = {k: scene[k].to(dev) for k in ("grad_color", "grad_depth", "grad_alpha")}
    g_obj = torch.rand(1, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
    white = (1.0, 1.0, 1.0)

    def call(rast, t, m2d, layers):
        return rast.forward_layers(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"], shs=t["shs"], scales=t["scales"],
                                   rotations=t["rotations"], layers=layers)

    full = {k: scene[k].to(dev).requires_grad_(True) for k in KEYS}
    m2d_full = torch.zeros(P, 3, device=dev, requires_grad=True)
    sinks_full = [torch.zeros(n_bkgd, 3, device=dev, requires_grad=True), torch.zeros(P - n_bkgd, 3, device=dev, requires_grad=True)]
    ref = call(sgb.GaussianRasterizer(st), full, m2d_full, [sgb.RenderLayer(0, n_bkgd, white, sinks_full[0]),
                                                             sgb.RenderLayer(n_bkgd, P, white, sinks_full[1])])
    torch.autograd.backward([ref[0], ref[2], ref[3], ref[5][1][2]], [up["grad_color"], up["grad_depth"], up["grad_alpha"], g_obj])
    rast = GaussianShardedRasterizer(st, capacity=sgb.InstanceCapacity(), exchange="p2p")
    worst = 0.0
    for rep in range(3):  # pass 1: plain (learns the capacities); passes 2-3: layered
        loc = {k: scene[k][lo:hi].to(dev).requires_grad_(True) for k in KEYS}
        m2d = torch.zeros(hi - lo, 3, device=dev, requires_grad=True)
        if rep == 0:
            got = rast(means3D=loc["means3D"], means2D=m2d, opacities=loc["opacities"], shs=loc["shs"], scales=loc["scales"],
                       rotations=loc["rotations"])
            torch.autograd.backward([got[0], got[2], got[3]], [up["grad_color"] * m, up["grad_depth"] * m, up["grad_alpha"] * m])
            rast.synchronize_capacity()
            continue
        rb, re = min(hi - lo, max(0, n_bkgd - lo)), hi - lo  # this rank's rows of each layer, in its own rows
        sinks = [torch.zeros(rb, 3, device=dev, requires_grad=True), torch.zeros(re - rb, 3, device=dev, requires_grad=True)]
        got = call(rast, loc, m2d, [sgb.RenderLayer(0, rb, white, sinks[0]), sgb.RenderLayer(rb, re, white, sinks[1])])
        torch.autograd.backward([got[0], got[2], got[3], got[5][1][2]], [up["grad_color"] * m, up["grad_depth"] * m, up["grad_alpha"] * m,
                                                                         g_obj * m])
        rast.synchronize_capacity()
        images = [(got[0], ref[0]), (got[2], ref[2]), (got[3], ref[3])] + [(a, b) for k in range(2) for a, b in zip(got[5][k], ref[5][k])]
        for i, (a, b) in enumerate(images):
            assert torch.equal(a.detach()[:, rows], b.detach()[:, rows]), f"image {i}: own rows differ"
            assert float(a.detach()[:, ~rows].abs().max()) == 0.0 if (~rows).any() else True, f"image {i}: foreign rows not zero"
        pairs = [(loc[k].grad, full[k].grad[lo:hi], k) for k in KEYS] + [(m2d.grad, m2d_full.grad[lo:hi], "means2D")]
        cut = lambda g, a, b: None if g is None else g[a:b]
        pairs += [(sinks[0].grad, cut(sinks_full[0].grad, lo, lo + rb), "background sink"),
                  (sinks[1].grad, cut(sinks_full[1].grad, max(0, lo - n_bkgd), hi - n_bkgd), "objects sink")]
        for a, b, name in pairs:
            if b is None:  # (the background layer has no gradient: neither call returns one for its sink)
                assert a is None, (name, "a gradient where the single-GPU call has none")
                continue
            if b.numel() == 0:
                continue
            e = util.rel_err(a.double().cpu().numpy(), b.double().cpu().numpy())
            worst = max(worst, e)
            assert e < GRAD_TOL, (name, e)
    return worst


def run_all(rank, world, dev, exchange):
    # the last case carries feature channels through the bounded path: with exchange=p2p its passes 2-4 are the fused step with
    # semantics (sgr_sharded_*_features, no NCCL), with exchange=nccl the staged one
    for S, P, W, H, bounded in ((0, 200_003, 1280, 720, False), (2, 60_001, 800, 608, False), (0, 200_003, 1280, 720, True),
                                (3 + 4, 60_001, 800, 608, True)):
        worst, floor = run_case(rank, world, dev, S, P, W, H, bounded, exchange)
        print(f"[rank {rank}/{world}] exchange={exchange} S={S} P={P} {W}x{H} bounded={bounded}: images bit-equal, worst grad rel err {worst:.2e} "
              f"(single-GPU run-to-run floor {floor:.2e})", flush=True)
    run_losses(rank, world, dev)
    print(f"[rank {rank}/{world}] band losses: the frame's values, gradient rows bit-equal to the single-GPU losses", flush=True)
    run_image_stages(rank, world, dev)
    print(f"[rank {rank}/{world}] band sky and colour correction: rows bit-equal to the single-GPU calls, parameter gradients the frame's",
          flush=True)
    run_features(rank, world, dev)
    print(f"[rank {rank}/{world}] band feature finishing: rows bit-equal to the single-GPU calls", flush=True)


def main():
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    ok = True
    try:
        mode = sys.argv[1] if len(sys.argv) > 1 else "nccl"
        if mode == "losses-p2p":
            run_losses(rank, world, dev, exchange="p2p")
            print(f"[rank {rank}/{world}] band losses over peer memory: the same values on every rank, the frame's, gradient rows bit-equal "
                  "to the single-GPU losses", flush=True)
        elif mode == "image-p2p":
            run_image_stages(rank, world, dev, exchange="p2p")
            print(f"[rank {rank}/{world}] sky and colour correction over peer memory: rows bit-equal to the single-GPU calls, parameter "
                  "gradients the frame's and the same bytes on every rank", flush=True)
        elif mode in ("compose", "compose-p2p"):
            P = run_compose(rank, world, dev, "p2p" if mode == "compose-p2p" else "nccl")
            print(f"[rank {rank}/{world}] compose ({mode}): {P} Gaussians, own rows bit-equal, dL/dposes and dL/dcorrection the same bytes on "
                  "every rank and the frame's", flush=True)
        elif mode == "layers":
            worst = run_layers(rank, world, dev)
            print(f"[rank {rank}/{world}] render layers (fused p2p step): own rows bit-equal, gradients rel err {worst:.2e}", flush=True)
        elif mode == "checkpoint":
            P, worst = run_checkpoint(rank, world, dev)
            print(f"[rank {rank}/{world}] checkpoint: saved at world {world} and resumed, {P} Gaussians, rows / moments / statistics bit for "
                  f"bit, the next step's own image rows bit-equal, gradients rel err {worst:.2e}", flush=True)
        elif mode == "rebalance":
            P_new = run_rebalance(rank, world, dev)
            print(f"[rank {rank}/{world}] rebalance: {P_new} Gaussians, rows / moments / statistics the even split's slice bit for bit, "
                  "own image rows bit-equal before and after", flush=True)
        else:
            run_all(rank, world, dev, mode)
    except AssertionError as e:
        ok = False
        print(f"[rank {rank}] FAILED: {e!r}", flush=True)
    if world > 1:
        flag = torch.tensor([0 if ok else 1], device=dev)
        dist.all_reduce(flag)
        ok = int(flag.item()) == 0
        dist.destroy_process_group()
    if rank == 0:
        print("GAUSSIAN_SHARDED_CHECK", "OK" if ok else "FAILED", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
