"""GPU: the block-masked Adam of the sky cube map (training.CubeMapSparseAdam over sgr_cube_sparse_adam_step) and the marks it consumes
(sky.sky_composite(blocks=): sgr_band_sky_composite_backward_or_marks, sgr_sky_grad_peer_sum_union, and the band path's summed marks).

  * Marked blocks get FusedAdam's update bit for bit; outside them grad, exp_avg and exp_avg_sq are seeded with NaN and param, exp_avg
    and exp_avg_sq keep their bits (so the kernel neither reads nor writes there); the map comes back all zero.  All blocks marked is
    FusedAdam over the whole tensor.
  * State dicts move FusedAdam -> CubeMapSparseAdam -> FusedAdam; the step count advances per call; no gradient, no change.
  * The whole-frame backward with blocks= gives the same dL/dacc and dL/dcube up to its atomics' order; its marks lie between the
    intersection and the union of tests/test_sky_p2p_gpu.py's _map_bounds, and two backward passes leave the OR of their marks.
  * A short training loop (compose -> rasterize -> sky -> losses -> backward -> step) against FusedAdam on a clone, taking the marked
    blocks from it and the rest from before the step.
  * Emulated ranks: over peer memory (world 2, 3, 8) and on the band path with an emulated all-reduce, every rank's map holds the same
    bytes, the OR of the ranks' band marks, and after the step every rank's cube and moments are the same bytes.
  * The step captured in a CUDA graph replays the eager step."""
import math

import pytest
import torch

import street_gaussians_b200 as sgb
from rank_threads import run_ranks
from street_gaussians_b200 import _capi, band_losses, losses, sky, synthetic
from street_gaussians_b200 import sharded as SH
from street_gaussians_b200._capi import ptr
from street_gaussians_b200.training import CubeMapSparseAdam, FusedAdam
from test_sky_p2p_gpu import (VARIANTS, W_OF, _frame, _map_bounds, _rows_of, _settings, _stand_in, _texel_terms, _warm_up,
                              _whole)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
F64 = torch.float64
U = 2.0 ** -24
BLOCK = 32
SETTINGS = [dict(lr=0.01, betas=(0.9, 0.999), eps=1e-15), dict(lr=0.3, betas=(0.5, 0.75), eps=1e-3)]


def bits(t):
    return t.contiguous().view(torch.int32)


def _nblk(R):
    return 6 * (-(-R // BLOCK)) ** 2


def _texel_blocks(R):
    nb = -(-R // BLOCK)
    f, r, c = torch.meshgrid(torch.arange(6), torch.arange(R), torch.arange(R), indexing="ij")
    return ((f * nb + r // BLOCK) * nb + c // BLOCK).to(DEV)


def _map(kind, R, gen):
    n, nb = _nblk(R), -(-R // BLOCK)
    m = torch.zeros(n, dtype=torch.uint8, device=DEV)
    if kind == "one":
        m[int(torch.randint(n, (1,), generator=gen, device=DEV))] = 1
    elif kind == "all":
        m.fill_(1)
    elif kind == "edge":  # every face's last block row and column (clipped when 32 does not divide R)
        v = m.view(6, nb, nb)
        v[:, -1, :] = 7
        v[:, :, -1] = 255
    elif kind == "random":
        m = (torch.rand(n, generator=gen, device=DEV) < 0.3).to(torch.uint8)
    return m


def _fused_step(p0, g, m0, v0, step, hp):
    """FusedAdam's step `step` (1-based) on clones of p0 / m0 / v0 with gradient g."""
    q = torch.nn.Parameter(p0.clone())
    q.grad = g.clone()
    fa = FusedAdam([q], **hp)
    fa.state[q] = dict(step=step - 1, exp_avg=m0.clone(), exp_avg_sq=v0.clone())
    fa.step()
    return q.detach(), fa.state[q]["exp_avg"], fa.state[q]["exp_avg_sq"]


@pytest.mark.parametrize("hp", range(len(SETTINGS)))
@pytest.mark.parametrize("R", [1, 31, 32, 40, 64, 1024])
def test_marked_blocks_are_fused_adam_and_the_rest_is_untouched(R, hp):
    hp = SETTINGS[hp]
    gen = torch.Generator(device=DEV).manual_seed(R * 7 + int(hp["lr"] * 100))
    tb = _texel_blocks(R).unsqueeze(-1).expand(6, R, R, 3)
    for kind in ("empty", "one", "all", "edge", "random"):
        for step in (1, 3, 7):
            p0 = torch.randn(6, R, R, 3, generator=gen, device=DEV)
            m0 = 0.1 * torch.randn(6, R, R, 3, generator=gen, device=DEV)
            v0 = 0.01 * torch.rand(6, R, R, 3, generator=gen, device=DEV)
            g = torch.randn(6, R, R, 3, generator=gen, device=DEV)
            blocks = _map(kind, R, gen)
            marked = blocks.bool()[tb]
            want_p, want_m, want_v = _fused_step(p0, g, m0, v0, step, hp)
            nan = torch.full_like(p0, float("nan"))
            p = torch.nn.Parameter(p0.clone())
            p.grad = torch.where(marked, g, nan)
            opt = CubeMapSparseAdam([p], **hp)
            opt.state[p] = dict(step=step - 1, exp_avg=torch.where(marked, m0, nan), exp_avg_sq=torch.where(marked, v0, nan))
            before = [bits(t).clone() for t in (p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])]
            opt.step(blocks)
            torch.cuda.synchronize()
            got = (p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])
            for name, x, want, b in zip(("param", "exp_avg", "exp_avg_sq"), got, (want_p, want_m, want_v), before):
                assert torch.equal(bits(x)[marked], bits(want)[marked]), (kind, step, name)
                assert torch.equal(bits(x)[~marked], b[~marked]), (kind, step, name)
                if kind == "all":
                    assert torch.equal(bits(x), bits(want)), (kind, step, name)
            assert not bool(torch.isnan(p.detach()[marked]).any())
            assert opt.state[p]["step"] == step
            assert not bool(blocks.any()), (kind, step)


def test_state_dict_round_trips_and_steps_count():
    R = 40
    gen = torch.Generator(device=DEV).manual_seed(3)
    p0 = torch.randn(6, R, R, 3, generator=gen, device=DEV)
    grads = [torch.randn(6, R, R, 3, generator=gen, device=DEV) for _ in range(4)]
    hp = SETTINGS[0]
    ref = torch.nn.Parameter(p0.clone())
    fr = FusedAdam([ref], **hp)
    for gr in grads:
        ref.grad = gr.clone()
        fr.step()
    p = torch.nn.Parameter(p0.clone())
    fa = FusedAdam([p], **hp)
    p.grad = grads[0].clone()
    fa.step()
    cs = CubeMapSparseAdam([p], **hp)
    cs.load_state_dict(fa.state_dict())
    blocks = sky.block_map(R, DEV)
    for k in (1, 2):
        p.grad = grads[k].clone()
        blocks.fill_(1)
        cs.step(blocks)
        assert cs.state[p]["step"] == k + 1
    fb = FusedAdam([p], **hp)
    fb.load_state_dict(cs.state_dict())
    p.grad = grads[3].clone()
    fb.step()
    assert fb.state[p]["step"] == 4
    assert torch.equal(bits(p.detach()), bits(ref.detach()))
    for k in ("exp_avg", "exp_avg_sq"):
        assert torch.equal(bits(fb.state[p][k]), bits(fr.state[ref][k]))
    # no gradient: nothing changes, the map included
    p.grad = None
    blocks.fill_(1)
    before = bits(p.detach()).clone()
    cs.step(blocks)
    assert cs.state[p]["step"] == 3 and torch.equal(bits(p.detach()), before) and bool(blocks.all())


def test_step_refuses_a_map_on_another_device_or_a_changed_cube():
    p = torch.nn.Parameter(torch.zeros(6, 8, 8, 3, device=DEV))
    p.grad = torch.ones_like(p)
    opt = CubeMapSparseAdam([p], eps=1e-15)
    with pytest.raises(_capi.SgrError):
        opt.step(sky.block_map(8, "cpu"))
    assert not opt.state


# ---- the marks --------------------------------------------------------------------------------------------------------------------
def _marked_whole(x, blocks):
    rgb, acc, cube = (x[k].clone().requires_grad_(True) for k in ("rgb", "acc", "cube"))
    if x["jitter"]:
        torch.manual_seed(x["seed"])
    out = sgb.sky_composite(rgb, acc, cube, x["K"], x["w2c"], sky_mask=x["mask"], perturb=x["jitter"], white_background=x["fill"] == 1.0,
                            blocks=blocks)
    out.backward(x["up"])
    return dict(out=out.detach(), rgb=rgb.grad, acc=acc.grad, cube=cube.grad)


@pytest.mark.parametrize("R", [16, 100, 1024])
@pytest.mark.parametrize("H", [375, 1280])
def test_whole_frame_marks(H, R):
    frames = [_frame(H, R, 3 * R + H, "edge", VARIANTS[(R + H) % 4]), _frame(H, R, 5 * R + H, "corner", VARIANTS[(R + H + 1) % 4])]
    acc_map = sky.block_map(R, DEV)
    singles = []
    for x in frames:
        ref = _whole(x)
        blocks = sky.block_map(R, DEV)
        got = _marked_whole(x, blocks)
        assert torch.equal(bits(got["out"]), bits(ref["out"])) and torch.equal(bits(got["rgb"]), bits(ref["rgb"]))
        assert torch.equal(bits(got["acc"]), bits(ref["acc"]))
        n, sabs = _texel_terms(x, ref)
        err = (got["cube"].to(F64) - ref["cube"].to(F64)).abs()
        assert bool((err <= 2 * n * U * sabs * (1 + 1e-3) + 1e-30).all())
        lo, hi = _map_bounds(x, ref, _rows_of(H, None))
        assert int(blocks.max()) == 1
        marked = set(torch.nonzero(blocks).view(-1).tolist())
        assert lo and lo <= marked <= hi, (len(lo - marked), len(marked - hi))
        # the map covers every texel the gradient moved
        assert not bool(got["cube"][~blocks.bool()[_texel_blocks(R)]].any())
        singles.append(blocks)
        _marked_whole(x, acc_map)  # accumulate both frames' marks into one map
    assert torch.equal(acc_map, singles[0] | singles[1])
    if R > 16:  # a face edge and a cube corner sample different blocks
        assert not torch.equal(singles[0], singles[1])


def test_no_blocks_without_a_cube_gradient():
    x = _frame(375, 64, 1, "edge", VARIANTS[0])
    blocks = sky.block_map(64, DEV)
    rgb, acc = x["rgb"].clone().requires_grad_(True), x["acc"].clone().requires_grad_(True)
    sgb.sky_composite(rgb, acc, x["cube"], x["K"], x["w2c"], blocks=blocks).backward(x["up"])
    assert not bool(blocks.any())
    with pytest.raises(ValueError, match="blocks"):
        sgb.sky_composite(rgb, acc, x["cube"], x["K"], x["w2c"], blocks=sky.block_map(65, DEV))


# ---- a short training loop ------------------------------------------------------------------------------------------------------
def _yaw(w2c, a):
    """w2c with the camera turned by `a` radians about its own vertical axis."""
    Rz = torch.eye(4, device=DEV)
    c, s = math.cos(a), math.sin(a)
    Rz[0, 0], Rz[0, 2], Rz[2, 0], Rz[2, 2] = c, s, -s, c
    return (Rz @ w2c).contiguous()


def test_training_loop_against_fused_adam_on_the_marked_blocks():
    """compose -> GaussianRasterizer -> sky_composite(blocks=) -> photometric + sky loss -> backward -> CubeMapSparseAdam.step, with the
    sky camera yawed between iterations, each step checked against FusedAdam on a clone of (p, m, v)."""
    Hs, Ws, R = 320, 480, 128
    sc = synthetic.make_scene(P=20000, width=Ws, height=Hs, sh_degree=3, seed=4, n_vehicles=2, per_vehicle=2000, with_raw=True, scale_med=0.05)
    raw, cam = sc["raw"], sc["cam"]
    st = sgb.GaussianRasterizationSettings(image_height=Hs, image_width=Ws, tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"], bg=torch.zeros(3, device=DEV),
                                           scale_modifier=1.0, viewmatrix=cam["viewmatrix"].to(DEV), projmatrix=cam["projmatrix"].to(DEV),
                                           sh_degree=cam["sh_degree"], campos=cam["campos"].to(DEV), prefiltered=False, debug=False)
    fx, fy = Ws / (2 * cam["tanfovx"]), Hs / (2 * cam["tanfovy"])
    K = torch.tensor([[fx, 0, Ws / 2], [0, fy, Hs / 2], [0, 0, 1.0]], device=DEV)
    w2c0 = cam["viewmatrix"].to(DEV).T.contiguous()
    g = torch.Generator(device=DEV).manual_seed(9)
    gt = torch.rand(3, Hs, Ws, generator=g, device=DEV)
    sky_mask = torch.rand(1, Hs, Ws, generator=g, device=DEV) < 0.3
    cube = torch.nn.Parameter(0.5 + 0.2 * torch.rand(6, R, R, 3, generator=g, device=DEV))
    opt = CubeMapSparseAdam([cube], lr=0.01, eps=1e-15)
    blocks = sky.block_map(R, DEV)
    rast = sgb.GaussianRasterizer(st)
    models = [{k: v.to(DEV) for k, v in m.items()} for m in raw["models"]]
    xyz, rot, scale, opac, sh = sgb.compose(models, raw["poses"].to(DEV), raw["idft"].to(DEV))
    tb = _texel_blocks(R).unsqueeze(-1).expand(6, R, R, 3)
    seen = []
    for it in range(4):
        w2c = _yaw(w2c0, 0.35 * it)
        res = rast(means3D=xyz, means2D=torch.zeros_like(xyz, requires_grad=True), opacities=opac, shs=sh, scales=scale, rotations=rot)
        rgb, acc = res[0], res[3]
        cube.grad = None
        out = sgb.sky_composite(rgb, acc, cube, K, w2c, sky_mask=sky_mask, blocks=blocks)
        loss = losses.photometric_loss(out, gt, None, 1.0, 0.2) + losses.sky_loss(acc, sky_mask, 1.0)
        loss.backward()
        marked = blocks.bool()[tb]
        seen.append(blocks.clone())
        p0 = cube.detach().clone()
        st_ = opt.state[cube]
        m0 = st_["exp_avg"].clone() if st_ else torch.zeros_like(p0)
        v0 = st_["exp_avg_sq"].clone() if st_ else torch.zeros_like(p0)
        want = _fused_step(p0, cube.grad, m0, v0, it + 1, dict(lr=0.01, eps=1e-15))
        opt.step(blocks)
        torch.cuda.synchronize()
        assert opt.state[cube]["step"] == it + 1 and not bool(blocks.any())
        for x, w, b in zip((cube.detach(), opt.state[cube]["exp_avg"], opt.state[cube]["exp_avg_sq"]), want, (p0, m0, v0)):
            assert torch.equal(bits(x), bits(torch.where(marked, w, b))), it
        assert 0 < int(marked.sum()) < marked.numel()
    assert not torch.equal(seen[0], seen[-1])  # the yaw moved the sampled blocks


# ---- emulated ranks ---------------------------------------------------------------------------------------------------------------
_warm = []


def _warm_up_union():
    """tests/test_sky_p2p_gpu.py's warm-up, plus the exchange that writes the union: two ranks' calls enqueued one after the other from
    this thread, so its gather kernel loads while no emulated rank spins in a barrier."""
    if _warm:
        return
    _warm_up()
    R = 16
    wss = SH.PeerWorkspace.emulate(_settings(375, W_OF[375]), 8, 2, DEV)
    skys = SH.SkyWorkspace.emulate(R, 2, DEV)
    g = [torch.zeros(6, R, R, 3, device=DEV) for _ in range(2)]
    u = [sky.block_map(R, DEV) for _ in range(2)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(2)]
    torch.cuda.synchronize()
    for r in range(2):
        with torch.cuda.stream(streams[r]):
            skys[r].block_map.zero_()
            sky.sky_grad_peer_sum(wss[r], skys[r], g[r], u[r])
    torch.cuda.synchronize()
    _warm.append(True)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_peer_memory_union_and_step_on_every_rank(world):
    _warm_up_union()
    H, R = 375, 100
    W = W_OF[H]
    wss = SH.PeerWorkspace.emulate(_settings(H, W), 8, world, DEV)
    skys = SH.SkyWorkspace.emulate(R, world, DEV)
    bands = [SH.cyclic_band(H, r, world) for r in range(world)]
    rows = [_rows_of(H, b) for b in bands]
    ris = [_stand_in(wss[r], skys[r], bands[r]) for r in range(world)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    frames = [_frame(H, R, 40 + world, "edge", VARIANTS[0]), _frame(H, R, 50 + world, "corner", VARIANTS[2])]
    cube0 = frames[0]["cube"]
    cubes = [torch.nn.Parameter(cube0.clone()) for _ in range(world)]
    opts = [CubeMapSparseAdam([c], lr=0.05, eps=1e-15) for c in cubes]
    blocks = [sky.block_map(R, DEV) for _ in range(world)]
    union = torch.zeros_like(blocks[0])
    for x in frames:  # two backward passes accumulate into the maps before one step
        torch.cuda.synchronize()
        per = []
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                rgb = torch.where(rows[r].view(1, -1, 1), x["rgb"], torch.zeros_like(x["rgb"])).requires_grad_(True)
                acc = torch.where(rows[r].view(1, -1, 1), x["acc"], torch.zeros_like(x["acc"])).requires_grad_(True)
                out = sgb.sky_composite(rgb, acc, cubes[r], x["K"], x["w2c"], sky_mask=x["mask"], white_background=x["fill"] == 1.0,
                                        rasterizer=ris[r], blocks=blocks[r])
                per.append((out, torch.where(rows[r].view(1, -1, 1), x["up"], torch.zeros_like(x["up"]))))
        torch.cuda.synchronize()

        def rank(r, _tr):
            with torch.cuda.stream(streams[r]):
                torch.autograd.backward([per[r][0]], [per[r][1]])

        run_ranks(world, rank)
        torch.cuda.synchronize()
        for r in range(world):  # the band's own marks of this pass
            union |= skys[r].block_map.bool().to(torch.uint8)
        for r in range(world):
            assert torch.equal(blocks[r], union), r
        assert int(union.max()) == 1 and bool(union.any())
    for r in range(world):
        assert torch.equal(bits(cubes[r].grad), bits(cubes[0].grad)), r

    def step(r, _tr):
        with torch.cuda.stream(streams[r]):
            opts[r].step(blocks[r])

    run_ranks(world, step)
    torch.cuda.synchronize()
    moved = (cubes[0].detach() != cube0).any(-1)
    assert bool(moved.any())
    for r in range(world):
        assert not bool(blocks[r].any())
        assert torch.equal(bits(cubes[r].detach()), bits(cubes[0].detach())), r
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(bits(opts[r].state[cubes[r]][k]), bits(opts[0].state[cubes[0]][k])), (r, k)


class _EmulatedAllReduce:
    """band_losses.all_reduce_sum for ranks emulated one after the other (autograd runs a CUDA backward on its device thread, so ranks
    in threads could not block on each other inside it).  A recording pass keeps every rank's tensor of every call; the second pass
    writes into each rank's tensor of call k the ascending-rank sum of the recorded tensors of call k, so every rank gets the same bytes."""

    def __init__(self):
        self.calls, self.totals, self.k = [], None, 0

    def next_rank(self):
        if self.totals is None:
            self.calls.append([])
        self.k = 0

    def freeze(self):
        self.totals = []
        for k in range(len(self.calls[0])):
            total = self.calls[0][k].clone()
            for rank_calls in self.calls[1:]:
                total += rank_calls[k]
            self.totals.append(total)

    def __call__(self, t, group=None):
        if self.totals is None:
            self.calls[-1].append(t.clone())
        else:
            t.copy_(self.totals[self.k])
            self.k += 1
        return t


@pytest.mark.parametrize("world", [2, 3, 5])
def test_band_path_leaves_the_union_on_every_rank(world, monkeypatch):
    H, R = 375, 96
    W = W_OF[H]
    reduce = _EmulatedAllReduce()
    monkeypatch.setattr(band_losses, "all_reduce_sum", reduce)
    bands = [SH.contiguous_band(H, r, world) for r in range(world)]  # bands of distinct rows see distinct blocks
    rows = [_rows_of(H, b) for b in bands]
    x = _frame(H, R, 70 + world, "corner", VARIANTS[3 if world % 2 else 2])
    mode = _capi.SKY_MASK_GIVEN if x["mask"] is not None else _capi.SKY_MASK_ACC
    mask = x["mask"].to(torch.uint8).contiguous() if x["mask"] is not None else None
    banded = lambda t, r: torch.where(rows[r].view(1, -1, 1), t, torch.zeros_like(t))  # noqa: E731
    own = []
    for r in range(world):  # each band's own marks through the marking entry
        m = torch.full((_nblk(R),), 0xff, dtype=torch.uint8, device=DEV)
        _capi.call("sgr_band_sky_composite_backward_marked", DEV, H, W, *bands[r], R, mode, x["fill"], ptr(banded(x["acc"], r)), ptr(mask),
                   ptr(x["cube"]), ptr(x["K"]), ptr(x["w2c"]), None, None, ptr(banded(x["up"], r)), None, ptr(torch.zeros_like(x["cube"])),
                   ptr(m))
        own.append(m)
    want = torch.stack(own).bool().any(0).to(torch.uint8)
    assert bool(want.any()) and not all(torch.equal(o, want) for o in own)

    def rank(r, blocks):
        reduce.next_rank()
        rgb, acc = banded(x["rgb"], r).requires_grad_(True), banded(x["acc"], r).requires_grad_(True)
        cube = x["cube"].clone().requires_grad_(True)
        out = sgb.sky_composite(rgb, acc, cube, x["K"], x["w2c"], sky_mask=x["mask"], white_background=x["fill"] == 1.0, band=bands[r],
                                blocks=blocks)
        torch.autograd.backward([out], [banded(x["up"], r)])
        return cube.grad

    for r in range(world):  # the recording pass, on throwaway maps
        rank(r, sky.block_map(R, DEV))
    reduce.freeze()
    assert len(reduce.totals) == 2  # the cube gradient, then the marks
    blocks = [sky.block_map(R, DEV) for _ in range(world)]
    grads = [rank(r, blocks[r]) for r in range(world)]
    torch.cuda.synchronize()
    for r in range(world):
        assert torch.equal(blocks[r], want), r
        assert torch.equal(bits(grads[r]), bits(grads[0])), r


# ---- CUDA graph -------------------------------------------------------------------------------------------------------------------
def test_step_captured_in_a_cuda_graph_replays_the_eager_step():
    R = 64
    gen = torch.Generator(device=DEV).manual_seed(11)
    p = torch.nn.Parameter(torch.randn(6, R, R, 3, generator=gen, device=DEV))
    p.grad = torch.randn(6, R, R, 3, generator=gen, device=DEV)
    opt = CubeMapSparseAdam([p], lr=0.02, eps=1e-15)
    blocks = sky.block_map(R, DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        blocks.fill_(1)
        opt.step(blocks)  # first step: the moments are allocated outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step(blocks)  # step 2 baked into the graph
    assert opt.state[p]["step"] == 2
    for kind in ("random", "edge"):
        g_new = torch.randn(6, R, R, 3, generator=gen, device=DEV)
        m_new = _map(kind, R, gen)
        ref_p = torch.nn.Parameter(p.detach().clone())
        ref_p.grad = g_new.clone()
        ref = CubeMapSparseAdam([ref_p], lr=0.02, eps=1e-15)
        ref.state[ref_p] = dict(step=1, exp_avg=opt.state[p]["exp_avg"].clone(), exp_avg_sq=opt.state[p]["exp_avg_sq"].clone())
        ref_map = m_new.clone()
        ref.step(ref_map)
        p.grad.copy_(g_new)
        blocks.copy_(m_new)
        graph.replay()
        torch.cuda.synchronize()
        assert not bool(blocks.any())
        assert torch.equal(bits(p.detach()), bits(ref_p.detach())), kind
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(bits(opt.state[p][k]), bits(ref.state[ref_p][k])), (kind, k)
