"""The fp64 per-element tier of the Gaussian-sharded step: the fused calls (sgr_sharded_forward / sgr_sharded_backward), the staged
calls (project -> forward_records -> backward_blend_records with a sum + slice standing in for the NCCL reduce-scatter, and the
peer-memory scatter_records / gather_grad2d) and the autograd module, with N ranks emulated on N streams of one GPU, on the scenes of
tests/sharded64_case.py (block run totals 0 .. 256 world, depth ties across ranks, empty bands, padding tail / middle / whole rank).

Exact (no tolerance), per rank: the status words (no barrier timeout, no overflow), n_sel = the visible Gaussians whose tile rectangle
meets the band (from the kernel's own records), the instance count = that of the single-GPU forward restricted to the same band (the
same exact tile culling) and at most the rectangles' pairs inside the band, radii, zero gradients of culled Gaussians, images zero
outside the band and summing over the ranks to the single-GPU render bit for bit.

Per element, against float64 (oracle/raster64.py).  blend64 is fed the kernel's own fp32 records and the rendered alpha image
(T_final), so it restates exactly the sums the ranks' blend_bwd2 computes.  Each rank's partial row of Gaussian g is an fp32 sum over
the pixels of its band; blend64's bound 2^-24 (kmass + ntiles mass) covers the per-pixel terms and the one float atomic per tile and
component, whichever band a tile falls in (the partial sums of the ranks partition the terms of the single-GPU sum).  The gather then
adds at most `world` partial rows in fp32 in ascending rank order: each addition rounds once, by at most 2^-24 of a partial sum's
magnitude <= mass.  So a grad2d element is within
    B2d = 2^-24 (kmass + ntiles mass + world mass)            (sharded64_case.sharded_bound)
and g_means2D = grad2d[0..2] is checked against it directly.  The chain rule (preprocess_bwd, K_CHAIN roundings) then runs on that
gathered row; chain64 carries B2d through the per-Gaussian Jacobian (mass2d = mass, kmass2d = kmass + (ntiles + world) mass), and
chain_bound adds the chain's own roundings: every parameter gradient is within chain_bound(chain64(pre, blend64 grad2d, ...)).
Dropping a round of the gather, reading a row from the wrong slot, adding a rank's partial twice or breaking a depth tie the other way
moves an element by a whole term, far above these bounds (test_sharded64_cpu.py shows the float64 side is that sensitive)."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

import sharded64_case as SC
import util
from oracle import raster64 as R64
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi, synthetic
from street_gaussians_b200 import rasterizer as R
from street_gaussians_b200 import sharded as SH

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
F64 = torch.float64
REPORT = {}
GRAD_NAMES = ["g_means3D", "g_means2D", "g_shs", "g_colors_precomp", "g_opacities", "g_scales", "g_rotations", "g_cov3D_precomp"]
_warm = []


def _warm_up_fused_path(dev):
    """Load every kernel of the fused Gaussian-sharded step BEFORE ranks are emulated on one GPU.  The emulation keeps the spinning
    barrier kernel of "rank 0" resident while the host enqueues "rank 1"; with CUDA's lazy module loading the first launch of a kernel
    loads it at launch time, which synchronises the context, i.e. waits for the spinning kernel, which waits for work the blocked host
    thread has not enqueued yet (resolved only by the barrier's 2 s bound).  Every gather variant is loaded here too: SH degree 3
    (TMA), 0 and 2 (staged), colors_precomp with cov3D_precomp (unstaged)."""
    if _warm:
        return
    for D, pre in ((3, False), (0, False), (2, False), (0, True)):
        scene = synthetic.make_scene(P=3000, width=160, height=96, sh_degree=D, seed=1, pose=True)
        if pre:
            scene = SC.to_precomp(scene)
        st = util.settings_from(sgb, scene["cam"], dev)
        dv = lambda k: scene[k].to(dev) if scene.get(k) is not None else None
        lt = SH._local_tensors(dv("means3D"), dv("shs"), dv("colors_precomp"), None, dv("opacities"), dv("scales"), dv("rotations"),
                               dv("cov3D_precomp"))
        up = [scene[k].to(dev) for k in ("grad_color", "grad_depth", "grad_alpha")]
        with torch.no_grad():
            for gcap in (3000, -1):
                ws = SH.PeerWorkspace.emulate(st, 3000, 1, dev)[0]
                col, dep, alp, _ = SH.sharded_forward_raw(st, None, ws, lt, 3000, 500_000, gcap)
                SH.sharded_backward_raw(st, None, ws, lt, 3000, 500_000, alp, *up)
    pair = SH.PeerWorkspace.emulate(st, 8, 2, dev)  # the barrier kernel itself: nothing spins yet when rank 0's launch loads it
    streams = [torch.cuda.Stream(device=dev) for _ in range(2)]
    torch.cuda.synchronize()
    for r in range(2):
        with torch.cuda.stream(streams[r]):
            _capi.check(_capi.lib().sgr_peer_barrier(C.byref(pair[r].peers), 1, C.c_void_p(streams[r].cuda_stream)), "sgr_peer_barrier")
    torch.cuda.synchronize()
    _warm.append(True)


def _dv(scene, k, lo=None, hi=None):
    v = scene.get(k)
    if v is None:
        return None
    return (v if lo is None else v[lo:hi]).to(DEV).contiguous().clone()  # a rank's own, separately allocated tensors


def _local(scene, lo, hi):
    return SH._local_tensors(*(_dv(scene, k, lo, hi) for k in ("means3D", "shs", "colors_precomp")), None,
                             *(_dv(scene, k, lo, hi) for k in ("opacities", "scales", "rotations", "cov3D_precomp")))


def _single(scene, st, band=None, semantics=None):
    with torch.no_grad():
        return R._forward_impl(_dv(scene, "means3D"), _dv(scene, "shs"), _dv(scene, "colors_precomp"), semantics, _dv(scene, "opacities"),
                               _dv(scene, "scales"), _dv(scene, "rotations"), _dv(scene, "cov3D_precomp"), st, band)


def gather_variant(lt, g_sh, no_tma):
    """Which kernel launch_preprocess_bwd runs with a peer table (bwd_rows_fit_tma restated): TMA rows for M in {4, 8, 12, 16} with 16-B aligned
    SH in / out, the staged kernel for the other M <= 16 (and under SGR_NO_TMA), the unstaged one without SH (colors_precomp)."""
    sh = lt["sh"]
    if sh is None:
        return "unstaged"
    M = int(sh.shape[1])
    if not no_tma and 0 < M <= 16 and (M * 12) % 16 == 0 and sh.data_ptr() % 16 == 0 and g_sh.data_ptr() % 16 == 0:
        return "tma"
    return "staged"


def band_mask(H, r, world):
    return SH.band_of_rows(H, r, world).to(DEV)


def _ratio(worst, key, err, bnd, what):
    r = float((err / (bnd + 1e-300)).max()) if err.numel() else 0.0
    worst[key] = max(worst.get(key, 0.0), r)
    assert bool((err <= bnd).all()), (what, key, r, torch.nonzero(err > bnd)[:6].tolist())


def check_against_fp64(tag, scene, rec, radii, alpha, kg, world, worst):
    """kg: the kernel's gradients of all Gaussians (rank-major) by GRAD_NAMES key.  Per element against chain64(blend64 grad2d)."""
    cam = scene["cam"]
    W, H = int(cam["image_width"]), int(cam["image_height"])
    up = dict(color=scene["grad_color"], depth=scene["grad_depth"], alpha=scene["grad_alpha"])
    bl = R64.blend64(rec.double(), radii, W, H, cam["bg"], upstream=up, alpha_img=alpha)
    pre = R64.preprocess64(scene, DEV, requires_grad=True)
    assert torch.equal(pre["radii"].to(torch.int32), radii), (tag, "radii vs preprocess64")
    vis = radii > 0
    nt = bl["ntiles"].to(F64)[:, None]
    ch = R64.chain64(pre, bl["grad2d"], bl["mass_grad2d"], bl["kmass_grad2d"] + (nt + world) * bl["mass_grad2d"])
    n = 0
    for key, got in kg.items():
        if got is None:
            continue
        assert bool((got[~vis] == 0).all()), (tag, key, "gradient of a culled Gaussian")
        if key == "g_means2D":
            err = (got.double() - bl["grad2d"][:, 0:3]).abs()
            bnd = SC.sharded_bound(bl, world)[:, 0:3]
        else:
            ref = ch[key]
            err = (got.double().reshape(ref.shape) - ref).abs()
            bnd = R64.chain_bound(ch, key)
        _ratio(worst, key, err, bnd, tag)
        n += 1
    assert n >= 5
    return bl


def tie_check(case, rec, radii, bl, alpha):
    """The depth ties of the case: bit-identical view depth in the kernel's records, different owners, and blending them in the other
    order moves the image by more than the bound (so a wrong tie order could not pass)."""
    cam = case["scene"]["cam"]
    W, H = case["W"], case["H"]
    for a, b in case["ties"]:
        assert rec[a, 7].item() == rec[b, 7].item() and int(case["owner_of"][a]) != int(case["owner_of"][b])
        perm = torch.arange(rec.shape[0], device=rec.device)
        perm[a], perm[b] = b, a
        sw = R64.blend64(rec[perm].double(), radii[perm], W, H, cam["bg"])
        gap = float(((sw["color"] - bl["color"]).abs() / (R64.bound(bl["kmass_color"]) + 1e-300)).max())
        assert gap > 1e3, ("tie swap is not detectable", a, b, gap)


def run_fused(name, D=3, precomp=False, compact=True, frames=2, no_tma=False, expect=None):
    """Two frames of `name` (seeds 0, 1; same chunk), each forward + backward on emulated ranks (compact: first with every
    depth-order slot, then with the learnt n_sel + 16), then two forwards in a row."""
    _warm_up_fused_path(DEV)
    cases = [SC.build(name, seed=f, D=D, device=DEV) for f in range(frames)]
    world, chunk, W, H = cases[0]["world"], cases[0]["chunk"], cases[0]["W"], cases[0]["H"]
    st = util.settings_from(sgb, cases[0]["scene"]["cam"], DEV)
    wss = SH.PeerWorkspace.emulate(st, chunk, world, DEV)
    for ws in wss:
        ws.buf[: ws.off_flags].fill_(0x7f)  # poison all but the barrier pads: no array needs a particular content on entry
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    worst, variants, classes = {}, set(), set()
    for fi, case in enumerate(cases):
        scene = dict(case["scene"])
        if precomp:
            scene, removed, _ = R64.margin_scene(SC.to_precomp(scene, seed=fi), device=DEV)
            assert removed == 0, (name, "the precomputed-covariance scene is not margin-clean", removed)
        classes |= SC.total_classes(case["totals"], world)
        assert SC.total_classes(case["totals"], world) >= case["claims"], (name, case["totals"])
        P_r = case["P_r"]
        offs = [sum(P_r[:r]) for r in range(world)]
        st = util.settings_from(sgb, scene["cam"], DEV)
        locs = [_local(scene, offs[r], offs[r] + P_r[r]) for r in range(world)]
        up = [scene[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
        col, rad, dep, alp, _, fst, _ = _single(scene, st)
        R_band = [int(_single(scene, st, SH.cyclic_band(H, r, world))[5].num_instances) for r in range(world)]
        capacity = int(fst.num_instances) + 1000
        n_sel_rank = [0] * world
        checked = False
        for ps in range(2 if compact else 1):
            tag = f"{name} frame {fi} pass {ps}"
            status = [torch.zeros(8, dtype=torch.int32).pin_memory() for _ in range(world)]
            outs = []
            torch.cuda.synchronize()
            with torch.no_grad():
                for r in range(world):
                    gcap = -1 if not compact else (chunk * world if ps == 0 else n_sel_rank[r] + 16)
                    with torch.cuda.stream(streams[r]):
                        outs.append(SH.sharded_forward_raw(st, SH.cyclic_band(H, r, world), wss[r], locs[r], P_r[r], capacity, gcap, status[r]))
                torch.cuda.synchronize()
                rec = torch.cat([o[3]["rec"][:n].clone() for o, n in zip(outs, P_r)])
                radii = torch.cat([o[3]["radii"][:n].clone() for o, n in zip(outs, P_r)])
                imgs = [torch.stack([o[i] for o in outs]) for i in range(3)]
            # ---- exact ----
            assert torch.equal(radii, rad), (tag, "radii")
            assert torch.equal(rec[:, 11].contiguous().view(torch.int32) >> 3, radii), (tag, "radius packed in the record")
            n_exp, pairs_exp = SC.expected_counts(rec[:, 0].cpu(), rec[:, 1].cpu(), radii.cpu(), W, H, world)
            for r in range(world):
                R_r, over, emitted, n_sel, timed_out = (int(v) for v in status[r][:5])
                assert timed_out == 0, f"{tag}, rank {r}: the device barrier of epoch {timed_out} timed out"
                assert over == 0, (tag, r, over)
                assert n_sel == n_exp[r], (tag, r, n_sel, n_exp[r])
                assert R_r == emitted == R_band[r] and R_r <= pairs_exp[r], (tag, r, R_r, emitted, R_band[r], pairs_exp[r])
                n_sel_rank[r] = n_sel
                outside = ~band_mask(H, r, world)
                for i in range(3):
                    assert float(imgs[i][r][:, outside].abs().max()) == 0.0 if bool(outside.any()) else True, (tag, r, "outside the band")
            for i, (ref, nm) in enumerate(zip((col, dep, alp), ("color", "depth", "alpha"))):
                assert torch.equal(imgs[i].sum(0), ref), f"{tag}: {nm} differs from the single-GPU render"
            assert sum(1 for n in n_exp if n == 0) >= case["empty_bands"]
            # ---- backward ----
            with torch.no_grad():
                grads = []
                for r in range(world):
                    with torch.cuda.stream(streams[r]):
                        grads.append(SH.sharded_backward_raw(st, SH.cyclic_band(H, r, world), wss[r], locs[r], P_r[r], capacity, outs[r][2], *up))
                torch.cuda.synchronize()
            for r in range(world):
                if P_r[r]:
                    variants.add(gather_variant(locs[r], grads[r][2], no_tma))
            # (a rank that owns nothing passes no SH tensor and gets None for g_shs: its zero rows add nothing)
            kg = {k: (torch.cat([g[i] for g in grads if g[i] is not None]) if any(g[i] is not None for g in grads) else None)
                  for i, k in enumerate(GRAD_NAMES)}
            bl = check_against_fp64(tag, scene, rec, radii, alp, kg, world, worst)
            if not checked:
                tie_check(case, rec, radii, bl, alp)
                checked = True
    assert variants == {expect}, (name, variants, expect)
    # a forward after a forward (no backward): the leading barrier is taken (epochs advance by 2), images stay exact
    with torch.no_grad():
        e0 = [ws.epoch for ws in wss]
        for rep in range(2):
            status = [torch.zeros(8, dtype=torch.int32).pin_memory() for _ in range(world)]
            outs = []
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    outs.append(SH.sharded_forward_raw(st, SH.cyclic_band(H, r, world), wss[r], locs[r], P_r[r], capacity, -1, status[r]))
            torch.cuda.synchronize()
            assert all(int(s[4]) == 0 and int(s[1]) == 0 for s in status), "forward after forward"
            assert torch.equal(sum(o[0] for o in outs), col)
        assert [ws.epoch - e for ws, e in zip(wss, e0)] == [3] * world
    REPORT[name] = dict(world=world, chunk=chunk, P_r=cases[0]["P_r"], totals=sorted(set(cases[0]["totals"].values())), classes=sorted(classes),
                        ties=len(cases[0]["ties"]), gather=sorted(variants), **{k: round(v, 4) for k, v in worst.items()})
    print(name, REPORT[name])


FUSED = [("w2_tail_M16", "w2_tail", dict(D=3, compact=True, expect="tma")),
         ("w3_middle_M4", "w3_middle", dict(D=1, compact=False, expect="tma")),
         ("w5_empty_rank_M1", "w5_empty_rank", dict(D=0, compact=True, expect="staged")),
         ("w8_empty_bands_M9", "w8_empty_bands", dict(D=2, compact=True, expect="staged")),
         ("w3_short_row_precomp", "w3_short_row", dict(D=0, precomp=True, compact=False, expect="unstaged"))]


@pytest.mark.parametrize("cid,name,kw", FUSED, ids=[c[0] for c in FUSED])
def test_fused_step_per_element(cid, name, kw):
    """sgr_sharded_forward / sgr_sharded_backward on emulated ranks, world 2, 3, 5, 8, every gather variant (M = 16 and 4: TMA rows;
    M = 1 and 9: the staged kernel; colors_precomp with cov3D_precomp: the unstaged one), compacted and uncompacted depth order."""
    run_fused(name, **kw)


VARIANT_SCRIPT = r"""
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import test_sharded64_gpu as T
T.run_fused("w3_middle", D=3, compact=True, no_tma=True, expect="staged")
print("OK")
"""


def test_fused_step_staged_gather_without_tma():
    """M = 16 under SGR_NO_TMA=1 (read once per process, so in a fresh interpreter): the staged gather kernel at the row width the TMA
    kernel normally takes."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = VARIANT_SCRIPT.format(root=os.path.dirname(here), tests=here)
    p = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, SGR_NO_TMA="1"), capture_output=True, text=True, timeout=900)
    print(p.stdout[-2000:])
    assert p.returncode == 0 and "OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]


STAGED = [("w3_middle", 3), ("w5_empty_rank", 17), ("w8_empty_bands", 0)]


@pytest.mark.parametrize("name,S", STAGED, ids=[f"{n}_S{s}" for n, s in STAGED])
def test_staged_paths_per_element(name, S):
    """The staged calls with feature channels: (1) project_records -> forward_records -> backward_blend_records per rank on the
    rank-major gathered records, partial grad2d / semantics gradients summed in fp32 in rank order and sliced (the NCCL reduce-scatter);
    (2) the peer-memory exchange, scatter_records then gather_grad2d.  Images bit-equal to the single-GPU render; all eleven grad2d
    components and grad_semantics per element against blend64 under the sharded bound; padding slots exactly zero."""
    case = SC.build(name, seed=3, D=1, device=DEV)
    scene = dict(case["scene"])
    world, chunk, W, H, P_r = case["world"], case["chunk"], case["W"], case["H"], case["P_r"]
    P = sum(P_r)
    g = torch.Generator().manual_seed(S + 5)
    sem = torch.rand(P, S, generator=g) if S else None
    gs = (torch.randn(S, H, W, generator=g) / (H * W)) if S else torch.zeros(0, H, W)
    st = util.settings_from(sgb, scene["cam"], DEV)
    offs = [sum(P_r[:r]) for r in range(world)]
    slot_of = torch.cat([r * chunk + torch.arange(n) for r, n in enumerate(P_r)]).to(DEV)
    P_total = chunk * world
    pad = torch.ones(P_total, dtype=torch.bool, device=DEV)
    pad[slot_of] = False
    up = [scene[k].to(DEV) for k in ("grad_color", "grad_depth", "grad_alpha")]
    sem_d = sem.to(DEV) if S else None
    col, rad, dep, alp, se, _, _ = _single(scene, st, semantics=sem_d)
    worst = {}
    with torch.no_grad():
        locs = [_local(scene, offs[r], offs[r] + P_r[r]) for r in range(world)]
        recs, radii = zip(*(SH.project_records(locs[r], st, chunk) for r in range(world)))
        rec_cat, radii_all = torch.cat(recs), torch.cat(radii)
        sem_all = None
        if S:
            sem_all = torch.zeros(P_total, S, device=DEV)
            sem_all[slot_of] = sem_d
        rec, rad_k = rec_cat[slot_of], radii_all[slot_of]
        assert torch.equal(rad_k, rad) and int(radii_all[pad].abs().sum()) == 0
        up_s = dict(color=scene["grad_color"], depth=scene["grad_depth"], alpha=scene["grad_alpha"], semantic=gs if S else None)
        bl = R64.blend64(rec.double(), rad_k, W, H, scene["cam"]["bg"], semantics=sem_d, upstream=up_s, alpha_img=alp)
        b2d = SC.sharded_bound(bl, world)[:, :11]
        # (1) NCCL stand-in
        imgs, g2, gsm = None, None, None
        for r in range(world):
            band = SH.cyclic_band(H, r, world)
            fs, rec_all, gb, ib = SH.alloc_gathered(st, P_total, S, DEV)
            rec_all.copy_(rec_cat)
            out = SH.forward_records(st, band, fs, (gb, ib), radii_all, sem_all)
            imgs = out if imgs is None else tuple(a + b for a, b in zip(imgs, out))
            part, part_sem = SH.backward_blend_records(st, band, fs, P_total, sem_all, out[2], *up, gs.to(DEV))
            g2 = part.clone() if g2 is None else g2 + part
            gsm = part_sem.clone() if gsm is None else gsm + part_sem
        for a, b, nm in zip(imgs, (col, dep, alp, se), ("color", "depth", "alpha", "semantic")):
            assert torch.equal(a, b), f"{name}: staged {nm} differs from the single-GPU render"
        assert float(g2[pad].abs().max()) == 0.0 if bool(pad.any()) else True
        _ratio(worst, "grad2d_nccl", (g2[slot_of, :11].double() - bl["grad2d"][:, :11]).abs(), b2d, name)
        if S:
            bs = R64.bound(bl["kmass_grad_semantics"], bl["mass_grad_semantics"], bl["ntiles"], extra=float(world))
            _ratio(worst, "grad_semantics", (gsm[slot_of].double() - bl["grad_semantics"]).abs(), bs, name)
            assert float(gsm[pad].abs().max()) == 0.0 if bool(pad.any()) else True
        # (2) peer-memory exchange
        wss = SH.PeerWorkspace.emulate(st, chunk, world, DEV)
        for ws in wss:
            ws.buf.fill_(0x7f)
        for r in range(world):
            SH.scatter_records(st, wss[r], recs[r], radii[r], P_r[r])
        imgs = None
        for r in range(world):
            ws = wss[r]
            fs = SH.peer_forward_state(ws)
            band = SH.cyclic_band(H, r, world)
            out = SH.forward_records(st, band, fs, (ws.geom_bytes, ws.img_bytes), ws.radii_all, sem_all)
            imgs = out if imgs is None else tuple(a + b for a, b in zip(imgs, out))
            SH.backward_blend_records(st, band, fs, P_total, sem_all, out[2], *up, gs.to(DEV), grad2d_out=ws.grad2d)
        for a, b, nm in zip(imgs, (col, dep, alp, se), ("color", "depth", "alpha", "semantic")):
            assert torch.equal(a, b), f"{name}: peer-exchange {nm} differs from the single-GPU render"
        g2p = torch.cat([SH.gather_grad2d(st, wss[r], recs[r], radii[r], P_r[r])[:P_r[r]] for r in range(world)])
        _ratio(worst, "grad2d_p2p", (g2p[:, :11].double() - bl["grad2d"][:, :11]).abs(), b2d, name)
    REPORT[f"staged_{name}_S{S}"] = dict(world=world, P_r=P_r, **{k: round(v, 4) for k, v in worst.items()})
    print(f"staged_{name}_S{S}", REPORT[f"staged_{name}_S{S}"])


def test_module_world1_three_frames_per_element():
    """GaussianShardedRasterizer(capacity=InstanceCapacity(), exchange="p2p") at world 1 through torch.autograd, three frames: the staged
    exact path, then the fused path compacted into all slots, then the fused path with the learnt Gaussian capacity.  Radii exact,
    images and every leaf gradient per element against render64 with the bound of test_raster64_gpu.test_end_to_end_autograd
    (t_rec covers the blend being fed fp32 rather than fp64 records)."""
    from street_gaussians_b200.sharded import GaussianShardedRasterizer
    case = SC.build("w2_tail", seed=4, D=3, device=DEV)
    sc = case["scene"]
    W, H = case["W"], case["H"]
    st = util.settings_from(sgb, sc["cam"], DEV)
    cap = sgb.InstanceCapacity()
    mod = GaussianShardedRasterizer(st, capacity=cap, exchange="p2p")
    paths, gcaps = [], []
    for frame in range(3):
        gcaps.append(cap.gaussian_capacity)
        leaves = {k: sc[k].to(DEV).clone().requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
        m2d = torch.zeros(sc["means3D"].shape[0], 3, device=DEV, requires_grad=True)
        color, radii, depth, alpha, _ = mod(means3D=leaves["means3D"], means2D=m2d, opacities=leaves["opacities"], shs=leaves["shs"],
                                            scales=leaves["scales"], rotations=leaves["rotations"])
        paths.append(bool(getattr(color.grad_fn, "fused", False)))
        loss = (color * sc["grad_color"].to(DEV)).sum() + (depth * sc["grad_depth"].to(DEV)).sum() + (alpha * sc["grad_alpha"].to(DEV)).sum()
        loss.backward()
        mod.synchronize_capacity()
        mine = dict(color=color.detach(), depth=depth.detach(), alpha=alpha.detach(), g_means2D=m2d.grad,
                    **{"g_" + k: v.grad for k, v in leaves.items()})
        r = R64.render64(sc, DEV, alpha_img=mine["alpha"])
        assert torch.equal(r["radii"].to(torch.int32), radii), (frame, "radii")
        cond = float(r["pre"]["cond"][r["pre"]["vis"]].max())
        t_rec = R64.EPS32 * 64.0 * (1 + cond) * (1 + max(W, H))
        worst = {}
        bl = r["blend"]
        for key in ("color", "depth", "alpha"):
            _ratio(worst, key, (mine[key].double() - r[key]).abs(), R64.bound(bl["kmass_" + key]) + t_rec * bl["mass_" + key], f"frame {frame}")
        for key in ("g_means3D", "g_means2D", "g_shs", "g_opacities", "g_scales", "g_rotations"):
            ref = r[key]
            got = mine[key].double().reshape(ref.shape)
            if key == "g_means2D":
                got, ref = got[:, :2], ref[:, :2]
                bnd0 = (R64.EPS32 * r["kmass_g_means2D"])[:, :2]
            else:
                bnd0 = R64.chain_bound(r, key)
            rowmax = ref.abs().reshape(ref.shape[0], -1).amax(1).reshape((-1,) + (1,) * (ref.dim() - 1))
            _ratio(worst, key, (got - ref).abs(), bnd0 + t_rec * rowmax, f"frame {frame}")
        REPORT[f"module_frame{frame}"] = dict(fused=paths[-1], **{k: round(v, 4) for k, v in worst.items()})
        print(f"module_frame{frame}", REPORT[f"module_frame{frame}"])
    assert paths == [False, True, True], paths
    assert gcaps[1] is None and gcaps[2] is not None, gcaps
