"""The sky composite and the colour correction on a tile-row band (sgr_band_sky_composite_* / sgr_band_color_correct_*) against the
whole-frame calls, with N ranks emulated on one GPU: every rank calls the library on its banded inputs (its rows, zeros elsewhere) and
the test sums the parameter partials as the all-reduce does.

Per case: the output and image-gradient rows of every rank equal the whole-frame call's bit for bit and its other rows are zero.
  dL/dcube   the texels take float atomics, so the summed partials and the whole-frame gradient are two orders of the same fp32 terms:
             each within (n - 1) u sum |term| of the exact sum for a texel of n terms, so they differ by at most 2 n u sum |term| (u = 2^-24;
             n and sum |term| from the fp64 restatement).  The sum is also held to tests/sky_oracle.py's per-texel bound.
  dL/daffine the band partials are fp64 sums of exact products, rounded once after the ranks' sum: within one fp32 ulp of the fp64
             restatement (tests/correction_oracle.py) at every world size.
Two mutation checks show that the comparison catches a kernel that indexes the band-local row instead of the global one, and one that
drops the last partial tile row."""
import numpy as np
import pytest
import torch

import correction_oracle as CCO
import sky_oracle as SO
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi, band_losses, corrections, synthetic
from street_gaussians_b200._capi import ptr
from street_gaussians_b200.rasterizer import TileRowBand
from street_gaussians_b200.sharded import contiguous_band, cyclic_band
from test_sky_gpu import _look_at

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
F64 = torch.float64
U = 2.0 ** -24
CASES = [(world, layout, H) for world in (1, 2, 3, 5, 8) for layout in ("cyclic", "contiguous") for H in (375, 1280)] + \
        [(8, "cyclic", 80), (8, "contiguous", 40)]  # more ranks than tile rows: empty bands
W_OF = {375: 200, 1280: 1920, 80: 64, 40: 48}
R_SKY = 96
# (mode, fill, jitter): both mask modes, fills 0 and 1, fixed jitter
SKY_VARIANTS = {"acc_fill1": (False, 1.0, False), "acc_fill0_jitter": (False, 0.0, True), "mask_fill1_jitter": (True, 1.0, True),
                "mask_fill0": (True, 0.0, False)}


def _bands(H, world, layout):
    mk = cyclic_band if layout == "cyclic" else contiguous_band
    return [mk(H, r, world) for r in range(world)]


def _rows_of(H, band):
    rows = torch.arange((H + 15) // 16)
    own = (rows >= band.begin) & (rows < band.end) & (((rows - band.begin) % max(band.step, 1)) == 0)
    return own.repeat_interleave(16)[:H].to(DEV)


def _banded(x, rows):
    return torch.where(rows.view(1, -1, 1), x, torch.zeros_like(x))


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---- sky ---------------------------------------------------------------------------------------------------------------------
def _sky_frame(H, W, seed, masked, jitter):
    g = torch.Generator(device=DEV).manual_seed(seed)
    cube = -0.2 + 1.4 * torch.rand(6, R_SKY, R_SKY, 3, generator=g, device=DEV)
    rgb = torch.rand(3, H, W, generator=g, device=DEV)
    acc = torch.rand(1, H, W, generator=g, device=DEV)
    acc = torch.where(torch.rand(1, H, W, generator=g, device=DEV) < 0.5, torch.zeros_like(acc), acc)
    up = torch.randn(3, H, W, generator=g, device=DEV)
    mask = (torch.rand(H, W, generator=g, device=DEV) < 0.3).to(torch.uint8) if masked else None
    jx = torch.rand(H, W, generator=g, device=DEV) if jitter else None
    jy = torch.rand(H, W, generator=g, device=DEV) if jitter else None
    f = 1.1 * W
    K = torch.tensor([[f, 0.0, W / 2], [0.0, f, H / 2], [0.0, 0.0, 1.0]], device=DEV)
    w2c = _look_at([1.0, -0.6, 1.0], 0.2).to(DEV)  # straddles a cube corner
    return dict(cube=cube, rgb=rgb, acc=acc, up=up, mask=mask, jx=jx, jy=jy, K=K, w2c=w2c)


def _sky_whole(f, fill):
    H, W = f["rgb"].shape[1:]
    mode = _capi.SKY_MASK_GIVEN if f["mask"] is not None else _capi.SKY_MASK_ACC
    out = torch.empty_like(f["rgb"])
    _capi.call("sgr_sky_composite_forward", DEV, H, W, R_SKY, mode, fill, ptr(f["rgb"]), ptr(f["acc"]), ptr(f["mask"]), ptr(f["cube"]), ptr(f["K"]),
               ptr(f["w2c"]), ptr(f["jx"]), ptr(f["jy"]), ptr(out))
    gacc, gcube = torch.empty_like(f["acc"]), torch.zeros_like(f["cube"])
    _capi.call("sgr_sky_composite_backward", DEV, H, W, R_SKY, mode, fill, ptr(f["acc"]), ptr(f["mask"]), ptr(f["cube"]), ptr(f["K"]), ptr(f["w2c"]),
               ptr(f["jx"]), ptr(f["jy"]), ptr(f["up"]), ptr(gacc), ptr(gcube))
    return out, gacc, gcube


def _sky_band(f, fill, band, rows):
    """One rank: the band entries on its banded rgb, acc and upstream gradient."""
    H, W = f["rgb"].shape[1:]
    mode = _capi.SKY_MASK_GIVEN if f["mask"] is not None else _capi.SKY_MASK_ACC
    rgb, acc, up = _banded(f["rgb"], rows), _banded(f["acc"], rows), _banded(f["up"], rows)
    b, e, s = band
    out = torch.zeros_like(rgb)
    _capi.call("sgr_band_sky_composite_forward", DEV, H, W, b, e, s, R_SKY, mode, fill, ptr(rgb), ptr(acc), ptr(f["mask"]), ptr(f["cube"]),
               ptr(f["K"]), ptr(f["w2c"]), ptr(f["jx"]), ptr(f["jy"]), ptr(out))
    gacc, gcube = torch.zeros_like(acc), torch.zeros_like(f["cube"])
    _capi.call("sgr_band_sky_composite_backward", DEV, H, W, b, e, s, R_SKY, mode, fill, ptr(acc), ptr(f["mask"]), ptr(f["cube"]), ptr(f["K"]),
               ptr(f["w2c"]), ptr(f["jx"]), ptr(f["jy"]), ptr(up), ptr(gacc), ptr(gcube))
    return out, gacc, gcube


def _texel_terms(f, fill):
    """Per texel of the cube: n, the number of per-pixel terms its atomics add, and sum |term| (fp64 restatement of the kernel's terms)."""
    H, W = f["rgb"].shape[1:]
    d = SO.rays(H, W, f["K"].to(F64), f["w2c"].to(F64), f["jx"], f["jy"])
    face, gx, gy = SO.face_coords(d)
    x, y = SO.tex_xy(gx, gy, R_SKY)
    idx, w = SO.effective(*SO.taps(face, x, y, R_SKY))
    sampled = SO.sky_mask_of(f["acc"], f["mask"].bool() if f["mask"] is not None else None)
    gt = (f["up"].to(F64) * (1 - f["acc"].to(F64))).permute(1, 2, 0) * sampled.unsqueeze(-1)  # [H, W, 3]
    term = (w.unsqueeze(-1) * gt.unsqueeze(-2)).abs()  # [H, W, 4, 3]
    live = (w > 0) & sampled.unsqueeze(-1)
    n = torch.zeros(6 * R_SKY * R_SKY, dtype=F64, device=DEV).index_add_(0, idx.reshape(-1), live.reshape(-1).to(F64))
    sabs = torch.zeros(6 * R_SKY * R_SKY, 3, dtype=F64, device=DEV).index_add_(0, idx.reshape(-1), term.reshape(-1, 3))
    return n.view(6, R_SKY, R_SKY, 1), sabs.view(6, R_SKY, R_SKY, 3)


def _sky_problems(f, fill, ranks, H, ref):
    """What is wrong with the ranks' (rows, out, dacc, dcube) against the whole-frame results `ref`: an empty list when nothing."""
    out_ref, gacc_ref, gcube_ref = ref
    bad = []
    covered = torch.zeros(H, dtype=torch.bool, device=DEV)
    for r, (rows, out, gacc, _) in enumerate(ranks):
        covered |= rows
        if not _bits_equal(out[:, rows], out_ref[:, rows]):
            bad.append(f"rank {r}: rgb_out rows differ")
        if not _bits_equal(gacc[:, rows], gacc_ref[:, rows]):
            bad.append(f"rank {r}: dL/dacc rows differ")
        if bool((~rows).any()) and (bool(out[:, ~rows].any()) or bool(gacc[:, ~rows].any())):
            bad.append(f"rank {r}: foreign rows written")
    if not bool(covered.all()):
        bad.append("rows not covered by any band")
    total = sum(g for _, _, _, g in ranks)
    n, sabs = _texel_terms(f, fill)
    bound = 2 * n * U * sabs * (1 + 1e-3) + 1e-30
    err = (total.to(F64) - gcube_ref.to(F64)).abs()
    if not bool((err <= bound).all()):
        bad.append(f"summed dL/dcube: {int((err > bound).sum())} texels outside the atomic-order bound, worst {float((err / bound).max()):.3g}x")
    return bad


def _sky_run(world, layout, H, variant, band_of=None):
    W = W_OF[H]
    masked, fill, jitter = SKY_VARIANTS[variant]
    f = _sky_frame(H, W, 7 * world + H, masked, jitter)
    ref = _sky_whole(f, fill)
    ranks = []
    for band in _bands(H, world, layout):
        rows = _rows_of(H, band)
        ranks.append((rows,) + _sky_band(f, fill, band_of(band) if band_of else band, rows))
    return f, fill, ranks, ref


@pytest.mark.parametrize("variant", list(SKY_VARIANTS))
@pytest.mark.parametrize("world,layout,H", CASES)
def test_sky_band_matches_whole_frame(world, layout, H, variant):
    f, fill, ranks, ref = _sky_run(world, layout, H, variant)
    assert _sky_problems(f, fill, ranks, H, ref) == []
    assert int((ref[2] != 0).sum()) > 100  # the cube gradient is not trivially zero
    if H == 375 or world == 8:  # the fp64 restatement (memory-heavy at 1280 x 1920: once per layout there)
        total = sum(g for _, _, _, g in ranks)
        r = SO.sky64(f["rgb"], f["acc"], f["cube"], f["K"], f["w2c"], f["up"], f["mask"].bool() if f["mask"] is not None else None, f["jx"], f["jy"],
                     fill)
        err = (total.to(F64) - r["dcube"]).abs()
        assert bool((err <= r["b_dcube"]).all()), f"{int((err > r['b_dcube']).sum())} texels outside the fp64 restatement's bound"


def test_sky_mask_rows_rule_is_global():
    """A band that owns tile rows 0-3 (rows 0-63, the 50-row rule inside it) and one that starts below it, in the mask mode."""
    H, W = 375, 200
    f = _sky_frame(H, W, 3, True, False)
    ref = _sky_whole(f, 0.0)
    bands = [TileRowBand(0, 4, 1), TileRowBand(4, 24, 1)]
    ranks = [(_rows_of(H, b),) + _sky_band(f, 0.0, b, _rows_of(H, b)) for b in bands]
    assert _sky_problems(f, 0.0, ranks, H, ref) == []
    assert not bool(f["mask"][:50].all())  # the rule, not the mask, makes rows 0-49 sample the cube


@pytest.mark.parametrize("world,layout", [(2, "cyclic"), (3, "contiguous"), (5, "cyclic")])
def test_sky_check_catches_band_local_rows(world, layout):
    """Mutation: a kernel that indexed its band's pixels by the band-local row (the band's rows packed into a frame of their own) gives
    other rays and, in the mask mode, another rows-0-49 rule; the comparison reports it."""
    H, W = 375, 200
    f = _sky_frame(H, W, 5, True, False)
    ref = _sky_whole(f, 1.0)
    ranks = []
    for band in _bands(H, world, layout):
        rows = _rows_of(H, band)
        idx = rows.nonzero().squeeze(1)
        Hl = int(idx.numel())
        local = dict(f, rgb=f["rgb"][:, idx].contiguous(), acc=f["acc"][:, idx].contiguous(), up=f["up"][:, idx].contiguous(),
                     mask=f["mask"][idx].contiguous())
        lb = TileRowBand(0, (Hl + 15) // 16, 1)
        out_l, gacc_l, gcube = _sky_band(local, 1.0, lb, _rows_of(Hl, lb)) if Hl else (None, None, torch.zeros_like(f["cube"]))
        out, gacc = torch.zeros_like(f["rgb"]), torch.zeros_like(f["acc"])
        if Hl:
            out[:, idx], gacc[:, idx] = out_l, gacc_l
        ranks.append((rows, out, gacc, gcube))
    assert _sky_problems(f, 1.0, ranks, H, ref) != []


@pytest.mark.parametrize("layout", ["cyclic", "contiguous"])
def test_sky_check_catches_a_dropped_partial_tile_row(layout):
    """Mutation: a kernel that skipped the last tile row when it is partial (H = 375: rows 368-374)."""
    H, rows_n = 375, (375 + 15) // 16
    f, fill, ranks, ref = _sky_run(3, layout, H, "acc_fill1", band_of=lambda b: TileRowBand(b.begin, min(b.end, rows_n - 1), b.step))
    assert _sky_problems(f, fill, ranks, H, ref) != []


# ---- colour correction -------------------------------------------------------------------------------------------------------
CC_CASES = [c + (W_OF[c[2]],) for c in CASES] + [(3, "cyclic", 375, 203), (2, "contiguous", 40, 51)]  # H W % 4 != 0: the scalar path


def _cc_inputs(H, W, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    img = torch.rand(3, H, W, generator=g, device=DEV)
    A = torch.eye(4, device=DEV)[:3] + 0.1 * torch.randn(3, 4, generator=g, device=DEV)
    up = torch.randn(3, H, W, generator=g, device=DEV)
    return img, A, up


def _cc_whole(img, A, up):
    H, W = img.shape[1:]
    out, gimg, gA = torch.empty_like(img), torch.empty_like(img), torch.empty(3, 4, device=DEV)
    _capi.call("sgr_color_correct_forward", DEV, H, W, ptr(img), ptr(A), ptr(out))
    nb = int(_capi.lib().sgr_color_correct_scratch_bytes(H, W))
    scratch = torch.empty(nb, device=DEV, dtype=torch.uint8)
    _capi.call("sgr_color_correct_backward", DEV, H, W, ptr(img), ptr(A), ptr(up), ptr(gimg), ptr(gA), ptr(scratch), nb)
    return out, gimg, gA


def _cc_band(img, A, up, band, rows):
    H, W = img.shape[1:]
    x, g = _banded(img, rows), _banded(up, rows)
    b, e, s = band
    out, gimg = torch.zeros_like(x), torch.zeros_like(x)
    _capi.call("sgr_band_color_correct_forward", DEV, H, W, b, e, s, ptr(x), ptr(A), ptr(out))
    nb = int(_capi.lib().sgr_band_color_correct_scratch_bytes(H, W))
    scratch = torch.empty(nb, device=DEV, dtype=torch.uint8)
    sums = torch.empty(12, device=DEV, dtype=F64)
    _capi.call("sgr_band_color_correct_backward", DEV, H, W, b, e, s, ptr(x), ptr(A), ptr(g), ptr(gimg), ptr(sums), ptr(scratch), nb)
    return out, gimg, sums


def _affine_grad(sums):
    gA = torch.empty(3, 4, device=DEV)
    _capi.call("sgr_band_color_correct_affine_grad", DEV, ptr(sums), ptr(gA))
    return gA


def _within_ulp(got, exact):
    """|got - exact| <= one fp32 ulp of |exact|, element by element."""
    e = exact.detach().cpu().double().numpy()
    sp = np.spacing(np.abs(e).astype(np.float32)).astype(np.float64)
    return bool((np.abs(got.detach().cpu().double().numpy() - e) <= sp).all())


def _cc_problems(img, A, up, ranks, H):
    out_ref, gimg_ref, _ = _cc_whole(img, A, up)
    bad = []
    covered = torch.zeros(H, dtype=torch.bool, device=DEV)
    for r, (rows, out, gimg, _) in enumerate(ranks):
        covered |= rows
        if not (_bits_equal(out[:, rows], out_ref[:, rows]) and _bits_equal(gimg[:, rows], gimg_ref[:, rows])):
            bad.append(f"rank {r}: rows differ")
        if bool((~rows).any()) and (bool(out[:, ~rows].any()) or bool(gimg[:, ~rows].any())):
            bad.append(f"rank {r}: foreign rows written")
    if not bool(covered.all()):
        bad.append("rows not covered by any band")
    gA = _affine_grad(sum(s for _, _, _, s in ranks))
    if not _within_ulp(gA, CCO.color64(img, A, up)["daffine"]):
        bad.append("summed dL/daffine is not within one ulp of the fp64 restatement")
    return bad


@pytest.mark.parametrize("world,layout,H,W", CC_CASES)
def test_color_correct_band_matches_whole_frame(world, layout, H, W):
    img, A, up = _cc_inputs(H, W, 3 * world + H)
    ranks = [(_rows_of(H, b),) + _cc_band(img, A, up, b, _rows_of(H, b)) for b in _bands(H, world, layout)]
    assert _cc_problems(img, A, up, ranks, H) == []


def test_color_correct_check_catches_a_dropped_partial_tile_row():
    H, W = 375, 200
    rows_n = (H + 15) // 16
    img, A, up = _cc_inputs(H, W, 1)
    ranks = [(_rows_of(H, b),) + _cc_band(img, A, up, TileRowBand(b.begin, min(b.end, rows_n - 1), b.step), _rows_of(H, b))
             for b in _bands(H, 3, "cyclic")]
    assert _cc_problems(img, A, up, ranks, H) != []


def test_band_entries_capture_in_a_cuda_graph():
    """No host synchronisation: the band calls of one rank replay from a CUDA graph with the eager results."""
    H, W = 375, 200
    band = cyclic_band(H, 1, 3)
    rows = _rows_of(H, band)
    f = _sky_frame(H, W, 2, True, True)
    img, A, up = _cc_inputs(H, W, 2)
    eager = _sky_band(f, 1.0, band, rows)[:2] + _cc_band(img, A, up, band, rows)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _sky_band(f, 1.0, band, rows), _cc_band(img, A, up, band, rows)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = _sky_band(f, 1.0, band, rows)[:2] + _cc_band(img, A, up, band, rows)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, captured):
        assert torch.equal(a, b)


# ---- autograd ----------------------------------------------------------------------------------------------------------------
def test_autograd_whole_image_band_one_rank():
    """band = the whole image, group = None: the whole-frame outputs and gradients; dL/dcube to the atomic-order bound, dL/daffine to the
    fp64 sums' rounding (within one ulp of the fp64 restatement, and within the whole-frame call's own bound of it)."""
    H, W = 375, 200
    whole = TileRowBand(0, (H + 15) // 16, 1)
    f = _sky_frame(H, W, 11, True, False)
    A = torch.eye(4, device=DEV)[:3] + 0.1 * torch.randn(3, 4, device=DEV)
    gt = torch.rand(3, H, W, device=DEV)
    res = []
    for band in (None, whole):
        rgb, acc, cube, aff = (t.clone().requires_grad_(True) for t in (f["rgb"], f["acc"], f["cube"], A))
        torch.manual_seed(5)
        sky = sgb.sky_composite(rgb, acc, cube, f["K"], f["w2c"], sky_mask=f["mask"].bool(), perturb=True, band=band)
        col = corrections.color_correct(sky, aff, band=band)
        ((col - gt) * f["up"]).sum().backward()
        res.append(dict(sky=sky.detach(), col=col.detach(), rgb=rgb.grad, acc=acc.grad, cube=cube.grad, aff=aff.grad))
    a, b = res
    for k in ("sky", "col", "rgb", "acc"):
        assert _bits_equal(a[k], b[k]), k
    torch.manual_seed(5)
    jx, jy = torch.rand(H, W, device=DEV), torch.rand(H, W, device=DEV)
    g_col = f["up"]
    # the sky's upstream gradient is the colour correction's dL/dimage, A^T g (its terms' magnitudes to fp32 rounding here)
    fj = dict(f, jx=jx, jy=jy, up=(A[:, :3].T @ g_col.reshape(3, -1)).reshape(3, H, W))
    n, sabs = _texel_terms(fj, 1.0)
    err = (a["cube"].double() - b["cube"].double()).abs()
    assert bool((err <= 2 * n * U * sabs * (1 + 1e-3) + 1e-30).all())
    r = CCO.color64(a["sky"], A, g_col)
    assert _within_ulp(b["aff"], r["daffine"])
    assert bool(((a["aff"].double() - b["aff"].double()).abs() <= 2 * r["b_daffine"]).all())


def test_chained_band_step_one_rank():
    """rasterizer (band) -> sky -> colour correction -> frame_losses -> backward on one rank (whole-image band, no process group)
    against the same step without a band."""
    Hs, Ws, R = 320, 480, 64
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
    cube0 = 0.5 + 0.4 * torch.rand(6, R, R, 3, generator=g, device=DEV)
    affine0 = torch.eye(4, device=DEV)[:3] + 0.05 * torch.randn(3, 4, generator=g, device=DEV)
    whole = TileRowBand(0, (Hs + 15) // 16, 1)

    def step(band):
        models = [{k: v.to(DEV).requires_grad_(True) for k, v in m.items()} for m in raw["models"]]
        cube, affine = cube0.clone().requires_grad_(True), affine0.clone().requires_grad_(True)
        xyz, rot, scale, opac, sh = sgb.compose(models, raw["poses"].to(DEV), raw["idft"].to(DEV))
        m2d = torch.zeros_like(xyz, requires_grad=True)
        rast = sgb.GaussianRasterizer(st, band=band)
        res = rast(means3D=xyz, means2D=m2d, opacities=opac, shs=sh, scales=scale, rotations=rot)
        rgb, acc = res[0], res[3]
        out = sgb.sky_composite(rgb, acc, cube, K, w2c, sky_mask=sky_mask, band=band)
        col = corrections.color_correct(out, affine, band=band)
        if band is None:
            from street_gaussians_b200 import losses
            vals = [losses.photometric_loss(col, gt, None, 1.0, 0.2), losses.sky_loss(acc, sky_mask, 1.0)]
        else:
            fl = band_losses.frame_losses(col, gt, None, 1.0, 0.2, acc=acc, sky_mask=sky_mask, band=band)
            vals = [fl["photometric"], fl["sky"]]
        sum(vals).backward()
        return dict(vals=[float(v.detach()) for v in vals], col=col.detach(), grads=[v.grad.clone() for m in models for v in m.values()], cube=cube.grad,
                    affine=affine.grad)

    a, b = step(None), step(whole)
    assert _bits_equal(a["col"], b["col"])
    for x, y in zip(a["vals"], b["vals"]):
        assert abs(x - y) <= 2 * float(np.spacing(np.float32(abs(x))))
    assert int((a["cube"] != 0).sum()) > 100
    assert float((a["cube"] - b["cube"]).abs().max()) <= 1e-5 * float(a["cube"].abs().max())
    assert float((a["affine"] - b["affine"]).abs().max()) <= 1e-5 * float(a["affine"].abs().max())
    for k, (x, y) in enumerate(zip(a["grads"], b["grads"])):
        assert float((x - y).abs().max()) <= 1e-3 * max(float(x.abs().max()), 1e-12), k
