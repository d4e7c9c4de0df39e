"""The evaluation metrics (metrics.py, include/sgr.h "Evaluation metrics") on one GPU.

Against the float64 restatement (eval_oracle.py): the L1 and MSE sums are formed from fp64 differences of the fp32 inputs and summed in
fp64, so L1 and PSNR are within ULPS fp32 ulps (the final fp32 rounding and the fp64 sums' own error, ~1e-12 relative); SSIM is within
eval_oracle.ssim_bound, the first-order bound of the fp32 evaluation of the map and its sum, plus the final rounding.

Exactness: identical calls give identical bits, and V views in one call the bits of V single-view calls.  With the masked SSIM and no
clamp or quantisation the SSIM sum is the image loss's (sgr_image_loss) up to the fp64 regrouping of the same tile partials:
|difference| <= 2 T 2^-53 sum |S| with T tiles (|S| <= 1 + 2^-20 in fp32).

Bands: ranks emulated on one GPU (the halo moved by the library's pack / unpack, the slots summed as the all-reduce does); the summed
sums equal the whole-frame sums up to the same regrouping bound, and the fp32 values to one ulp.  Two mutations fail the same check:
dropping the halo, and scoring each band's rows as a frame of their own (band-local row indexing)."""
import numpy as np
import pytest
import torch

import eval_oracle as EO
from street_gaussians_b200 import _capi, band_losses, losses, metrics
from street_gaussians_b200.rasterizer import TileRowBand
from street_gaussians_b200.sharded import band_of_rows, contiguous_band, cyclic_band

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ULPS = 4
EPS64 = 2.0 ** -53
SIZES = [(375, 200), (1280, 1920), (40, 48)]
FLAGS = {"raw": (False, False, False), "clamp": (True, False, False), "png": (True, True, False), "masked_ssim": (False, False, True),
         "train_report": (True, False, True), "png_masked": (True, True, True)}
MASKS = ["none", "all_true", "all_false", "random"]


def _flags(name):
    return metrics._flags(*FLAGS[name])


def _inputs(V, H, W, seed, mask_kind):
    g = torch.Generator(device=DEV).manual_seed(seed)
    img = torch.rand(V, 3, H, W, device=DEV, generator=g) * 1.2 - 0.1  # outside [0, 1] in places: the clamp matters
    gt = torch.rand(V, 3, H, W, device=DEV, generator=g)
    gt = torch.where(torch.rand(V, 1, H, W, device=DEV, generator=g) < 0.5, img + 0.05 * torch.randn(V, 3, H, W, device=DEV, generator=g), gt)
    if mask_kind == "none":
        m = None
    elif mask_kind == "all_true":
        m = torch.ones(V, H * W, device=DEV, dtype=torch.uint8)
    elif mask_kind == "all_false":
        m = torch.zeros(V, H * W, device=DEV, dtype=torch.uint8)
    else:
        m = (torch.rand(V, H * W, device=DEV, generator=g) > 0.3).to(torch.uint8)
    return img, gt, m


def _score(img, gt, m, flags, band=None):
    sums = torch.zeros(img.shape[0], 5, device=DEV, dtype=torch.float64)
    metrics.accumulate(img.contiguous(), gt.contiguous(), m, sums, flags, band)
    return sums


def _ulps(a, b):
    a, b = np.float32(a), np.float32(b)
    if np.isnan(a) or np.isnan(b):
        return 0 if (np.isnan(a) and np.isnan(b)) else np.inf
    if np.isinf(a) or np.isinf(b):
        return 0 if a == b else np.inf
    return abs(float(a) - float(b)) / float(np.spacing(np.float32(max(abs(a), abs(b)))))


ORACLE_CASES = [(H, W, f, mk) for (H, W) in SIZES for f in FLAGS for mk in MASKS
                if (H, W) != (1280, 1920) or (f in ("train_report", "png") and mk in ("random", "none"))]


@pytest.mark.parametrize("H,W,flag,mask_kind", ORACLE_CASES)
def test_against_fp64_restatement(H, W, flag, mask_kind):
    img, gt, m = _inputs(1, H, W, H + W, mask_kind)
    clamp, quant, ssim_masked = FLAGS[flag]
    out = metrics.finish(_score(img, gt, m, _flags(flag))).cpu().numpy()
    mask = None if m is None else m[0].view(H, W).bool().cpu().numpy()
    ref = EO.view_metrics(img[0].cpu().numpy(), gt[0].cpu().numpy(), mask, clamp, quant, ssim_masked)
    psnr, ssim, l1, n = out[0]
    assert int(n) == ref["n"]
    assert _ulps(l1, ref["l1"]) <= ULPS, (l1, ref["l1"])
    assert _ulps(psnr, ref["psnr"]) <= ULPS, (psnr, ref["psnr"])
    assert abs(float(ssim) - ref["ssim"]) <= ref["ssim_bound"] + float(np.spacing(np.float32(ref["ssim"]))), (ssim, ref["ssim"], ref["ssim_bound"])
    if mask_kind == "all_false":
        assert np.isnan(psnr) and np.isnan(l1)
    # the means row of one view is the view
    assert _ulps(out[1, 0], psnr) == 0 and _ulps(out[1, 2], l1) == 0 and out[1, 1] == ssim and out[1, 3] == 1


def test_psnr_edges_and_masks():
    """metrics.psnr: +inf for identical images, NaN for an empty mask, [1, H, W] and [H, W] bool / uint8 masks alike."""
    img, gt, m = _inputs(1, 40, 48, 3, "random")
    x, y = img[0], gt[0]
    assert float(metrics.psnr(x, x)) == float("inf")
    assert np.isnan(float(metrics.psnr(x, y, torch.zeros(1, 40, 48, dtype=torch.bool, device=DEV))))
    mb = m[0].view(40, 48).bool()
    vals = {float(metrics.psnr(x, y, mm)) for mm in (mb, mb[None], mb.to(torch.uint8), mb[None].to(torch.uint8))}
    assert len(vals) == 1
    ref = EO.view_metrics(x.cpu().numpy(), y.cpu().numpy(), mb.cpu().numpy(), clamp=False)
    assert _ulps(vals.pop(), ref["psnr"]) <= ULPS


def test_quantize8_on_device_at_level_boundaries():
    """Each value a 1x1 view against gt 0: the view's abs_diff is the device's quantised value itself, bit for bit the oracle's."""
    v = EO.quant_boundary_values()
    x = torch.from_numpy(v).to(DEV).view(-1, 1, 1, 1)
    sums = _score(x, torch.zeros_like(x), None, _flags("png"))
    assert np.array_equal(sums[:, 0].cpu().numpy(), EO.prepare(v, True, True).astype(np.float64))


def test_psnr_skips_the_ssim():
    """metrics.psnr scores without the SSIM map: the same L1 / MSE sums bit for bit, no SSIM sum, ssim NaN."""
    img, gt, m = _inputs(1, 375, 200, 4, "random")
    full = _score(img, gt, m, 0)
    lean = _score(img, gt, m, _capi.EVAL_NO_SSIM)
    assert torch.equal(_bits(lean[:, [0, 1, 3]]), _bits(full[:, [0, 1, 3]]))
    assert float(lean[0, 2]) == 0.0 and float(lean[0, 4]) == 0.0
    out = metrics.finish(lean).cpu()
    assert np.isnan(float(out[0, 1])) and float(out[0, 0]) == float(metrics.finish(full)[0, 0])
    assert float(metrics.psnr(img[0], gt[0], m[0].view(375, 200))) == float(out[0, 0])


def _bits(t):
    return t.contiguous().view(torch.int64)


@pytest.mark.parametrize("flag", ["train_report", "png"])
def test_identical_calls_and_batches_give_identical_bits(flag):
    V, H, W = 4, 375, 200
    img, gt, m = _inputs(V, H, W, 7, "random")
    a, b = _score(img, gt, m, _flags(flag)), _score(img, gt, m, _flags(flag))
    assert torch.equal(_bits(a), _bits(b))
    singles = torch.cat([_score(img[v:v + 1], gt[v:v + 1], m[v:v + 1], _flags(flag)) for v in range(V)])
    assert torch.equal(_bits(a), _bits(singles))
    vm = metrics.ViewMetrics(*FLAGS[flag])
    for v in range(V):
        vm.add(img[v], gt[v], m[v].view(1, H, W).bool())
    r = vm.result()
    out = metrics.finish(a).cpu()
    assert torch.equal(r["psnr"], out[:V, 0]) and torch.equal(r["ssim"], out[:V, 1]) and torch.equal(r["l1"], out[:V, 2])
    assert torch.equal(r["n"], a[:, 3].cpu().to(torch.int64))
    assert r["mean"]["psnr"] == float(out[V, 0]) and r["mean"]["ssim"] == float(out[V, 1])


def test_view_metrics_grows_past_its_first_buffer():
    V, H, W = 40, 40, 48
    img, gt, m = _inputs(V, H, W, 8, "random")
    vm = metrics.ViewMetrics()
    for v in range(V):
        vm.add(img[v], gt[v], m[v].view(H, W))
    r = vm.result()
    ref = metrics.finish(_score(img, gt, m, _flags("train_report"))).cpu()
    assert torch.equal(r["psnr"], ref[:V, 0]) and len(vm) == 0


@pytest.mark.parametrize("H,W", [(375, 200), (1280, 1920), (40, 48)])
def test_masked_ssim_is_the_image_loss_ssim(H, W):
    img, gt, m = _inputs(1, H, W, 5, "random")
    sums = _score(img, gt, m, _flags("masked_ssim"))
    partials, _ = band_losses.image_loss_stats(img[0].contiguous(), gt[0].contiguous(), m[0], TileRowBand(0, (H + 15) // 16, 1))
    T = 3 * ((H + 15) // 16) * ((W + 15) // 16)
    bound = 2 * T * EPS64 * 3 * H * W * (1 + 2.0 ** -20)
    assert abs(float(sums[0, 2]) - float(partials[0])) <= bound
    ref = losses.ssim(img[0], gt[0], mask=m[0].view(1, H, W).bool())
    assert _ulps(metrics.finish(sums)[0, 1].item(), ref.item()) <= 1


# ---- bands ---------------------------------------------------------------------------------------------------------------------
BAND_CASES = [(world, layout, H) for world in (1, 2, 3, 5, 8) for layout in ("cyclic", "contiguous") for H in (375, 1280)] + \
             [(8, "cyclic", 80), (8, "contiguous", 40)]  # more ranks than tile rows: empty bands
W_OF = {375: 200, 1280: 1920, 80: 64, 40: 48}


def _bands(H, world, layout):
    mk = cyclic_band if layout == "cyclic" else contiguous_band
    return [mk(H, r, world) for r in range(world)]


def _banded(x, rows):
    return torch.where(rows.view(1, -1, 1), x, torch.zeros_like(x))


def _emulated(img, gt, m, flags, H, world, layout, halo=True, local_rows=False):
    """The summed slots of `world` ranks, each scoring the rendered rows of its band (zero elsewhere) plus, with `halo`, the rows the
    library's halo exchange brings.  local_rows: the mutation of a kernel indexing band-local rows (the band's rows packed as a frame)."""
    bands = _bands(H, world, layout)
    rows = [band_of_rows(H, r, world, layout).to(DEV) for r in range(world)]
    xs = [_banded(img[0], rows[r]) for r in range(world)]
    filled = [x.clone() for x in xs]
    if halo:
        for r in range(world):
            up, down = band_losses.halo_peers(r, world)
            for side, src, src_side in ((band_losses.RECV_UP, up, band_losses.SEND_DOWN), (band_losses.RECV_DOWN, down, band_losses.SEND_UP)):
                buf = band_losses.halo_pack(xs[src], bands[src], src_side)
                if buf.numel():
                    band_losses.halo_unpack(filled[r], bands[r], side, buf)
    total = torch.zeros(1, 5, device=DEV, dtype=torch.float64)
    for r in range(world):
        if local_rows:
            idx = rows[r].nonzero().squeeze(1)
            if idx.numel() == 0:
                continue
            Hl = int(idx.numel())
            ml = None if m is None else m[0].view(H, -1)[idx].reshape(1, -1).contiguous()
            total += _score(filled[r][:, idx][None], gt[0][:, idx][None], ml, flags, TileRowBand(0, (Hl + 15) // 16, 1))
        else:
            total += _score(filled[r][None], gt, m, flags, bands[r])
    return total


def _band_problems(total, whole, H, W):
    """What differs between the summed band slots and the whole-frame slot beyond the regrouping bound."""
    T = 3 * ((H + 15) // 16) * ((W + 15) // 16)
    probs = []
    for k, scale in ((0, abs(float(whole[0, 0]))), (1, abs(float(whole[0, 1]))), (2, 3 * H * W * (1 + 2.0 ** -20))):
        if not abs(float(total[0, k]) - float(whole[0, k])) <= 2 * T * EPS64 * scale:
            probs.append((k, float(total[0, k]), float(whole[0, k])))
    if float(total[0, 3]) != float(whole[0, 3]) or float(total[0, 4]) != 3 * H * W:
        probs.append(("counts", total[0, 3:].tolist(), whole[0, 3:].tolist()))
    a, b = metrics.finish(total).cpu().numpy(), metrics.finish(whole).cpu().numpy()
    for k in range(3):
        if _ulps(a[0, k], b[0, k]) > 1:
            probs.append(("value", k, a[0, k], b[0, k]))
    return probs


@pytest.mark.parametrize("world,layout,H", BAND_CASES)
@pytest.mark.parametrize("flag", ["train_report", "png"])
def test_band_sums_are_the_whole_frame_sums(world, layout, H, flag):
    W = W_OF[H]
    img, gt, m = _inputs(1, H, W, 31 + world, "random")
    whole = _score(img, gt, m, _flags(flag))
    assert _band_problems(_emulated(img, gt, m, _flags(flag), H, world, layout), whole, H, W) == []


@pytest.mark.parametrize("world,layout", [(2, "cyclic"), (3, "contiguous"), (5, "cyclic")])
def test_band_check_catches_a_dropped_halo(world, layout):
    H, W = 375, 200
    img, gt, m = _inputs(1, H, W, 4, "random")
    whole = _score(img, gt, m, _flags("train_report"))
    assert _band_problems(_emulated(img, gt, m, _flags("train_report"), H, world, layout, halo=False), whole, H, W) != []


@pytest.mark.parametrize("world,layout", [(2, "cyclic"), (3, "contiguous"), (5, "cyclic")])
def test_band_check_catches_band_local_rows(world, layout):
    H, W = 375, 200
    img, gt, m = _inputs(1, H, W, 6, "random")
    whole = _score(img, gt, m, _flags("train_report"))
    assert _band_problems(_emulated(img, gt, m, _flags("train_report"), H, world, layout, local_rows=True), whole, H, W) != []


def test_view_metrics_band_one_rank_and_capture():
    """ViewMetrics with the whole-image band and no process group gives the single-GPU bits; the accumulate calls replay from a graph."""
    H, W, V = 375, 200, 3
    img, gt, m = _inputs(V, H, W, 9, "random")
    band = TileRowBand(0, (H + 15) // 16, 1)
    a, b = metrics.ViewMetrics(), metrics.ViewMetrics(band=band)
    for v in range(V):
        a.add(img[v], gt[v], m[v].view(1, H, W).bool())
        b.add(img[v], gt[v], m[v].view(1, H, W).bool())
    ra, rb = a.result(), b.result()
    assert torch.equal(ra["psnr"], rb["psnr"]) and torch.equal(ra["ssim"], rb["ssim"]) and torch.equal(ra["l1"], rb["l1"])
    # capture: scratch allocated outside, the same sums after a replay
    sums = torch.zeros(V, 5, device=DEV, dtype=torch.float64)
    nb = int(_capi.lib().sgr_eval_metrics_scratch_bytes(V, 3, H, W))
    scratch = torch.empty(nb, device=DEV, dtype=torch.uint8)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        _capi.call("sgr_eval_metrics_accumulate", DEV, V, 3, H, W, _flags("train_report"), _capi.ptr(img), _capi.ptr(gt), _capi.ptr(m),
                   _capi.ptr(sums), _capi.ptr(scratch), nb)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(sums), _bits(_score(img, gt, m, _flags("train_report"))))
