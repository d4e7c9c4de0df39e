"""The feature maps' finishing on a tile-row band (features.finish_features(band=), sgr_band_finish_features_*) against the whole-frame
call, with N ranks emulated on one GPU: every rank finishes its banded feature image (its rows, zeros elsewhere, as a sharded rasterizer
returns it) and back-propagates the whole frame's upstream gradient.

Per case: the rows of the band in the normals, the semantics and dL/drendered equal the whole-frame call's bit for bit, every other row is
zero, and the ranks' results summed equal the whole-frame results bit for bit (the rows are disjoint and the inputs hold no -0).  The
cases cover both normal-channel counts, both semantic modes and pixels whose normal is zero (F.normalize's 1e-12 clamp).  Two mutation
checks show that the comparison catches a kernel that indexes the band-local row instead of the frame's, and one that drops the last
partial tile row."""
import pytest
import torch

from street_gaussians_b200 import _capi, features
from street_gaussians_b200._capi import ptr
from street_gaussians_b200.rasterizer import TileRowBand
from street_gaussians_b200.sharded import contiguous_band, cyclic_band

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
K_SEM = 4
CASES = [(world, layout, H) for world in (1, 2, 3, 5, 8) for layout in ("cyclic", "contiguous") for H in (375, 1280)] + \
        [(8, "cyclic", 80), (8, "contiguous", 40)]  # more ranks than tile rows: empty bands
W_OF = {375: 200, 1280: 96, 80: 64, 40: 48}
VARIANTS = [(nc, mode) for nc in (0, 3) for mode in ("logits", "probabilities")]


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


def _frame(H, W, nc, mode, seed):
    """rendered [nc + K, H, W], upstream gradients of the normals and the semantics.  The semantics are positive in 'probabilities' mode
    (accumulated probabilities); one pixel in 50 has a zero normal."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.rand(nc + K_SEM, H, W, generator=g, device=DEV)
    if mode == "logits":
        x[nc:] = 4 * x[nc:] - 2
    if nc:
        x[:nc] = 2 * x[:nc] - 1
        x[:nc, torch.rand(H, W, generator=g, device=DEV) < 0.02] = 0.0
        assert int((x[:nc].abs().sum(0) == 0).sum()) > 0
    gn = torch.randn(nc, H, W, generator=g, device=DEV)
    gs = torch.randn(K_SEM, H, W, generator=g, device=DEV)
    return x, gn, gs


def _finish(x, nc, mode, gn, gs, band=None):
    """(normals or None, semantic, dL/drendered) through the autograd wrapper."""
    x = x.detach().clone().requires_grad_(True)
    n, s = features.finish_features(x, nc, mode, band=band)
    outs, grads = [s], [gs]
    if n is not None:
        outs.append(n)
        grads.append(gn)
    (g,) = torch.autograd.grad(outs, x, grads)
    return n, s.detach(), g


def _run(world, layout, H, nc, mode, band_of=lambda b: b, seed=3):
    W = W_OF[H]
    x, gn, gs = _frame(H, W, nc, mode, seed)
    ref = _finish(x, nc, mode, gn, gs)
    ranks = []
    for band in _bands(H, world, layout):
        rows = _rows_of(H, band)
        ranks.append((rows,) + _finish(_banded(x, rows), nc, mode, gn, gs, band=band_of(band)))
    return ref, ranks


def _problems(ref, ranks):
    """What is wrong with the ranks' (rows, normals, semantic, dL/drendered) against the whole-frame results: an empty list when nothing."""
    out = []
    sums = [None, torch.zeros_like(ref[1]), torch.zeros_like(ref[2])]
    if ref[0] is not None:
        sums[0] = torch.zeros_like(ref[0])
    for r, (rows, *res) in enumerate(ranks):
        for k, name in enumerate(("normals", "semantic", "dL/drendered")):
            if ref[k] is None:
                if res[k] is not None:
                    out.append((r, name, "unexpected"))
                continue
            own, other = res[k][:, rows], res[k][:, ~rows]
            if not _bits_equal(own, ref[k][:, rows]):
                out.append((r, name, "band rows"))
            if bool(other.any()):
                out.append((r, name, "foreign rows"))
            sums[k] += res[k]
    for k, name in enumerate(("normals", "semantic", "dL/drendered")):
        if ref[k] is not None and not _bits_equal(sums[k], ref[k]):
            out.append(("sum", name))
    return out


@pytest.mark.parametrize("nc,mode", VARIANTS)
@pytest.mark.parametrize("world,layout,H", CASES)
def test_band_matches_whole_frame(world, layout, H, nc, mode):
    ref, ranks = _run(world, layout, H, nc, mode)
    assert bool(torch.isfinite(ref[2]).all())
    assert _problems(ref, ranks) == []


def test_zero_normal_takes_the_clamp():
    """A zero normal pixel finishes to 0 (0 / 1e-12) and its gradient is g / 1e-12 on every rank that owns it."""
    H, W = 375, 200
    x, gn, gs = _frame(H, W, 3, "logits", 11)
    zero = x[:3].abs().sum(0) == 0
    ref, ranks = _run(3, "cyclic", H, 3, "logits", seed=11)
    assert bool((ref[0][:, zero] == 0).all())
    eps = torch.full_like(gn[:, zero], 1e-12)  # a tensor divisor: true division, as in the kernel
    assert torch.equal(ref[2][:3, zero], gn[:, zero] / eps)
    assert _problems(ref, ranks) == []


@pytest.mark.parametrize("world,layout", [(2, "cyclic"), (3, "contiguous"), (5, "cyclic")])
def test_check_catches_band_local_rows(world, layout):
    """Mutation: a kernel that indexed its band's pixels by the band-local row (read and wrote the band's rows as if they were the first
    rows of the frame); the comparison reports it."""
    H, W, nc, mode = 375, 200, 3, "probabilities"
    x, gn, gs = _frame(H, W, nc, mode, 5)
    ref = _finish(x, nc, mode, gn, gs)
    ranks = []
    for band in _bands(H, world, layout):
        rows = _rows_of(H, band)
        idx = rows.nonzero().squeeze(1)
        Hl = int(idx.numel())
        res = [torch.zeros_like(ref[0]), torch.zeros_like(ref[1]), torch.zeros_like(ref[2])]
        if Hl:
            local = _finish(x[:, idx].contiguous(), nc, mode, gn[:, idx].contiguous(), gs[:, idx].contiguous())
            for k in range(3):
                res[k][:, :Hl] = local[k]
        ranks.append((rows, *res))
    assert _problems(ref, ranks) != []


@pytest.mark.parametrize("layout", ["cyclic", "contiguous"])
def test_check_catches_a_dropped_partial_tile_row(layout):
    """Mutation: a kernel that skipped the last tile row when it is partial (H = 375: rows 368-374)."""
    H, rows_n = 375, (375 + 15) // 16
    ref, ranks = _run(3, layout, H, 3, "logits", band_of=lambda b: TileRowBand(b.begin, min(b.end, rows_n - 1), b.step))
    assert _problems(ref, ranks) != []


def test_band_entries_capture_in_a_cuda_graph():
    """No host synchronisation: one rank's band forward and backward replay from a CUDA graph with the eager results."""
    H, W, nc, mode = 375, 200, 3, _capi.SEMANTIC_PROBABILITIES
    S = nc + K_SEM
    x, gn, gs = _frame(H, W, nc, "probabilities", 9)
    band = cyclic_band(H, 1, 3)
    x = _banded(x, _rows_of(H, band)).contiguous()
    n, s, g = torch.zeros(nc, H, W, device=DEV), torch.zeros(K_SEM, H, W, device=DEV), torch.zeros(S, H, W, device=DEV)

    def step():
        _capi.call("sgr_band_finish_features_forward", DEV, S, H, W, nc, mode, *band, ptr(x), ptr(n), ptr(s))
        _capi.call("sgr_band_finish_features_backward", DEV, S, H, W, nc, mode, *band, ptr(x), ptr(gn), ptr(gs), ptr(g))

    step()
    torch.cuda.synchronize()
    eager = (n.clone(), s.clone(), g.clone())
    for t in (n, s, g):
        t.zero_()
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        step()  # warm-up on a side stream, as torch.cuda.graph expects
    torch.cuda.current_stream(DEV).wait_stream(side)
    for t in (n, s, g):
        t.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip((n, s, g), eager):
        assert _bits_equal(a, b)
    assert bool(eager[2].any())
