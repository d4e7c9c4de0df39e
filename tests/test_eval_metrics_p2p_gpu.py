"""GPU: metrics.ViewMetrics(rasterizer=) of a GaussianShardedRasterizer(exchange="p2p") stand-in, with 1, 2, 3, 5 and 8 ranks emulated
by threads (tests/rank_threads.py) on streams of one GPU through PeerWorkspace.emulate (loss sections poisoned with 0x7f): the halo goes
through sgr_band_halo_exchange_peers and the [V, 5] slots through sgr_band_peer_sum.  Every rank's numbers are the same bytes, and each
view's PSNR, SSIM and L1 are within the band cases' bound of tests/test_eval_metrics_gpu.py (one fp32 ulp) of the whole-frame
single-GPU call, with the masked-element count exact.  A stand-in with exchange="nccl" and no process group takes the NCCL path's
single-rank case and gives the single-GPU bits."""
import types

import pytest
import torch

from rank_threads import run_ranks
from street_gaussians_b200 import metrics
from street_gaussians_b200 import sharded as SH
from test_band_losses_p2p_gpu import _settings, _warm_up
from test_eval_metrics_gpu import W_OF, _inputs, _ulps

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
CASES = [(1, 375), (2, 375), (3, 1280), (5, 375), (8, 80)]
V = 3


def _stand_in(ws, band, exchange="p2p"):
    """What ViewMetrics reads of a GaussianShardedRasterizer, around an emulated workspace."""
    return types.SimpleNamespace(exchange=exchange, group=None, band=band, loss_workspace=lambda: ws)


def _rank_metrics(world, H, W, img, gt, m, flags):
    wss = SH.PeerWorkspace.emulate(_settings(H, W), 8, world, DEV)
    for ws in wss:
        ws.buf[ws.off_loss: ws.off_loss + ws.loss_bytes].fill_(0x7f)
    rows = [SH.band_of_rows(H, r, world).to(DEV) for r in range(world)]
    ris = [_stand_in(wss[r], SH.cyclic_band(H, r, world) if world > 1 else None) for r in range(world)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
    torch.cuda.synchronize()

    def rank(r, _tr):
        with torch.cuda.stream(streams[r]):
            vm = metrics.ViewMetrics(*flags, rasterizer=ris[r])
            for v in range(V):
                banded = torch.where(rows[r].view(1, -1, 1), img[v], torch.zeros_like(img[v]))
                vm.add(banded, gt[v], m[v].view(1, H, W).bool())
            return vm.result()

    out = run_ranks(world, rank)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("world,H", CASES)
@pytest.mark.parametrize("flags", [(True, False, True), (True, True, False)], ids=["train_report", "png"])
def test_view_metrics_over_peer_memory_are_the_whole_frame(world, H, flags):
    _warm_up()
    W = W_OF[H]
    img, gt, m = _inputs(V, H, W, 17 + world, "random")
    ref = metrics.ViewMetrics(*flags)
    for v in range(V):
        ref.add(img[v], gt[v], m[v].view(1, H, W).bool())
    want = ref.result()
    res = _rank_metrics(world, H, W, img, gt, m, flags)
    for r in range(world):
        for key in ("psnr", "ssim", "l1", "n"):
            assert torch.equal(res[r][key].view(torch.int32 if key != "n" else torch.int64), res[0][key].view(torch.int32 if key != "n" else torch.int64)), (r, key)
    assert torch.equal(res[0]["n"], want["n"])
    for key in ("psnr", "ssim", "l1"):
        for v in range(V):
            assert _ulps(float(res[0][key][v]), float(want[key][v])) <= 1, (key, v, float(res[0][key][v]), float(want[key][v]))


def test_view_metrics_with_an_nccl_rasterizer_at_one_rank():
    """exchange="nccl" resolves to the band= / group= path: at one rank without a process group, the whole image and no collective."""
    H, W = 375, W_OF[375]
    img, gt, m = _inputs(V, H, W, 5, "random")
    a = metrics.ViewMetrics()
    b = metrics.ViewMetrics(rasterizer=_stand_in(None, None, exchange="nccl"))
    for v in range(V):
        a.add(img[v], gt[v], m[v].view(1, H, W).bool())
        b.add(img[v], gt[v], m[v].view(1, H, W).bool())
    ra, rb = a.result(), b.result()
    for key in ("psnr", "ssim", "l1", "n"):
        assert torch.equal(ra[key], rb[key]), key
