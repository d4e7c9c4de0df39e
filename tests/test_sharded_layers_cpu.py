"""Render layers of the fused Gaussian-sharded step, checked without a GPU: the C ABI (symbols, struct layouts, argument checks that come
back before any CUDA call), the peer workspace's layer sections, and the host restatement of which slot of which rank receives which
layer bit (tests/sharded_layers_case.py, used by tests/test_sharded_layers_gpu.py)."""
import ctypes as C
import os
import subprocess

import pytest
import torch

import sharded_layers_case as LC
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi
from street_gaussians_b200.sharded import PeerWorkspace

EINVAL, ENOMEM = -1, -3  # SGR_EINVAL, SGR_ENOMEM of include/sgr.h
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _settings(H=480, W=640):
    return sgb.GaussianRasterizationSettings(H, W, 0.5, 0.4, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3, torch.zeros(3), False, False)


def test_layer_structs_match_the_header(tmp_path):
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "sgr.h"', 'int main(void) {']
    for name in ("SgrShardedLayer", "SgrLayerPeers"):
        body.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        body += [f'  printf("{name}.{f[0]} %zu\\n", offsetof({name}, {f[0]}));' for f in getattr(_capi, name)._fields_]
    body += ['  printf("SGR_MAX_SHARDED_LAYERS %d\\n", SGR_MAX_SHARDED_LAYERS);', '  return 0;', '}']
    src = tmp_path / "layers.c"
    src.write_text("\n".join(body))
    exe = tmp_path / "layers"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(line.rsplit(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for name in ("SgrShardedLayer", "SgrLayerPeers"):
        ct = getattr(_capi, name)
        assert int(out[name]) == C.sizeof(ct), name
        for f in ct._fields_:
            assert int(out[f"{name}.{f[0]}"]) == getattr(ct, f[0]).offset, (name, f[0])
    assert int(out["SGR_MAX_SHARDED_LAYERS"]) == _capi.MAX_SHARDED_LAYERS == 2
    for s in ("sgr_sharded_layer_state_sizes", "sgr_sharded_forward_layers", "sgr_sharded_backward_layers"):
        assert s in _capi.SYMBOLS and hasattr(_capi.lib(), s)


def _frame(P=100):
    fr = _capi.SgrFrame()
    fr.P, fr.width, fr.height, fr.D, fr.M = P, 64, 64, 0, 1
    fr.tan_fovx, fr.tan_fovy, fr.scale_modifier = 0.5, 0.5, 1.0
    fr.row_begin, fr.row_end, fr.row_step = 0, 4, 1
    return fr


@pytest.mark.parametrize("direction", ["forward", "backward"])
def test_bad_layer_arguments_return_einval_before_any_cuda_call(direction):
    """Every pointer below is fake: a check that let a call through would touch the device (there is none here) or fault."""
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    ok = C.c_void_p(1 << 20)
    fr = _frame()
    nb = C.c_size_t(0)
    assert L.sgr_sharded_layer_state_sizes(C.byref(fr), 1000, C.byref(nb)) == 0 and nb.value > 64 * 64 * 4 + 1000 * 4 + 100 * 60

    def good():
        t = (_capi.SgrShardedLayer * 2)()
        for k in range(2):
            t[k] = _capi.SgrShardedLayer(10 * k, 50, ok.value, ok.value, nb.value, ok.value, ok.value, ok.value)
        return t

    peers, lpeers = _capi.SgrPeers(), _capi.SgrLayerPeers()

    def call(table, n):
        if direction == "forward":
            return L.sgr_sharded_forward_layers(C.byref(fr), C.byref(peers), *[ok] * 12, 0, ok, 0, ok, 0, 1000, -1, 0, 0, C.byref(lpeers), table, n, None)
        return L.sgr_sharded_backward_layers(C.byref(fr), C.byref(peers), 1000, *[ok] * 22, 0, C.byref(lpeers), table, n, None)

    assert call(None, 1) == EINVAL and "layer table is NULL" in err()
    assert call(good(), 3) == EINVAL and "3 layers" in err()
    assert call(good(), 0) == EINVAL and "0 layers" in err()
    t = good()
    t[1].begin, t[1].end = 60, 50
    assert call(t, 2) == EINVAL and "bad layer 1 range [60, 50)" in err()
    t = good()
    t[0].end = 101
    assert call(t, 2) == EINVAL and "bad layer 0 range [0, 101)" in err()
    t = good()
    t[1].bg = None
    assert call(t, 2) == EINVAL and "layer 1 bg is NULL" in err()
    t = good()
    t[0].state_bytes = nb.value - 1
    assert call(t, 2) == ENOMEM and "state too small" in err()
    fr.S = 3
    assert call(good(), 2) == EINVAL and "no feature channels" in err()
    fr.S = 0
    if direction == "backward":
        t = good()
        t[0].dL_dcolor = ok.value
        assert call(t, 2) == EINVAL and "1 of its 3 upstream gradients" in err()
    # a well-formed table reaches the peer table's checks (an empty one here), still before any CUDA call
    assert call(good(), 2) == EINVAL and "bad peer table" in err()
    # a valid one-rank peer table: the layer sections are checked in both directions, and their layer count against the call's
    peers.world, peers.rank, peers.chunk = 1, 0, 100
    peers.records[0] = peers.radii[0] = peers.grad2d[0] = peers.flags[0] = ok.value
    lpeers.layers, lpeers.layer_mask[0] = 2, ok.value

    def live():  # (a backward without any layer gradient is the plain fused one, which reads no layer section)
        t = good()
        t[0].dL_dcolor = t[0].dL_ddepth = t[0].dL_dalpha = ok.value
        return t

    assert call(live(), 2) == EINVAL and "entry 0 has no layer section" in err()
    lpeers.layer_grad2d[0], lpeers.layers = ok.value, 1
    assert call(live(), 2) == EINVAL and "hold 1 layers, the call has 2" in err()


def test_workspace_layer_sections_are_aligned_ordered_and_optional():
    st = _settings()
    P_total = 8 * 12_501
    cpu = torch.device("cpu")
    base = PeerWorkspace.layout(st, P_total, cpu)
    assert PeerWorkspace.layout(st, P_total, cpu, layers=0) == base
    gb, ib, off_radii, off_grad, off_flags, total = PeerWorkspace.layout(st, P_total, cpu, layers=2)
    assert (gb, ib, off_radii, off_grad) == base[:4]
    loss_end = PeerWorkspace.loss_offset(off_grad, P_total, 0) + PeerWorkspace.loss_section_bytes(st)
    assert base[4] == (loss_end + 255) // 256 * 256  # without layers the pad follows the loss section, as before
    off_mask, off_lgrad = PeerWorkspace.layer_offsets(st, off_grad, P_total, 0)
    assert off_mask % 256 == 0 and off_lgrad % 256 == 0 and off_flags % 256 == 0
    assert loss_end <= off_mask and off_mask + P_total <= off_lgrad and off_lgrad + 2 * 48 * P_total <= off_flags and total == off_flags + 256
    wss = PeerWorkspace.emulate(_settings(96, 128), 11, 3, cpu, layers=2)
    for r, ws in enumerate(wss):
        assert ws.layer_grad2d.shape == (2, 33, 12) and ws.layer_mask.shape == (33,) and ws.layer_mask.dtype == torch.uint8
        assert ws.layer_mask.data_ptr() == ws.buf.data_ptr() + ws.off_layer_mask
        assert ws.layer_grad2d.data_ptr() == ws.buf.data_ptr() + ws.off_layer_grad
        for p in range(3):
            assert ws.layer_peers.layer_mask[p] == wss[p].buf.data_ptr() + ws.off_layer_mask
            assert ws.layer_peers.layer_grad2d[p] == wss[p].buf.data_ptr() + ws.off_layer_grad
    plain = PeerWorkspace.emulate(_settings(96, 128), 11, 3, cpu)[0]
    assert plain.layers == 0 and plain.layer_peers.layer_mask[0] is None and plain.layer_grad2d.numel() == 0


def test_mask_restatement_on_a_hand_checked_case():
    """world 2, chunk 300: rank 0 owns 300 rows, rank 1 owns 263.  Rows go to rank 0 (mask 1), rank 1 (mask 2) or both (3)."""
    P_r, chunk, world = [300, 263], 300, 2
    masks = torch.tensor([(i % 3) + 1 for i in range(sum(P_r))])
    ranges = [[(0, 0), (260, 300)], [(0, 263), (5, 7)]]
    out = LC.mask_slots(masks, P_r, chunk, world, ranges)
    for d in range(world):
        slots, gids, bits = out[d]
        # every Gaussian d needs, once, in ascending global order; block b of owner s fills the first slots of [s chunk + 256 b, +256)
        assert torch.equal(gids, torch.nonzero((masks >> d) & 1).flatten())
        for s in range(world):
            for b0 in range(0, P_r[s], 256):
                n = int(((masks[sum(P_r[:s]) + b0: sum(P_r[:s]) + min(P_r[s], b0 + 256)] >> d) & 1).sum())
                g0 = sum(P_r[:s]) + b0
                blk = (gids >= g0) & (gids < g0 + 256) & (gids < sum(P_r[:s + 1]))
                assert torch.equal(slots[blk], s * chunk + b0 + torch.arange(n))
    # bits: rank 0 rows 260..299 are layer 1; rank 1 rows are all layer 0, rows 5, 6 also layer 1
    slots, gids, bits = out[1]
    expect = torch.where(gids < 300, torch.where(gids >= 260, 2, 0), torch.where((gids - 300 >= 5) & (gids - 300 < 7), 3, 1))
    assert torch.equal(bits, expect)
    assert int(bits[(gids == 301)]) == 1 and int(bits[gids == 305]) == 3 and int(bits[gids == 262]) == 2
    assert torch.equal(LC.layer_rows(P_r, ranges, 1), torch.cat([torch.arange(260, 300), torch.arange(305, 307)]))
    assert torch.equal(LC.layer_rows(P_r, ranges, 0), torch.arange(300, 563))


def test_module_refuses_unsupported_configurations_without_a_gpu():
    from street_gaussians_b200.sharded import GaussianShardedRasterizer, ShardedGaussianRasterizer
    st = _settings(64, 64)
    m = torch.zeros(4, 3)
    kw = dict(means3D=m, means2D=None, opacities=torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), scales=torch.ones(4, 3),
              rotations=torch.ones(4, 4), layers=[sgb.RenderLayer(0, 4, (1, 1, 1))])
    with pytest.raises(_capi.SgrError, match="exchange='p2p'.*exchange='nccl'"):
        GaussianShardedRasterizer(st, capacity=sgb.InstanceCapacity()).forward_layers(**kw)
    with pytest.raises(_capi.SgrError, match="fused=False"):
        GaussianShardedRasterizer(st, capacity=sgb.InstanceCapacity(), exchange="p2p", fused=False).forward_layers(**kw)
    with pytest.raises(_capi.SgrError, match="InstanceCapacity"):
        GaussianShardedRasterizer(st, exchange="p2p").forward_layers(**kw)
    with pytest.raises(_capi.SgrError, match="capacity is known"):
        GaussianShardedRasterizer(st, capacity=sgb.InstanceCapacity(), exchange="p2p").forward_layers(**kw)
    cap = sgb.InstanceCapacity()
    cap.observe(1000)
    mod = GaussianShardedRasterizer(st, capacity=cap, exchange="p2p")
    with pytest.raises(_capi.SgrError, match="no feature channels"):
        mod.forward_layers(**kw, semantics=torch.zeros(4, 3))
    with pytest.raises(_capi.SgrError, match="at most 2 layers"):
        mod.forward_layers(**dict(kw, layers=[sgb.RenderLayer(0, 1, (1, 1, 1))] * 3))
    with pytest.raises(_capi.SgrError, match="single-GPU only"):
        ShardedGaussianRasterizer(st).forward_layers(**kw)
