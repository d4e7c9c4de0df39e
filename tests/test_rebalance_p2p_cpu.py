"""CPU: rebalance's row moves over the Gaussian-sharded rasterizer's peer memory (sharded.PeerTransport, sharded.peer_rounds,
include/sgr.h sgr_peer_exchange_round) and ViewMetrics(rasterizer=).

  * peer_rounds at world 2, 3, 5, 8 and 16, with ranks that send nothing and moves larger than the staging region: every float of every
    pair moves exactly once, each round's pieces of a source fit its staging region without overlapping, every offset is a multiple of
    4 floats, and every rank issues the same barriers;
  * PeerTransport's all_gather and exchange on workspaces emulated on CPU buffers, with the library's calls replaced by a Python
    restatement (stage, barrier, pull; threads for the ranks): every buffer arrives, and every rank makes the same calls;
  * the refusals (exchange="nccl", no workspace yet, a forward in flight, sums that do not fit the loss section) raise before any call;
  * the new struct against the header, and the entry's argument checks before anything is enqueued."""
import ctypes as C
import os
import subprocess
import threading
import types

import numpy as np
import pytest
import torch

import street_gaussians_b200 as sgb
from rank_threads import run_ranks
from street_gaussians_b200 import _capi, metrics
from street_gaussians_b200 import sharded as SH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK = C.c_void_p(1 << 20)  # a 16-byte aligned address: validation fails before anything dereferences it


def _err():
    return _capi.lib().sgr_last_error().decode()


def _sizes(world, seed, big=0, empty=()):
    """[world][world] float counts: random, ranks in `empty` send nothing, pair (0, world - 1) gets `big` floats more."""
    rng = np.random.default_rng(seed)
    s = rng.integers(0, 50, size=(world, world)) * (rng.random((world, world)) < 0.6)
    np.fill_diagonal(s, 0)
    for r in empty:
        s[r, :] = 0
    s[0, world - 1] += big
    return s.tolist()


def _check_schedule(sizes, cap):
    world = len(sizes)
    rounds = SH.peer_rounds(sizes, cap)
    cover = {(s, d): np.zeros(sizes[s][d], dtype=np.int64) for s in range(world) for d in range(world)}
    C4 = cap // 4 * 4
    for pieces in rounds:
        used = {}
        for p in pieces:
            assert p.floats > 0 and p.stage_at % 4 == 0 and p.buf_at % 4 == 0, p
            assert 0 <= p.stage_at and p.stage_at + p.floats <= C4, p
            cover[(p.src, p.dst)][p.buf_at:p.buf_at + p.floats] += 1
            used.setdefault(p.src, []).append((p.stage_at, p.stage_at + p.floats))
        for spans in used.values():  # a source's pieces of one round never overlap in its staging region
            spans.sort()
            assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), spans
        for r in range(world):  # at most one piece per peer on each side: the kernel's table holds SGR_MAX_PEERS
            assert sum(p.src == r for p in pieces) <= world - 1 and sum(p.dst == r for p in pieces) <= world - 1
    for key, c in cover.items():
        assert bool((c == 1).all()), (key, c)
    # every rank computes the schedule from the same table: the same rounds, hence 1 + 2 rounds barriers, also without a piece of its own
    per_rank = [1 + 2 * len(SH.peer_rounds([list(row) for row in sizes], cap)) for _ in range(world)]
    assert len(set(per_rank)) == 1
    return rounds


@pytest.mark.parametrize("world", [2, 3, 5, 8, 16])
def test_rounds_move_every_float_once(world):
    for seed in range(4):
        sizes = _sizes(world, seed + 10 * world, big=1000 + seed, empty=(1,))
        assert not any(sizes[1])
        total = max(sum(row) for row in sizes)
        for cap in (16, 64, 4 * total, 4 * total + 3):
            rounds = _check_schedule(sizes, cap)
            if cap == 16:
                assert len(rounds) > 1000 // 16  # the big move takes many rounds
            if cap >= 4 * total:
                assert len(rounds) == 1
    assert SH.peer_rounds([[0] * world for _ in range(world)], 64) == []


def test_rounds_reject_bad_tables():
    with pytest.raises(ValueError):
        SH.peer_rounds([[1, 2], [3, 0]], 64)  # a rank sending to itself
    with pytest.raises(ValueError):
        SH.peer_rounds([[0, -1], [0, 0]], 64)
    with pytest.raises(ValueError):
        SH.peer_rounds([[0, 1, 0], [0, 0]], 64)
    with pytest.raises(ValueError):
        SH.peer_rounds([[0, 5], [0, 0]], 3)  # not even one aligned piece fits


def _st(H=96, W=128):
    return sgb.GaussianRasterizationSettings(H, W, 0.5, 0.4, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)


def _rasterizers(world, chunk=6):
    wss = SH.PeerWorkspace.emulate(_st(), chunk, world, torch.device("cpu"))
    return [types.SimpleNamespace(exchange="p2p", _ws=ws) for ws in wss], wss


class _Library:
    """sgr_peer_exchange_round and sgr_peer_barrier restated on CPU buffers, the ranks being threads: a barrier is a thread barrier,
    and the pieces are copied with memmove at the addresses the library would use.  Records every rank's calls."""

    def __init__(self, world):
        self.bar = threading.Barrier(world, timeout=60)
        self.calls = [[] for _ in range(world)]

    def __call__(self, name, device, *args):
        peers = args[0]._obj
        rank = peers.rank
        if name == "sgr_peer_barrier":
            self.calls[rank].append("barrier")
            self.bar.wait()
            return
        assert name == "sgr_peer_exchange_round", name
        staging, stage, n_stage, pull, n_pull = args[1:]
        self.calls[rank].append(("round", n_stage, n_pull))
        for i in range(n_stage):
            p = stage[i]
            assert p.rank == rank and p.offset % 4 == 0 and 4 * (p.offset + p.floats) <= staging
            C.memmove(peers.records[rank] + 4 * p.offset, p.local, 4 * p.floats)
        self.bar.wait()
        for i in range(n_pull):
            p = pull[i]
            assert p.offset % 4 == 0 and 4 * (p.offset + p.floats) <= staging and p.local % 16 == 0
            C.memmove(p.local, peers.records[p.rank] + 4 * p.offset, 4 * p.floats)


@pytest.mark.parametrize("world,chunk", [(2, 1), (3, 2), (5, 6), (8, 1)])
def test_transport_moves_every_buffer(world, chunk, monkeypatch):
    """all_gather and exchange through emulated CPU workspaces, the rounds at `chunk` slots per rank (chunk 1: the moves need several
    rounds).  Rank 1 sends nothing; every rank makes the same barrier calls."""
    rasts, wss = _rasterizers(world, chunk)
    for ws in wss:
        ws.buf[: ws.off_flags].fill_(0x7f)
    lib = _Library(world)
    monkeypatch.setattr(_capi, "call", lib)
    cap = SH.PeerTransport(rasts[0]).staging_bytes // 4
    sizes = _sizes(world, world, big=3 * cap + 5, empty=(1,))
    g = torch.Generator().manual_seed(world)
    data = [[torch.randn(sizes[s][d], generator=g) for d in range(world)] for s in range(world)]
    tables = [torch.arange(33, dtype=torch.int64).view(3, 11) * (r + 1) for r in range(world)]

    def rank(r, _tr):
        tr = SH.PeerTransport(rasts[r])
        assert (tr.world, tr.rank) == (world, r)
        got = tr.all_gather(tables[r])
        assert rasts[r]._ws.fwd_pending  # the next forward waits for the peers' reads of the table
        recvs = {s: torch.full((sizes[s][r],), float("nan")) for s in range(world) if sizes[s][r]}
        tr.exchange({d: data[r][d] for d in range(world) if sizes[r][d]}, recvs, sizes)
        assert not rasts[r]._ws.fwd_pending
        return got, recvs

    out = run_ranks(world, rank)
    for r, (got, recvs) in enumerate(out):
        assert all(torch.equal(a, b) for a, b in zip(got, tables)) and all(a.dtype == torch.int64 for a in got)
        for s in range(world):
            if sizes[s][r]:
                assert torch.equal(recvs[s], data[s][r]), (r, s)
    n_rounds = len(SH.peer_rounds(sizes, cap))
    assert n_rounds > 1
    barriers = [sum(c == "barrier" for c in calls) for calls in lib.calls]
    assert barriers == [1 + n_rounds] * world  # + one inside each round call: 1 + 2 rounds in all
    assert [sum(isinstance(c, tuple) for c in calls) for calls in lib.calls] == [1 + n_rounds] * world
    assert all(c[1] == 0 for c in lib.calls[1][1:] if isinstance(c, tuple))  # the empty sender stages nothing in the exchange, yet takes part
    assert all(ws.epoch == 1 + 1 + 2 * n_rounds for ws in wss)


def test_exchange_checks_the_buffers_against_the_table(monkeypatch):
    rasts, _ = _rasterizers(2)
    monkeypatch.setattr(_capi, "call", lambda *a: pytest.fail("no call may be made"))
    tr = SH.PeerTransport(rasts[0])
    with pytest.raises(ValueError, match="send buffer of rank 1"):
        tr.exchange({1: torch.zeros(3)}, {}, [[0, 4], [0, 0]])
    with pytest.raises(ValueError, match="receive buffer of rank 1"):
        tr.exchange({}, {}, [[0, 0], [2, 0]])
    with pytest.raises(ValueError, match="send buffer"):
        tr.exchange({1: torch.zeros(4, dtype=torch.float64)}, {}, [[0, 4], [0, 0]])


def test_refusals_raise_before_any_call(monkeypatch):
    rasts, wss = _rasterizers(2)
    monkeypatch.setattr(_capi, "call", lambda *a: pytest.fail("no call may be made"))
    with pytest.raises(_capi.SgrError, match="exchange='nccl'"):
        SH.PeerTransport(SH.GaussianShardedRasterizer(_st(), exchange="nccl"))
    with pytest.raises(_capi.SgrError, match="forward and backward first"):
        SH.PeerTransport(SH.GaussianShardedRasterizer(_st(), exchange="p2p"))
    wss[0].in_flight = True
    with pytest.raises(_capi.SgrError, match="backward"):
        SH.PeerTransport(rasts[0])
    wss[1].in_flight = False
    tr = SH.PeerTransport(rasts[1])
    wss[1].in_flight = True  # a forward between making the transport and using it
    with pytest.raises(_capi.SgrError, match="backward"):
        tr.all_gather(torch.zeros(2, 11, dtype=torch.int64))
    with pytest.raises(_capi.SgrError, match="backward"):
        tr.exchange({}, {}, [[0, 0], [0, 0]])
    # rebalance with a refused transport: the transport raises while it is made, before rebalance runs
    m = types.SimpleNamespace(_xyz=torch.zeros(0, 3))
    with pytest.raises(_capi.SgrError):
        SH.rebalance([m], transport=SH.PeerTransport(rasts[0]))
    assert not torch.cuda.is_initialized()


def test_transport_keeps_its_workspace_across_repartition(monkeypatch):
    """rebalance repartitions the rasterizer before it exchanges: the transport keeps the workspace it was made with."""
    rast = SH.GaussianShardedRasterizer(_st(), exchange="p2p", chunk=6)
    rast._ws = SH.PeerWorkspace.emulate(_st(), 6, 1, torch.device("cpu"))[0]
    tr = SH.PeerTransport(rast)
    ws = rast._ws
    monkeypatch.setattr(SH.PeerWorkspace, "__init__", lambda *a, **k: pytest.fail("no workspace may be set up"))
    assert rast.repartition(9, chunk=9) == 9
    assert tr.ws is ws and rast._ws is ws
    t = torch.arange(22, dtype=torch.int64).view(2, 11)
    assert tr.all_gather(t)[0] is t  # world 1: nothing to move


def test_view_metrics_refuses_sums_that_do_not_fit(monkeypatch):
    H = 96
    ws = SH.PeerWorkspace.emulate(_st(H), 6, 2, torch.device("cpu"))[0]
    ri = types.SimpleNamespace(exchange="p2p", group=None, band=SH.cyclic_band(H, 0, 2), loss_workspace=lambda: ws)
    vm = metrics.ViewMetrics(rasterizer=ri)
    V = ws.loss_bytes // (8 * _capi.EVAL_SUMS) + 1
    vm._n, vm._sums, vm._H = V, torch.zeros(V, _capi.EVAL_SUMS, dtype=torch.float64), H
    monkeypatch.setattr(_capi, "call", lambda *a: pytest.fail("no call may be made"))
    with pytest.raises(ValueError, match="do not fit"):
        vm.result()
    assert len(vm) == V  # nothing was dropped


def test_struct_layout_compiled_from_the_header(tmp_path):
    src = tmp_path / "layout.c"
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "sgr.h"', 'int main(void) {',
            '  printf("size %zu\\n", sizeof(SgrPeerPiece));']
    body += [f'  printf("{f[0]} %zu\\n", offsetof(SgrPeerPiece, {f[0]}));' for f in _capi.SgrPeerPiece._fields_] + ['  return 0;', '}']
    src.write_text("\n".join(body))
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(line.rsplit(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["size"]) == C.sizeof(_capi.SgrPeerPiece)
    for f in _capi.SgrPeerPiece._fields_:
        assert int(out[f[0]]) == getattr(_capi.SgrPeerPiece, f[0]).offset, f[0]
    assert "sgr_peer_exchange_round" in _capi.SYMBOLS


def test_round_validates_before_launch():
    L = _capi.lib()
    pe = _capi.SgrPeers()
    pe.world, pe.rank, pe.chunk = 2, 1, 8
    for p in range(2):
        pe.records[p], pe.flags[p] = OK.value, OK.value
    P = _capi.SgrPeerPiece

    def call(stage=(), pull=(), peers=pe, staging=4096):
        ts = (P * max(1, len(stage)))(*stage)
        tp = (P * max(1, len(pull)))(*pull)
        return L.sgr_peer_exchange_round(C.byref(peers) if peers is not None else None, staging, ts, len(stage), tp, len(pull), None)

    assert call(peers=None) == -1 and "peers is NULL" in _err()
    bad = _capi.SgrPeers()
    bad.world, bad.rank = 2, 2
    assert call(peers=bad) == -1 and "bad peer table" in _err()
    nopad = _capi.SgrPeers()
    nopad.world, nopad.rank = 2, 0
    nopad.records[0] = nopad.records[1] = OK.value
    assert call(peers=nopad) == -1 and "barrier pad" in _err()
    noreg = _capi.SgrPeers()
    noreg.world, noreg.rank = 2, 0
    noreg.flags[0] = noreg.flags[1] = OK.value
    noreg.records[0] = OK.value
    assert call(peers=noreg) == -1 and "staging region" in _err()
    noreg.records[1] = OK.value + 4
    assert call(peers=noreg) == -1 and "16-byte aligned" in _err()
    assert call(stage=[P(0, 0, 0, 4, OK.value)]) == -1 and "names rank 0" in _err()  # a rank stages into its own region only
    assert call(pull=[P(2, 0, 0, 4, OK.value)]) == -1 and "names rank 2" in _err()
    assert call(pull=[P(0, 0, 2, 4, OK.value)]) == -1 and "16-byte aligned inside" in _err()
    assert call(pull=[P(0, 0, 1020, 8, OK.value)]) == -1 and "inside" in _err()
    assert call(pull=[P(0, 0, -4, 4, OK.value)]) == -1 and "inside" in _err()
    assert call(pull=[P(0, 0, 0, 4, None)]) == -1 and "NULL buffer" in _err()
    assert call(pull=[P(0, 0, 0, 4, OK.value + 8)]) == -1 and "16-byte aligned" in _err()
    assert call(pull=[P(0, 0, 0, 1, OK.value)] * 17) == -1 and "at most 16" in _err()
