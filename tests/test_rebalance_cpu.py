"""CPU checks of rebalancing Gaussian ownership across ranks: sharded.rebalance_plan against a numpy restatement that assigns every
global row to its new owner, on hand-picked and random splits, and the argument validation of sgr_rebalance_pack / sgr_rebalance_splice,
which must reject bad ranges, buffer sizes and pointers before anything is launched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from street_gaussians_b200 import _capi
from street_gaussians_b200.sharded import rebalance_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def restate(counts):
    """Global rows (model-major; within a model rank-major) of every (rank, model) before, and after the even split of the global rows."""
    counts = np.asarray(counts, dtype=np.int64).reshape(len(counts), -1)
    world, nm = counts.shape
    P = int(counts.sum())
    old, g = {}, 0
    for m in range(nm):
        for r in range(world):
            old[r, m] = np.arange(g, g + counts[r, m])
            g += counts[r, m]
    base, extra = divmod(P, world)
    B = np.array([r * base + min(r, extra) for r in range(world + 1)])
    owner = np.searchsorted(B, np.arange(P), side="right") - 1
    model_of = np.concatenate([np.full(int(counts[:, m].sum()), m) for m in range(nm)]) if nm else np.zeros(0, np.int64)
    new = {(r, m): np.nonzero((owner == r) & (model_of == m))[0] for r in range(world) for m in range(nm)}
    return old, new, owner


def check_plan(counts):
    plan = rebalance_plan(counts)
    world, nm = len(counts), len(counts[0])
    old, new, owner = restate(counts)
    got = {(r, m): np.full(plan.counts[r][m], -1, dtype=np.int64) for r in range(world) for m in range(nm)}
    for mv in plan.moves + plan.kept:
        assert 0 <= mv.src_row_begin < mv.src_row_end <= counts[mv.src][mv.model]
        rows = old[mv.src, mv.model][mv.src_row_begin:mv.src_row_end]
        dst = got[mv.dst, mv.model][mv.dst_row_begin:mv.dst_row_begin + len(rows)]
        assert len(dst) == len(rows) and (dst == -1).all(), ("rows written twice or past the new count", mv)
        got[mv.dst, mv.model][mv.dst_row_begin:mv.dst_row_begin + len(rows)] = rows
    for key in got:
        assert np.array_equal(got[key], new[key]), (key, got[key], new[key])
    totals = [sum(c) for c in plan.counts]
    assert max(totals) - min(totals) <= 1
    # a row moves exactly when its owner changes; rows that stay are never part of a move
    moved = np.concatenate([old[mv.src, mv.model][mv.src_row_begin:mv.src_row_end] for mv in plan.moves]) if plan.moves else np.zeros(0, np.int64)
    old_owner = np.empty(len(owner), dtype=np.int64)
    for (r, m), rows in old.items():
        old_owner[rows] = r
    assert all(mv.src != mv.dst for mv in plan.moves) and all(mv.src == mv.dst for mv in plan.kept)
    assert np.array_equal(np.sort(moved), np.nonzero(old_owner != owner)[0])
    # the rank-major concatenation of the new rows is the global array
    cat = np.concatenate([got[r, m] for r in range(world) for m in range(nm)])
    assert np.array_equal(cat, np.arange(len(owner)))
    # every move lands in its destination's own range
    for mv in plan.moves:
        assert (owner[old[mv.src, mv.model][mv.src_row_begin:mv.src_row_end]] == mv.dst).all()
    return plan


CASES = {
    "world1": [[7, 0, 3]],
    "balanced": [[5, 0, 0], [1, 4, 0], [0, 2, 3]],
    "one_rank_holds_everything": [[100, 20, 30], [0, 0, 0], [0, 0, 0], [0, 0, 0]],
    "empty_ranks": [[0, 0], [40, 3], [0, 0], [0, 9], [0, 0]],
    "model_empty_everywhere": [[10, 0, 0], [6, 0, 4], [0, 0, 0]],
    "model_spans_three_ranks": [[2, 0], [30, 0], [1, 0], [0, 1]],
    "skew_past_neighbour": [[90, 0, 0], [0, 5, 0], [0, 0, 3], [0, 0, 2]],
    "last_rank_heavy": [[1, 0], [0, 1], [0, 1], [0, 61]],
    "single_model": [[3], [17], [0], [8], [1], [0], [0], [40]],
    "nothing": [[0, 0], [0, 0]],
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_plan_matches_restatement(name):
    plan = check_plan(CASES[name])
    if name in ("world1", "balanced", "nothing"):
        assert plan.moves == []
    if name == "skew_past_neighbour":
        assert any(mv.src == 0 and mv.dst == 3 for mv in plan.moves)
    if name == "one_rank_holds_everything":
        assert {mv.dst for mv in plan.moves} == {1, 2, 3} and {mv.src for mv in plan.moves} == {0}


def _random_split(rng, world, nm):
    """A valid split: per-model totals, then the ranks' global ranges cut at random points."""
    totals = rng.integers(0, 50, nm) * (rng.random(nm) > 0.2)
    P = int(totals.sum())
    cuts = np.sort(rng.integers(0, P + 1, world - 1))
    B = np.concatenate([[0], cuts, [P]])
    G = np.concatenate([[0], np.cumsum(totals)])
    return [[max(0, min(B[r + 1], G[m + 1]) - max(B[r], G[m])) for m in range(nm)] for r in range(world)]


def test_plan_matches_restatement_on_random_splits():
    rng = np.random.default_rng(5)
    for _ in range(300):
        check_plan(_random_split(rng, int(rng.integers(1, 9)), int(rng.integers(1, 6))))


def test_plan_rejects_splits_that_break_the_global_order():
    with pytest.raises(ValueError, match="rank-major split"):
        rebalance_plan([[5, 3], [2, 4]])  # rank 1 holds model-0 rows after rank 0 held model-1 rows
    with pytest.raises(ValueError):
        rebalance_plan([[5, -1]])
    with pytest.raises(ValueError):
        rebalance_plan([[5, 1], [2]])
    with pytest.raises(ValueError):
        rebalance_plan([])


# ---- the C ABI ----
def test_rebalance_struct_matches_ctypes(tmp_path):
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "sgr.h"', 'int main(void) {',
            '  printf("SgrRebalanceRange %zu\\n", sizeof(SgrRebalanceRange));']
    body += [f'  printf("{f[0]} %zu\\n", offsetof(SgrRebalanceRange, {f[0]}));' for f in _capi.SgrRebalanceRange._fields_]
    body += ['  printf("moments %zu\\n", offsetof(SgrDensifySegment, moments));', '  return 0;', '}']
    src = tmp_path / "rebalance_layout.c"
    src.write_text("\n".join(body))
    exe = tmp_path / "rebalance_layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(line.rsplit(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["SgrRebalanceRange"]) == C.sizeof(_capi.SgrRebalanceRange)
    for f in _capi.SgrRebalanceRange._fields_:
        assert int(out[f[0]]) == getattr(_capi.SgrRebalanceRange, f[0]).offset, f[0]
    assert int(out["moments"]) == _capi.SgrDensifySegment.moments.offset


def _segment(count=10, moments=0b111111):
    """A segment of fake device addresses (never dereferenced: every call below fails validation first)."""
    s = _capi.SgrDensifySegment()
    s.count, s.dc_width, s.rest_width, s.semantic_width, s.moments = count, 3, 45, 0, moments
    for a in range(6):
        s.param[a] = 0x10000 * (a + 1)
        if (moments >> a) & 1:
            s.exp_avg[a], s.exp_avg_sq[a] = 0x100000 * (a + 1), 0x200000 * (a + 1)
    s.max_radii2D, s.xyz_gradient_accum, s.denom = 0x9000, 0xA000, 0xB000
    return s


def _ranges(*rows):
    t = (_capi.SgrRebalanceRange * len(rows))()
    for i, (seg, buf, src, dst, n) in enumerate(rows):
        t[i].segment, t[i].buffer, t[i].src_row, t[i].dst_row, t[i].rows = seg, buf, src, dst, n
    return t


def test_row_floats():
    L = _capi.lib()
    s = _segment()
    assert L.sgr_rebalance_row_floats(C.byref(s)) == 3 * (3 + 3 + 45 + 1 + 3 + 4) + 4
    s.moments = 0
    assert L.sgr_rebalance_row_floats(C.byref(s)) == 59 + 4
    s.semantic_width, s.moments = 5, 1 << 6
    assert L.sgr_rebalance_row_floats(C.byref(s)) == 64 + 5 * 2 + 4
    s.semantic_width = 0
    assert L.sgr_rebalance_row_floats(C.byref(s)) == -1 and b"moment bit 6" in L.sgr_last_error()
    assert L.sgr_rebalance_scratch_bytes(4) >= 4 * 24 * 24


def test_pack_validates_before_any_launch():
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    segs = (_capi.SgrDensifySegment * 2)(_segment(10), _segment(0))
    rf = 181
    bufs = (C.c_void_p * 2)(0x5000000, 0x6000000)
    size = (C.c_int64 * 2)(4 * rf, 10 * rf)
    pack = lambda r, n, b=bufs, sz=size, nb=2, scratch=None, sb=0: L.sgr_rebalance_pack(segs, 2, r, n, b, sz, nb, scratch, sb, None)
    ok = _ranges((0, 0, 6, 0, 4), (0, 1, 0, 0, 6))
    assert L.sgr_rebalance_pack(None, 0, ok, 2, bufs, size, 2, None, 0, None) == -1 and "segment table is empty" in err()
    assert pack(_ranges((2, 0, 0, 0, 1)), 1) == -1 and "names segment 2" in err()
    assert pack(_ranges((0, 2, 0, 0, 1)), 1) == -1 and "names buffer 2" in err()
    assert pack(_ranges((0, -1, 0, 0, 1)), 1) == -1 and "names buffer -1" in err()  # only splice reads old rows directly
    assert pack(_ranges((0, 0, 7, 0, 4)), 1) == -1 and "reads rows [7, 11) of segment 0, which has 10" in err()
    assert pack(_ranges((1, 0, 0, 0, 1)), 1) == -1 and "segment 1, which has 0" in err()
    assert pack(_ranges((0, 0, -1, 0, 1)), 1) == -1 and "reads rows" in err()
    assert pack(_ranges((0, 0, 0, 0, -1)), 1) == -1 and "reads rows" in err()
    # two blocks in one buffer need both blocks' floats
    assert pack(_ranges((0, 0, 0, 0, 4), (0, 0, 4, 0, 1)), 2) == -3 and "buffer 0 holds 724 floats" in err()
    nul = (C.c_void_p * 2)(None, 0x6000000)
    assert pack(ok, 2, b=nul) == -1 and "buffer 0 is NULL" in err()
    assert pack(ok, 2, nb=-1) == -1 and "bad buffer table" in err()
    assert pack(None, 2) == -1 and "bad range table" in err()
    segs[0].exp_avg[2] = None
    assert pack(ok, 2) == -1 and "Adam moments of features_rest" in err()
    segs[0].exp_avg[2] = 0x300000
    segs[0].param[1] = None
    assert pack(ok, 2) == -1 and "features_dc is NULL" in err()
    segs[0].param[1] = 0x20000
    segs[0].denom = None
    assert pack(ok, 2) == -1 and "statistics" in err()
    segs[0].denom = 0xB000
    segs[0].rest_width = -1
    assert pack(ok, 2) == -1 and "row widths" in err()
    segs[0].rest_width = 45
    # everything valid: the scratch is checked before the launch
    assert pack(ok, 2) == -3 and "scratch too small" in err()
    assert pack(ok, 2, scratch=0x7000000, sb=L.sgr_rebalance_scratch_bytes(2) - 1) == -3 and "scratch too small" in err()


def test_splice_validates_before_any_launch():
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    segs = (_capi.SgrDensifySegment * 2)(_segment(10), _segment(0))
    outs = (_capi.SgrDensifyOutput * 2)()
    for k, n in enumerate((8, 5)):
        o = outs[k]
        o.count = n
        for a in range(6):
            o.param[a], o.exp_avg[a], o.exp_avg_sq[a] = 0x1000 * (a + 1), 0x2000 * (a + 1), 0x3000 * (a + 1)
        o.max_radii2D, o.xyz_gradient_accum, o.denom = 0x10, 0x20, 0x30
    bufs = (C.c_void_p * 1)(0x5000000)
    size = (C.c_int64 * 1)(10 * 181)
    splice = lambda r, n, o=outs, scratch=None: L.sgr_rebalance_splice(segs, o, 2, r, n, bufs, size, 1, scratch, 0, None)
    ok = _ranges((0, -1, 2, 0, 8), (1, 0, 0, 0, 5))
    assert splice(ok, 2, o=None) == -1 and "output table is NULL" in err()
    assert splice(_ranges((0, -1, 4, 0, 8), (1, 0, 0, 0, 5)), 2) == -1 and "reads rows [4, 12)" in err()
    assert splice(_ranges((0, -1, 2, 1, 8), (1, 0, 0, 0, 5)), 2) == -1 and "writes rows [1, 9) of output 0, which has 8" in err()
    assert splice(_ranges((0, -1, 2, 0, 7), (1, 0, 0, 0, 5)), 2) == -1 and "write 7 of its 8 rows" in err()
    assert splice(_ranges((0, -1, 2, 0, 4), (0, -1, 0, 3, 5), (1, 0, 0, 0, 5)), 3) == -1 and "not written exactly once" in err()
    assert splice(_ranges((0, -1, 2, 0, 8), (1, 0, 0, 0, 5), (1, 0, 0, 0, 6)), 3) == -1 and "writes rows [0, 6)" in err()
    assert splice(_ranges((0, 0, 0, 0, 8), (1, 0, 0, 0, 5)), 2) == -3 and "buffer 0 holds 1810 floats" in err()
    outs[1].exp_avg_sq[4] = None
    assert splice(ok, 2) == -1 and "output 1: the Adam moments of scaling" in err()
    outs[1].exp_avg_sq[4] = 0x5000
    outs[1].param[6] = 0x7000
    assert splice(ok, 2) == -1 and "output 1: semantic is given for a zero row width" in err()
    outs[1].param[6] = None
    outs[0].xyz_gradient_accum = None
    assert splice(ok, 2) == -1 and "output 0 has a NULL statistics array" in err()
    outs[0].xyz_gradient_accum = 0x20
    outs[0].count = -1
    assert splice(ok, 2) == -1 and "output 0: count -1" in err()
    outs[0].count = 8
    assert splice(ok, 2) == -3 and "scratch too small" in err()
