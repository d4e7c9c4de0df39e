"""CPU checks of checkpoints under Gaussian sharding and of the sky's lat-long export: sharded.even_slices against rebalance_plan,
sharded.gather_pieces (every row exactly once, rank-major, no piece over its limit), the PNG writer decoded with zlib, argument checks
that fire before anything touches CUDA, training.adam_state_dict against torch.optim.Adam.state_dict, and the ctypes mirror of
sgr_sky_cube_to_latlong."""
import ctypes as C
import os
import re
import struct
import types
import zlib

import numpy as np
import pytest
import torch

from street_gaussians_b200 import _capi, sky, training
from street_gaussians_b200 import sharded as SH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def random_tables(seed=0, n=300):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        world, nm = int(rng.integers(1, 10)), int(rng.integers(1, 6))
        totals = [int(rng.integers(0, 4) and rng.integers(0, 40)) for _ in range(nm)]
        yield world, totals


@pytest.mark.parametrize("seed", [0, 1])
def test_even_slices_are_the_split_rebalance_leaves(seed):
    for world, totals in random_tables(seed):
        sl = SH.even_slices(totals, world)
        # every row once, in rank-major order within each model
        for k, n in enumerate(totals):
            at = 0
            for r in range(world):
                lo, hi = sl[r][k]
                assert lo == at and lo <= hi
                at = hi
            assert at == n
        # rebalance() from any split of the same global rows ends with these counts (all rows on rank 0, and on the last rank)
        for start in ([totals] + [[0] * len(totals)] * (world - 1), [[0] * len(totals)] * (world - 1) + [totals]):
            assert SH.rebalance_plan(start).counts == [[hi - lo for lo, hi in row] for row in sl], (world, totals)
        P = sum(totals)
        per = [sum(hi - lo for lo, hi in row) for row in sl]
        assert per == [P // world + (r < P % world) for r in range(world)]


def test_even_slices_more_ranks_than_rows():
    sl = SH.even_slices([2, 0, 3], 8)
    assert [sum(hi - lo for lo, hi in row) for row in sl] == [1, 1, 1, 1, 1, 0, 0, 0]
    assert sl[5] == [(2, 2), (0, 0), (3, 3)]
    with pytest.raises(ValueError):
        SH.even_slices([1], 0)
    with pytest.raises(ValueError):
        SH.even_slices([1, -1], 2)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gather_pieces_cover_every_row_once_in_rank_major_order(seed):
    rng = np.random.default_rng(seed)
    for _ in range(200):
        world, nm = int(rng.integers(1, 9)), int(rng.integers(1, 5))
        counts = [[int(rng.integers(0, 3) and rng.integers(0, 30)) for _ in range(nm)] for _ in range(world)]
        row_bytes = [int(rng.integers(1, 8)) * 4 for _ in range(nm)]
        piece = int(rng.integers(max(row_bytes), 80))
        pieces = SH.gather_pieces(counts, row_bytes, piece)
        seen = []
        for s, ranges in pieces:
            assert ranges and sum(rows * row_bytes[k] for k, _, rows in ranges) <= piece
            for k, first, rows in ranges:
                assert rows > 0
                seen += [(s, k, first + i) for i in range(rows)]
        assert seen == [(s, k, i) for s in range(world) for k in range(nm) for i in range(counts[s][k])]
        assert [s for s, _ in pieces] == sorted(s for s, _ in pieces)


def test_gather_pieces_limits():
    assert SH.gather_pieces([[3, 0], [0, 2]], [8, 4], 1 << 30) == [(0, [(0, 0, 3)]), (1, [(1, 0, 2)])]
    assert SH.gather_pieces([[3]], [8], 8) == [(0, [(0, 0, 1)]), (0, [(0, 1, 1)]), (0, [(0, 2, 1)])]
    # a model nobody holds rows of does not bound the piece
    assert SH.gather_pieces([[0, 1]], [1000, 4], 4) == [(0, [(1, 0, 1)])]
    with pytest.raises(ValueError, match="smaller than one row"):
        SH.gather_pieces([[1]], [16], 8)


def decode_png(data: bytes):
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    at, chunks = 8, []
    while at < len(data):
        n, = struct.unpack(">I", data[at:at + 4])
        kind, body = data[at + 4:at + 8], data[at + 8:at + 8 + n]
        crc, = struct.unpack(">I", data[at + 8 + n:at + 12 + n])
        assert crc == zlib.crc32(kind + body) & 0xFFFFFFFF
        chunks.append((kind, body))
        at += 12 + n
    assert [k for k, _ in chunks] == [b"IHDR", b"IDAT", b"IEND"]
    W, H, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", chunks[0][1])
    assert (depth, ctype, comp, filt, inter) == (8, 2, 0, 0, 0)
    raw = np.frombuffer(zlib.decompress(chunks[1][1]), np.uint8).reshape(H, 1 + 3 * W)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(H, W, 3)


@pytest.mark.parametrize("shape", [(1, 1), (7, 13), (16, 32), (3, 200)])
def test_png_writer_round_trips(shape):
    a = np.random.default_rng(shape[0]).integers(0, 256, shape + (3,), dtype=np.uint8)
    assert np.array_equal(decode_png(sky.png_bytes(a)), a)
    assert np.array_equal(decode_png(sky.png_bytes(torch.from_numpy(a))), a)


def test_png_writer_rejects_other_arrays():
    for bad in (np.zeros((2, 2, 3), np.float32), np.zeros((2, 2), np.uint8), np.zeros((0, 2, 3), np.uint8), np.zeros((2, 2, 4), np.uint8)):
        with pytest.raises(ValueError):
            sky.png_bytes(bad)


def test_latlong_argument_checks():
    cube = torch.zeros(6, 4, 4, 3)
    with pytest.raises(_capi.SgrError, match="no CPU fallback"):
        sky.cubemap_to_latlong(cube, (4, 8))
    for bad in (torch.zeros(6, 4, 5, 3), torch.zeros(5, 4, 4, 3), torch.zeros(6, 4, 4, 4)):
        with pytest.raises(ValueError, match="6, R, R, 3"):
            sky.cubemap_to_latlong(bad, (4, 8))
    with pytest.raises(ValueError, match="float32"):
        sky.cubemap_to_latlong(cube.double(), (4, 8))


def test_latlong_entry_validates_before_touching_cuda():
    L = _capi.lib()
    for args in ((0, 1, 4, 8, 1, 1), (16385, 1, 4, 8, 1, 1), (4, 1, 0, 8, 1, 1), (4, 1, 4, -1, 1, 1), (4, None, 4, 8, 1, 1), (4, 1, 4, 8, None, None), (4, 1, 65536, 65536 * 128, 1, 1)):
        R, cube, H, W, out, u8 = args
        rc = L.sgr_sky_cube_to_latlong(R, cube, H, W, out, u8, None)
        assert rc != 0
        assert b"sgr_sky_cube_to_latlong" in L.sgr_last_error()


def test_latlong_ctypes_mirror_matches_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "sgr.h")).read(), flags=re.S)
    decl = re.search(r"int\s+sgr_sky_cube_to_latlong\s*\(([^)]*)\)", src).group(1)
    params = [p.strip() for p in decl.split(",")]
    L = _capi.lib()
    fn = L.sgr_sky_cube_to_latlong
    assert "sgr_sky_cube_to_latlong" in _capi.SYMBOLS
    assert fn.restype is C.c_int and len(fn.argtypes) == len(params) == 7
    kinds = [C.c_int32 if p.startswith("int32_t") else C.c_void_p for p in params]
    assert list(fn.argtypes) == kinds


def test_gather_state_argument_checks():
    tr = types.SimpleNamespace(world=2, rank=0)
    with pytest.raises(ValueError, match="sub-models"):
        SH.gather_state([], transport=tr)
    m = {a: torch.zeros(0, 3) for a in training.PARAM_NAMES}
    with pytest.raises(ValueError, match="dst=2"):
        SH.gather_state([m], dst=2, transport=tr)
    with pytest.raises(ValueError, match="piece_bytes"):
        SH.gather_state([m], piece_bytes=0, transport=tr)


def reference_model(n=5, M=4, S=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.nn.Parameter(torch.randn(*s, generator=g))
    return types.SimpleNamespace(_xyz=r(n, 3), _features_dc=r(n, 1, 3), _features_rest=r(n, M - 1, 3), _opacity=r(n, 1), _scaling=r(n, 3),
                                 _rotation=r(n, 4), _semantic=r(n, S))


def reference_optimizer(m, lrs=(1.6e-4, 2.5e-3, 1.25e-4, 0.05, 5e-3, 1e-3, 1e-3)):
    """GaussianModel.training_setup's torch.optim.Adam (gaussian_model.py:286-303)."""
    return torch.optim.Adam([{"params": [getattr(m, a)], "lr": lr, "name": n} for a, n, lr in zip(training.PARAM_NAMES, training.ADAM_GROUP_NAMES, lrs)],
                            lr=0.0, eps=1e-15)


def test_adam_state_dict_is_torch_adams_state_dict():
    m = reference_model()
    opt = reference_optimizer(m)
    fresh = training.adam_state_dict(m, opt)
    assert fresh["state"] == {} and fresh["param_groups"] == opt.state_dict()["param_groups"]
    for it in range(3):
        for a in training.PARAM_NAMES[:-1]:  # the semantic tensor gets no gradient: it keeps no state, as in torch
            getattr(m, a).grad = torch.randn_like(getattr(m, a)) * (it + 1)
        opt.step()
    want, got = opt.state_dict(), training.adam_state_dict(m, opt)
    assert got["param_groups"] == want["param_groups"]
    assert list(got["state"]) == list(want["state"]) == list(range(6))
    for i, st in want["state"].items():
        assert list(got["state"][i]) == list(st)
        for k, v in st.items():
            assert got["state"][i][k].dtype == v.dtype and torch.equal(got["state"][i][k], v), (i, k)
    # the reference's optimizer takes it back
    m2 = reference_model(seed=1)
    opt2 = reference_optimizer(m2)
    opt2.load_state_dict(got)
    assert int(opt2.state[m2._xyz]["step"]) == 3 and torch.equal(opt2.state[m2._xyz]["exp_avg"], opt.state[m._xyz]["exp_avg"])


def test_adam_state_dict_over_one_optimizer_of_several_models():
    ms = [reference_model(seed=s) for s in range(2)]
    opt = training.FusedAdam([{"params": [getattr(m, a) for m in ms], "lr": 1e-3 * (i + 1), "name": n}
                              for i, (a, n) in enumerate(zip(training.PARAM_NAMES, training.ADAM_GROUP_NAMES))], eps=1e-15)
    for m in ms:
        opt.state[m._xyz] = dict(step=4, exp_avg=torch.ones(5, 3), exp_avg_sq=torch.full((5, 3), 2.0))
    sd = training.adam_state_dict(ms[1], opt)
    assert [g["name"] for g in sd["param_groups"]] == list(training.ADAM_GROUP_NAMES)
    assert [g["params"] for g in sd["param_groups"]] == [[i] for i in range(7)]
    assert [g["lr"] for g in sd["param_groups"]] == [1e-3 * (i + 1) for i in range(7)]
    assert list(sd["state"]) == [0] and float(sd["state"][0]["step"]) == 4.0 and sd["state"][0]["step"].dtype == torch.float32
    with pytest.raises(ValueError, match="not held by the optimizer"):
        training.adam_state_dict(reference_model(seed=9), opt)
