"""CPU checks of the block-masked Adam of the sky cube map: sgr_cube_sparse_adam_step's and the accumulating marks' argument checks
without a GPU, the new sgr.h declarations against their ctypes prototypes, sky.block_map's size against the block formula, and the
checks training.CubeMapSparseAdam makes before anything touches a device."""
import ctypes as C
import os
import re

import pytest
import torch

from street_gaussians_b200 import _capi, sky, training

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("sgr_cube_sparse_adam_step", "sgr_band_sky_composite_backward_or_marks", "sgr_sky_grad_peer_sum_union")
C_TYPES = {"int32_t": C.c_int32, "float": C.c_float, "double": C.c_double}


def _blocks(R):
    return 6 * (-(-R // 32)) ** 2


def _declarations():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "sgr.h")).read(), flags=re.S)
    out = {}
    for name in ENTRIES:
        m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
        assert m, name
        out[name] = [p.strip() for p in m.group(1).replace("\n", " ").split(",")]
    return out


def test_header_declarations_match_ctypes_prototypes():
    L = _capi.lib()
    for name, params in _declarations().items():
        assert name in _capi.SYMBOLS
        fn = getattr(L, name)
        assert fn.restype is C.c_int, name
        assert len(fn.argtypes) == len(params), (name, len(fn.argtypes), len(params))
        for p, t in zip(params, fn.argtypes):
            if "*" in p:
                assert t is C.c_void_p or issubclass(t, C._Pointer), (name, p, t)
            else:
                assert t is C_TYPES[p.split()[0]], (name, p, t)
    assert L.sgr_cube_sparse_adam_step.argtypes[1] is C.POINTER(_capi.SgrAdamTensor)


@pytest.mark.parametrize("R", [1, 16, 31, 32, 33, 40, 64, 100, 1024, 16384])
def test_block_map_size_is_the_block_formula(R):
    m = sky.block_map(R, "cpu")
    assert m.dtype == torch.uint8 and m.shape == (_blocks(R),) and not bool(m.any())
    assert int(_capi.lib().sgr_sky_grad_blocks(R)) == _blocks(R)


@pytest.mark.parametrize("R", [0, -3, 16385])
def test_block_map_refuses_bad_sizes(R):
    with pytest.raises(ValueError):
        sky.block_map(R, "cpu")


def _rec(R, numel=None, step=1, lr=1e-3):
    t = _capi.SgrAdamTensor()
    t.param, t.grad, t.exp_avg, t.exp_avg_sq = 0x1000, 0x2000, 0x3000, 0x4000
    t.numel = 18 * R * R if numel is None else numel
    t.lr, t.step = lr, step
    return t


def test_cube_step_validates_before_touching_cuda():
    """Every call below fails its checks, so nothing is enqueued on the made-up device addresses."""
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    fn = L.sgr_cube_sparse_adam_step
    call = lambda R, rec, m=0x5000, b1=0.9, b2=0.999: fn(R, None if rec is None else C.byref(rec), m, b1, b2, 1e-15, None)
    for R in (0, -1, 16385):
        assert call(R, _rec(8)) == -1 and "R=" in err()
    assert call(8, None) == -1 and "NULL" in err()
    assert call(8, _rec(8), m=None) == -1 and "NULL" in err()
    for field in ("param", "grad", "exp_avg", "exp_avg_sq"):
        r = _rec(8)
        setattr(r, field, None)
        assert call(8, r) == -1 and "NULL" in err(), field
    assert call(8, _rec(8, numel=18 * 64 - 3)) == -1 and "numel" in err()
    assert call(9, _rec(8)) == -1 and "numel" in err()
    assert call(8, _rec(8, step=0)) == -1 and "step" in err()
    for lr in (float("nan"), float("inf")):
        assert call(8, _rec(8, lr=lr)) == -1 and "lr" in err()
    for b1, b2 in ((1.0, 0.999), (-0.1, 0.999), (0.9, 1.0), (0.9, float("nan"))):
        assert call(8, _rec(8), b1=b1, b2=b2) == -1 and "betas" in err()


def test_accumulating_entries_validate_before_touching_cuda():
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    p = 0x1000
    marks = lambda m, R=16, rows=(0, 2, 1): L.sgr_band_sky_composite_backward_or_marks(32, 32, *rows, R, 0, 1.0, p, None, p, p, p, None, None, p,
                                                                                       p, p, m, None)
    assert marks(None) == -1 and "NULL" in err()
    assert marks(p, R=0) == -1
    assert marks(p, rows=(3, 1, 1)) == -1 and "band" in err()
    peers, skyp = _capi.SgrPeers(), _capi.SgrSkyPeers()
    peers.world, peers.rank = 2, 0
    union = lambda u, m=p: L.sgr_sky_grad_peer_sum_union(C.byref(peers), C.byref(skyp), 16, m, p, u, None)
    assert union(None) == -1 and "union_map" in err()
    assert union(p) == -1 and "must not be block_map" in err()
    assert union(0x9000) == -1 and "section" in err()  # the sky section table is empty
    peers.world = 0
    assert union(0x9000) == -1 and "peer table" in err()


# ---- training.CubeMapSparseAdam -------------------------------------------------------------------------------------------------
def _cube(R=40, grad=True):
    p = torch.nn.Parameter(torch.zeros(6, R, R, 3))
    if grad:
        p.grad = torch.ones_like(p)
    return p


@pytest.mark.parametrize("shape", [(6, 8, 8), (5, 8, 8, 3), (6, 8, 9, 3), (6, 8, 8, 4), (1, 6, 8, 8, 3)])
def test_optimizer_refuses_a_cube_of_the_wrong_shape(shape):
    with pytest.raises(ValueError, match="6, R, R, 3"):
        training.CubeMapSparseAdam([torch.nn.Parameter(torch.zeros(shape))])


def test_optimizer_refuses_wrong_dtype_layout_and_count():
    with pytest.raises(ValueError, match="fp32"):
        training.CubeMapSparseAdam([torch.nn.Parameter(torch.zeros(6, 8, 8, 3, dtype=torch.float64))])
    with pytest.raises(ValueError, match="contiguous"):
        training.CubeMapSparseAdam([torch.nn.Parameter(torch.zeros(6, 8, 3, 8).transpose(2, 3))])
    with pytest.raises(ValueError, match="exactly one"):
        training.CubeMapSparseAdam([_cube(8), _cube(8)])
    with pytest.raises(ValueError, match="exactly one"):
        training.CubeMapSparseAdam([{"params": [_cube(8)]}, {"params": [_cube(8)], "lr": 0.1}])
    with pytest.raises(ValueError, match="R=16385"):
        training.CubeMapSparseAdam([torch.nn.Parameter(torch.empty(6, 16385, 16385, 3, device="meta"))])


def test_step_needs_a_map_of_the_cube_size():
    p = _cube(40)
    opt = training.CubeMapSparseAdam([p], lr=0.1, eps=1e-15)
    with pytest.raises(TypeError, match="dense fallback"):
        opt.step()
    for bad in (torch.zeros(_blocks(40) + 1, dtype=torch.uint8), torch.zeros(_blocks(40) - 1, dtype=torch.uint8),
                torch.zeros(_blocks(40), dtype=torch.int32), torch.zeros(_blocks(40), dtype=torch.bool),
                torch.zeros(2 * _blocks(40), dtype=torch.uint8)[::2]):
        with pytest.raises(ValueError, match="blocks"):
            opt.step(bad)
    assert not opt.state and bool((p == 0).all())


def test_step_refuses_cpu_tensors_and_changes_nothing():
    p = _cube(40)
    opt = training.CubeMapSparseAdam([p], lr=0.1, eps=1e-15)
    m = sky.block_map(40, "cpu")
    m[3] = 1
    with pytest.raises(_capi.SgrError, match="CUDA"):
        opt.step(m)
    assert not opt.state and bool((p == 0).all()) and int(m.sum()) == 1


def test_step_without_a_gradient_changes_nothing():
    p = _cube(40, grad=False)
    opt = training.CubeMapSparseAdam([p], lr=0.1, eps=1e-15)
    m = sky.block_map(40, "cpu")
    m[:5] = 1
    assert opt.step(m) is None
    assert not opt.state and bool((p == 0).all()) and int(m.sum()) == 5


def test_step_refuses_bad_hyper_parameters_before_any_state_changes():
    p = _cube(8)
    m = sky.block_map(8, "cpu")
    for kw in (dict(lr=float("nan")), dict(lr=float("inf")), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.5))):
        opt = training.CubeMapSparseAdam([p], **kw)
        with pytest.raises(ValueError, match="lr|betas"):
            opt.step(m)
        assert not opt.state
