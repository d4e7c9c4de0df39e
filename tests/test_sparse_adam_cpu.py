"""CPU checks of the visibility-masked Adam: the SgrSparseAdamSegment layout against its ctypes mirror, argument validation of
sgr_sparse_adam_step without a GPU, and the shape / length / device checks of training.SparseAdam."""
import ctypes as C
import os
import subprocess
import types

import pytest
import torch

from street_gaussians_b200 import _capi, training

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sparse_adam_struct_matches_ctypes(tmp_path):
    name = "SgrSparseAdamSegment"
    ct = _capi.SgrSparseAdamSegment
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "sgr.h"', 'int main(void) {',
            f'  printf("{name} %zu\\n", sizeof({name}));']
    body += [f'  printf("{name}.{f[0]} %zu\\n", offsetof({name}, {f[0]}));' for f in ct._fields_]
    body += ['  printf("ABI %d\\n", SGR_ABI_VERSION);', '  printf("MAXW %d\\n", SGR_SPARSE_ADAM_MAX_WIDTH);', '  return 0;', '}']
    src = tmp_path / "sparse_adam_layout.c"
    src.write_text("\n".join(body))
    exe = tmp_path / "sparse_adam_layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(line.rsplit(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out[name]) == C.sizeof(ct)
    for f in ct._fields_:
        assert int(out[f"{name}.{f[0]}"]) == getattr(ct, f[0]).offset, f[0]
    assert int(out["ABI"]) == _capi.ABI_VERSION == 7
    assert int(out["MAXW"]) == _capi.SPARSE_ADAM_MAX_WIDTH and 256 * _capi.SPARSE_ADAM_MAX_WIDTH < 2 ** 31


def _segment(start, count, widths=(3, 3, 45, 1, 3, 4, 0)):
    s = _capi.SgrSparseAdamSegment()
    s.start, s.count = start, count
    for a, w in enumerate(widths):
        s.width[a] = w
        if w:
            s.param[a], s.grad[a], s.exp_avg[a], s.exp_avg_sq[a] = (0x1000 * (4 * a + j + 1) for j in range(4))
            s.lr[a], s.step[a] = 1e-3, 1
    return s


def test_sparse_adam_step_validates_before_touching_cuda():
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    radii = 0x9000
    call = lambda segs, n, r=radii, b1=0.9, b2=0.999: L.sgr_sparse_adam_step(segs, n, r, b1, b2, 1e-15, None)
    assert call(None, 0) == -1 and "empty" in err()

    def table():
        return (_capi.SgrSparseAdamSegment * 3)(_segment(0, 10), _segment(10, 0), _segment(10, 7, (3, 15, 45, 1, 3, 4, 3)))

    t = table()
    t[0].count = -1
    assert call(t, 3) == -1 and "segment 0" in err() and "count -1" in err()
    t = table()
    t[0].start = -2
    assert call(t, 3) == -1 and "segment 0: start -2" in err()
    t = table()
    t[2].start = 12                      # a gap after segment 1
    assert call(t, 3) == -1 and "segment 2: start 12 (expected 10)" in err()
    t = table()
    t[2].start = 4                       # not ascending
    assert call(t, 3) == -1 and "segment 2: start 4" in err()
    t = table()
    t[2].width[6] = -3
    assert call(t, 3) == -1 and "semantic has width -3" in err()
    t = table()
    t[2].width[2] = _capi.SPARSE_ADAM_MAX_WIDTH + 1   # 256 rows of it would overflow the kernel's int span
    assert call(t, 3) == -4 and "features_rest has width 8388608 > 8388607" in err()
    t[2].width[2] = _capi.SPARSE_ADAM_MAX_WIDTH
    assert call(t, 3, r=None) == -1 and "radii is NULL" in err()
    for field in ("param", "grad", "exp_avg", "exp_avg_sq"):
        t = table()
        getattr(t[2], field)[1] = None
        assert call(t, 3) == -1 and "segment 2: features_dc has a NULL pointer" in err(), field
    t = table()
    t[1].param[0] = None                 # no rows: NULL pointers are fine
    t[0].param[6] = None                 # width 0: NULL pointers are fine
    t[2].step[3] = 0
    assert call(t, 3) == -1 and "opacity has step 0" in err()
    t = table()
    t[1].step[0] = -4                    # step is checked even where there are no rows
    assert call(t, 3) == -1 and "segment 1: xyz has step -4" in err()
    for bad in (float("nan"), float("inf"), float("-inf")):
        t = table()
        t[0].lr[5] = bad
        assert call(t, 3) == -1 and "rotation has a non-finite lr" in err(), bad
    t = table()
    assert call(t, 3, b1=1.0) == -1 and "betas" in err()
    assert call(t, 3, r=None) == -1 and "radii is NULL" in err()
    # nothing to update: no rows at all needs no radii and no CUDA
    empty = (_capi.SgrSparseAdamSegment * 2)(_segment(0, 0), _segment(0, 0))
    assert call(empty, 2, r=None) == 0


def _model(n, dc=1, rest=15, sem=0, grad=True):
    shapes = ((n, 3), (n, dc, 3), (n, rest, 3), (n, 1), (n, 3), (n, 4), (n, sem))
    m = types.SimpleNamespace()
    for name, s in zip(training.PARAM_NAMES, shapes):
        p = torch.nn.Parameter(torch.zeros(s))
        if grad:
            p.grad = torch.zeros(s)
        setattr(m, name, p)
    return m


def _optimizer(models):
    return training.SparseAdam([{"params": [getattr(m, n)], "lr": 1e-3} for m in models for n in training.PARAM_NAMES], eps=1e-15)


def test_sparse_adam_python_checks():
    bg, act = _model(20), _model(5, dc=5)
    opt = _optimizer([bg, act])
    r = torch.ones(25, dtype=torch.int32)
    with pytest.raises(TypeError, match="dense"):
        opt.step()
    with pytest.raises(TypeError, match="dense"):
        opt.step([bg, act])
    with pytest.raises(ValueError, match=r"radii must be an int32 tensor of shape \[25\]"):
        opt.step([bg, act], torch.ones(24, dtype=torch.int32))
    with pytest.raises(ValueError, match="int32"):
        opt.step([bg, act], torch.ones(25, dtype=torch.int64))
    with pytest.raises(ValueError, match=r"\[25\]"):
        opt.step([bg, act], torch.ones(25, 1, dtype=torch.int32))
    bad = _model(5, dc=5)
    bad._opacity = torch.nn.Parameter(torch.zeros(4, 1))
    with pytest.raises(ValueError, match="model 1: _opacity has shape"):
        opt.step([bg, bad], r)
    with pytest.raises(_capi.SgrError, match="CUDA"):
        opt.step([bg, act], r)
    # nothing was touched by the failed calls
    assert len(opt.state) == 0 and not any(getattr(bg, n).any() for n in training.PARAM_NAMES)
