"""CPU-side checks of the render layers (include/sgr.h, SgrLayer): the entry points are exported, the C structs match their ctypes
mirrors, and bad layers and CPU tensors are rejected before anything is launched."""
import ctypes as C
import os
import subprocess

import pytest
import torch

import street_gaussians_b200 as sgb
import util
from street_gaussians_b200 import _capi, synthetic
from street_gaussians_b200.sharded import GaussianShardedRasterizer, ShardedGaussianRasterizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("sgr_layer_state_sizes", "sgr_forward_layer", "sgr_backward_blend_layer", "sgr_backward_geom_layered")


def _frame(P=100, W=64, H=48):
    fr = _capi.SgrFrame()
    fr.P, fr.width, fr.height, fr.D, fr.M = P, W, H, 0, 0
    fr.tan_fovx, fr.tan_fovy, fr.scale_modifier = 0.5, 0.4, 1.0
    return fr


def test_layer_symbols_exported():
    lib = C.CDLL(_capi.LIB_PATH)
    for s in NEW:
        assert s in _capi.SYMBOLS and hasattr(lib, s), s
    assert _capi.lib().sgr_abi_version() == 7


def test_layer_struct_layouts_match_ctypes(tmp_path):
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "sgr.h"', 'int main(void) {']
    for name in ("SgrLayer", "SgrLayerGrad"):
        body.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        body += [f'  printf("{name}.{f[0]} %zu\\n", offsetof({name}, {f[0]}));' for f in getattr(_capi, name)._fields_]
    body += ['  return 0;', '}']
    src, exe = tmp_path / "layers.c", tmp_path / "layers"
    src.write_text("\n".join(body))
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(line.rsplit(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for name in ("SgrLayer", "SgrLayerGrad"):
        ct = getattr(_capi, name)
        assert int(out[name]) == C.sizeof(ct), name
        for f in ct._fields_:
            assert int(out[f"{name}.{f[0]}"]) == getattr(ct, f[0]).offset, (name, f[0])


def test_layer_entry_points_validate_before_touching_cuda():
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    fr = _frame()
    nb = C.c_size_t(0)
    assert L.sgr_layer_state_sizes(C.byref(fr), 1000, C.byref(nb)) == 0
    assert nb.value >= 1000 * 4 + 64 * 48 * 4 and nb.value % 256 == 0
    assert L.sgr_layer_state_sizes(C.byref(fr), -1, C.byref(nb)) == -1
    bg = C.c_void_p(16)  # never dereferenced: every call below fails its checks first
    for b, e in ((-1, 5), (6, 5), (0, 101)):
        lay = _capi.SgrLayer(b, e, bg)
        assert L.sgr_forward_layer(C.byref(fr), C.byref(lay), 0, None, None, None, None, 0, None, None, None, None) == -1
        assert "bad layer range" in err()
        assert L.sgr_backward_blend_layer(C.byref(fr), C.byref(lay), None, None, None, None, None, None, None, None) == -1
    lay = _capi.SgrLayer(0, 5, None)
    assert L.sgr_forward_layer(C.byref(fr), C.byref(lay), 0, None, None, None, None, 0, None, None, None, None) == -1 and "bg" in err()
    fr.row_begin, fr.row_end, fr.row_step = 0, 2, 1
    lay = _capi.SgrLayer(0, 5, bg)
    assert L.sgr_forward_layer(C.byref(fr), C.byref(lay), 0, None, None, None, None, 0, None, None, None, None) == -4 and "whole image" in err()
    fr = _frame()
    grads = (_capi.SgrLayerGrad * 1)(_capi.SgrLayerGrad(3, 200, None, None))
    assert L.sgr_backward_geom_layered(C.byref(fr), *([None] * 9), grads, 1, None, *([None] * 8), None) == -1 and "range" in err()


def _cpu_call(layers, rast_cls=sgb.GaussianRasterizer, **kw):
    scene = synthetic.make_scene(P=40, width=64, height=48, sh_degree=1, seed=3)
    st = util.settings_from(sgb, scene["cam"], "cpu")
    rast = rast_cls(st, **kw)
    return rast.forward_layers(means3D=scene["means3D"], means2D=torch.zeros(40, 3), opacities=scene["opacities"], shs=scene["shs"],
                               scales=scene["scales"], rotations=scene["rotations"], layers=layers)


def test_bad_layers_are_rejected_before_any_launch():
    for layers in ([sgb.RenderLayer(-1, 3, (1.0, 1.0, 1.0))], [sgb.RenderLayer(5, 4, (1.0, 1.0, 1.0))],
                   [sgb.RenderLayer(0, 41, (1.0, 1.0, 1.0))], [sgb.RenderLayer(0, 40, (1.0, 1.0))],
                   [sgb.RenderLayer(0, 40, torch.ones(4))], [sgb.RenderLayer(0, 40, torch.ones(3), torch.zeros(39, 3))],
                   [(0, 40, (1.0, 1.0, 1.0)), (10, 50, (0.0, 0.0, 0.0))]):
        with pytest.raises(ValueError):
            _cpu_call(layers)


def test_cpu_tensors_and_sharded_rasterizers_raise():
    with pytest.raises(_capi.SgrError, match="CUDA"):
        _cpu_call([sgb.RenderLayer(10, 40, (1.0, 1.0, 1.0))])
    with pytest.raises(_capi.SgrError, match="whole image"):
        _cpu_call([sgb.RenderLayer(10, 40, (1.0, 1.0, 1.0))], band=sgb.TileRowBand(0, 2, 1))
    with pytest.raises(_capi.SgrError, match="single-GPU"):
        _cpu_call([sgb.RenderLayer(10, 40, (1.0, 1.0, 1.0))], rast_cls=ShardedGaussianRasterizer)
    scene = synthetic.make_scene(P=40, width=64, height=48, sh_degree=1, seed=3)
    rast = GaussianShardedRasterizer.__new__(GaussianShardedRasterizer)
    with pytest.raises(_capi.SgrError, match="single-GPU"):
        GaussianShardedRasterizer.forward_layers(rast, scene["means3D"], None, scene["opacities"], shs=scene["shs"], scales=scene["scales"],
                                                 rotations=scene["rotations"], layers=[sgb.RenderLayer(0, 40, (1.0, 1.0, 1.0))])
    assert "layers" not in __import__("inspect").signature(sgb.GaussianRasterizer.forward).parameters
