"""CPU checks of densification: the torch oracle against the reference's own densify_and_prune (fixture), the mapping of the
reference's draw order onto the per-parent layout, the new C structs against their ctypes mirrors, and argument validation of
the new entry points without a GPU."""
import ctypes as C
import os
import subprocess

import torch

import densify_case as DC
from oracle import densify_oracle as DO
from street_gaussians_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_reproduces_reference_fixture():
    models, min_opacity = DC.load()
    assert [m["kind"] for m in models] == ["background", "actor", "actor"]
    for k, m in enumerate(models):
        out, scalars, mask, _, _ = DO.densify_model(m["in"], m["kind"], m["draws"], **DC.oracle_kwargs(m, min_opacity))
        ref = m["out"]
        for key, v in m["scalars"].items():
            assert scalars[key] == v, (k, key, scalars[key], v)
        assert out["xyz"].shape[0] == ref["xyz"].shape[0]
        assert int((mask & 1).count_nonzero() + ((mask >> 1) & 1).sum() + ((mask >> 2) & 1).sum() + ((mask >> 3) & 1).sum()) == ref["xyz"].shape[0]
        for a in DC.NAMES:
            assert out[a].shape == ref[a].shape, (k, a)
            assert torch.allclose(out[a], ref[a], rtol=0, atol=1e-6), (k, a, float((out[a] - ref[a]).abs().max()))
            for mk in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(out[mk][a], ref[mk][a]), (k, a, mk)
        for s in ("xyz_gradient_accum", "denom", "max_radii2D"):
            assert out[s].shape == ref[s].shape and not ref[s].any()
        # the fixture exercises every section and both prune causes
        assert scalars["points_clone"] > 0 and scalars["points_split"] > 0 and scalars["points_pruned"] > 0
        assert set(mask.unique().tolist()) >= {0, 1, 3, 12}


def test_reference_draw_order_round_trips_through_the_layout():
    models, _ = DC.load()
    for m in models:
        t = m["in"]
        _, clone, split = DO.decisions(t, m["grad_col"], m["grad_threshold"], m["extent"], m["percent_dense"])
        box = m["kind"] == "actor"
        z_split, z_box = DO.layout_to_reference_draws(m["draws"], clone, split, box)
        assert z_split.shape == (2 * int(split.sum()), 3)
        back = DO.reference_draws_to_layout(t["xyz"].shape[0], z_split, z_box, clone, split)
        assert torch.equal(back, m["draws"])
        if box:
            assert z_box.shape == (int((~split).sum() + clone.sum() + 2 * split.sum()), 2, 3)
        # slots a parent does not use stay zero
        unused = ~split
        assert not m["draws"][unused, 0:6].any()
        if box:
            assert not m["draws"][~clone & ~split, 12:18].any()


def test_densify_structs_match_ctypes(tmp_path):
    structs = ["SgrDensifySegment", "SgrDensifyOutput"]
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "sgr.h"', 'int main(void) {']
    for name in structs:
        body.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        body += [f'  printf("{name}.{f[0]} %zu\\n", offsetof({name}, {f[0]}));' for f in getattr(_capi, name)._fields_]
    body += ['  printf("T %d\\n", SGR_DENSIFY_TENSORS);', '  printf("D %d\\n", SGR_DENSIFY_DRAWS);', '  printf("R %d\\n", SGR_DENSIFY_RESULT);',
             '  printf("B %d\\n", SGR_DENSIFY_BACKGROUND);', '  printf("A %d\\n", SGR_DENSIFY_ACTOR);', '  return 0;', '}']
    src = tmp_path / "densify_layout.c"
    src.write_text("\n".join(body))
    exe = tmp_path / "densify_layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(line.rsplit(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for name in structs:
        ct = getattr(_capi, name)
        assert int(out[name]) == C.sizeof(ct), name
        for f in ct._fields_:
            assert int(out[f"{name}.{f[0]}"]) == getattr(ct, f[0]).offset, (name, f[0])
    assert (int(out["T"]), int(out["D"]), int(out["R"])) == (_capi.DENSIFY_TENSORS, _capi.DENSIFY_DRAWS, _capi.DENSIFY_RESULT)
    assert (int(out["B"]), int(out["A"])) == (_capi.DENSIFY_BACKGROUND, _capi.DENSIFY_ACTOR)


def _valid_segment(count=10):
    s = _capi.SgrDensifySegment()
    s.kind, s.count, s.dc_width, s.rest_width, s.semantic_width = _capi.DENSIFY_BACKGROUND, count, 3, 9, 0
    for a in (0, 1, 2, 3, 4, 5):
        s.param[a] = 0x1000 * (a + 1)
    s.max_radii2D, s.xyz_gradient_accum, s.denom = 0x9000, 0xA000, 0xB000
    return s


def test_densify_entry_points_validate_before_touching_cuda():
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    res = (C.c_int64 * 16)()
    assert L.sgr_densify_plan(None, 0, 0, None, None, 0, res, None) == -1 and "empty" in err()
    segs = (_capi.SgrDensifySegment * 2)(_valid_segment(), _valid_segment())
    segs[1].kind = 7
    assert L.sgr_densify_plan(segs, 2, 0, None, None, 0, res, None) == -1 and "unknown kind" in err()
    segs[1].kind = _capi.DENSIFY_ACTOR
    segs[1].grad_col = 2
    assert L.sgr_densify_plan(segs, 2, 0, None, None, 0, res, None) == -1 and "grad_col" in err()
    segs[1].grad_col = 0
    segs[0].param[2] = None
    assert L.sgr_densify_plan(segs, 2, 0, None, None, 0, res, None) == -1 and "features_rest is NULL" in err()
    segs[0].param[2] = 0x3000
    segs[0].param[6] = 0x7000
    assert L.sgr_densify_plan(segs, 2, 0, None, None, 0, res, None) == -1 and "zero row width" in err()
    segs[0].param[6] = None
    segs[0].exp_avg[0] = 0xC000
    assert L.sgr_densify_plan(segs, 2, 0, None, None, 0, res, None) == -1 and "both Adam moments" in err()
    segs[0].exp_avg[0] = None
    segs[1].denom = None
    assert L.sgr_densify_plan(segs, 2, 0, None, None, 0, res, None) == -1 and "statistics" in err()
    segs[1].denom = 0xB000
    assert L.sgr_densify_plan(segs, 2, 0, None, None, 0, None, None) == -1 and "result is NULL" in err()
    need = L.sgr_densify_scratch_bytes(2, 20)
    assert need > 20 * 17
    assert L.sgr_densify_plan(segs, 2, 0, None, None, 0, res, None) == -3 and "scratch too small" in err()
    # apply: the output table must match the inputs' tensors and moments
    assert L.sgr_densify_apply(segs, None, 2, 0, None, None, 0, None) == -1 and "output table" in err()
    outs = (_capi.SgrDensifyOutput * 2)()
    outs[0].count = 5
    assert L.sgr_densify_apply(segs, outs, 2, 0, None, None, 0, None) == -1 and "output 0: xyz is NULL" in err()
    for a in (0, 1, 2, 3, 4, 5):
        outs[0].param[a] = 0x1000
    outs[0].exp_avg[1] = outs[0].exp_avg_sq[1] = 0x2000
    assert L.sgr_densify_apply(segs, outs, 2, 0, None, None, 0, None) == -1 and "exactly where the input" in err()
    outs[0].exp_avg[1] = outs[0].exp_avg_sq[1] = None
    outs[0].max_radii2D, outs[0].xyz_gradient_accum, outs[0].denom = 1, 2, 3
    assert L.sgr_densify_apply(segs, outs, 2, 0, None, None, 0, None) == -3 and "scratch too small" in err()
    # reset_opacity
    assert L.sgr_reset_opacity(None, 0, None) == -1 and "empty" in err()
    segs[0].param[3] = None
    assert L.sgr_reset_opacity(segs, 2, None) == -1 and "opacity is NULL" in err()
