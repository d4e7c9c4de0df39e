"""CPU: the restated sky cube map composite (tests/sky_oracle.py) against the reference's own outputs (tests/golden/callsite/sky.npz),
the restated cube lookup's geometry (texel centres, the 12 edges, the adjacency table, the corner rule), and argument checks of
street_gaussians_b200.sky and its C entries that run before anything touches CUDA."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest
import torch

import sky_oracle as SO
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi

F64 = torch.float64
FIX = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "callsite", "sky.npz")
CASES = ("train_mask", "train_acc", "eval_acc")


def load(case):
    z = np.load(FIX)
    t = lambda k: torch.from_numpy(z[k])
    mask = t(f"{case}_sky_mask") if f"{case}_sky_mask" in z else None
    jx = t(f"{case}_jx") if f"{case}_jx" in z else None
    jy = t(f"{case}_jy") if f"{case}_jy" in z else None
    return z, dict(rgb=t(f"{case}_rgb"), acc=t(f"{case}_acc"), cube=t("cube_map"), K=t("K"), w2c=t(f"{case}_w2c"), g=t(f"{case}_g"),
                   sky_mask=mask, jx=jx, jy=jy, fill=float(z[f"{case}_fill"]))


@pytest.mark.parametrize("case", CASES)
def test_restatement_reproduces_reference_fixture(case):
    z, a = load(case)
    r = SO.sky64(a["rgb"], a["acc"], a["cube"], a["K"], a["w2c"], a["g"], a["sky_mask"], a["jx"], a["jy"], a["fill"])
    ref = lambda k: torch.from_numpy(z[f"{case}_{k}"]).to(F64)
    # the reference rounds its rays in fp32 through K^-1 and the camera origin; R = 16 keeps that far below 1e-5
    assert float((r["out"] - ref("ref_out")).abs().max()) < 1e-5
    assert float((r["dacc"] - ref("ref_dacc")).abs().max()) < 1e-5
    assert float((r["dcube"] - ref("ref_dcube")).abs().max()) < 1e-4 * float(ref("ref_dcube").abs().max())
    assert torch.equal(ref("ref_drgb"), a["g"].to(F64))
    # the case exercises what it is meant to: sampled and filled pixels, the clamp at both ends, several faces
    mask = SO.sky_mask_of(a["acc"], a["sky_mask"])
    assert 0 < int(mask.sum()) < mask.numel()
    s = SO.lookup(a["cube"].to(F64), SO.rays(64, 80, a["K"].to(F64), a["w2c"].to(F64), a["jx"], a["jy"]))[mask]
    assert bool((s < 0).any()) and bool((s > 1).any())
    assert len(set(r["face"][mask].tolist())) >= 3
    if a["sky_mask"] is not None:  # the reference wrote rows 0-49 into the mask it was given
        after = torch.from_numpy(z[f"{case}_mask_after"])
        assert bool(after[0, :50].all()) and torch.equal(after[0, 50:], a["sky_mask"][0, 50:])


def test_fp32_restatement_matches_float64():
    _, a = load("train_mask")
    o = SO.composite(a["rgb"], a["acc"], a["cube"], a["K"], a["w2c"], a["sky_mask"], a["jx"], a["jy"], a["fill"])
    r = SO.sky64(a["rgb"], a["acc"], a["cube"], a["K"], a["w2c"], a["g"], a["sky_mask"], a["jx"], a["jy"], a["fill"])
    assert bool(((o.to(F64) - r["out"]).abs() <= r["b_out"]).all())


@pytest.mark.parametrize("R", [1, 2, 16])
def test_every_texel_centre_returns_its_texel(R):
    cube = torch.randn(6, R, R, 3, dtype=F64, generator=torch.Generator().manual_seed(R))
    g = (2 * torch.arange(R, dtype=F64) + 1) / R - 1
    gy, gx = torch.meshgrid(g, g, indexing="ij")
    for s in range(6):
        got = SO.lookup(cube, SO.cube_to_dir(s, gx, gy))
        assert torch.equal(got, cube[s]), s


def _edge_points(f, edge, R, n=7):
    """Directions on the seam of face f's edge and their unit normal across it (pointing off the face)."""
    t = torch.linspace(-0.9, 0.9, n, dtype=F64)
    one = torch.ones_like(t)
    gx, gy = {0: (-one, t), 1: (one, t), 2: (t, -one), 3: (t, one)}[edge]
    d = SO.cube_to_dir(f, gx, gy)
    Uv, Vv = torch.tensor(SO.FACE_U[f], dtype=F64), torch.tensor(SO.FACE_V[f], dtype=F64)
    out = {0: -Uv, 1: Uv, 2: -Vv, 3: Vv}[edge]
    return d, out


@pytest.mark.parametrize("f,edge", list(itertools.product(range(6), range(4))))
def test_each_edge_is_continuous(f, edge):
    R = 16
    cube = torch.rand(6, R, R, 3, dtype=F64, generator=torch.Generator().manual_seed(7 * f + edge))
    d, out = _edge_points(f, edge, R)
    for eps in (1e-3, 1e-5, 1e-7):
        a, b = SO.lookup(cube, d - eps * out), SO.lookup(cube, d + eps * out)
        # first order: the lookup's slope is at most R / 2 texel differences (<= 1) per unit of face coordinate, times 2 faces
        assert float((a - b).abs().max()) <= 2 * R * eps, (eps, float((a - b).abs().max()))
    # the two sides choose different faces
    fa, _, _ = SO.face_coords(d - 1e-7 * out)
    fb, _, _ = SO.face_coords(d + 1e-7 * out)
    assert bool((fa == f).all()) and not bool((fb == f).any())


@pytest.mark.parametrize("R", [2, 5, 16])
def test_adjacency_table_agrees_with_geometry(R):
    """For every out-of-face tap, the direction of its extrapolated centre lands, on the face it selects, nearest to the texel ADJ
    maps the tap to."""
    for f in range(6):
        t = torch.arange(R)
        for edge, (c, r) in enumerate([(torch.full_like(t, -1), t), (torch.full_like(t, R), t), (t, torch.full_like(t, -1)), (t, torch.full_like(t, R))]):
            gx, gy = (2 * c.to(F64) + 1) / R - 1, (2 * r.to(F64) + 1) / R - 1
            face, hx, hy = SO.face_coords(SO.cube_to_dir(f, gx, gy))
            col = torch.floor((hx + 1) / 2 * R).long().clamp(0, R - 1)
            row = torch.floor((hy + 1) / 2 * R).long().clamp(0, R - 1)
            want = (face * R + row) * R + col
            got = SO.tap_texels(torch.full_like(t, f), c, r, R)
            assert torch.equal(got, want), (f, edge)
            assert bool((face == SO.ADJ[f][edge][0]).all())
    # every edge is shared by exactly two faces, and the table is symmetric
    for f, edge in itertools.product(range(6), range(4)):
        nf = SO.ADJ[f][edge][0]
        assert nf != f and nf // 2 != f // 2 and sum(e[0] == f for e in SO.ADJ[nf]) == 1


def test_corner_taps_take_the_mean_of_the_three_and_are_continuous():
    R = 8
    cube = torch.rand(6, R, R, 3, dtype=F64, generator=torch.Generator().manual_seed(3))
    for sx, sy, sz in itertools.product((-1.0, 1.0), repeat=3):
        corner = torch.tensor([sx, sy, sz], dtype=F64)
        # a fine grid of directions around the corner, crossing the corner region, its edges and the three faces
        s = torch.linspace(-0.2, 0.2, 81, dtype=F64)
        a, b = torch.meshgrid(s, s, indexing="ij")
        e1 = torch.tensor([1.0, -1.0, 0.0], dtype=F64) / 2 ** 0.5
        e2 = torch.tensor([1.0, 1.0, -2.0], dtype=F64) / 6 ** 0.5
        d = corner + a.unsqueeze(-1) * e1 + b.unsqueeze(-1) * e2
        v = SO.lookup(cube, d)
        step = float(s[1] - s[0])
        # Lipschitz across neighbouring grid points: a texel difference (<= 1) per texel of distance, R / 2 texels per unit
        lip = 2 * R * step
        assert float((v[1:] - v[:-1]).abs().max()) <= lip and float((v[:, 1:] - v[:, :-1]).abs().max()) <= lip
    # at the very corner the three faces' corner texels are averaged; the corner tap holds their mean
    d = torch.tensor([[1.0, 1.0, 1.0]], dtype=F64)
    face, gx, gy = SO.face_coords(d)
    x, y = SO.tex_xy(gx, gy, R)
    idx, w = SO.taps(face, x, y, R)
    assert int((idx < 0).sum()) == 1 and float(w[idx < 0]) == 0.25
    ie, we = SO.effective(idx, w)
    assert abs(float(we.sum()) - 1.0) < 1e-15
    flat = cube.reshape(-1, 3)
    assert torch.allclose(SO.lookup(cube, d)[0], flat[ie[0][idx[0] >= 0]].mean(0), rtol=0, atol=1e-15)


def _args(**over):
    a = dict(rgb=torch.rand(3, 6, 8), acc=torch.rand(1, 6, 8), cube_map=torch.rand(6, 4, 4, 3), K=torch.eye(3), w2c=torch.eye(4))
    a.update(over)
    return a


@pytest.mark.parametrize("over,match", [
    (dict(rgb=torch.rand(4, 6, 8)), r"rgb must be \[3, H, W\]"),
    (dict(acc=torch.rand(6, 8)), r"acc must be \[1, 6, 8\]"),
    (dict(cube_map=torch.rand(6, 4, 5, 3)), "square"),
    (dict(cube_map=torch.rand(5, 4, 4, 3)), r"\[6, R, R, 3\]"),
    (dict(K=torch.eye(4)), r"K must be \[3, 3\]"),
    (dict(rgb=torch.rand(3, 6, 8, dtype=F64)), "float32"),
])
def test_wrapper_rejects_bad_shapes_without_cuda(over, match):
    a = _args(**over)
    with pytest.raises(ValueError, match=match):
        sgb.sky_composite(a["rgb"], a["acc"], a["cube_map"], a["K"], a["w2c"])


def test_wrapper_rejects_cpu_tensors_and_bad_masks():
    a = _args()
    with pytest.raises(_capi.SgrError, match="no CPU fallback"):
        sgb.sky_composite(a["rgb"], a["acc"], a["cube_map"], a["K"], a["w2c"])
    with pytest.raises(ValueError, match="sky_mask"):
        sgb.sky_composite(a["rgb"], a["acc"], a["cube_map"], a["K"], a["w2c"], sky_mask=torch.ones(1, 6, 8))
    with pytest.raises(ValueError, match="sky_mask"):
        sgb.sky_composite(a["rgb"], a["acc"], a["cube_map"], a["K"], a["w2c"], sky_mask=torch.ones(1, 5, 8, dtype=torch.bool))


def test_c_entries_validate_before_touching_cuda():
    L = _capi.lib()
    p = C.c_void_p(16)
    err = lambda: L.sgr_last_error().decode()
    fwd = lambda H, W, R, mode, mask=p, jx=None, jy=None, rgb=p: L.sgr_sky_composite_forward(H, W, R, mode, C.c_float(1.0), rgb, p, mask, p, p, p,
                                                                                              jx, jy, p, None)
    bwd = lambda H, W, R, mode, mask=p: L.sgr_sky_composite_backward(H, W, R, mode, C.c_float(1.0), p, mask, p, p, p, None, None, p, p, p, None)
    for H, W, R in ((0, 4, 4), (4, 0, 4), (4, 4, 0), (-1, 4, 4), (4, 4, 16385)):
        assert fwd(H, W, R, 0) == -1 and "bad sizes" in err()
        assert bwd(H, W, R, 0) == -1 and "bad sizes" in err()
    for mode in (2, -1, 7):
        assert fwd(4, 4, 4, mode) == -1 and "unknown mask mode" in err()
        assert bwd(4, 4, 4, mode) == -1 and "unknown mask mode" in err()
    assert fwd(4, 4, 4, _capi.SKY_MASK_GIVEN, mask=None) == -1 and "needs sky_mask" in err()
    assert bwd(4, 4, 4, _capi.SKY_MASK_GIVEN, mask=None) == -1 and "needs sky_mask" in err()
    assert fwd(4, 4, 4, 0, rgb=None) == -1 and "NULL" in err()
    assert fwd(4, 4, 4, 0, jx=p) == -1 and "both jitters" in err()
