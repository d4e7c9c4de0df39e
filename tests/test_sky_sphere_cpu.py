"""CPU: the whole-sphere views of the sky cube map (tests/sky_sphere_case.py) and tests/sky_oracle.py's bounds on them.

  * Each family reaches what it claims, on all pixels and on the pixels each mask mode samples: the sphere family every face, side and
    corner tap (up to R = 16; the sides at R = 37), every R = 1 sample with a corner tap; the exact family every corner tap at every R;
    the rig exactly +x, +-y and the +x / +-y edges.
  * The exact family is exact in fp32: the kernel's adjugate K^-1, Rm^T K^-1 and the rays restated in float32 equal float64, the centre
    pixel is a three-way tie the x face takes, its row and column are two-way ties, and where the largest component is +-1 the texel
    coordinates are exact too.
  * sky64's bounds hold the fp32 torch restatement (sky_oracle.composite in float32) at these edges: seams hit exactly, a corner tap on
    every R = 1 sample, exact three-way ties; and its largest error / bound is above 1e-3, so the bounds are not empty."""
import numpy as np
import pytest
import torch

import sky_oracle as SO
import sky_sphere_case as SC

F64 = torch.float64


@pytest.mark.parametrize("family,R", SC.family_cases(), ids=lambda v: str(v))
def test_family_covers_what_it_claims(family, R):
    vs = SC.views(family, R)
    rays = [SC.rays64(v) for v in vs]
    SC.assert_coverage(family, R, SC.union_coverage([SC.coverage(d, R) for d in rays]))
    if family == "rig":  # its frames (2.4 M pixels each) are checked on their sampled pixels in tests/test_sky_sphere_gpu.py
        return
    for mode in SC.MODES:
        frs = SC.frames(family, R, mode)
        got = SC.union_coverage([SC.coverage(d, R, SC.sampled(fr)) for d, fr in zip(rays, frs)])
        SC.assert_coverage(family, R, got)
        assert all(0 < int(SC.sampled(fr).sum()) < fr["acc"].numel() for fr in frs)
    if R == 1:  # every sample's taps leave the face across a column and a row: one of them is past a corner
        for d in rays:
            face, gx, gy = SO.face_coords(d)
            idx, _ = SO.taps(face, *SO.tex_xy(gx, gy, 1), 1)
            assert bool((idx < 0).any(-1).all())


@pytest.mark.parametrize("R", SC.EXACT_R)
def test_exact_family_is_exact_in_fp32(R):
    I0, J0 = SC.EXACT_IJ
    corners = set()
    for v in SC.exact_views(R):
        e = SC.exact_rays_fp32(v)
        for k in ("kinv", "m", "d"):
            assert np.array_equal(e[k + "32"].astype(np.float64), e[k + "64"]), (v["name"], k)
        d = e["d64"]
        # the centre pixel looks along a cube corner: a three-way tie, which the x face takes
        assert np.array_equal(np.abs(d[J0, I0]), np.ones(3)), v["name"]
        face, _, _ = SO.face_coords(torch.from_numpy(d[J0, I0]))
        assert int(face) in (0, 1)
        # its row to the left and its column above lie on two cube edges (two components tied at |1|, the third below) until the
        # camera's third component reaches -1, 2 f pixels away
        n = int(SC.exact_focal(R)) * 2
        for line in (d[J0, max(I0 - n + 1, 0):I0], d[max(J0 - n + 1, 0):J0, I0]):
            a = np.sort(np.abs(line), -1)
            assert np.array_equal(a[:, 1:], np.ones_like(a[:, 1:])) and bool((a[:, 0] < 1).all())
        # where the largest component is +-1 (the seams and the corner), the face and texel coordinates are exact too
        sel = np.abs(d).max(-1) == 1
        _, xy = SC.exact_texel_coords_fp32(d[sel], R)
        for a, b in zip(xy["32"], xy["64"]):
            assert np.array_equal(a.astype(np.float64), b), v["name"]
        # the centre and its neighbours (I0 - 1, J0), (I0 - 1, J0 - 1) each have a corner tap of nonzero weight (f > R)
        three = torch.from_numpy(np.stack([d[J0, I0], d[J0, I0 - 1], d[J0 - 1, I0 - 1]]))
        face3, gx, gy = SO.face_coords(three)
        idx, w = SO.taps(face3, *SO.tex_xy(gx, gy, R), R)
        assert bool(((idx < 0) & (w > 0)).any(-1).all()), v["name"]
        corners |= SC.coverage(three, R)[2]
    # over the 24 rotations those three pixels alone put a corner tap on every face at every corner
    assert corners == SC.ALL_CORNERS, sorted(SC.ALL_CORNERS - corners)


def _fp32_within(fr, worst):
    rgb, acc, cube = (fr[k].clone().requires_grad_(True) for k in ("rgb", "acc", "cube"))
    out = SO.composite(rgb, acc, cube, fr["K"], fr["w2c"], fr["mask"], None, None, fr["fill"])
    dacc, dcube = torch.autograd.grad(out, [acc, cube], fr["up"])
    r = SO.sky64(fr["rgb"], fr["acc"], fr["cube"], fr["K"], fr["w2c"], fr["up"], fr["mask"], None, None, fr["fill"])
    for k, got in (("out", out.detach()), ("dacc", dacc), ("dcube", dcube)):
        err = (got.to(F64) - r[k]).abs()
        assert bool((err <= r["b_" + k]).all()), (k, float((err / r["b_" + k]).max()))
        worst[k] = max(worst[k], float((err / r["b_" + k]).max()))


# the seams and ties: the sphere at R = 1 (a corner tap on every sample), the exact family at small R (corners, edges and ties on
# exact rays) and at R = 1000 on a third of the rotations (the corner inside a clipped 8-texel block)
BOUND_CASES = [("sphere", 1, None), ("sphere", 3, None), ("exact", 1, None), ("exact", 2, None), ("exact", 3, None), ("exact", 1000, 3)]


def test_fp32_restatement_inside_sky64_bounds():
    """Every element inside its bound in every case; the largest error / bound over the cases above 1e-3 for each output."""
    worst = dict(out=0.0, dacc=0.0, dcube=0.0)
    for family, R, every in BOUND_CASES:
        case = dict(out=0.0, dacc=0.0, dcube=0.0)
        for mode in SC.MODES:
            for fr in SC.frames(family, R, mode)[::every or 1]:
                _fp32_within(fr, case)
        print(family, R, {k: round(v, 4) for k, v in case.items()})
        worst = {k: max(v, case[k]) for k, v in worst.items()}
    assert all(v > 1e-3 for v in worst.values()), worst
