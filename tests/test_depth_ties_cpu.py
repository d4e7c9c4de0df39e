"""CPU tier of the depth-tie checks (tests/tie_case.py, tests/test_depth_ties_gpu.py): the builders place every tie they claim on
the post-margin scene, and the float64 reference is sensitive to the order of a tie: blending each group's rows reversed moves some
pixel and some grad2d row by more than raster64.bound, so a kernel that orders equal depths any other way than by ascending index
could not pass the GPU tier."""
import pytest
import torch

import tie_case as TC
from oracle import raster64 as R64


@pytest.fixture(scope="module", params=sorted(TC.BUILDERS))
def case(request):
    return TC.BUILDERS[request.param]()


def test_builders_place_their_ties(case):
    sc = case["scene"]
    pre = R64.preprocess64(sc)
    groups = TC.tie_groups(pre["rec"], pre["radii"])
    assert [m.tolist() for m in groups] == [m.tolist() for m in case["groups"]]
    assert len(groups) >= 1 and all(len(m) >= 2 for m in groups)
    # identity camera: the view depth is the fp32 z bit for bit
    vis = pre["radii"] > 0
    assert torch.equal(pre["rec"][vis, 7].float(), sc["means3D"][vis, 2])
    rc = TC.rects(pre)
    for m in groups:
        z = sc["means3D"][m, 2]
        assert bool((z == z[0]).all())
        # colour and opacity differ inside a group (except a clone and its parent)
        assert len(torch.unique(sc["opacities"][m, 0])) >= 2 or case["name"] == "clones"
        assert any(TC.common_tile(rc, m[[i, j]]) for i in range(len(m)) for j in range(i + 1, len(m)))
    assert R64.margins(pre["rec"], pre["radii"], pre["cam"]["W"], pre["cam"]["H"], pre=pre).numel() == 0


def test_group_sizes_and_edges():
    g = TC.groups_case()
    assert g["sizes"] == [2, 3, 5, 9, 17, 40]
    p = TC.partition_case()
    lo, hi = p["positions"]
    assert lo < TC.PARTITION < hi and p["E"] < 396 * TC.PARTITION
    b = TC.big_case()
    pre = R64.preprocess64(b["scene"])
    rc = TC.rects(pre)
    assert all(int((rc[i, 2] - rc[i, 0]) * (rc[i, 3] - rc[i, 1])) > TC.BIG_TILES for i in b["big"])
    c = TC.clone_case()
    sc = c["scene"]
    for k in ("means3D", "shs", "opacities", "scales", "rotations"):
        assert torch.equal(sc[k][c["parents"]], sc[k][c["clones"]]), k
    assert bool((c["clones"] > c["parents"]).all())


def test_fp64_reference_is_sensitive_to_tie_order(case):
    """blend64 with every tie group's rows reversed against blend64 in index order: some pixel and some grad2d row move by more
    than the per-element bound of the index-order blend."""
    sc = case["scene"]
    pre = R64.preprocess64(sc)
    W, H = pre["cam"]["W"], pre["cam"]["H"]
    up = dict(color=sc["grad_color"], depth=sc["grad_depth"], alpha=sc["grad_alpha"])
    bl = R64.blend64(pre["rec"], pre["radii"], W, H, pre["cam"]["bg"], upstream=up)
    perm = TC.reversed_ties(pre["rec"].shape[0], case["groups"])
    assert not torch.equal(perm, torch.arange(len(perm)))
    rv = R64.blend64(pre["rec"][perm], pre["radii"][perm], W, H, pre["cam"]["bg"], upstream=up)
    if case["name"] != "clones":  # (a clone and its parent are the same Gaussian: only the gradients tell them apart)
        moved = False
        for key in ("color", "depth", "alpha"):
            moved |= bool(((rv[key] - bl[key]).abs() > R64.bound(bl["kmass_" + key])).any())
        assert moved, "no pixel notices the reversed ties"
    g_rev = rv["grad2d"][perm]  # back to the original rows
    bnd = R64.bound(bl["kmass_grad2d"], bl["mass_grad2d"], bl["ntiles"])
    over = ((g_rev - bl["grad2d"]).abs() > bnd)[:, :11]
    rows = torch.nonzero(over.any(1)).reshape(-1)
    tied = torch.cat(case["groups"])
    assert bool(torch.isin(rows, tied).any())  # (a Gaussian in front of a group moves too: the value behind it changes)
    if case["name"] == "clones":  # every parent / clone pair swaps its gradients
        assert bool(torch.isin(case["parents"], rows).all())
