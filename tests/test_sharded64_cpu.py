"""CPU tier of the Gaussian-sharded fp64 checks (tests/sharded64_case.py, tests/test_sharded64_gpu.py): the builders place every edge
they claim on the post-margin scene, the expected per-rank counts agree with an independent per-Gaussian loop, and the float64
reference is sensitive enough that a wrong tie order or a missing rank partial could not pass the GPU tier's bound."""
import pytest
import torch

import sharded64_case as SC
from oracle import raster64 as R64

ALL_CLASSES = {"0", "1-255", "256", "257", "512", ">=768", "256w"}


@pytest.fixture(scope="module")
def cases():
    return {n: SC.build(n, seed=0, D=0) for n in SC.CASES}


def test_builders_place_every_edge(cases):
    seen = set()
    for name, c in cases.items():
        sc, world, chunk, P_r = c["scene"], c["world"], c["chunk"], c["P_r"]
        _, removed, _ = R64.margin_scene(sc)
        assert removed == 0, (name, "not margin-clean")
        assert sc["means3D"].shape[0] == sum(P_r) and all(0 <= p <= chunk for p in P_r)
        pre = R64.preprocess64(sc)
        mask = SC.masks(pre["rec"][:, 0], pre["rec"][:, 1], pre["radii"], c["W"], c["H"], world)
        assert torch.equal(mask, c["mask"])
        cl = SC.total_classes(SC.block_totals(mask, P_r, chunk), world)
        assert cl >= c["claims"], (name, cl, c["claims"])
        seen |= cl
        assert max(SC.block_totals(mask, P_r, chunk).values()) <= 256 * world
        for a, b in c["ties"]:  # bit-identical view depth, different owners, overlapping
            assert pre["rec"][a, 7].item() == pre["rec"][b, 7].item()
            assert int(c["owner_of"][a]) != int(c["owner_of"][b])
            assert abs(pre["rec"][a, 0].item() - pre["rec"][b, 0].item()) < 2 and int(pre["radii"][a]) > 0 and int(pre["radii"][b]) > 0
        n_sel, _ = SC.expected_counts(pre["rec"][:, 0], pre["rec"][:, 1], pre["radii"], c["W"], c["H"], world)
        assert sum(1 for n in n_sel if n == 0) >= SC.CASES[name].get("empty_bands", 0)
    assert seen == ALL_CLASSES, seen
    # ownership layouts: tail padding, padding in the middle, an empty rank; chunk not a multiple of 256 and below 256
    layouts = {SC.CASES[n]["layout"] for n in cases}
    assert layouts == {"tail", "middle", "empty"}
    assert any(c["chunk"] % 256 for c in cases.values()) and any(c["chunk"] < 256 for c in cases.values())
    assert cases["w3_middle"]["P_r"][0] < cases["w3_middle"]["chunk"] and 0 in cases["w5_empty_rank"]["P_r"]
    assert sum(len(c["ties"]) for c in cases.values()) >= 4
    assert {c["world"] for c in cases.values()} == {2, 3, 5, 8}


def test_expected_counts_against_a_per_gaussian_loop(cases):
    for name, c in cases.items():
        pre = R64.preprocess64(c["scene"])
        px, py, radii = pre["rec"][:, 0], pre["rec"][:, 1], pre["radii"]
        W, H, world = c["W"], c["H"], c["world"]
        gx, gy = (W + 15) // 16, (H + 15) // 16
        n_sel, pairs = [0] * world, [0] * world
        for i in range(len(radii)):
            r = int(radii[i])
            if r <= 0:
                continue
            x, y = float(torch.tensor(float(px[i]), dtype=torch.float32)), float(torch.tensor(float(py[i]), dtype=torch.float32))
            f = lambda v, g: min(max(int(float(torch.tensor(v, dtype=torch.float32))), 0), g)  # fp32 value, truncated, clamped
            x0, x1 = f((x - r) / 16, gx), f((x + r + 15) / 16, gx)
            y0, y1 = f((y - r) / 16, gy), f((y + r + 15) / 16, gy)
            if x1 <= x0 or y1 <= y0:
                continue
            for k in range(world):
                rows = sum(1 for yy in range(y0, y1) if yy % world == k)
                n_sel[k] += rows > 0
                pairs[k] += rows * (x1 - x0)
        assert (n_sel, pairs) == tuple(map(list, SC.expected_counts(px, py, radii, W, H, world))), name


def test_fp64_reference_is_sensitive(cases):
    """On the smallest case: swapping one tie pair moves the image by far more than its bound, and a Gaussian's grad2d row with one
    rank's partial dropped (the band partials from blend64 with the upstream zeroed outside each band) leaves the sharded bound."""
    c = cases["w2_tail"]
    sc, world = c["scene"], c["world"]
    pre = R64.preprocess64(sc)
    cam = pre["cam"]
    W, H = cam["W"], cam["H"]
    up = dict(color=sc["grad_color"], depth=sc["grad_depth"], alpha=sc["grad_alpha"])
    bl = R64.blend64(pre["rec"], pre["radii"], W, H, cam["bg"], upstream=up)
    a, b = c["ties"][0]
    perm = torch.arange(pre["rec"].shape[0])
    perm[a], perm[b] = b, a
    sw = R64.blend64(pre["rec"][perm], pre["radii"][perm], W, H, cam["bg"])
    assert float(((sw["color"] - bl["color"]).abs() / (R64.bound(bl["kmass_color"]) + 1e-300)).max()) > 1e3
    parts = [R64.blend64(pre["rec"], pre["radii"], W, H, cam["bg"], upstream=SC.band_upstream(sc, r, world), alpha_img=bl["alpha"])["grad2d"]
             for r in range(world)]
    total = sum(parts)
    assert float((total - bl["grad2d"]).abs().max()) <= 1e-12 * float(bl["mass_grad2d"].max())  # the partials add up
    bnd = SC.sharded_bound(bl, world)
    two = torch.nonzero((c["mask"] == 3) & (pre["radii"] > 0)).reshape(-1)
    assert len(two) > 0
    dropped = 0
    for g in two.tolist():
        for r in range(world):
            e = (total[g] - parts[r][g] - bl["grad2d"][g]).abs()[:11]
            dropped += bool((e > bnd[g, :11]).any())
    assert dropped >= 0.9 * world * len(two), (dropped, len(two))
