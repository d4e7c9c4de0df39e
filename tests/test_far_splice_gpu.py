"""The far pass of the saturation split buckets only the far instances [E_near, E) of the emitted sequence and splices each tile's
near list and far list into the final one (csrc/binning.cu launch_far_binning).  At the edges of that splice the lists must still
be the stable bucketing of the whole emitted sequence (test_binning_gpu.check_lists) and the images those of the unsplit frame:
  * an empty far slab (every tile saturates in the near one), and a far slab that is the whole sequence (E_near = 0);
  * tiles with far instances only, next to tiles with near ones only;
  * E_near at every offset modulo 8 (the far bucketing starts its partitions at E_near rounded down to whole 16-B key loads);
  * a bounded frame that overflows inside the far slab;
  * a far slab of more partitions than one round of the bucketing."""
import pytest
import torch

from street_gaussians_b200 import _capi, synthetic
from street_gaussians_b200._capi import STATUS_EMITTED, STATUS_FAR_END, STATUS_INSTANCES, STATUS_NEAR_END, STATUS_OVERFLOW
from test_binning_gpu import bin_lists, capacity_of, check_lists, single_tile_scene
from test_saturation_split_gpu import assert_same, render, scene_of, splats, wall_scene

pytestmark = pytest.mark.gpu
ALL, AUTO = _capi.NEAR_BUDGET_ALL, _capi.NEAR_BUDGET_AUTO


def split_lists(scene, budget, capacity=None):
    with _capi.near_budget(budget):
        d = bin_lists(scene, capacity=capacity_of(capacity) if capacity else None)
    check_lists(d)
    return d


def status(scene, budget, capacity=None):
    return render(scene, budget, capacity=capacity, backward=False)["status"]


def test_empty_far_slab():
    sc, walls = wall_scene(640, 480)
    R_wall = int(status(walls, ALL)[STATUS_INSTANCES])
    st = status(sc, R_wall)
    assert int(st[STATUS_NEAR_END]) == R_wall and int(st[STATUS_EMITTED]) == R_wall and int(st[STATUS_FAR_END]) == 0
    d = split_lists(sc, R_wall)
    assert d["E"] == R_wall
    assert_same(render(sc, ALL), render(sc, R_wall), what="empty far slab")


def test_whole_sequence_far():
    sc, _ = wall_scene(640, 480, seed=1, layers=2)
    st = status(sc, 0)
    assert int(st[STATUS_NEAR_END]) == 0 and int(st[STATUS_FAR_END]) == int(st[STATUS_EMITTED]) == int(st[STATUS_INSTANCES])
    split_lists(sc, 0)
    assert_same(render(sc, ALL), render(sc, 0), what="B = 0")


def test_far_only_tiles():
    """Opaque walls over the left half only, random splats everywhere behind them: with the walls as the near slab, the right half's
    tiles have far instances only and the left half's near ones only."""
    W, H = 640, 480
    cam = synthetic.make_camera(W, H, sh_degree=0)
    gy, gx = torch.meshgrid(torch.arange(0, H, 4), torch.arange(0, W // 2 - 24, 4), indexing="ij")
    walls = [splats(cam, gx.flatten(), gy.flatten(), torch.full((gx.numel(),), 2.0 + 0.1 * k), 4.0, 0.99, k) for k in range(3)]
    gen = torch.Generator().manual_seed(9)
    n = 8000
    bg = splats(cam, torch.rand(n, generator=gen) * W, torch.rand(n, generator=gen) * H, 5 + 40 * torch.rand(n, generator=gen),
                1 + 6 * torch.rand(n, generator=gen), 0.3 + 0.6 * torch.rand(n, generator=gen), 50)
    sc, wall_sc = scene_of(cam, *walls, bg), scene_of(cam, *walls)
    R_wall = int(status(wall_sc, ALL)[STATUS_INSTANCES])
    full = render(sc, ALL)
    for b in (R_wall, R_wall + 1, AUTO):
        d = split_lists(sc, b)
        assert_same(full, render(sc, b), what=f"B={b}")
    st = status(sc, R_wall)
    assert int(st[STATUS_NEAR_END]) == R_wall and int(st[STATUS_FAR_END]) > 0
    d = split_lists(sc, R_wall)
    near_tiles = torch.bincount(d["keys"][:R_wall], minlength=d["ntile"]) > 0
    far_tiles = torch.bincount(d["keys"][R_wall:], minlength=d["ntile"]) > 0
    assert bool((far_tiles & ~near_tiles).any()) and bool((near_tiles & ~far_tiles).any())


def test_near_end_at_every_alignment():
    """Single-instance Gaussians, so the budget sets E_near exactly: E_near = 8 k + r for every r."""
    gen = torch.Generator().manual_seed(4)
    W, H = 1920, 1280
    ntile = (W // 16) * (H // 16)
    n = 30000
    sc = single_tile_scene(torch.randint(0, ntile, (n,), generator=gen), torch.rand(n, generator=gen) * 40 + 5, W, H)
    full = render(sc, ALL)
    for b in range(4096, 4096 + 9):
        st = status(sc, b)
        assert int(st[STATUS_NEAR_END]) == b and int(st[STATUS_EMITTED]) == n
        split_lists(sc, b)
        assert_same(full, render(sc, b), what=f"B={b}")


def test_overflow_inside_the_far_slab():
    """A capacity between E_near and the emitted sequence: the frame keeps the Gaussians whose whole instance counts fit, as the
    one-pass binning with that capacity does."""
    sc = synthetic.make_config("B", seed=2)
    st = status(sc, AUTO)
    E_near, E = int(st[STATUS_NEAR_END]), int(st[STATUS_EMITTED])
    assert E > E_near + 16
    far_emitted = False
    for cap in (E_near + 1, (E_near + E) // 2, E - 1):
        split = render(sc, AUTO, capacity=cap)
        s = split["status"]
        assert int(s[STATUS_OVERFLOW]) & 1 and int(s[STATUS_EMITTED]) <= cap
        assert int(s[STATUS_FAR_END]) == int(s[STATUS_EMITTED]) - int(s[STATUS_NEAR_END])
        far_emitted |= int(s[STATUS_FAR_END]) > 0
        split_lists(sc, AUTO, capacity=cap)
        assert_same(render(sc, ALL, capacity=cap), split, what=f"cap={cap}")
    assert far_emitted


def test_many_far_partitions():
    """Config C at a small budget: the far slab spans several partitions of the bucketing."""
    sc = synthetic.make_config("C", seed=0)
    R_ = int(status(sc, ALL)[STATUS_INSTANCES])
    b = R_ // 64
    st = status(sc, b)
    assert int(st[STATUS_FAR_END]) > 4 * 2048
    split_lists(sc, b)
