"""The tile bucketing at the edges of its per-frame partition size, and the far count of the saturation split against the row walk.

The bucketing cuts the E emitted instances into partitions of bucket_part(E) instances (csrc/binning.cu): about E / TARGET_PARTS in
whole rounds of 2048, at least one round and at most 32768.  part_size() restates that rule, so each case asserts which edge it
hits; the lists are checked with test_binning_gpu's restatement (vals_out = the stable sort of the emitted sequence by tile, ranges
from bincount / cumsum).

The far count (far_count_kernel) skips the row walk of a far Gaussian whose tile rectangle holds no tile the near blend left
unsaturated.  Its counts (geom state `iota`, per depth slot) are checked against the walk: a tile is unsaturated exactly when its
split list is its whole one-pass list, and a far Gaussian's count is the number of its one-pass instances in such tiles."""
import pytest
import torch

import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi
from street_gaussians_b200 import rasterizer as R
from street_gaussians_b200 import synthetic
from street_gaussians_b200._capi import STATUS_EMITTED, STATUS_INSTANCES, STATUS_NEAR_END, STATUS_SPLIT_K
import util
from test_binning_gpu import bin_lists, capacity_of, check_lists, single_tile_scene
from test_saturation_split_gpu import render, scene_of, splats

pytestmark = pytest.mark.gpu
DEV = "cuda"
ALL, AUTO = _capi.NEAR_BUDGET_ALL, _capi.NEAR_BUDGET_AUTO
TARGET_PARTS = 396   # csrc/binning.cu kBucketTargetParts
ROUND = 2048         # kPassRound
MAX_PART = 32768     # kBucketMaxPart


def part_size(E):
    per = -(-E // TARGET_PARTS)
    return min(max(-(-per // ROUND) * ROUND, ROUND), MAX_PART)


def n_parts(E):
    return -(-E // part_size(E))


def lists(scene, budget=ALL, **kw):
    with _capi.near_budget(budget):
        return bin_lists(scene, **kw)


def spread_scene(n, width=1920, height=1280, rows=None, seed=11):
    """n single-instance Gaussians (one tile each) on random tiles of a 1920x1280 frame, or of the tile rows `rows` only."""
    gen = torch.Generator().manual_seed(seed)
    gx, gy = (width + 15) // 16, (height + 15) // 16
    rows = torch.arange(gy) if rows is None else torch.as_tensor(rows)
    ty = rows[torch.randint(0, rows.numel(), (n,), generator=gen)]
    tiles = ty * gx + torch.randint(0, gx, (n,), generator=gen)
    return single_tile_scene(tiles, torch.rand(n, generator=gen) * 40 + 5, width, height)


@pytest.fixture(scope="module")
def big_spread():
    return spread_scene(TARGET_PARTS * 2 * ROUND + 1000)


# (E, the partition size it must get)
EDGES = [(1, ROUND), (ROUND - 1, ROUND), (ROUND, ROUND), (ROUND + 1, ROUND),             # around one multiple of one round
         (2 * ROUND - 1, ROUND), (2 * ROUND, ROUND), (2 * ROUND + 1, ROUND),           # ... and two
         (TARGET_PARTS * ROUND - 1, ROUND), (TARGET_PARTS * ROUND, ROUND),             # the last E with one round per partition
         (TARGET_PARTS * ROUND + 1, 2 * ROUND),
         ((TARGET_PARTS - 1) * 2 * ROUND - 1, 2 * ROUND), ((TARGET_PARTS - 1) * 2 * ROUND, 2 * ROUND),  # around a multiple of two rounds
         ((TARGET_PARTS - 1) * 2 * ROUND + 1, 2 * ROUND), (TARGET_PARTS * 2 * ROUND, 2 * ROUND)]


@pytest.mark.parametrize("E,part", EDGES)
def test_partition_edges(big_spread, E, part):
    assert part_size(E) == part and n_parts(E) <= TARGET_PARTS
    d = lists(big_spread, capacity=capacity_of(E))
    check_lists(d, expect_E=E)


def test_no_instances():
    sc = single_tile_scene(torch.arange(50), -torch.ones(50), 256, 256)  # all behind the camera
    for budget in (ALL, AUTO):
        d = lists(sc, budget, capacity=capacity_of(1000))
        check_lists(d, expect_E=0)
        assert not d["ranges"].any()
    assert n_parts(0) == 0


def test_size_capped_at_32768():
    """Up to E = TARGET_PARTS * 32768 the partitions number at most the target; one instance more and the size stays at its cap, so
    the partitions outnumber the target and the grid follows the capacity."""
    E = TARGET_PARTS * MAX_PART
    assert part_size(E - 1) == part_size(E) == part_size(E + 1) == MAX_PART
    assert n_parts(E) == TARGET_PARTS and n_parts(E + 1) == TARGET_PARTS + 1
    sc = spread_scene(E + 1000, seed=12)
    for e in (E - 1, E, E + 1):
        check_lists(lists(sc, capacity=capacity_of(e)), expect_E=e)


@pytest.mark.parametrize("budget", [ALL, AUTO])
def test_bounded_overflow(budget):
    sc = synthetic.make_config("B", seed=1)
    R_ = check_lists(lists(sc))
    cap = R_ // 2 + 3
    d = lists(sc, budget, capacity=capacity_of(cap))
    E = check_lists(d)
    assert 0 < E <= cap < R_


@pytest.mark.parametrize("B", [ROUND - 1, ROUND + 1, 2 * ROUND, TARGET_PARTS * ROUND + 1])
def test_split_frame(B):
    """Single-instance Gaussians never saturate a tile, so the near bucketing runs over exactly [0, B) and the final one over every
    instance.  The final lists are checked directly; the near lists are what the near blend reads, so the images, n_contrib and
    tile_max_contrib equal the one-pass frame's only if they were right."""
    sc = spread_scene(TARGET_PARTS * ROUND + 6000, width=1280, height=720, seed=4)
    n = sc["means3D"].shape[0]
    d = lists(sc, B)
    check_lists(d, expect_E=n)
    full, got = render(sc, ALL, backward=False), render(sc, B, backward=False)
    assert int(got["status"][STATUS_NEAR_END]) == B and int(got["status"][STATUS_EMITTED]) == n
    for k in ("color", "depth", "alpha", "radii", "n_contrib", "tile_max"):
        assert torch.equal(full[k], got[k]), k
    assert part_size(n) == 2 * ROUND and part_size(B) == (2 * ROUND if B > TARGET_PARTS * ROUND else ROUND)


@pytest.mark.parametrize("E", [ROUND - 1, 3 * ROUND + 1])
def test_cyclic_band(E):
    """A rank of eight on a cyclic band (rows 3, 11, 19, ...): every Gaussian sits on an owned row, so the band emits all of them."""
    band = R.TileRowBand(3, 80, 8)
    sc = spread_scene(E, rows=list(range(3, 80, 8)), seed=6)
    d = lists(sc, band=band)
    check_lists(d, expect_E=E)
    check_lists(lists(sc, band=band, capacity=capacity_of(E + 100)), expect_E=E)
    rows = torch.arange(80, device=DEV).repeat_interleave(120)
    assert not d["ranges"][(rows - 3) % 8 != 0].any()


# ---- far count ----

def split_state(scene, budget):
    """Forward at `budget`: status words, depth order (perm), counts per depth slot (iota), emitted sequence and lists."""
    cam = scene["cam"]
    st = util.settings_from(sgb, cam, DEV)
    dv = lambda k: scene[k].to(DEV) if scene.get(k) is not None else None
    P = scene["means3D"].shape[0]
    with torch.no_grad(), _capi.near_budget(budget):
        out = R._forward_impl(dv("means3D"), dv("shs"), None, None, dv("opacities"), dv("scales"), dv("rotations"), None, st, None, None)
    fst = out[5]
    torch.cuda.synchronize()
    v = R.state_views(st, fst, P)
    status = v["status"].long().cpu()
    E = int(status[STATUS_EMITTED])
    return dict(status=status, iota=v["iota"].long(), perm=v["perm"].long(), ntile=v["ranges"].shape[0], E=E,
                keys=v["keys_in"][:E].long() & 0xFFFF, vals=v["vals_in"][:E].long(), out=v["vals_out"][:E].long(), ranges=v["ranges"].long())


def check_far_counts(scene, budget):
    """Every far Gaussian's count equals the row walk's over the unsaturated tiles; returns (unsaturated tile mask, expected counts)."""
    full, split = split_state(scene, ALL), split_state(scene, budget)
    check_lists(full)
    check_lists(split)
    P, ntile = scene["means3D"].shape[0], full["ntile"]
    K = int(split["status"][STATUS_SPLIT_K])
    slot = torch.empty(P, dtype=torch.long, device=DEV)
    slot[split["perm"]] = torch.arange(P, device=DEV)
    far_pair = slot[full["vals"]] >= K
    len_a = full["ranges"][:, 1] - full["ranges"][:, 0]
    len_s = split["ranges"][:, 1] - split["ranges"][:, 0]
    near_len = torch.bincount(full["keys"][~far_pair], minlength=ntile)
    # each split list is the one-pass list (unsaturated tile) or its near part (saturated tile)
    assert bool(((len_s == len_a) | (len_s == near_len)).all())
    tile = torch.repeat_interleave(torch.arange(ntile, device=DEV), len_s)
    j = torch.arange(split["E"], device=DEV) - split["ranges"][tile, 0]
    assert torch.equal(split["out"], full["out"][full["ranges"][tile, 0] + j])
    unsat = (len_s == len_a) & (len_a > near_len)
    walk = torch.bincount(full["vals"][far_pair & unsat[full["keys"]]], minlength=P)
    assert torch.equal(split["iota"][K:], walk[split["perm"][K:]])
    return unsat, walk


def holed_wall_scene(W, H, holes, probes):
    """Three opaque walls of small splats (2 px apart, sigma 2 px) over every tile but `holes`, in front of random background
    splats of all sizes and of `probes` (px, py, sigma) far splats."""
    cam = synthetic.make_camera(W, H, sh_degree=0)
    gy, gx = torch.meshgrid(torch.arange(1, H, 2), torch.arange(1, W, 2), indexing="ij")
    gx, gy = gx.flatten(), gy.flatten()
    keep = torch.ones_like(gx, dtype=torch.bool)
    for tx, ty in holes:
        keep &= ~((gx // 16 == tx) & (gy // 16 == ty))
    gx, gy = gx[keep], gy[keep]
    walls = [splats(cam, gx, gy, torch.full((gx.numel(),), 2.0 + 0.1 * k), 2.0, 0.99, k) for k in range(3)]
    gen = torch.Generator().manual_seed(100)
    n = 20000
    bg = splats(cam, torch.rand(n, generator=gen) * W, torch.rand(n, generator=gen) * H, 5 + 40 * torch.rand(n, generator=gen),
                1 + 30 * torch.rand(n, generator=gen) ** 3, 0.3 + 0.6 * torch.rand(n, generator=gen), 200)
    px, py, sg = (torch.tensor(c, dtype=torch.float64) for c in zip(*probes))
    pr = splats(cam, px, py, torch.full((px.numel(),), 4.0), sg, 0.5, 300)
    return scene_of(cam, *walls, bg, pr), sum(w["means3D"].shape[0] for w in walls), bg["means3D"].shape[0]


def test_far_count_holes_at_corners_and_edge():
    W, H = 640, 480
    gx, gy = W // 16, H // 16
    holes = [(0, 0), (gx - 1, 0), (0, gy - 1), (gx - 1, gy - 1), (gx // 2, 0)]
    hx = 16 * (gx // 2)  # left edge of the mid-edge hole
    probes = [(hx - 2.5, 6.5, 1.5),             # rectangle reaches the hole in its last column only
              (hx + 17.5, 6.5, 1.5),            # ... in its first column only
              (6.5, 16 * (gy - 1) - 2.5, 1.5),  # ... in its last row only (bottom-left corner)
              (W - 8.5, 17.5, 1.5),             # ... in its first row only (top-right corner)
              (W - 40.5, H - 40.5, 30.0),       # a large rectangle (warp-cooperative walk) over the bottom-right hole
              (W / 2, H / 2, 60.0)]             # a large rectangle around the middle, far from every hole
    sc, n_wall_gauss, n_bg = holed_wall_scene(W, H, holes, probes)
    B = int(render(scene_of(sc["cam"], *[{k: sc[k][:n_wall_gauss] for k in ("means3D", "scales", "rotations", "opacities", "shs")}]),
                   ALL, backward=False)["status"][STATUS_INSTANCES])
    unsat, walk = check_far_counts(sc, B)
    for tx, ty in holes:
        assert bool(unsat[ty * gx + tx]), (tx, ty)
    assert int(unsat.sum()) < gx * gy // 4  # the walls saturate almost every other tile
    probe_ids = torch.arange(len(probes), device=DEV) + n_wall_gauss + n_bg
    assert (walk[probe_ids[:5]] > 0).all(), walk[probe_ids]  # the edge probes do reach their hole
    assert int(walk[probe_ids[5]]) == 0


def test_far_count_nothing_saturates():
    cam = synthetic.make_camera(640, 480, sh_degree=0)
    gen = torch.Generator().manual_seed(5)
    n = 3000
    sc = scene_of(cam, splats(cam, torch.rand(n, generator=gen) * 640, torch.rand(n, generator=gen) * 480, 3 + 30 * torch.rand(n, generator=gen),
                              2 + 6 * torch.rand(n, generator=gen), 0.05))
    unsat, walk = check_far_counts(sc, AUTO)
    assert int(walk.sum()) > 0
