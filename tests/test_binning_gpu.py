"""The per-tile lists against a torch restatement of the bucketing, from the library's own emitted sequence: vals_out[:E] must be
vals_in[:E] stably sorted by keys_in[:E], and ranges[t] = (start, start + count) from bincount / cumsum, (0, 0) for a tile without
instances.  E = status word 3 (the instances actually emitted; R in exact mode).  Covers the tile-bucketing path (frames of at most
16384 tiles) at multiples of its largest partition (32768 instances) and the tile radix sort of larger frames.  tools/ab_binning.py
compares the lists, images and gradients of two builds of the library frame by frame, layered renders included."""
import pytest
import torch

import util
import street_gaussians_b200 as sgb
from street_gaussians_b200 import rasterizer as R
from street_gaussians_b200 import synthetic
from street_gaussians_b200._capi import STATUS_EMITTED

pytestmark = pytest.mark.gpu
DEV = "cuda"
K = 32768           # largest bucketing partition (csrc/binning.cu kBucketMaxPart; a frame's partitions hold bucket_part(E) instances)
MAX_TILES = 16384   # largest frame that buckets (csrc/binning.cu kBucketMaxTiles)


def bin_lists(scene, band=None, capacity=None):
    cam = scene["cam"]
    st = util.settings_from(sgb, cam, DEV)
    dv = lambda k: scene[k].to(DEV) if scene.get(k) is not None else None
    P = scene["means3D"].shape[0]
    with torch.no_grad():
        out = R._forward_impl(dv("means3D"), dv("shs"), dv("colors_precomp"), dv("semantics"), dv("opacities"), dv("scales"),
                              dv("rotations"), dv("cov3D_precomp"), st, band, capacity)
    fst = out[5]
    torch.cuda.synchronize()
    v = R.state_views(st, fst, P)
    E = int(v["status"][STATUS_EMITTED])
    ranges, ntile = v["ranges"].long(), v["ranges"].shape[0]
    if fst.num_instances == 0:
        empty = torch.zeros(0, dtype=torch.long, device=DEV)
        return dict(E=E, ntile=ntile, keys=empty, vals=empty, out=empty, ranges=ranges)
    keys = v["keys_in"][:E].long() & (0xFFFF if v["keys_in"].dtype == torch.int16 else 0xFFFFFFFF)
    return dict(E=E, ntile=ntile, keys=keys, vals=v["vals_in"][:E].long(), out=v["vals_out"][:E].long(), ranges=ranges)


def check_lists(d, expect_E=None):
    E, ntile = d["E"], d["ntile"]
    if expect_E is not None:
        assert E == expect_E, (E, expect_E)
    keys, vals = d["keys"], d["vals"]
    assert int(keys.max()) < ntile if E else True
    order = torch.sort(keys, stable=True).indices
    assert torch.equal(d["out"], vals[order]), "vals_out[:E] differs from the stable sort of the emitted sequence"
    cnt = torch.bincount(keys, minlength=ntile)
    start = torch.cumsum(cnt, 0) - cnt
    exp = torch.stack([torch.where(cnt > 0, start, 0), torch.where(cnt > 0, start + cnt, 0)], 1)
    assert torch.equal(d["ranges"], exp), "ranges differ from bincount / cumsum"
    return E


def capacity_of(n):
    return sgb.InstanceCapacity(initial=n)


def single_tile_scene(tiles, z, width, height):
    """One Gaussian per entry, projected onto the centre of tile `tiles[i]` at depth z[i] with a footprint inside that tile
    (radius 2 px): every Gaussian emits exactly one instance."""
    cam = synthetic.make_camera(width, height, sh_degree=0)
    gx = (width + 15) // 16
    tx, ty = (tiles % gx).double(), (tiles // gx).double()
    px, py = tx * 16 + 8, ty * 16 + 8
    z = z.double()
    x = ((2 * px + 1) / width - 1) * z * cam["tanfovx"]
    y = ((2 * py + 1) / height - 1) * z * cam["tanfovy"]
    n = tiles.numel()
    gen = torch.Generator().manual_seed(3)
    npx = width * height
    return dict(cam=cam, means3D=torch.stack([x, y, z], 1).float().contiguous(), scales=torch.full((n, 3), 1e-4),
                rotations=torch.tensor([[1.0, 0, 0, 0]]).repeat(n, 1), opacities=torch.full((n, 1), 0.5),
                shs=torch.rand(n, 1, 3, generator=gen), grad_color=torch.randn(3, height, width, generator=gen) / npx,
                grad_depth=torch.randn(1, height, width, generator=gen) / npx, grad_alpha=torch.randn(1, height, width, generator=gen) / npx)


@pytest.fixture(scope="module")
def edge_scene():
    """3K + 500 single-instance Gaussians on a 1920x1280 frame (9600 tiles); the K + 100 nearest, and only they, sit on tile 17,
    so the first partition holds one tile only."""
    gen = torch.Generator().manual_seed(11)
    n_hot, n = K + 100, 3 * K + 500
    W, H = 1920, 1280
    ntile = (W // 16) * (H // 16)
    tiles = torch.randint(0, ntile - 1, (n,), generator=gen)
    tiles[tiles >= 17] += 1
    tiles[:n_hot] = 17
    z = torch.rand(n, generator=gen) * 40 + 5
    z[:n_hot] = 2 + torch.rand(n_hot, generator=gen)
    return single_tile_scene(tiles, z, W, H)


def test_single_tile_scene_emits_one_instance_each(edge_scene):
    d = bin_lists(edge_scene)
    assert d["E"] == edge_scene["means3D"].shape[0]
    check_lists(d)


@pytest.mark.parametrize("cap", [1, K - 1, K, K + 1, 2 * K, 2 * K + 7])
def test_partition_edges(edge_scene, cap):
    d = bin_lists(edge_scene, capacity=capacity_of(cap))
    check_lists(d, expect_E=cap)
    lo, hi = d["ranges"][17].tolist()
    assert hi - lo == min(cap, K + 100)


def test_no_instances():
    sc = single_tile_scene(torch.arange(50), -torch.ones(50), 256, 256)  # all behind the camera
    d = bin_lists(sc, capacity=capacity_of(1000))
    check_lists(d, expect_E=0)
    assert not d["ranges"].any()
    check_lists(bin_lists(sc))


def test_config_C_exact_and_bounded():
    sc = synthetic.make_config("C", seed=0)
    d = bin_lists(sc)
    R_ = check_lists(d)
    assert R_ > 10 * K
    cap = int(R_ * 1.25) + 4096
    check_lists(bin_lists(sc, capacity=capacity_of(cap)), expect_E=R_)
    # twice: the lists do not depend on the order of atomics
    d2 = bin_lists(sc, capacity=capacity_of(cap))
    assert torch.equal(d2["out"], d["out"]) and torch.equal(d2["ranges"], d["ranges"])


def test_bounded_overflow_drops_whole_gaussians():
    sc = synthetic.make_config("B", seed=1)
    R_ = check_lists(bin_lists(sc))
    d = bin_lists(sc, capacity=capacity_of(R_ // 2 + 3))
    E = check_lists(d)
    assert 0 < E <= R_ // 2 + 3 and E < R_


@pytest.mark.parametrize("band", [R.TileRowBand(1, 80, 3), R.TileRowBand(10, 50, 1)])
def test_bands(band):
    sc = synthetic.make_scene(P=300_000, width=1920, height=1280, sh_degree=1, seed=5)
    d = bin_lists(sc, band=band)
    check_lists(d)
    rows = torch.arange(80, device=DEV).repeat_interleave(120)
    inband = (rows >= band.begin) & (rows < band.end) & ((rows - band.begin) % band.step == 0)
    assert not d["ranges"][~inband].any()
    check_lists(bin_lists(sc, band=band, capacity=capacity_of(d["E"] + 5000)), expect_E=d["E"])


@pytest.mark.parametrize("W,H", [(2048, 2048), (2064, 2048), (5000, 4000)])
def test_both_sides_of_the_tile_threshold(W, H):
    """128 x 128 = 16384 tiles buckets; 129 x 128 takes the tile radix sort on 16-bit ids, 313 x 250 on 32-bit ids."""
    sc = synthetic.make_scene(P=200_000, width=W, height=H, sh_degree=0, seed=2, scale_med=0.02)
    d = bin_lists(sc)
    assert (d["ntile"] <= MAX_TILES) == (W == 2048)
    R_ = check_lists(d)
    check_lists(bin_lists(sc, capacity=capacity_of(R_ + 1000)), expect_E=R_)
