"""Depth ties on the GPU: the binning's list order among Gaussians of equal view depth, and the blend of tied Gaussians against
float64, on every binning path.

csrc/binning.cu promises the reference's order: ascending tile, then ascending depth bits, then ascending Gaussian index among equal
depths.  A tie is common in real frames (every clone of densify_and_prune is an exact copy of its parent, at a higher index), and
the order of a tie decides which of two tied Gaussians blends in front and so which takes the front splat's gradient.
  1. the list-order invariant: in every tile's list, (depth bits from the kernel's own records, index) strictly increases, on the
     bucketed one-pass binning, the tile radix sort on 16- and 32-bit tile ids, a cyclic band, a bounded frame, a split frame and
     config C;
  2. per element against blend64 (test_raster64_gpu.check) on the tie scenes of tests/tie_case.py under the same modes (the
     tile radix sort on 16-bit ids);
  3. the saturation split swept over every budget of a tied stack, with the split inside a tie group;
  4. a render layer whose first row cuts a tie group;
  5. clones written by densify_and_prune;
  6. the reference itself (tests/golden/live/ties.npz, tests/golden/make_tie_golden.py)."""
import os

import numpy as np
import pytest
import torch

import tie_case as TC
import util
import test_raster64_gpu as T64
from oracle import raster64 as R64
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi, synthetic, training
from street_gaussians_b200 import rasterizer as R
from street_gaussians_b200._capi import STATUS_EMITTED, STATUS_INSTANCES, STATUS_NEAR_END, STATUS_OVERFLOW, STATUS_SPLIT_K
from test_bucket_partitions_gpu import part_size, split_state
from test_saturation_split_gpu import assert_same, render

pytestmark = pytest.mark.gpu
DEV = "cuda"
ALL, AUTO = _capi.NEAR_BUDGET_ALL, _capi.NEAR_BUDGET_AUTO
MAX_BUCKET_TILES = 16384       # csrc/binning.cu kBucketMaxTiles
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live", "ties.npz")
REPORT = {}


def frame_lists(scene, band=None, capacity=None, budget=ALL):
    """Forward of `scene`: the final per-tile lists, their ranges, the status words and each Gaussian's depth bits from the
    kernel's records (rec[:, 7])."""
    cam = scene["cam"]
    st = util.settings_from(sgb, cam, DEV)
    dv = lambda k: scene[k].to(DEV) if scene.get(k) is not None else None
    P = scene["means3D"].shape[0]
    with torch.no_grad(), _capi.near_budget(budget):
        out = R._forward_impl(dv("means3D"), dv("shs"), dv("colors_precomp"), None, dv("opacities"), dv("scales"), dv("rotations"),
                              None, st, band, capacity)
    fst = out[5]
    torch.cuda.synchronize()
    v = R.state_views(st, fst, P)
    status = v["status"].long().cpu()
    E = int(status[STATUS_EMITTED])
    bits = v["rec"][:, 7].contiguous().view(torch.int32).long()
    return dict(list=v["vals_out"][:E].long(), ranges=v["ranges"].long(), status=status, E=E, bits=bits, radii=out[1],
                ntile=v["ranges"].shape[0])


def check_order(d):
    """(depth bits, index) strictly increases along every tile's list.  Returns the number of adjacent tied pairs."""
    ln = d["ranges"][:, 1] - d["ranges"][:, 0]
    assert int(ln.sum()) == d["E"]
    starts = d["ranges"][:, 0][ln > 0]
    assert torch.equal(starts, (torch.cumsum(ln, 0) - ln)[ln > 0]), "the lists are laid out in tile order"
    tile = torch.repeat_interleave(torch.arange(d["ntile"], device=DEV), ln)
    ids = d["list"]
    dep = d["bits"][ids]
    assert bool((dep >= 0).all()) and bool((d["radii"][ids] > 0).all())
    same = tile[1:] == tile[:-1]
    tie = dep[1:] == dep[:-1]
    up = (dep[1:] > dep[:-1]) | (tie & (ids[1:] > ids[:-1]))
    bad = torch.nonzero(same & ~up).reshape(-1)
    assert len(bad) == 0, f"{len(bad)} adjacent pairs out of (depth, index) order, first at {bad[:4].tolist()}: " \
                          f"ids {[(int(ids[i]), int(ids[i + 1])) for i in bad[:4].tolist()]}"
    return int((same & tie).sum())


def quantized_scene(W, H, P=200_000, seed=2, step=1.0 / 64):
    """A random scene whose depths are rounded to multiples of `step`: nearly every Gaussian shares its depth with others."""
    sc = synthetic.make_scene(P=P, width=W, height=H, sh_degree=0, seed=seed, scale_med=0.02)
    sc["means3D"][:, 2] = torch.round(sc["means3D"][:, 2] / step) * step
    return sc


@pytest.fixture(scope="module")
def cases():
    out = {name: make(device=DEV) for name, make in TC.BUILDERS.items()}
    return out


@pytest.fixture(scope="module")
def wide():
    return {16: TC.wide_case(2064, 2048, device=DEV), 32: TC.wide_case(5000, 4000, device=DEV)}


# ------------------------------------------------------------------------------------------------ 1. list order
def _path(d, ntile_cond, split=False):
    st = d["status"]
    assert ntile_cond(d["ntile"]), d["ntile"]
    if split:
        assert int(st[STATUS_NEAR_END]) < int(st[STATUS_INSTANCES]), "the split took effect: the near pass holds part of the frame"
    else:
        assert int(st[STATUS_EMITTED]) == int(st[STATUS_INSTANCES]), "one pass: every instance emitted"


MODES = ["bucketed", "sort16", "sort32", "band", "bounded", "split"]


@pytest.mark.parametrize("mode", MODES)
def test_list_order(mode, cases, wide):
    bucketed = lambda n: n <= MAX_BUCKET_TILES
    scenes = []
    if mode == "sort16":
        for sc in (wide[16]["scene"], quantized_scene(2064, 2048)):
            d = frame_lists(sc)
            _path(d, lambda n: MAX_BUCKET_TILES < n <= 65535)
            scenes.append(check_order(d))
    elif mode == "sort32":
        for sc in (wide[32]["scene"], quantized_scene(5000, 4000)):
            d = frame_lists(sc)
            _path(d, lambda n: n > 65536)
            scenes.append(check_order(d))
    elif mode == "band":
        for sc in (cases["groups"]["scene"], quantized_scene(1920, 1280)):
            gy = (sc["cam"]["image_height"] + 15) // 16
            band = R.TileRowBand(1, gy, 2)
            d = frame_lists(sc, band=band)
            rows = torch.arange(d["ntile"], device=DEV) // ((sc["cam"]["image_width"] + 15) // 16)
            assert not d["ranges"][(rows - 1) % 2 != 0].any() and d["E"] > 0
            scenes.append(check_order(d))
    elif mode == "bounded":
        for sc in [c["scene"] for c in cases.values()] + [quantized_scene(1920, 1280)]:
            R_ = frame_lists(sc)["E"]
            d = frame_lists(sc, capacity=sgb.InstanceCapacity(initial=R_ + 100))
            assert int(d["status"][STATUS_OVERFLOW]) == 0 and d["E"] == R_
            scenes.append(check_order(d))
    elif mode == "split":
        for sc in [cases["groups"]["scene"], cases["stack"]["scene"], quantized_scene(1920, 1280)]:
            R_ = frame_lists(sc)["E"]
            for budget in (AUTO, R_ // 3):
                d = frame_lists(sc, budget=budget)
                _path(d, bucketed, split=True)
                scenes.append(check_order(d))
    else:
        for c in cases.values():
            d = frame_lists(c["scene"])
            _path(d, bucketed)
            scenes.append(check_order(d))
        d = frame_lists(quantized_scene(1920, 1280))
        _path(d, bucketed)
        scenes.append(check_order(d))
    # every frame holds adjacent ties (a split frame's ties may all lie behind its saturated tiles, as on config C)
    assert all(n > 0 for n in scenes) if mode != "split" else sum(scenes) > 0, scenes
    REPORT[mode] = scenes
    print(mode, "adjacent tied pairs per frame:", scenes)


def test_list_order_partition_boundary(cases):
    """The tie group of the partition case takes positions across the first partition boundary of the emitted sequence."""
    c = cases["partition"]
    with _capi.near_budget(ALL):
        s = split_state(c["scene"], ALL)
    E = s["E"]
    assert part_size(E) == TC.PARTITION
    grp = c["groups"][0].to(DEV)
    pos = torch.nonzero(torch.isin(s["vals"], grp)).reshape(-1)
    assert len(pos) == len(grp) and int(pos.min()) < TC.PARTITION <= int(pos.max()), pos.tolist()
    d = frame_lists(c["scene"])
    assert check_order(d) >= len(grp) - 1


def test_list_order_config_C():
    """Config C under its identity view: the view depth is means3D[:, 2] exactly, and tied pairs share tile lists."""
    sc = synthetic.make_config("C", seed=0)
    n = {}
    for name, kw in (("one_pass", {}), ("auto_split", dict(budget=AUTO))):
        d = frame_lists(sc, **kw)
        n[name] = check_order(d)
    R_ = frame_lists(sc)["E"]
    d = frame_lists(sc, capacity=sgb.InstanceCapacity(initial=R_ + 4096))
    n["bounded"] = check_order(d)
    REPORT["config_C"] = n
    print("config C adjacent tied pairs in the tile lists:", n)
    assert n["one_pass"] > 0


# ------------------------------------------------------------------------------------------------ 2. per element
@pytest.mark.parametrize("name", sorted(TC.BUILDERS))
def test_per_element_one_pass(name, cases):
    T64.check(f"ties_{name}", cases[name]["scene"], max_removed=0.0)


def test_per_element_tile_sort(wide):
    """The 16-bit tile radix sort (2064 x 2048).  (32-bit ids are covered by the list-order invariant: at 5000 x 4000 the pixel
    positions carry an fp32 rounding that puts a few rectangle edges of any random placement inside the per-element margin.)"""
    c = wide[16]
    W, H = c["scene"]["cam"]["image_width"], c["scene"]["cam"]["image_height"]
    assert MAX_BUCKET_TILES < ((W + 15) // 16) * ((H + 15) // 16) <= 65535
    T64.check("ties_wide16", c["scene"], max_removed=0.0)


def test_per_element_band_bounded_split(cases):
    sc = cases["groups"]["scene"]
    gy = (sc["cam"]["image_height"] + 15) // 16
    T64.check("ties_band", sc, band=R.TileRowBand(1, gy, 2), max_removed=0.0)
    R_ = frame_lists(sc)["E"]
    T64.check("ties_bounded", sc, capacity=R.InstanceCapacity(initial=R_ + 64), max_removed=0.0)
    for budget in (AUTO, R_ // 3):
        with _capi.near_budget(budget):
            assert int(frame_lists(sc, budget=budget)["status"][STATUS_NEAR_END]) < R_
            T64.check(f"ties_split{budget}", sc, max_removed=0.0)


# ------------------------------------------------------------------------------------------------ 3. saturation split
def test_every_split_of_a_tied_stack(cases):
    """Every budget from 0 to R over a stack of tie groups: images, n_contrib and tile_max_contrib bit-equal to the one-pass
    binning.  Some budget puts the split strictly inside a group, and some leaves a tile unsaturated that holds near and far
    members of one group, so the spliced list joins them; those frames are checked against blend64 per element."""
    c = cases["stack"]
    sc = c["scene"]
    P = sc["means3D"].shape[0]
    full = render(sc, ALL)
    Rn = int(full["status"][STATUS_INSTANCES])
    # depth-order slot of every Gaussian: (depth, index) order; all of the stack is visible
    z = sc["means3D"][:, 2].double()
    slot = torch.empty(P, dtype=torch.long)
    slot[torch.from_numpy(np.lexsort((np.arange(P), z.numpy())))] = torch.arange(P)
    spans = [(int(slot[m].min()), int(slot[m].max()) + 1) for m in c["groups"]]
    assert all(hi - lo == len(m) for (lo, hi), m in zip(spans, c["groups"]))
    inside, joined = [], []
    for b in range(Rn + 1):
        got = render(sc, b)
        assert_same(full, got, what=f"B={b}")
        K = int(got["status"][STATUS_SPLIT_K])
        if not any(lo < K < hi for lo, hi in spans):
            continue
        inside.append(b)
        s = split_state(sc, b)
        assert int(s["status"][STATUS_SPLIT_K]) == K
        assert torch.equal(s["perm"][:K].cpu().sort().values, torch.nonzero(slot < K).reshape(-1).sort().values)
        ln = s["ranges"][:, 1] - s["ranges"][:, 0]
        tile = torch.repeat_interleave(torch.arange(s["ntile"], device=DEV), ln)
        sl = slot.to(DEV)[s["out"]]
        for m in c["groups"]:
            inm = torch.isin(s["out"], m.to(DEV))
            near_t = torch.zeros(s["ntile"], dtype=torch.bool, device=DEV)
            far_t = torch.zeros_like(near_t)
            near_t[tile[inm & (sl < K)]] = True
            far_t[tile[inm & (sl >= K)]] = True
            if bool((near_t & far_t).any()):
                joined.append(b)
                break
    assert inside, "no budget splits inside a tie group"
    assert joined, "no unsaturated tile holds near and far members of one tie group"
    for b in sorted({inside[0], joined[0], joined[-1]}):
        with _capi.near_budget(b):
            T64.check(f"ties_stack_B{b}", sc, max_removed=0.0)
    REPORT["stack"] = dict(R=Rn, inside=len(inside), joined=len(joined))
    print("tied stack:", REPORT["stack"])


# ------------------------------------------------------------------------------------------------ 4. render layers
def test_layer_cuts_a_tie_group(cases):
    """The layer [b, P) with b inside the largest tie group: the layered render and its gradients against render64 on the
    subset (test_layers_gpu.check_layered)."""
    import test_layers_gpu as TL
    c = cases["groups"]
    sc = dict(c["scene"])
    m = max(c["groups"], key=len)
    b0 = int(m[len(m) // 2])
    sc2, b = TL._margin_pair(sc, b0)
    pre = R64.preprocess64(sc2, DEV)
    gs = TC.tie_groups(pre["rec"], pre["radii"])
    assert any(bool((g < b).any()) and bool((g >= b).any()) and len(g) >= 3 for g in gs), "b cuts a tie group"
    TL.check_layered(sc2, b)


# ------------------------------------------------------------------------------------------------ 5. clones
def _model(raw, parents):
    n = raw["xyz"].shape[0]
    acc = torch.zeros(n, 2)
    acc[parents] = 1.0
    m = {"_" + k: v.to(DEV).contiguous() for k, v in raw.items()}
    m.update(_semantic=torch.zeros(n, 0, device=DEV), max_radii2D=torch.zeros(n, device=DEV), xyz_gradient_accum=acc.to(DEV),
             denom=torch.ones(n, 1, device=DEV), percent_dense=0.01, percent_big_ws=0.1, scene_radius=torch.tensor([1000.0]),
             sphere_center=torch.zeros(3), sphere_radius=torch.tensor([1000.0]))
    return m


def test_clones(cases):
    """densify_and_prune with a threshold that clones the parents only: the clones are exact copies at higher indices, their
    depths equal their parents' bit for bit, every grad2d row is within blend64's bound, and parent and clone take different
    gradients, the parent the front one."""
    c = cases["clones"]
    raw, parents, clones = c["raw"], c["parents"], c["clones"]
    model = _model(raw, parents)
    sc = training.densify_and_prune([model], 0.5, 0.0, False, seed=11)
    assert sc[0]["points_clone"] == len(parents) and sc[0]["points_split"] == 0 and sc[0]["points_pruned"] == 0
    new = {k: model["_" + k].detach().cpu() for k in raw}
    for k, v in raw.items():
        assert torch.equal(new[k], torch.cat([v, v[parents]])), k
    scene = TC.scene_of_raw(new, c["scene"])
    for k in ("means3D", "shs", "opacities", "scales", "rotations"):
        assert torch.equal(scene[k], c["scene"][k]), k
    bl, k = T64.check("ties_clones", scene, max_removed=0.0)
    p, q = parents.to(DEV), clones.to(DEV)
    bits = k["rec"][:, 7].contiguous().view(torch.int32)
    assert torch.equal(bits[p], bits[q]) and bool((k["radii"][p] > 0).all())
    g = k["grad2d"].double()[:, :11]
    bnd = R64.bound(bl["kmass_grad2d"], bl["mass_grad2d"], bl["ntiles"])[:, :11]
    # different gradients: every pair differs by more than both bounds in some component
    assert bool((((g[p] - g[q]).abs() > bnd[p] + bnd[q]).any(1)).all())
    # the parent takes the front one: blend64's front row (its own, index order), not the clone's
    assert bool((((g[p] - bl["grad2d"][q][:, :11]).abs() > bnd[p] + bnd[q]).any(1)).all())


# ------------------------------------------------------------------------------------------------ 6. the reference
def golden_scenes():
    """The two seeded scenes of tests/golden/live/ties.npz, built on the CPU."""
    return dict(groups=TC.groups_case(), clones=TC.clone_case())


def test_against_reference_golden():
    """The reference's outputs on the tie scenes: radii and view depths bit-equal, images within 1e-4, and every tied row's
    gradients row by row (relative to that row), so that two tied rows whose gradients are swapped fail."""
    z = np.load(GOLDEN)
    for name, c in golden_scenes().items():
        sc = c["scene"]
        mine = util.run_api(sgb, sc)
        d = frame_lists(sc)
        assert (mine["radii"] == z[f"{name}_radii"]).all(), name
        vis = mine["radii"] > 0
        assert (d["bits"].cpu().numpy()[vis] == z[f"{name}_depth_bits"][vis]).all(), name
        for key in ("color", "depth", "alpha"):
            err = float(np.abs(mine[key] - z[f"{name}_{key}"]).max())
            assert err <= 1e-4, (name, key, err)
        rows = torch.cat(c["groups"]).numpy()
        worst = 0.0
        for key in ("g_means3D", "g_means2D", "g_shs", "g_opacities", "g_scales", "g_rotations"):
            ref = z[f"{name}_{key}"].reshape(len(vis), -1)[rows]
            got = mine[key].reshape(len(vis), -1)[rows]
            tol = 2e-3 * np.abs(ref).max(1, keepdims=True) + 1e-12
            worst = max(worst, float((np.abs(got - ref) / tol).max()))
            assert (np.abs(got - ref) <= tol).all(), (name, key, float((np.abs(got - ref) / tol).max()))
            if name == "clones" and key == "g_shs":
                # the bar tells a parent from its clone: their reference colour gradients (alpha T against alpha (1 - alpha) T)
                # differ by more than it
                full = z[f"{name}_{key}"].reshape(len(vis), -1)
                pr, cl = full[c["parents"].numpy()], full[c["clones"].numpy()]
                bar = 2e-3 * np.maximum(np.abs(pr).max(1), np.abs(cl).max(1))
                assert (np.abs(pr - cl).max(1) > bar).all()
        REPORT[f"golden_{name}"] = worst
        print(name, "worst gradient row error / bar:", round(worst, 4))
