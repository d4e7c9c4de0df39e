"""Scene builders for the depth-tie checks (tests/test_depth_ties_*.py): groups of Gaussians with bit-identical view depth.

The binning promises the reference's list order (csrc/binning.cu): ascending tile, then ascending depth bits, then ascending
Gaussian index among equal depths.  Every scene here is built under the identity camera, so a Gaussian's fp32 view depth is its
z bit for bit, and a tie group is a set of Gaussians given the same fp32 z.  Members of a group differ in colour and opacity, so
their blend order shows in the images and in the gradients.  Every builder runs raster64.margin_scene and then asserts the ties it
claims on what survived; when the margin pass breaks a claim, the builder places the scene again with the next seed.

Each builder returns dict(name, scene, groups = [ascending index tensors of the tie groups], ...case-specific fields)."""
from __future__ import annotations

import torch

import raster64_case as RC
from oracle import raster64 as R64

F64 = torch.float64
TILE = 16
BIG_TILES = 64          # csrc/binning.cu: a Gaussian of more than 64 tiles takes emit_big_kernel
PARTITION = 2048        # test_bucket_partitions_gpu.part_size(E) for every E of the partition case
ATTEMPTS = 12


def _r(g, n, lo, hi):
    return torch.rand(n, generator=g, dtype=F64) * (hi - lo) + lo


def tie_groups(rec, radii):
    """The tie groups of the visible Gaussians: index tensors (ascending, at least two members) of equal fp32 view depth."""
    vis = torch.as_tensor(radii).cpu() > 0
    idx = torch.nonzero(vis).reshape(-1)
    bits = rec[:, 7].cpu().to(torch.float32).view(torch.int32)[idx]
    u, inv, cnt = torch.unique(bits, return_inverse=True, return_counts=True)
    return [idx[inv == k] for k in torch.nonzero(cnt >= 2).reshape(-1).tolist()]


def rects(pre):
    W, H = pre["cam"]["W"], pre["cam"]["H"]
    x0, y0, x1, y1 = R64.tile_rect(pre["rec"][:, 0].cpu(), pre["rec"][:, 1].cpu(), pre["radii"].cpu(), W, H)
    return torch.stack([x0, y0, x1, y1], 1)


def common_tile(rc, members):
    """Whether the tile rectangles of all `members` share a tile."""
    r = rc[members]
    return bool((r[:, 0].max() < r[:, 2].min()) and (r[:, 1].max() < r[:, 3].min()))


def group(W, H, cx, cy, n, z, g, sigma=(5.0, 9.0), opac=None, jitter=3.0, sh_degree=0):
    """n Gaussians around pixel (cx, cy) at the one view depth z (fp32-exact), of distinct opacity and colour."""
    hi = min(0.45, 3.0 / n)
    o = _r(g, n, 0.4 * hi, hi) if opac is None else _r(g, n, *opac)
    seed = int(torch.randint(0, 1 << 30, (1,), generator=g))
    return RC.screen_scene(W, H, cx + _r(g, n, -jitter, jitter), cy + _r(g, n, -jitter, jitter), _r(g, n, *sigma),
                           torch.full((n,), float(z), dtype=F64), o, seed=seed, sh_degree=sh_degree)


def _cat(parts):
    sc = parts[0]
    for p in parts[1:]:
        sc = RC.cat_scenes(sc, p)
    return sc


def _aniso(sc, g):
    """Raw, non-normalised quaternions and anisotropic scales (as test_raster64_gpu.preprocess_scene): no gradient of a rotation
    vanishes identically, as it does for an isotropic splat."""
    P = sc["means3D"].shape[0]
    q = torch.randn(P, 4, generator=g)
    sc = dict(sc)
    sc["rotations"] = (q / q.norm(dim=1, keepdim=True) * (0.8 + 0.4 * torch.rand(P, 1, generator=g))).float()
    sc["scales"] = (sc["scales"] * (0.6 + 0.8 * torch.rand(P, 3, generator=g))).float()
    return sc


def _shuffle(sc, g):
    """The rows in a random order: a group's indices end up interleaved with the other Gaussians'."""
    return R64.subset(sc, torch.randperm(sc["means3D"].shape[0], generator=g))


def _settle(sc, device):
    sc, removed, keep = R64.margin_scene(sc, device=device)
    pre = R64.preprocess64(sc, device)
    return sc, removed, keep, pre


def _retry(name, make, claims, seed, device):
    """make(seed) -> (scene, extra); claims(scene, pre, extra) -> (ok, info).  The first seed whose margin scene keeps the claims."""
    why = None
    for a in range(ATTEMPTS):
        sc0, extra = make(seed + 7919 * a)
        sc, removed, keep, pre = _settle(sc0, device)
        ok, info = claims(sc, pre, keep, extra)
        if ok:
            info.update(name=name, scene=sc, removed=removed, seed=seed + 7919 * a, groups=tie_groups(pre["rec"], pre["radii"]))
            return info
        why = info
    raise AssertionError(f"{name}: no placement in {ATTEMPTS} attempts keeps its ties ({why})")


def _interleaved(groups):
    return all(int(m[-1] - m[0]) + 1 > len(m) for m in groups)


# ------------------------------------------------------------------------------------------------ cases
def groups_case(W=160, H=96, sizes=(2, 3, 5, 9, 17, 40), n_fill=150, seed=1, device="cpu", sh_degree=0):
    """Tie groups of `sizes` members, each stacked over one tile, placed so that neighbouring groups overlap, over random filler
    at other depths; rows shuffled, so every group's indices are interleaved with other Gaussians'."""
    def make(s):
        g = torch.Generator().manual_seed(s)
        parts = []
        for k, n in enumerate(sizes):
            cx = float(_r(g, 1, 24, W - 24)); cy = float(_r(g, 1, 24, H - 24))
            parts.append(group(W, H, cx, cy, n, 3.0 + 0.5 * k, g, sh_degree=sh_degree))
        parts.append(RC.filler(W, H, n_fill, seed=s, sh_degree=sh_degree))
        return _shuffle(_aniso(_cat(parts), g), g), None

    def claims(sc, pre, keep, extra):
        gs = tie_groups(pre["rec"], pre["radii"])
        rc = rects(pre)
        sz = sorted(len(m) for m in gs)
        ok = sz == sorted(sizes) and all(common_tile(rc, m) for m in gs) and _interleaved(gs)
        return ok, dict(sizes=sz)
    return _retry("groups", make, claims, seed, device)


def wide_case(W, H, n_groups=24, n_fill=1500, seed=5, device="cpu"):
    """groups_case spread over a frame of more than 16384 tiles (the tile radix sort): n_groups tie groups of 2 to 40 members."""
    def make(s):
        g = torch.Generator().manual_seed(s)
        sizes = [2, 3, 40] + torch.randint(2, 25, (n_groups - 3,), generator=g).tolist()
        parts = [group(W, H, float(_r(g, 1, 24, W - 24)), float(_r(g, 1, 24, H - 24)), n, 3.0 + 0.25 * k, g) for k, n in enumerate(sizes)]
        parts.append(RC.filler(W, H, n_fill, seed=s))
        return _shuffle(_cat(parts), g), sizes

    def claims(sc, pre, keep, sizes):
        gs = tie_groups(pre["rec"], pre["radii"])
        rc = rects(pre)
        ok = len(gs) == len(sizes) and max(len(m) for m in gs) == 40 and all(common_tile(rc, m) for m in gs) and _interleaved(gs)
        return ok, dict(n_groups=len(gs))
    return _retry(f"wide{W}x{H}", make, claims, seed, device)


def big_case(W=640, H=96, seed=2, device="cpu"):
    """A Gaussian whose tile rectangle holds more than 64 tiles (emit_big_kernel) tied with small ones inside its footprint, at both
    sides of its index; a second wide one tied with another group; filler in front and behind."""
    def make(s):
        g = torch.Generator().manual_seed(s)
        big = RC.screen_scene(W, H, [320.3, 150.7], [47.1, 40.2], [45.13, 38.3], [4.0, 6.0], [0.25, 0.2], seed=s)
        smalls = [group(W, H, 320.0 + dx, 48.0, 3, 4.0, g, sigma=(3.0, 6.0)) for dx in (-60.0, 0.0, 70.0)]
        smalls.append(group(W, H, 150.0, 40.0, 4, 6.0, g, sigma=(3.0, 6.0)))
        return _shuffle(_aniso(_cat([big] + smalls + [RC.filler(W, H, 200, seed=s)]), g), g), None

    def claims(sc, pre, keep, extra):
        gs = tie_groups(pre["rec"], pre["radii"])
        rc = rects(pre)
        area = (rc[:, 2] - rc[:, 0]) * (rc[:, 3] - rc[:, 1])
        big_in = [m for m in gs if int(area[m].max()) > BIG_TILES]
        ok = len(big_in) == 2 and all(len(m) >= 3 for m in big_in) and _interleaved(gs)
        for m in big_in:
            b = m[int(torch.argmax(area[m]))]
            small = [i for i in m.tolist() if i != int(b)]
            ok &= int(area[small].max()) <= BIG_TILES and any(common_tile(rc, torch.tensor([int(b), i])) for i in small)
            ok &= any(i < int(b) for i in small) and any(i > int(b) for i in small)
        return ok, dict(big=[int(m[int(torch.argmax(area[m]))]) for m in big_in])
    return _retry("big", make, claims, seed, device)


def partition_case(W=1280, H=512, front=PARTITION - 5, n_group=12, n_back=800, seed=3, device="cpu"):
    """Single-tile Gaussians: `front` of them in front of a tie group of n_group single-tile members that share one tile, and
    n_back behind it.  Every Gaussian emits one instance in depth order, so the group takes positions [front, front + n_group) of the
    emitted sequence, across the bucketing partition boundary at 2048 (E < 396 x 2048: partitions of 2048 instances)."""
    gx, gy = W // TILE, H // TILE

    def make(s):
        g = torch.Generator().manual_seed(s)
        nf = front + 40
        tiles = torch.randperm(gx * gy, generator=g)[:nf]
        cx = (tiles % gx).to(F64) * TILE + 8 + _r(g, nf, -0.5, 0.5)
        cy = (tiles // gx).to(F64) * TILE + 8 + _r(g, nf, -0.5, 0.5)
        f = RC.screen_scene(W, H, cx, cy, 1.0, _r(g, nf, 2.0, 3.0), _r(g, nf, 0.2, 0.6), seed=s)
        t0 = int(tiles[0])
        grp = group(W, H, (t0 % gx) * TILE + 8.0, (t0 // gx) * TILE + 8.0, n_group, 3.5, g, sigma=(0.9, 1.1), opac=(0.08, 0.3), jitter=0.5)
        tb = torch.randint(0, gx * gy, (n_back,), generator=g)
        b = RC.screen_scene(W, H, (tb % gx).to(F64) * TILE + 8 + _r(g, n_back, -0.5, 0.5), (tb // gx).to(F64) * TILE + 8 + _r(g, n_back, -0.5, 0.5),
                            1.0, _r(g, n_back, 4.0, 10.0), _r(g, n_back, 0.2, 0.6), seed=s + 1)
        sc = _shuffle(_cat([f, grp, b]), g)
        # trim the front to `front` visible Gaussians after the margin pass (removing a lone single-tile splat changes no other decision)
        sc1, _, _, pre = _settle(sc, device)
        d, vis = pre["rec"][:, 7].cpu(), pre["radii"].cpu() > 0
        fr = torch.nonzero(vis & (d < 3.5)).reshape(-1)
        if len(fr) < front:
            return sc1, None
        drop = torch.zeros(len(d), dtype=torch.bool)
        drop[fr[front:]] = True
        return R64.subset(sc1, torch.nonzero(~drop).reshape(-1)), None

    def claims(sc, pre, keep, extra):
        rc = rects(pre)
        vis = pre["radii"].cpu() > 0
        d = pre["rec"][:, 7].cpu()
        area = (rc[:, 2] - rc[:, 0]) * (rc[:, 3] - rc[:, 1])
        gs = tie_groups(pre["rec"], pre["radii"])
        n_front = int((vis & (d < 3.5)).sum())
        E = int(area[vis].sum())
        ok = (len(gs) == 1 and len(gs[0]) == n_group and common_tile(rc, gs[0]) and bool((area[vis] == 1).all())
              and n_front < PARTITION < n_front + n_group and E < 396 * PARTITION and _interleaved(gs))
        return ok, dict(front=n_front, E=E, positions=(n_front, n_front + n_group))
    return _retry("partition", make, claims, seed, device)


def stack_case(W=64, H=48, sizes=(3, 4, 4, 3), seed=4, device="cpu"):
    """Screen-wide splats stacked one group behind the other, every group a tie: the centre tiles saturate inside the third group,
    the corner tiles never do.  For the saturation split swept over every budget."""
    def make(s):
        g = torch.Generator().manual_seed(s)
        parts = [group(W, H, 31.5, 23.5, n, 1.0 + 0.5 * k, g, sigma=(28.0, 32.0), opac=(0.55, 0.8), jitter=1.0) for k, n in enumerate(sizes)]
        return _shuffle(_cat(parts), g), None

    def claims(sc, pre, keep, extra):
        gs = tie_groups(pre["rec"], pre["radii"])
        bl = R64.blend64(pre["rec"], pre["radii"], W, H, pre["cam"]["bg"])
        ok = sorted(len(m) for m in gs) == sorted(sizes) and bool(bl["stopped"].any()) and not bool(bl["stopped"].all())
        return ok, dict(sizes=[len(m) for m in gs])
    return _retry("stack", make, claims, seed, device)


# ------------------------------------------------------------------------------------------------ clones
def raw_of(sc):
    """The model parameters (log scale, logit opacity, SH split into dc / rest) of a scene."""
    o = sc["opacities"].double()
    return dict(xyz=sc["means3D"].clone(), features_dc=sc["shs"][:, :1].clone(), features_rest=sc["shs"][:, 1:].clone(),
                opacity=torch.log(o / (1 - o)).float(), scaling=torch.log(sc["scales"]), rotation=sc["rotations"].clone())


def scene_of_raw(raw, like):
    """The rendered scene of model parameters (the activations of GaussianModel: exp, sigmoid), with `like`'s camera and upstream."""
    out = dict(like)
    out.update(means3D=raw["xyz"].contiguous(), shs=torch.cat([raw["features_dc"], raw["features_rest"]], 1).contiguous(),
               opacities=torch.sigmoid(raw["opacity"]).contiguous(), scales=torch.exp(raw["scaling"]).contiguous(),
               rotations=raw["rotation"].contiguous())
    return out


def clone_case(W=128, H=80, n_parents=10, seed=6, device="cpu"):
    """A densification clone pass: n_parents Gaussians (members of tie groups and plain filler) and their exact copies appended
    at higher indices, in ascending parent order (the layout densify_and_prune writes).  Every parent ties with its copy in every
    tile it touches.  Returns also raw (the model before cloning), parents and clones (indices in the scene)."""
    def make(s):
        g = torch.Generator().manual_seed(s)
        parts = [group(W, H, float(_r(g, 1, 20, W - 20)), float(_r(g, 1, 20, H - 20)), n, 3.0 + 0.5 * k, g, sh_degree=1)
                 for k, n in enumerate((2, 3, 5))]
        parts.append(RC.filler(W, H, 100, seed=s, sh_degree=1))
        base = _shuffle(_aniso(_cat(parts), g), g)
        raw = raw_of(base)
        P0 = base["means3D"].shape[0]
        base = scene_of_raw(raw, base)
        sc0, _, keep0, _ = _settle(base, device)
        raw = {k: v[keep0] for k, v in raw.items()}
        P0 = len(keep0)
        pre0 = R64.preprocess64(sc0, device)
        vis = torch.nonzero(pre0["radii"].cpu() > 0).reshape(-1)
        grp = torch.cat(tie_groups(pre0["rec"], pre0["radii"]))
        others = vis[~torch.isin(vis, grp)]
        parents = torch.sort(torch.cat([grp[torch.randperm(len(grp), generator=g)[:n_parents // 2]],
                                        others[torch.randperm(len(others), generator=g)[:n_parents - n_parents // 2]]])).values
        full = {k: torch.cat([v, v[parents]]) for k, v in raw.items()}
        sc = scene_of_raw(full, sc0)
        return sc, dict(raw=raw, parents=parents, P0=P0)

    def claims(sc, pre, keep, extra):
        P0, parents = extra["P0"], extra["parents"]
        m = len(parents)
        ok = len(keep) == P0 + m  # the margin pass removed none of the model or its clones
        clones = torch.arange(P0, P0 + m)
        rec = pre["rec"].cpu()
        if ok:
            ok &= bool(torch.equal(rec[parents], rec[clones])) and bool((pre["radii"].cpu()[parents] > 0).all())
            gs = tie_groups(pre["rec"], pre["radii"])
            ok &= any(len(gg) > 2 for gg in gs)  # a clone of a member of a tie group of distinct Gaussians
        return ok, dict(raw=extra["raw"], parents=parents, clones=clones)
    return _retry("clones", make, claims, seed, device)


BUILDERS = dict(groups=groups_case, big=big_case, partition=partition_case, stack=stack_case, clones=clone_case)


def reversed_ties(P, groups):
    """A permutation of P rows that reverses the rows of every tie group (its own inverse)."""
    perm = torch.arange(P)
    for m in groups:
        perm[m] = m.flip(0)
    return perm
