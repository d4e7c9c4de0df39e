"""Scene and ownership builders for the fp64 tier of the Gaussian-sharded step (tests/test_sharded64_*.py).

A case is a global scene under the identity camera of raster64_case.screen_scene (view depth = the z that was set), split into
per-rank parts: rank r owns P_r <= chunk Gaussians, in global slots r*chunk + i, and the rank-major concatenation of the real
Gaussians is the single-GPU scene (ascending slot = ascending global id, so blend64's (depth, index) tie order is the order the
kernels claim).  Every edge is placed on purpose and asserted on the post-margin scene:

  block run totals  the rows a block of 256 owned slots sends, summed over the destination ranks (sum of popcount(mask)): 0
                    (padding), 1..255 (a partial block), 256, 257, 512, 3*256 and above (wide splats crossing every band);
  depth ties        pairs of strongly overlapping, opaque, contrasting splats with bit-identical z, owned by different ranks;
  empty bands       more ranks than tile rows;
  ownership         tail padding, padding in the middle (rank 0 short), a rank owning nothing, chunk not a multiple of 256, chunk < 256.
"""
from __future__ import annotations

import torch

import raster64_case as RC
from oracle import raster64 as R64

F64 = torch.float64
TILE = 16

# name: world, W, H, chunk, layout, block recipes (consumed in (rank, block) order by the full blocks; partial blocks take
# class-1 splats, or wide ones for "wide_part"), totals the case must contain
CASES = {
    "w2_tail": dict(world=2, W=48, H=64, chunk=300, layout="tail", recipes=["wide", "t257"],
                    totals={"1-255", "257", "512", "256w"}),
    "w3_middle": dict(world=3, W=48, H=96, chunk=549, layout="middle", recipes=["wide", "t257", "t512", "t768", "t256", "t256"],
                      totals={"0", "1-255", "256", "257", "512", ">=768", "256w"}),
    "w5_empty_rank": dict(world=5, W=48, H=96, chunk=256, layout="empty", recipes=["wide", "t257", "t512", "t768"],
                          totals={"0", "257", "512", ">=768", "256w"}),
    "w8_empty_bands": dict(world=8, W=32, H=80, chunk=200, layout="tail", recipes=[], part=["wide_part"],
                           totals={"1-255", ">=768"}, empty_bands=3),
    "w3_short_row": dict(world=3, W=48, H=17, chunk=300, layout="middle", recipes=["wide", "t257", "t256"],
                         totals={"1-255", "256", "257", "512"}, empty_bands=1),
}


def owned_counts(layout, world, chunk):
    """P_r per rank: (a) 'tail': the last rank is 37 short; (b) 'middle': rank 0 is 37 short (padding inside the global array,
    as after densification when chunk is the maximum of the ranks' counts); (c) 'empty': rank 1 owns nothing."""
    P = [chunk] * world
    if layout == "tail":
        P[-1] = chunk - 37
    elif layout == "middle":
        P[0] = chunk - 37
    elif layout == "empty":
        P[1] = 0
    else:
        raise ValueError(layout)
    return P


def dest_mask(y0, y1, world):
    """Ranks whose cyclic band (tile row y -> rank y % world) meets tile rows [y0, y1) (touched_ranks of sgr_common.cuh)."""
    if y1 <= y0:
        return 0
    if y1 - y0 >= world:
        return (1 << world) - 1
    m = 0
    for y in range(y0, y1):
        m |= 1 << (y % world)
    return m


def masks(px, py, radii, W, H, world):
    """Destination mask of every Gaussian from its tile rectangle (0 for culled ones)."""
    x0, y0, x1, y1 = R64.tile_rect(px, py, radii, W, H)
    vis = (torch.as_tensor(radii) > 0) & ((x1 - x0) * (y1 - y0) > 0)
    y0, y1, vis = y0.tolist(), y1.tolist(), vis.tolist()
    return torch.tensor([dest_mask(a, b, world) if v else 0 for a, b, v in zip(y0, y1, vis)], dtype=torch.int64)


def popcount(m):
    return torch.tensor([bin(int(v)).count("1") for v in m.tolist()], dtype=torch.int64)


def block_totals(mask, P_r, chunk):
    """{(rank, block): rows the block sends} over every block of every rank's chunk (padding slots send nothing)."""
    nblk = (chunk + 255) // 256
    pc = popcount(mask)
    out, o = {}, 0
    for r, n in enumerate(P_r):
        for b in range(nblk):
            lo, hi = min(n, 256 * b), min(n, 256 * (b + 1))
            out[(r, b)] = int(pc[o + lo:o + hi].sum())
        o += n
    return out


def total_classes(totals, world):
    cl = set()
    for t in totals.values():
        if t == 0:
            cl.add("0")
        elif t < 256:
            cl.add("1-255")
        elif t in (256, 257, 512):
            cl.add(str(t))
        if t >= 768:
            cl.add(">=768")
        if t == 256 * world:
            cl.add("256w")
    return cl


def _pool(W, H, world, seed, D, n_small, n_wide, n_ties):
    """Candidates: class-k splats span exactly k tile rows (k = 1, 2, 3), wide faint splats span every row, tie pairs.  n_small: {1: n, 2: n, 3: n} candidates per class."""
    g = torch.Generator().manual_seed(seed)
    gy = (H + TILE - 1) // TILE
    U = lambda n, lo, hi: torch.rand(n, generator=g, dtype=F64) * (hi - lo) + lo
    row = lambda n, top: torch.randint(0, max(1, top), (n,), generator=g).to(F64)
    parts, tags = [], []
    # class 1: radius 4-5 around a tile-row centre; class 2: across a row boundary; class 3: radius 11 from row y to y + 2
    for k, (off, jit, sig) in {1: (8.0, 2.0, (0.9, 1.4)), 2: (16.0, 2.0, (0.9, 1.4)), 3: (24.0, 1.5, (3.3, 3.3))}.items():
        if gy < k:
            continue
        n = n_small[k]
        py = TILE * row(n, gy - k + 1) + off + U(n, -jit, jit)
        parts.append(RC.screen_scene(W, H, U(n, 0, W), py, U(n, *sig), U(n, 3.0, 30.0), U(n, 0.05, 0.5), sh_degree=D, seed=seed + k))
        tags += [f"c{k}"] * n
    if n_wide:
        parts.append(RC.stack(W, H, W / 2, H / 2, n_wide, seed=seed + 7, opac=(0.004, 0.008), sigma=40.0, z0=2.0, sh_degree=D))
        tags += ["wide"] * n_wide
    for i in range(n_ties):  # two splats 1 px apart, bit-identical z, opacity 0.6, red against blue
        y = int(torch.randint(0, max(1, H // TILE), (1,), generator=g))  # a full tile row: the pair blends on visible pixels
        cx, cy = float(U(1, 6, W - 6)), TILE * y + 8.0 + float(U(1, -1.5, 1.5))
        z = float(U(1, 2.2, 2.9))
        for j, rgb in enumerate(([0.9, 0.1, 0.1], [0.1, 0.15, 0.9])):
            parts.append(RC.screen_scene(W, H, [cx + (j - 0.5)], [cy], [1.2], [z], [0.6], rgb=torch.tensor(rgb, dtype=F64), sh_degree=D,
                                         seed=seed + 100 + 2 * i + j))
            tags.append(f"tie{i}{'ab'[j]}")
    sc = parts[0]
    for p in parts[1:]:
        sc = RC.cat_scenes(sc, p)
    # mildly anisotropic splats under raw, non-normalised quaternions: with isotropic ones the rotation gradient is a sum of terms that
    # cancel exactly in fp64 and not in fp32, which no relative bound can cover
    P = sc["means3D"].shape[0]
    q = torch.randn(P, 4, generator=g)
    sc["rotations"] = (q / q.norm(dim=1, keepdim=True) * (0.9 + 0.2 * torch.rand(P, 1, generator=g))).float()
    sc["scales"] = (sc["scales"] * (0.85 + 0.3 * torch.rand(P, 3, generator=g))).float()
    return sc, tags


def _classify(sc, tags, world, device):
    pre = R64.preprocess64(sc, device)
    cam = pre["cam"]
    m = masks(pre["rec"][:, 0].cpu(), pre["rec"][:, 1].cpu(), pre["radii"].cpu(), cam["W"], cam["H"], world)
    return m, popcount(m)


def build(name, seed=0, D=3, device="cpu", max_tries=4):
    """The case `name` of CASES: returns dict(scene (global, rank-major), P_r, chunk, world, W, H, mask, totals, ties [(a, b) global
    indices], owner_of [global index -> rank], tags)."""
    spec = CASES[name]
    world, W, H, chunk = spec["world"], spec["W"], spec["H"], spec["chunk"]
    P_r = owned_counts(spec["layout"], world, chunk)
    gy = (H + TILE - 1) // TILE
    nblk = (chunk + 255) // 256
    plan = []  # per (rank, block): recipe
    recipes = list(spec["recipes"])
    for r in range(world):
        for b in range(nblk):
            n = max(0, min(P_r[r], 256 * (b + 1)) - 256 * b)
            if n == 256:
                plan.append((r, b, n, recipes.pop(0) if recipes else "t256"))
            elif n > 0:
                parts = spec.get("part", [])
                plan.append((r, b, n, parts[(r * nblk + b) % len(parts)] if parts and r == 0 else "small"))
            else:
                plan.append((r, b, 0, None))
    need = {"c1": 0, "c2": 0, "c3": 0, "wide": 0}
    for _, _, n, rc in plan:
        if rc == "wide" or rc == "wide_part":
            need["wide"] = max(need["wide"], n)
        elif rc == "t256" or rc == "small":
            need["c1"] += n
        elif rc == "t257":
            need["c1"] += 255; need["c2"] += 1
        elif rc == "t512":
            need["c2"] += 256
        elif rc == "t768":
            need["c3"] += 256
    n_ties = 2 if sum(1 for p in P_r if p > 0) >= 2 else 0
    n_small = {k: int(1.3 * need[f"c{k}"]) + 40 for k in (1, 2, 3)}
    pool, tags = _pool(W, H, world, seed * 7919 + len(name), D, n_small, need["wide"] + 80 if need["wide"] else 0, n_ties)
    excluded = torch.zeros(len(tags), dtype=torch.bool)
    for _ in range(max_tries):
        keep0 = torch.nonzero(~excluded).reshape(-1)
        sc, _, kept = R64.margin_scene(R64.subset(pool, keep0), device=device)
        kept = keep0[kept.cpu()]
        kt = [tags[i] for i in kept.tolist()]
        m, pc = _classify(sc, kt, world, device)
        full = min(gy, world)
        by = {"c1": [], "c2": [], "c3": [], "wide": []}
        ties = {}
        for i, (t, c) in enumerate(zip(kt, pc.tolist())):
            if t.startswith("tie"):
                ties.setdefault(t[:-1], {})[t[-1]] = i
            elif t == "wide" and c == full:
                by["wide"].append(i)
            elif t.startswith("c") and c == int(t[1]):
                by[t].append(i)
        pairs = [(v["a"], v["b"]) for v in ties.values() if len(v) == 2 and pc[v["a"]] == 1 and pc[v["b"]] == 1]
        owners = [r for r in range(world) if P_r[r] > 0]
        ranks = {r: [] for r in range(world)}
        cur = {k: 0 for k in by}
        tie_for = {r: [] for r in range(world)}
        for k, (a, b) in enumerate(pairs):  # the two splats of a pair go to two different ranks
            tie_for[owners[k % len(owners)]].append(a)
            tie_for[owners[(k + 1) % len(owners)]].append(b)

        def take(cls, n, r=None):
            out = []
            if cls == "c1" and r is not None:
                while tie_for[r] and len(out) < n:
                    out.append(tie_for[r].pop(0))
            lst = by[cls]
            while len(out) < n:
                if cur[cls] >= len(lst):
                    raise RuntimeError(f"{name}: not enough {cls} splats survived")
                out.append(lst[cur[cls]]); cur[cls] += 1
            return out

        for r, b, n, rc in plan:
            if rc is None:
                continue
            if rc in ("wide", "wide_part"):
                cur["wide"] = 0  # (each wide block reuses the same stack: at most one per case)
                ranks[r] += take("wide", n)
            elif rc in ("t256", "small"):
                ranks[r] += take("c1", n, r)
            elif rc == "t257":
                ranks[r] += take("c1", 255, r) + take("c2", 1)
            elif rc == "t512":
                ranks[r] += take("c2", 256)
            elif rc == "t768":
                ranks[r] += take("c3", 256)
        order = torch.tensor([i for r in range(world) for i in ranks[r]], dtype=torch.int64)
        scene = R64.subset(sc, order)
        scene2, removed, kept2 = R64.margin_scene(scene, device=device)
        if removed == 0:
            break
        bad = torch.ones(len(order), dtype=torch.bool)
        bad[kept2.cpu()] = False
        excluded[kept[order[bad]]] = True  # drop them from the pool and assemble again
    else:
        raise RuntimeError(f"{name}: the assembled scene is not margin-clean after {max_tries} tries")
    pos = {int(g): k for k, g in enumerate(order.tolist())}
    tie_pairs = [(pos[a], pos[b]) for a, b in pairs if a in pos and b in pos]
    owner_of = torch.cat([torch.full((n,), r, dtype=torch.int64) for r, n in enumerate(P_r)])
    mask = m[order]
    return dict(name=name, scene=scene, P_r=P_r, chunk=chunk, world=world, W=W, H=H, gy=gy, mask=mask,
                totals=block_totals(mask, P_r, chunk), ties=tie_pairs, owner_of=owner_of, tags=[kt[i] for i in order.tolist()],
                claims=spec["totals"], empty_bands=max(0, world - gy))


def band_of(gy, rank, world):
    return list(range(rank, gy, world))


def expected_counts(px, py, radii, W, H, world):
    """Per rank: n_sel (visible Gaussians whose tile rectangle meets the band) and the (Gaussian, tile) pairs of the rectangles inside
    the band (before the kernels' exact tile culling, which can only drop pairs)."""
    x0, y0, x1, y1 = R64.tile_rect(px, py, radii, W, H)
    vis = (torch.as_tensor(radii) > 0) & ((x1 - x0) * (y1 - y0) > 0)
    gy = (H + TILE - 1) // TILE
    n_sel, pairs = [], []
    for r in range(world):
        rows = torch.zeros(gy + 1, dtype=torch.int64)
        rows[1:][torch.arange(gy) % world == r] = 1
        cum = torch.cumsum(rows, 0)  # cum[y] = band rows < y
        nr = (cum[y1.clamp(0, gy)] - cum[y0.clamp(0, gy)]) * vis
        n_sel.append(int((nr > 0).sum()))
        pairs.append(int((nr * (x1 - x0)).sum()))
    return n_sel, pairs


def to_precomp(scene, seed=0):
    """colors_precomp and cov3D_precomp in place of SH and scale / rotation (the unstaged gather)."""
    sc = dict(scene)
    g = torch.Generator().manual_seed(seed)
    P = sc["means3D"].shape[0]
    # the degree-0 colour of the SH (the tie pairs keep their contrast), jittered
    sc["colors_precomp"] = (R64.SH_C0 * sc["shs"][:, 0].double() + 0.5 + 0.05 * torch.rand(P, 3, generator=g, dtype=F64)).clamp(min=0.0).float()
    s_, qq = sc["scales"].double(), sc["rotations"].double()
    rr, x, y, z = qq.unbind(1)
    Rm = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + rr * z), 2 * (x * z - rr * y)], -1),
                      torch.stack([2 * (x * y - rr * z), 1 - 2 * (x * x + z * z), 2 * (y * z + rr * x)], -1),
                      torch.stack([2 * (x * z + rr * y), 2 * (y * z - rr * x), 1 - 2 * (x * x + y * y)], -1)], -2)
    Mm = s_[:, :, None] * Rm
    Sg = Mm.transpose(1, 2) @ Mm
    sc["cov3D_precomp"] = torch.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]], 1).float()
    for k in ("shs", "scales", "rotations"):
        sc.pop(k)
    return sc


def sharded_bound(bl, world, key="grad2d"):
    """Per-element bound of a cross-rank sum of per-band partial sums: the single-GPU bound plus world 2^-24 mass (one fp32 add per rank)."""
    return R64.bound(bl["kmass_" + key], bl["mass_" + key], bl["ntiles"], extra=float(world))


def band_upstream(scene, rank, world):
    """The upstream image gradients zeroed outside the cyclic band of `rank`: blend64 with them gives that rank's partial grad2d."""
    H = int(scene["cam"]["image_height"])
    gy = (H + TILE - 1) // TILE
    rows = torch.zeros(H, dtype=torch.bool)
    for y in band_of(gy, rank, world):
        rows[y * TILE:min(H, y * TILE + TILE)] = True
    return {k: scene["grad_" + k] * rows[None, :, None].to(scene["grad_" + k].dtype) for k in ("color", "depth", "alpha")}
