"""Scenes for the fp64 densification tier (oracle/densify64.py, tests/test_densify64_*.py), in tests/densify_case.py's per-model
format.  Every builder returns (models, claims): claims name the edges the scene is built to reach, and claim_holds() re-derives
each one from the inputs with a plain per-parent fp32 loop, so a scene that stops reaching its edge fails on the CPU.

Claims: ("sizes", [segment sizes]); ("multi_segment_warp", None); (kind, k, l, expected 4-bit mask or None) for a designed parent
l of model k, where kind is one of the names in _PARENT_CHECKS; ("tile", k, tile, pattern) for a whole apply tile of model k."""
from __future__ import annotations

import math

import numpy as np
import torch

NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic")
F = np.float32


def model(n, kind, g, *, M=4, S=0, C=1, state=True, grad_col=None, extent=None, percent_dense=0.01, percent_big_ws=0.1,
          grad_threshold=None, box=2.0):
    """A random sub-model like test_densify_gpu._synthetic's, with every field this tier edits."""
    bk = kind == "background"
    rn = lambda *s: torch.randn(*s, generator=g)
    t = dict(xyz=rn(n, 3) * (torch.tensor([8.0, 3.0, 10.0]) if bk else torch.tensor([1.2, 0.5, 0.4])) + (torch.tensor([0.0, 0.0, 20.0]) if bk else 0),
             f_dc=rn(n, C, 3), f_rest=rn(n, M - 1, 3) * 0.2, opacity=rn(n, 1) * 3.0,
             scaling=math.log(0.1 if bk else 0.03) + rn(n, 3) * 0.6, rotation=rn(n, 4), semantic=torch.rand(n, S, generator=g))
    denom = torch.randint(0, 6, (n, 1), generator=g).float()
    t["xyz_gradient_accum"] = denom * torch.rand(n, 2, generator=g) * (1.6e-3 if bk else 4e-4)
    t["denom"], t["max_radii2D"] = denom, torch.rand(n, generator=g) * 20
    for mk in ("exp_avg", "exp_avg_sq"):
        t[mk] = {a: (rn(*t[a].shape).abs() * 1e-3 if state else None) for a in NAMES}
    t["step"] = {a: 7.0 for a in NAMES}
    m = dict(kind=kind, grad_col=(1 if bk else 0) if grad_col is None else grad_col,
             grad_threshold=(6e-4 if bk else 2e-4) if grad_threshold is None else grad_threshold,
             extent=torch.tensor([(20.0 if bk else 3.375) if extent is None else extent]), percent_dense=percent_dense,
             percent_big_ws=percent_big_ws, draws=rn(n, 18), **{"in": t})
    if bk:
        m.update(sphere_center=torch.tensor([0.0, 0.0, 20.0]), sphere_radius=torch.tensor([12.0]))
    else:
        m.update(min_xyz=torch.tensor([-box, -box / 2, -box / 2.5]), max_xyz=torch.tensor([box, box / 2, box / 2.5]))
    return m


def thresholds(m):
    """The fp32 thresholds the kernel compares against (training._densify forms them the same way)."""
    ext = F(float(m["extent"].reshape(-1)[0]))
    return dict(g=F(m["grad_threshold"]), dense=F(ext * F(m["percent_dense"])), big=F(ext * F(m["percent_big_ws"])))


def _set(m, l, **fields):
    for a, v in fields.items():
        tgt = m["in"][a]
        tgt[l] = torch.as_tensor(v, dtype=torch.float32).reshape(tgt[l].shape)


# ---- segment tables ----
def segments(sizes, seed=0, bkgd_at=1, bkgd=3000):
    g = torch.Generator().manual_seed(seed)
    models = [model(s, "actor", g) for s in sizes]
    models.insert(bkgd_at, model(bkgd, "background", g))
    return models, [("sizes", [bkgd if k == bkgd_at else sizes[k - (k > bkgd_at)] for k in range(len(models))]),
                    ("multi_segment_warp", None)]


def edge_sizes():
    """Sizes 0, 1, 2, 31, 33, 255, 256, 257 and 513, with empty actors first, in the middle and last."""
    return segments([0, 1, 2, 0, 31, 33, 255, 256, 257, 513, 0], seed=1)


def many_actors(n_act, seed):
    """1 background + n_act actors of 0-40 Gaussians (a fifth empty): several launches of reset_opacity, warps over many segments."""
    rs = np.random.RandomState(seed)
    sizes = [0 if rs.rand() < 0.2 else int(rs.randint(1, 41)) for _ in range(n_act)]
    return segments(sizes, seed=seed, bkgd_at=0, bkgd=2000)


# ---- apply tiles ----
def tiles():
    """An actor of four 256-parent tiles: all kept, all clones, all split, and one row of each section (one parent clones, one
    splits, the other 254 are pruned as big).  Nothing else in the actor is near a threshold: its box is 1e3 wide."""
    g = torch.Generator().manual_seed(5)
    a = model(1024, "actor", g, extent=10.0, box=1e3)     # dense 0.1, big 1.0
    thr = thresholds(a)
    t = a["in"]
    t["opacity"][:] = 4.0
    t["denom"][:] = 1.0
    acc = t["xyz_gradient_accum"]
    acc[:, 0] = 0.0
    t["scaling"][:] = math.log(0.05)                       # < dense
    acc[256:512, 0] = float(thr["g"]) * 2                  # tile 1: clones
    acc[512:768, 0] = float(thr["g"]) * 2                  # tile 2: split (scale 0.5: children 0.3125, not big)
    t["scaling"][512:768] = math.log(0.5)
    t["scaling"][768:1024] = math.log(2.0)                 # tile 3: big, pruned ...
    t["scaling"][768] = math.log(0.05)                     # ... but one clone
    acc[768, 0] = float(thr["g"]) * 2
    t["scaling"][769] = math.log(0.5)                      # and one split
    acc[769, 0] = float(thr["g"]) * 2
    bk = model(600, "background", g)
    return [bk, a], [("tile", 1, 0, "kept"), ("tile", 1, 1, "clone"), ("tile", 1, 2, "split"), ("tile", 1, 3, "one_each")]


# ---- exact thresholds, overflow and degenerate inputs ----
def edges(grad_col_bkgd=1, M=4, S=0, C_act=1, state=True):
    """Designed parents appended to a random background and actor, each on one threshold or overflow.  The background and the
    actor use extent 2 with percent_dense = percent_big_ws = 0.5, so the dense and big thresholds are exactly 1.0 = expf(0)."""
    g = torch.Generator().manual_seed(7)
    bk = model(700, "background", g, grad_col=grad_col_bkgd, extent=2.0, percent_dense=0.5, percent_big_ws=0.5, M=M, S=S, state=state)
    ac = model(700, "actor", g, grad_col=1 - grad_col_bkgd, extent=2.0, percent_dense=0.5, percent_big_ws=0.5, M=M, S=S, C=C_act,
               state=state, box=4.0)
    claims = []
    designs = []

    def add(m, k, kind, expect, **fields):
        designs.append((m, k, kind, expect, fields))

    for k, m in ((0, bk), (1, ac)):
        thr = thresholds(m)
        gc = m["grad_col"]
        base = dict(opacity=4.0, rotation=[1.0, 0.0, 0.0, 0.0], scaling=[math.log(0.1)] * 3, denom=1.0)
        x0 = [0.0, 0.0, 20.0] if k == 0 else [0.0, 0.0, 0.0]

        def acc(v):
            a = [0.0, 0.0]
            a[gc] = float(v)
            return a

        gt, below = float(thr["g"]), float(np.nextafter(thr["g"], F(0)))
        add(m, k, "g_on_threshold", 3, xyz=x0, xyz_gradient_accum=acc(gt), **base)           # |g| = thr: clone
        add(m, k, "g_below_threshold", 1, xyz=x0, xyz_gradient_accum=acc(below), **base)
        add(m, k, "neg_g_on_threshold", 3, xyz=x0, xyz_gradient_accum=acc(-gt), **base)      # clone takes |g|
        add(m, k, "split_on_threshold", None, xyz=x0, xyz_gradient_accum=acc(gt), **dict(base, scaling=[0.5, 0.0, 0.0]))
        add(m, k, "neg_g_split_side", None, xyz=x0, xyz_gradient_accum=acc(-gt), **dict(base, scaling=[0.5, 0.0, 0.0]))
        add(m, k, "smax_on_dense", 3, xyz=x0, xyz_gradient_accum=acc(gt), **dict(base, scaling=[0.0, -1.0, -2.0]))  # 1 <= 1: clone, not big
        add(m, k, "denom_zero_acc_zero", 1, xyz=x0, xyz_gradient_accum=[0.0, 0.0], **dict(base, denom=0.0))
        add(m, k, "denom_zero_acc_pos", 3, xyz=x0, xyz_gradient_accum=acc(1e-3), **dict(base, denom=0.0))   # +inf: clone
        add(m, k, "zero_quaternion", None, xyz=x0, xyz_gradient_accum=acc(gt), **dict(base, rotation=[0.0] * 4, scaling=[0.5, 0.0, 0.0]))
        add(m, k, "exp_overflow", None, xyz=x0, xyz_gradient_accum=acc(gt), **dict(base, scaling=[100.0, 0.0, -1.0]))
        add(m, k, "opacity_plus_100", 1, xyz=x0, xyz_gradient_accum=[0.0, 0.0], **dict(base, opacity=100.0))
        add(m, k, "opacity_minus_100", 0, xyz=x0, xyz_gradient_accum=[0.0, 0.0], **dict(base, opacity=-100.0))
        mo = float(F(0.005))
        lo = float(np.log(mo / (1 - mo)))
        ops = [F(lo)]
        for _ in range(2):
            ops = [np.nextafter(ops[0], F(-np.inf))] + ops + [np.nextafter(ops[-1], F(np.inf))]
        for v in ops:   # sigmoid within a few ulps of min_opacity on both sides
            add(m, k, "sigmoid_near_min_opacity", None, xyz=x0, xyz_gradient_accum=[0.0, 0.0], **dict(base, opacity=float(v)))
        if k == 0:   # sphere: a big parent at the diameter's distance stays big (pruned), a bigger distance is spared
            add(m, k, "distance_on_diameter", 0, xyz=[24.0, 0.0, 20.0], xyz_gradient_accum=[0.0, 0.0], **dict(base, scaling=[1.0, 0.0, 0.0]))
            add(m, k, "distance_beyond_diameter", 1, xyz=[25.0, 0.0, 20.0], xyz_gradient_accum=[0.0, 0.0], **dict(base, scaling=[1.0, 0.0, 0.0]))
            add(m, k, "distance_within_diameter", 0, xyz=[23.0, 0.0, 20.0], xyz_gradient_accum=[0.0, 0.0], **dict(base, scaling=[1.0, 0.0, 0.0]))
        else:        # box: scale expf(-200) = 0, so both samples are the centre itself; faces are inclusive
            lo3, hi3 = m["min_xyz"].numpy(), m["max_xyz"].numpy()
            for a in range(3):
                for face, out in ((lo3, float(np.nextafter(F(lo3[a]), F(-np.inf)))), (hi3, float(np.nextafter(F(hi3[a]), F(np.inf))))):
                    on = [0.0, 0.0, 0.0]
                    on[a] = float(face[a])
                    off = list(on)
                    off[a] = out
                    add(m, k, "sample_on_face", 3, xyz=on, xyz_gradient_accum=acc(gt), **dict(base, scaling=[-200.0] * 3))
                    add(m, k, "sample_past_face", 0, xyz=off, xyz_gradient_accum=acc(gt), **dict(base, scaling=[-200.0] * 3))
    n0 = {0: bk["in"]["xyz"].shape[0], 1: ac["in"]["xyz"].shape[0]}
    grow = {0: 0, 1: 0}
    for m, k, _, _, _ in designs:
        grow[k] += 1
    for k, m in ((0, bk), (1, ac)):
        _grow(m, grow[k])
    at = dict(n0)
    for m, k, kind, expect, fields in designs:
        _set(m, at[k], **fields)
        claims.append((kind, k, at[k], expect))
        at[k] += 1
    return [bk, ac], claims


def _grow(m, extra):
    """Append `extra` rows (copies of row 0) to every per-Gaussian tensor of m."""
    t = m["in"]
    rep = lambda v: torch.cat([v, v[:1].repeat(extra, *([1] * (v.dim() - 1)))]) if v.shape[0] else v
    for a in list(t):
        v = t[a]
        if torch.is_tensor(v):
            t[a] = rep(v).clone()
        elif isinstance(v, dict) and a != "step":
            t[a] = {b: (None if x is None else rep(x).clone()) for b, x in v.items()}
    m["draws"] = rep(m["draws"]).clone()


def box_sensitive(seed=9):
    """An actor whose clones and split children sit near its box faces with scales of the box's order, so which draws a row's box
    samples take decides its survival on many rows (a wrong draw slot changes masks)."""
    g = torch.Generator().manual_seed(seed)
    a = model(4000, "actor", g, extent=3.0, box=1.0, percent_dense=0.05, percent_big_ws=1.0)
    t = a["in"]
    t["opacity"][:] = 4.0
    t["denom"][:] = 1.0
    t["xyz_gradient_accum"][:, 0] = 1e-3
    lo, hi = a["min_xyz"], a["max_xyz"]
    t["xyz"] = (torch.rand(4000, 3, generator=g) * 0.3 + 0.7) * torch.where(torch.rand(4000, 3, generator=g) < 0.5, lo, hi)
    t["scaling"] = torch.log(torch.rand(4000, 3, generator=g) * 0.25 + 0.02)
    return [model(500, "background", g), a], []


def readout(n_seg=6, per=50_000, seed=3):
    """Every parent splits with identity rotation, scale expf(0) = 1 and xyz 0, so child c's xyz is draws [3c, 3c + 3) exactly; with
    prune_big_points off nothing is pruned.  Several segments, so the Philox subsequence must be the composed index."""
    g = torch.Generator().manual_seed(seed)
    models = []
    for k in range(n_seg):
        m = model(per, "background" if k == 0 else "actor", g, extent=1.0, percent_dense=0.5)
        t = m["in"]
        t["xyz"].zero_()
        t["scaling"].zero_()
        t["rotation"][:] = torch.tensor([1.0, 0.0, 0.0, 0.0])
        t["opacity"][:] = 4.0
        t["denom"][:] = 1.0
        t["xyz_gradient_accum"][:] = 1.0
        models.append(m)
    return models, []


# ---- the claims, re-derived per parent ----
def _parent(m, l):
    t = m["in"]
    f = lambda a: t[a][l].numpy().astype(np.float32).reshape(-1)
    thr = thresholds(m)
    with np.errstate(all="ignore"):
        g = F(f("xyz_gradient_accum")[m["grad_col"]]) / F(f("denom")[0])
        g = F(0) if np.isnan(g) else g
        s = np.exp(f("scaling").astype(np.float64))
        sig = 1.0 / (1.0 + np.exp(-float(f("opacity")[0])))
    return dict(g=g, s=s, smax=s.max(), sig=sig, x=f("xyz"), q=f("rotation"), thr=thr)


def _parent_check(kind, m, p):
    thr = p["thr"]
    if kind == "g_on_threshold":
        return p["g"] == thr["g"] and p["smax"] < thr["dense"]
    if kind == "g_below_threshold":
        return p["g"] < thr["g"] and p["g"] == np.nextafter(thr["g"], F(0))
    if kind == "neg_g_on_threshold":
        return -p["g"] == thr["g"] and p["smax"] < thr["dense"]
    if kind == "split_on_threshold":
        return p["g"] == thr["g"] and p["smax"] > thr["dense"]
    if kind == "neg_g_split_side":
        return -p["g"] == thr["g"] and p["smax"] > thr["dense"]
    if kind == "smax_on_dense":
        return p["smax"] == 1.0 == thr["dense"] == thr["big"] and p["g"] >= thr["g"]
    if kind == "denom_zero_acc_zero":
        return float(m["in"]["denom"][p["l"], 0]) == 0 and p["g"] == 0
    if kind == "denom_zero_acc_pos":
        return float(m["in"]["denom"][p["l"], 0]) == 0 and p["g"] == np.inf
    if kind == "zero_quaternion":
        return not p["q"].any() and p["g"] >= thr["g"] and p["smax"] > thr["dense"]
    if kind == "exp_overflow":
        return p["s"].max() > float(np.finfo(np.float32).max) and p["g"] >= thr["g"]
    if kind == "opacity_plus_100":
        return float(m["in"]["opacity"][p["l"], 0]) == 100.0
    if kind == "opacity_minus_100":
        return float(m["in"]["opacity"][p["l"], 0]) == -100.0
    if kind == "sigmoid_near_min_opacity":
        mo = float(F(0.005))
        return abs(p["sig"] - mo) <= 24 * np.spacing(F(mo))
    if kind in ("distance_on_diameter", "distance_beyond_diameter", "distance_within_diameter"):
        d = float(np.sqrt(np.sum((p["x"] - m["sphere_center"].numpy()) ** 2)))
        d2 = float(F(2 * float(m["sphere_radius"][0])))
        rel = {"distance_on_diameter": d == d2, "distance_beyond_diameter": d > d2, "distance_within_diameter": d < d2}[kind]
        return rel and p["smax"] > thr["big"] and p["g"] == 0
    if kind in ("sample_on_face", "sample_past_face"):
        lo, hi = m["min_xyz"].numpy(), m["max_xyz"].numpy()
        on = ((p["x"] == lo) | (p["x"] == hi)).sum() == 1
        inside = bool(((p["x"] >= lo) & (p["x"] <= hi)).all())
        return F(p["s"].max()) == 0 and (on and inside if kind == "sample_on_face" else not inside)
    raise KeyError(kind)


def claim_holds(models, claim):
    kind = claim[0]
    if kind == "sizes":
        return [m["in"]["xyz"].shape[0] for m in models] == claim[1]
    if kind == "multi_segment_warp":   # some warp of the plan kernel holds rows of three or more segments
        starts = np.cumsum([0] + [m["in"]["xyz"].shape[0] for m in models])
        nonempty = [(a, b) for a, b in zip(starts[:-1], starts[1:]) if b > a]
        per_warp = {}
        for a, b in nonempty:
            for w in range(a // 32, (b - 1) // 32 + 1):
                per_warp[w] = per_warp.get(w, 0) + 1
        return max(per_warp.values()) >= 3
    if kind == "tile":
        _, k, tile, pattern = claim
        m = models[k]
        ps = []
        for l in range(256 * tile, 256 * tile + 256):
            p = _parent(m, l)
            thr = p["thr"]
            ps.append(("clone" if p["g"] >= thr["g"] and p["smax"] <= thr["dense"] else
                       "split" if p["g"] >= thr["g"] else "big" if p["smax"] > thr["big"] else "kept"))
        if pattern in ("kept", "clone", "split"):
            return all(x == pattern for x in ps)
        return ps[0] == "clone" and ps[1] == "split" and all(x == "big" for x in ps[2:])
    _, k, l, _ = claim
    p = _parent(models[k], l)
    p["l"] = l
    return bool(_parent_check(kind, models[k], p))
