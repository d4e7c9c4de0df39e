"""Float64 restatement of densification (clone / split / prune) and of the opacity reset, with a bound on every value the fp32
kernels compute (street_gaussians_b200/csrc/densify.cu), and of the Philox normal draws the trainer's path uses.

Test-only code (the product never imports oracle/).  It follows oracle/densify_oracle.py (itself pinned bit for bit to the
reference's densify_and_prune on tests/golden/callsite/densify.npz), one parent at a time and in numpy, so that every decision
carries its fp64 margin and every output row its parent, its section and its bound.  u = 2^-24 below; each constant in a bound
is a count of roundings.

Draws.  The kernel takes the 18 normals of composed parent i from Philox4x32-10 (curand_init(seed, i, 0); five curand_normal4):
block n is Philox of counter (n, 0, i_lo, i_hi) under key (seed_lo, seed_hi), and each block's words (x, y, z, w) give
z[4n] = s(x) sin v(y), z[4n+1] = s(x) cos v(y), z[4n+2] = s(z) sin v(w), z[4n+3] = s(z) cos v(w) with
u(x) = x 2^-32 + 2^-33 and v(y) = y 2^-32 2pi + 2^-32 pi formed in fp32 (_curand_box_muller), s = sqrt(-2 ln u).  The words are
exact here (integer arithmetic, pinned to tests/golden/curand/philox.npz).  Whether nvcc contracts u and v into one FMA is not fixed,
so both roundings are evaluated and the bound covers their spread.  Then:
  * logf: <= 1 ulp (CUDA documents 1), sqrtf correctly rounded: s within 3u s;
  * __sincosf: absolute error 2^-21.41 is documented on [-pi, pi] only and v reaches 2pi: 2^-19 is taken, NOT measured
    (tests/test_densify64_gpu.py prints the largest error / bound it sees on the device);
  * the product s sin v: one rounding.
  bound = half the spread of the candidates + s (2^-19 + 8u).

Children (densify_and_split).  xyz = R (z (*) s) + x, R from the normalised quaternion, s = expf(scaling): the error budget is
that of tests/test_densify_gpu.py, 16 u (sum_k |z_k s_k| + |x|) (R's entries carry a few u absolute and |R_rk| <= 1: expf 4u,
z s 1u, R 4u, three products and three sums), plus the draws' own error sum_k dz_k s_k and 8 2^-149 for subnormal products.
Raw scaling = logf(expf(scaling) / 1.6f): the quotient carries 4u (expf) + 1u (division) + 2^-149 / s relative, logf 1 ulp:
bound = 8u + 2^-149 / s + 4u |r|.  Non-finite results (expf overflowing to inf, a zero quaternion's NaN) are exact classes.

Decisions.  g = accum / denom is one IEEE division in the kernel, so it is decided exactly here in fp32 (NaN -> 0, x/0 -> inf).
Every other decision (max scale against the dense and big thresholds, sigmoid(opacity) against min_opacity, the distance against
the sphere diameter, each box coordinate against its face) gets a margin: its distance to the threshold beyond the value's own
error bound, relative to the larger of the two.  A parent's margin is the smallest over every decision its rows depend on.
`decisions=` forces the 4-bit masks of chosen parents (the test forces the kernel's own on parents whose margin is below delta),
and the output rows are rebuilt from the masks as the apply kernel does: per section, in parent order.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -149
DRAWS = 18
SINCOS_ABS = 2.0 ** -19     # assumed bound of __sincosf on [0, 2pi]; see the module docstring
NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic")
SCALARS = ("points_total", "points_clone", "points_split", "points_below_min_opacity", "points_big_ws", "points_pruned")
_M32 = np.uint64(0xFFFFFFFF)
_F32_OVERFLOW = float(np.finfo(np.float32).max) * (1 + 2.0 ** -25)   # exp(x) rounds to +inf in fp32 at and above this
_INV = np.float32(2.3283064e-10)                    # CURAND_2POW32_INV
_INV_2PI = np.float32(_INV * np.float32(6.2831855))  # CURAND_2POW32_INV_2PI, folded in fp32


def _np(v):
    if hasattr(v, "detach"):
        v = v.detach().cpu()
        if v.dtype.is_floating_point:
            v = v.double()
        v = v.numpy()
    return np.asarray(v)


# ---- Philox4x32-10 ----
def philox_words(seed, idx, blocks=5):
    """The curand4 words of curand_init(seed, idx, 0), blocks of four: uint32 [n, blocks, 4]."""
    idx = np.asarray(idx, dtype=np.uint64).reshape(-1)
    seed = int(seed)
    out = np.empty((idx.size, blocks, 4), dtype=np.uint32)
    for n in range(blocks):
        c = [np.full(idx.size, n, np.uint64), np.zeros(idx.size, np.uint64), idx & _M32, idx >> np.uint64(32)]
        k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
        for r in range(10):
            if r:
                k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
            p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
            c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        out[:, n] = np.stack(c, axis=1).astype(np.uint32)
    return out


def _uniform_candidates(w, scale):
    """w * scale + scale / 2 in fp32, rounded after the product and the sum, and as one FMA."""
    wf = w.astype(np.float32)
    half = np.float32(scale / np.float32(2))
    two = (wf * scale).astype(np.float32) + half
    fma = (wf.astype(np.float64) * float(scale) + float(half)).astype(np.float32)
    return two.astype(np.float64), fma.astype(np.float64)


def philox_normals64(seed, idx):
    """The kernel's 18 draws of composed parents idx under seed: (z [n, 18] fp64, bound [n, 18])."""
    w = philox_words(seed, idx, 5)
    zs = []
    for a, b in ((0, 1), (2, 3)):
        us, vs = _uniform_candidates(w[:, :, a], _INV), _uniform_candidates(w[:, :, b], _INV_2PI)
        cand = []
        for uu in us:
            with np.errstate(invalid="ignore"):
                s = np.sqrt(-2.0 * np.log(uu))
            for vv in vs:
                cand.append((s * np.sin(vv), s * np.cos(vv), s))
        zs.append(cand)
    z = np.empty((w.shape[0], 5, 4))
    bound = np.empty_like(z)
    for h, cand in enumerate(zs):
        for j in range(2):
            c = np.stack([x[j] for x in cand])
            smax = np.max(np.stack([x[2] for x in cand]), axis=0)
            lo, hi = c.min(axis=0), c.max(axis=0)
            z[:, :, 2 * h + j] = 0.5 * (lo + hi)
            bound[:, :, 2 * h + j] = 0.5 * (hi - lo) + smax * (SINCOS_ABS + 8 * U)
    return z.reshape(-1, 20)[:, :DRAWS], bound.reshape(-1, 20)[:, :DRAWS]


# ---- densification ----
def _exp32(x):
    """expf's value in fp64, with fp32's overflow to +inf and underflow to 0, and its error bound (4u relative + 2^-149)."""
    with np.errstate(over="ignore"):
        e = np.exp(x)
    e = np.where(e >= _F32_OVERFLOW, np.inf, np.where(e < TINY / 2, 0.0, e))
    return e, 4 * U * e + TINY


def _quat_matrix(q, twice):
    with np.errstate(invalid="ignore", divide="ignore"):
        if twice:   # get_rotation = F.normalize(_rotation): x / max(||x||, 1e-12)
            q = q / np.maximum(np.linalg.norm(q, axis=1), 1e-12)[:, None]
        q = q / np.linalg.norm(q, axis=1)[:, None]
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], axis=1).reshape(-1, 3, 3)


def _sample(R, z, dz, s, ds, x, dx):
    """R (z (*) s) + x and its bound (module docstring)."""
    with np.errstate(invalid="ignore"):
        v = z * s
        y = np.einsum("nij,nj->ni", R, v) + x
        mag = np.abs(v).sum(axis=1, keepdims=True) + np.abs(x)
        err = 16 * U * mag + (dz * s + np.abs(z) * ds).sum(axis=1, keepdims=True) * 1.01 + dx + 8 * TINY
    return y, err


def _margin(v, e, thr):
    """Distance of v from thr beyond v's error bound e, relative to max(|v|, |thr|); NaN v has nothing to decide (+inf)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        m = (np.abs(v - thr) - e) / np.maximum(np.maximum(np.abs(v), abs(thr)), 1e-300)
    return np.where(np.isnan(v) | (np.isinf(v) & ~np.isinf(thr)), np.inf, m)


def densify64(t, kind, draws, *, grad_threshold, grad_col, extent, percent_dense, percent_big_ws, min_opacity, prune_big_points,
              sphere_center=None, sphere_radius=None, min_xyz=None, max_xyz=None, draw_bound=None, decisions=None):
    """One sub-model, with densify_oracle.densify_model's arguments (t: {name: tensor}, the statistics, "exp_avg" / "exp_avg_sq").
    draws [n, 18] (given or philox_normals64's) with draw_bound [n, 18] (None: exact).  decisions: (parents, masks) to force.

    Returns a dict: mask [n] (after forcing), natural [n] (before), margin [n], clone, split [n] bool, scalars (natural decisions),
    parent, section [rows], rows {name: fp64 [rows, ...]}, bound {"xyz", "scaling": [rows, 3]} (0 on copied rows),
    moments {name: bool [rows]} (True where the row carries its parent's moments)."""
    f32 = lambda v: float(np.float32(v))
    ext = float(_np(extent).reshape(-1)[0])
    dense_thr, big_thr = f32(np.float32(ext) * np.float32(percent_dense)), f32(np.float32(ext) * np.float32(percent_big_ws))
    g_thr, op_thr = f32(grad_threshold), f32(min_opacity)
    x, sc, q = _np(t["xyz"]), _np(t["scaling"]), _np(t["rotation"])
    o = _np(t["opacity"])[:, 0]
    n = x.shape[0]
    z = _np(draws).reshape(n, DRAWS)
    dz = np.zeros_like(z) if draw_bound is None else _np(draw_bound).reshape(n, DRAWS)
    # gradient: one fp32 division, exact
    with np.errstate(invalid="ignore", divide="ignore"):
        g = (_np(t["xyz_gradient_accum"])[:, grad_col].astype(np.float32) / _np(t["denom"])[:, 0].astype(np.float32)).astype(np.float64)
    g = np.where(np.isnan(g), 0.0, g)
    s, ds = _exp32(sc)
    smax, dsmax = s.max(axis=1), ds.max(axis=1)
    clone = (np.abs(g) >= g_thr) & (smax <= dense_thr)
    split = (g >= g_thr) & (smax > dense_thr)
    margin = np.where(np.abs(g) >= g_thr, _margin(smax, dsmax, dense_thr), np.inf)
    with np.errstate(over="ignore"):
        e_o, de_o = _exp32(-o)
        sig = 1.0 / (1.0 + e_o)
    with np.errstate(invalid="ignore"):
        dsig = np.where(np.isinf(e_o), 0.0, (8 * U + de_o / np.maximum(1.0 + e_o, 1.0)) * sig) + TINY
    below = sig < op_thr
    margin = np.minimum(margin, _margin(sig, dsig, op_thr))
    # children: xyz and raw scaling of both, from draws [0:3] and [3:6]
    R = _quat_matrix(q, False)
    xz = np.zeros_like(x)
    child_x, child_dx = [], []
    for c in range(2):
        y, e = _sample(R, z[:, 3 * c:3 * c + 3], dz[:, 3 * c:3 * c + 3], s, ds, x, xz)
        child_x.append(y)
        child_dx.append(e)
    with np.errstate(divide="ignore", invalid="ignore"):
        q16 = s / float(np.float32(1.6))
        child_raw = np.log(q16)
        child_draw = (8 * U + TINY / s) + 4 * U * np.abs(child_raw)
    child_s = q16                       # exp(log(s / 1.6)): the child's get_scaling
    child_ds = 12 * U * child_s + TINY
    # every candidate row of every parent: (slot, xyz, dxyz, scale, dscale)
    rows_of = [(0, x, xz, s, ds), (1, x, xz, s, ds), (0, child_x[0], child_dx[0], child_s, child_ds),
               (1, child_x[1], child_dx[1], child_s, child_ds)]
    survive = np.zeros((n, 4), dtype=bool)
    big_c, below_c = np.zeros((n, 4), dtype=bool), np.zeros((n, 4), dtype=bool)
    row_margin = np.full((n, 4), np.inf)
    actor = kind == "actor"
    Rb = _quat_matrix(q, True) if actor and prune_big_points else None
    for sec, (slot, xr, dxr, sr, dsr) in enumerate(rows_of):
        pruned = below.copy()
        big = np.zeros(n, dtype=bool)
        m = np.full(n, np.inf)
        if prune_big_points:
            smr = sr.max(axis=1)
            big = smr > big_thr
            m = np.minimum(m, _margin(smr, dsr.max(axis=1), big_thr))
            if not actor:
                c = _np(sphere_center).reshape(1, 3)
                d2 = float(np.float32(2 * float(_np(sphere_radius).reshape(-1)[0])))
                with np.errstate(invalid="ignore"):
                    dist = np.linalg.norm(xr - c, axis=1)
                ed = 8 * U * (dist + np.abs(c).sum()) + dxr.max(axis=1)
                m = np.minimum(m, np.where(big, _margin(dist, ed, d2), np.inf))
                big = big & ~(dist > d2)
                pruned |= big
            else:
                lo, hi = _np(min_xyz).reshape(-1), _np(max_xyz).reshape(-1)
                outside = np.zeros(n, dtype=bool)
                for j in range(2):
                    cols = slice(6 + 3 * (2 * slot + j), 9 + 3 * (2 * slot + j))
                    y, e = _sample(Rb, z[:, cols], dz[:, cols], sr, dsr, xr, dxr)
                    with np.errstate(invalid="ignore"):
                        outside |= ~((y >= lo) & (y <= hi)).all(axis=1)
                    for a in range(3):
                        m = np.minimum(m, np.minimum(_margin(y[:, a], e[:, a], lo[a]), _margin(y[:, a], e[:, a], hi[a])))
                pruned |= big | outside
        survive[:, sec] = ~pruned
        big_c[:, sec], below_c[:, sec] = big, below
        row_margin[:, sec] = m
    exists = np.stack([~split, clone, split, split], axis=1)
    natural = ((exists & survive) * (1 << np.arange(4))).sum(axis=1)
    margin = np.minimum(margin, np.where(exists | (np.abs(g) >= g_thr)[:, None], row_margin, np.inf).min(axis=1))
    scalars = dict(points_total=n, points_clone=int(clone.sum()), points_split=int(split.sum()),
                   points_below_min_opacity=int((below_c & exists).sum()), points_pruned=int((~survive & exists).sum()))
    if prune_big_points:
        scalars["points_big_ws"] = int((big_c & exists).sum())
    mask = natural.copy()
    if decisions is not None:
        fp, fm = decisions
        mask[_np(fp).astype(np.int64)] = _np(fm).astype(np.int64)
    parent = np.concatenate([np.nonzero(mask & (1 << k))[0] for k in range(4)])
    section = np.concatenate([np.full(int(((mask >> k) & 1).sum()), k) for k in range(4)])
    child = section >= 2
    cidx = np.clip(section - 2, 0, 1)
    rows = {a: _np(t[a])[parent].astype(np.float64) for a in NAMES}
    bound = {"xyz": np.zeros((parent.size, 3)), "scaling": np.zeros((parent.size, 3))}
    cx = np.stack(child_x, axis=0)[cidx, parent]
    cdx = np.stack(child_dx, axis=0)[cidx, parent]
    rows["xyz"][child], bound["xyz"][child] = cx[child], cdx[child]
    rows["scaling"][child], bound["scaling"][child] = child_raw[parent][child], child_draw[parent][child]
    return dict(mask=mask, natural=natural, margin=margin, clone=clone, split=split, g=g, scalars=scalars, parent=parent,
                section=section, rows=rows, bound=bound, carries=section == 0)


# ---- opacity reset ----
def reset_opacity64(o):
    """inverse_sigmoid(min(sigmoid(o), 0.01f)) in fp64 and its bound, and the mask of the region where sigmoid(o) is subnormal or 0
    in fp32 (o below about -87.3): there the fp32 value is decided by how expf overflows and how the division rounds, and the test
    holds the kernel to the reference's own torch expression on the same device instead (bound +inf here)."""
    o = _np(o).astype(np.float64)
    e, de = _exp32(-o)
    with np.errstate(divide="ignore"):
        sig = 1.0 / (1.0 + e)
    cap = float(np.float32(0.01))
    p = np.minimum(sig, cap)
    with np.errstate(divide="ignore"):
        r = np.log(p / (1.0 - p))
    region = sig < 2.0 ** -126
    bound = np.where(region, np.inf, 12 * U + 3 * U * np.abs(r))
    return r, bound, region
