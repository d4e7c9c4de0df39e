"""Views of the sky cube map over the whole sphere, for tests/test_sky_sphere_*.py.

The sky kernels (csrc/sky.cu) carry their own copy of the cube's geometry: the face frames kFaceN / kFaceU / kFaceV and the
integer-lattice wrap of a tap past a face edge in sky_texel.  tests/sky_oracle.py's ADJ table is a separate copy.  A sign error in one
face's frame only shows where a sample lands on that face or wraps into it, so these families put samples on every face, across every
face side and on every cube corner, and each asserts what it covers (`coverage`):
  sphere  26 look-at directions (6 face centres, 12 edge midpoints, 8 corners), a wide K (fx = fy = 0.3 W, about 118 degrees) at
          96 x 64, a different roll per view; R in SPHERE_R.  All 6 faces, 24 sides and 24 corner taps up to R = 16 (at R = 1 every
          sample has a corner tap), all 24 sides at R = 37.
  exact   rays that are exact in fp32: K = [[f, 0, cx], [0, f, cy], [0, 0, 1]] with f a power of two above R and the pixel (I0, J0)
          looking along (1, 1, 1), and w2c the 24 proper rotations of the cube.  The kernel's adjugate K^-1, Rm^T K^-1 and every ray
          are exact (`exact_rays_fp32` restates the kernel's fp32 steps), so the centre pixel sits on a cube corner with an exact
          three-way tie (the x face takes it), its row and column lie on two cube edges, and (I0 - 1, J0), (I0 - 1, J0 - 1) put corner
          taps on the other two faces of the corner (f > R).  All 24 corner taps at every R in EXACT_R.
  rig     five z-up cameras of a Waymo-like rig (front, front-left / -right at +-45 degrees, side-left / -right at +-90 degrees) with
          test_sky_gpu's K at 1920 x 1280 (1920 x 886 for the sides), R = 1024: faces +x, +y, -y and the +x / +-y edges, the
          configuration a z-up world trains in.  Its vertical half-FoV is about 17 degrees: no +-z, no -x, no corner.
`frame` gives each view seeded inputs for the two mask modes, with a sparse pattern of pixels left unsampled that keeps the coverage."""
from __future__ import annotations

import functools
import itertools
import math
from typing import Dict, List, Set, Tuple

import numpy as np
import torch

import sky_oracle as SO

F64 = torch.float64
SPHERE_HW = (64, 96)
SPHERE_R = (1, 2, 3, 5, 16, 37)
EXACT_HW = (64, 64)
EXACT_IJ = (40, 56)  # (I0, J0): column and row of the pixel looking along (1, 1, 1); J0 >= 50 so the mask mode decides it
EXACT_R = (1, 2, 3, 1000, 1024)
RIG_R = 1024
K_WAYMO = ((2055.6, 0.0, 939.7), (0.0, 2051.3, 641.1), (0.0, 0.0, 1.0))  # test_sky_gpu.K_WAYMO
RIG = (("front", 0.0, 1280), ("front_left", 45.0, 1280), ("front_right", -45.0, 1280), ("side_left", 90.0, 886),
       ("side_right", -90.0, 886))
MODES = ("acc", "sky_mask")


# ---- coverage ---------------------------------------------------------------------------------------------------------------
def coverage(d: torch.Tensor, R: int, sel=None) -> Tuple[Set[int], Set[Tuple[int, int]], Set[Tuple[int, int]]]:
    """What the samples along directions d [..., 3] (those where `sel` is set) reach on a cube of R x R faces, counting taps of
    nonzero bilinear weight: (faces sampled, (face, side) crossings, (face, corner) corner taps).  Side 0: column -1, 1: column R,
    2: row -1, 3: row R; corner (c >= R) + 2 (r >= R)."""
    face, gx, gy = SO.face_coords(d.to(F64))
    x, y = SO.tex_xy(gx, gy, R)
    idx, w = SO.taps(face, x, y, R)
    if sel is not None:
        face, x, y, idx, w = face[sel], x[sel], y[sel], idx[sel], w[sel]
    face, idx, w = face.reshape(-1), idx.reshape(-1, 4), w.reshape(-1, 4)
    x0, y0 = torch.floor(x).long().reshape(-1), torch.floor(y).long().reshape(-1)
    faces = set(torch.unique(face).tolist())
    sides, corners = set(), set()
    for k in range(4):
        c, r = x0 + (k & 1), y0 + (k >> 1)
        oc, orow = (c < 0) | (c >= R), (r < 0) | (r >= R)
        live = w[:, k] > 0
        assert bool(((idx[:, k] < 0) == (oc & orow)).all())
        side = torch.where(oc, (c >= R).long(), 2 + (r >= R).long())
        one = live & (oc ^ orow)
        sides |= set(zip(face[one].tolist(), side[one].tolist()))
        cor = live & oc & orow
        corners |= set(zip(face[cor].tolist(), ((c >= R).long() + 2 * (r >= R).long())[cor].tolist()))
    return faces, sides, corners


def union_coverage(parts):
    faces, sides, corners = set(), set(), set()
    for f, s, c in parts:
        faces |= f
        sides |= s
        corners |= c
    return faces, sides, corners


ALL_SIDES = set(itertools.product(range(6), range(4)))
ALL_CORNERS = set(itertools.product(range(6), range(4)))


# ---- views ------------------------------------------------------------------------------------------------------------------
def _w2c(right, down, forward, centre=(3.0, -2.0, 5.0)) -> torch.Tensor:
    Rc = torch.stack([right, down, forward], 1)  # camera-to-world rotation (x right, y down, z forward)
    w2c = torch.eye(4, dtype=F64)
    w2c[:3, :3] = Rc.T
    w2c[:3, 3] = -Rc.T @ torch.tensor(centre, dtype=F64)
    return w2c.float()


def look(direction, roll: float) -> torch.Tensor:
    """w2c of a camera looking along `direction`, rolled by `roll` radians about it.  The helper up axis is the world axis least
    aligned with the view, so it is never parallel to it."""
    z = torch.tensor(direction, dtype=F64)
    z = z / z.norm()
    a = torch.zeros(3, dtype=F64)
    a[int(z.abs().argmin())] = 1.0
    x0 = torch.linalg.cross(a, z)
    x0 = x0 / x0.norm()
    y0 = torch.linalg.cross(z, x0)
    x = math.cos(roll) * x0 + math.sin(roll) * y0
    y = torch.linalg.cross(z, x)
    return _w2c(x, y, z)


def sphere_directions() -> List[Tuple[float, float, float]]:
    """6 face centres, 12 edge midpoints, 8 corners."""
    dirs = []
    for n in (1, 2, 3):
        for v in itertools.product((-1.0, 0.0, 1.0), repeat=3):
            if sum(c != 0 for c in v) == n:
                dirs.append(v)
    return dirs


@functools.lru_cache(maxsize=None)
def sphere_views():
    H, W = SPHERE_HW
    f = 0.3 * W
    K = torch.tensor([[f, 0.0, W / 2], [0.0, f, H / 2], [0.0, 0.0, 1.0]])
    return [dict(name=f"sphere{k}", H=H, W=W, K=K, w2c=look(d, 0.3 + 0.7 * k)) for k, d in enumerate(sphere_directions())]


def cube_rotations() -> List[torch.Tensor]:
    """The 24 proper rotations of the cube: signed permutation matrices of determinant +1."""
    out = []
    for p in itertools.permutations(range(3)):
        for s in itertools.product((-1.0, 1.0), repeat=3):
            m = torch.zeros(3, 3, dtype=F64)
            for a in range(3):
                m[a, p[a]] = s[a]
            if float(torch.linalg.det(m)) > 0:
                out.append(m)
    assert len(out) == 24
    return out


def exact_focal(R: int) -> float:
    """The smallest power of two above R."""
    return float(2 ** (int(R).bit_length()))


@functools.lru_cache(maxsize=None)
def exact_views(R: int):
    H, W = EXACT_HW
    I0, J0 = EXACT_IJ
    f = exact_focal(R)
    K = torch.tensor([[f, 0.0, I0 + 0.5 - f], [0.0, f, J0 + 0.5 - f], [0.0, 0.0, 1.0]])
    views = []
    for k, Rm in enumerate(cube_rotations()):
        w2c = torch.eye(4)
        w2c[:3, :3] = Rm.float()
        w2c[:3, 3] = torch.tensor([0.25, -1.5, 2.0])
        views.append(dict(name=f"exact{k}", H=H, W=W, K=K, w2c=w2c))
    return views


@functools.lru_cache(maxsize=None)
def rig_views():
    K = torch.tensor(K_WAYMO)
    views = []
    for name, yaw, H in RIG:
        p = math.radians(yaw)
        fwd = torch.tensor([math.cos(p), math.sin(p), 0.0], dtype=F64)
        down = torch.tensor([0.0, 0.0, -1.0], dtype=F64)
        views.append(dict(name=name, H=H, W=1920, K=K, w2c=_w2c(torch.linalg.cross(down, fwd), down, fwd, (10.0, 4.0, 1.8))))
    return views


def views(family: str, R: int):
    return {"sphere": sphere_views, "exact": lambda: exact_views(R), "rig": rig_views}[family]()


def family_cases():
    """(family, R) of every case the value checks run."""
    return [("sphere", R) for R in SPHERE_R] + [("exact", R) for R in EXACT_R] + [("rig", RIG_R)]


def rays64(view, device=None) -> torch.Tensor:
    return SO.rays(view["H"], view["W"], view["K"].to(device, F64), view["w2c"].to(device, F64))


# ---- the exact family's fp32 steps ------------------------------------------------------------------------------------------
def exact_rays_fp32(view) -> Dict[str, np.ndarray]:
    """The kernel's fp32 steps (sky_camera, sky_pixel, sky_taps) restated in numpy float32 beside float64, for the exactness check:
    K^-1 by the adjugate and 1 / det, M = Rm^T K^-1, the ray M (i + 0.5, j + 0.5, 1), and the texel coordinates where the largest
    component is +-1."""
    f32, f64 = np.float32, np.float64
    k = view["K"].numpy().astype(f32).reshape(-1)
    r = view["w2c"].numpy().astype(f32)[:3, :3].reshape(-1)
    out = {}
    for name, t in (("32", f32), ("64", f64)):
        kk, rr = k.astype(t), r.astype(t)
        inv = np.array([kk[4] * kk[8] - kk[5] * kk[7], kk[2] * kk[7] - kk[1] * kk[8], kk[1] * kk[5] - kk[2] * kk[4],
                        kk[5] * kk[6] - kk[3] * kk[8], kk[0] * kk[8] - kk[2] * kk[6], kk[2] * kk[3] - kk[0] * kk[5],
                        kk[3] * kk[7] - kk[4] * kk[6], kk[1] * kk[6] - kk[0] * kk[7], kk[0] * kk[4] - kk[1] * kk[3]], dtype=t)
        det = kk[0] * inv[0] + kk[1] * inv[3] + kk[2] * inv[6]
        inv = (inv * (t(1) / det)).astype(t)
        m = np.array([[rr[0 * 3 + a] * inv[0 * 3 + b] + rr[1 * 3 + a] * inv[1 * 3 + b] + rr[2 * 3 + a] * inv[2 * 3 + b] for b in range(3)]
                      for a in range(3)], dtype=t)
        j, i = np.meshgrid(np.arange(view["H"]), np.arange(view["W"]), indexing="ij")
        px, py = (i.astype(t) + t(0.5)).astype(t), (j.astype(t) + t(0.5)).astype(t)
        d = np.stack([(m[a, 0] * px + m[a, 1] * py + m[a, 2]).astype(t) for a in range(3)], -1)
        out[f"kinv{name}"], out[f"m{name}"], out[f"d{name}"] = inv, m, d
    return out


def exact_texel_coords_fp32(d: np.ndarray, R: int):
    """The face of rays d [..., 3] whose largest |component| is 1 (so g = c / 1 is exact), and sky_taps' texel coordinates
    x = fl(fl(fl(g + 1) / 2) R - 0.5) and y in float32 and in float64: {"32": [x, y], "64": [x, y]}."""
    face, gx, gy = SO.face_coords(torch.from_numpy(d.astype(np.float64)))
    res = {}
    for name, t in (("32", np.float32), ("64", np.float64)):
        g = [np.asarray(v.numpy(), dtype=t) for v in (gx, gy)]
        res[name] = [((((g_ + t(1)) * t(0.5)).clip(0, 1) * t(R)) - t(0.5)).astype(t) for g_ in g]
    return face.numpy(), res


# ---- frames -----------------------------------------------------------------------------------------------------------------
def keep_pixels(family: str, view) -> List[Tuple[int, int]]:
    """(row, column) of pixels sampled in every mode: the exact family's corner pixel and its two neighbours."""
    if family != "exact":
        return []
    I0, J0 = EXACT_IJ
    return [(J0, I0), (J0, I0 - 1), (J0 - 1, I0 - 1)]


def cube_of(R: int, seed: int, device=None) -> torch.Tensor:
    """Seeded texels in [-0.2, 1.2], so the clamp acts at both ends."""
    return (-0.2 + 1.4 * torch.rand(6, R, R, 3, generator=torch.Generator().manual_seed(seed))).to(device)


def frame(family: str, view, cube: torch.Tensor, mode: str, seed: int, fill: float = 1.0, device=None):
    """Seeded inputs of one view on `cube` (generated on the CPU, so every device sees the same numbers): acc in [0, 0.95] with 30 %
    exact zeros, and 12 % of the pixels left unsampled: acc 1 or 0.9995 in the acc mode (1 - acc at or below 1e-3), unset in the given
    sky mask (rows 0-49 are sampled anyway)."""
    H, W = view["H"], view["W"]
    g = torch.Generator().manual_seed(seed)
    rgb = torch.rand(3, H, W, generator=g)
    acc = 0.95 * torch.rand(1, H, W, generator=g)
    acc = torch.where(torch.rand(1, H, W, generator=g) < 0.3, torch.zeros_like(acc), acc)
    off = torch.rand(1, H, W, generator=g) < 0.12
    for j, i in keep_pixels(family, view):
        off[0, j, i] = False
    up = torch.randn(3, H, W, generator=g)
    mask = None
    if mode == "acc":
        acc = torch.where(off, torch.where(torch.rand(1, H, W, generator=g) < 0.5, 1.0, 0.9995), acc)
    else:
        mask = ~off
    to = lambda t: t.to(device) if t is not None else None
    return dict(cube=cube, rgb=to(rgb), acc=to(acc), up=to(up), mask=to(mask), K=to(view["K"]), w2c=to(view["w2c"]), fill=fill)


def sampled(fr) -> torch.Tensor:
    return SO.sky_mask_of(fr["acc"], fr["mask"])


def fill_of(k: int) -> float:
    """White and black fills alternate over a family's views."""
    return 1.0 if k % 2 == 0 else 0.0


def seed_of(family: str, R: int, mode: str, k: int) -> int:
    return {"sphere": 1, "exact": 2, "rig": 3}[family] * 100003 + R * 101 + MODES.index(mode) * 53 + k


def frames(family: str, R: int, mode: str, device=None):
    """Every view of the family at R on one cube."""
    cube = cube_of(R, seed_of(family, R, mode, 99), device)
    return [frame(family, v, cube, mode, seed_of(family, R, mode, k), fill_of(k), device) for k, v in enumerate(views(family, R))]


# ---- what each family must cover --------------------------------------------------------------------------------------------
def expected(family: str, R: int):
    """(faces, sides, corners) the family must reach at R; None where nothing is required."""
    if family == "sphere":
        return set(range(6)), ALL_SIDES, (ALL_CORNERS if R <= 16 else None)
    if family == "exact":
        return set(range(6)), ALL_SIDES, ALL_CORNERS
    return {0, 2, 3}, {(0, 2), (0, 3), (2, 1), (3, 1)}, set()


def assert_coverage(family: str, R: int, got) -> None:
    faces, sides, corners = got
    want_f, want_s, want_c = expected(family, R)
    if family == "rig":  # the rig reaches exactly these and nothing else
        assert (faces, sides, corners) == (want_f, want_s, want_c), (faces, sides, corners)
        return
    assert faces == want_f, (family, R, faces)
    assert sides >= want_s, (family, R, sorted(want_s - sides))
    if want_c is not None:
        assert corners >= want_c, (family, R, sorted(want_c - corners))
