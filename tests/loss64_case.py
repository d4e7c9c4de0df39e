"""Inputs for the fp64 tier of the sky, object-accumulation and LiDAR depth losses (tests/test_loss64_cpu.py, test_loss64_gpu.py).

Every builder returns a dict of CPU tensors plus `edge(case, r)`, which asserts, on the restatement's result r (oracle/step64.py
acc_loss64 / lidar64), the edge the case was built around: a launch geometry, a tie layout, where the k-th key sits in the radix
digits, a keep that rounds, a mask, an autograd path or a clamp edge.  The CPU suite runs every edge check; the GPU suite then
compares the kernels with the restatement on the same inputs.

LiDAR keys are placed exactly: with acc in {0.25, 0.5, 1}, acc + 1e-10f == acc, so e = depth / b == z for depth = acc z with small
integer z, and lidar = z + q / 4 gives key |q| / 4 exactly; with depth = 0, e = 0 and the key is lidar itself, bit for bit.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import step64 as S64

F32 = torch.float32
NONEMPTY = lambda N, chunk: -(-N // chunk)  # blocks that hold pixels


def _require(cond):
    assert cond


def _bits(x: int) -> float:
    return float(np.array([x], np.uint32).view(np.float32)[0])


def _shape(N):
    return (1, N[0], N[1]) if isinstance(N, tuple) else (1, 1, N)


def _quantised(N, seed, qfrac=0.8, masked=True):
    """A mix of exactly quantised keys (multiples of 1/4 up to 10, acc in {0.25, 0.5, 1}) and rasterizer-like pixels with continuous
    errors (acc ~ U(0, 1) with exact zeros, 3 % outliers), ~85 % LiDAR density and an optional 80 % mask."""
    sh = _shape(N)
    g = torch.Generator().manual_seed(seed)
    z = torch.randint(2, 80, sh, generator=g).to(F32)
    aq = torch.tensor([0.25, 0.5, 1.0])[torch.randint(0, 3, sh, generator=g)]
    q = torch.randint(-40, 41, sh, generator=g).to(F32) * 0.25
    ac = torch.rand(sh, generator=g)
    ac[torch.rand(sh, generator=g) < 0.02] = 0.0
    dc = ac * z * (1.0 + 0.01 * torch.randn(sh, generator=g))
    lc = z + 0.5 * torch.randn(sh, generator=g) + torch.where(torch.rand(sh, generator=g) < 0.03, 30.0, 0.0)
    quant = torch.rand(sh, generator=g) < qfrac
    acc = torch.where(quant, aq, ac)
    depth = torch.where(quant, aq * z, dc)
    lidar = torch.where(quant, z + q, lc.clamp_min(0.0))
    lidar[torch.rand(sh, generator=g) > 0.85] = 0.0
    mask = (torch.rand(sh, generator=g) > 0.2) if masked else None
    return dict(depth=depth, acc=acc, lidar=lidar, mask=mask)


def _lidar(name, base, keep=0.95, weight=0.3, g_out=2.5, need=("depth", "acc"), edge=None):
    return dict(name=name, keep=keep, weight=weight, g_out=g_out, need=need, edge=edge or (lambda c, r: None), **base)


def _placed(keys, N, seed):
    """Pixels whose keys are exactly `keys` (floats, placed at random positions of an N-pixel map), the rest invalid (lidar = 0).
    depth = 0 makes the key the lidar value itself; acc ~ U(0.1, 1] varies dL/ddepth = g / b."""
    g = torch.Generator().manual_seed(seed)
    sh = _shape(N)
    n = len(keys)
    pos = torch.randperm(int(np.prod(sh)), generator=g)[:n]
    lidar = torch.zeros(sh).reshape(-1)
    lidar[pos] = torch.from_numpy(np.asarray(keys, np.float32))
    acc = (0.1 + 0.9 * torch.rand(sh, generator=g)).reshape(-1)
    depth = torch.zeros_like(acc)
    return dict(depth=depth.reshape(sh), acc=acc.reshape(sh), lidar=lidar.reshape(sh), mask=None)


def _keep_for(k, n):
    """A keep with int(keep n) == k."""
    keep = (k + 0.5) / n
    assert int(keep * n) == k
    return keep


def _geometry_edge(N, blocks, chunk, empty):
    def edge(c, r):
        n = int(np.prod(_shape(N)))
        assert S64.lidar_grid(n) == (blocks, chunk), S64.lidar_grid(n)
        assert blocks - NONEMPTY(n, chunk) == empty
        assert r["k"] >= 1
        if n > 10_000:
            assert r["ties"] > 1 and r["take"] >= 1
    return edge


def lidar_cases():
    cs = []
    # ---- launch geometry: lidar_grid(N) = (min(ceil(N / 256), 528), ceil(tiles / blocks) 256)
    for N, blocks, chunk, empty, keep in ((1, 1, 256, 0, 1.0), (255, 1, 256, 0, 0.95), (256, 1, 256, 0, 0.95), (257, 2, 256, 0, 0.95),
                                          (135168, 528, 256, 0, 0.95), (135169, 528, 512, 263, 0.95), ((1280, 1920), 528, 4864, 22, 0.95),
                                          ((1279, 1921), 528, 4864, 22, 0.95)):
        base = _quantised(N, seed=int(np.prod(_shape(N))) % 9973, masked=N != 256)
        if N == 1:
            base["lidar"][:] = 7.0
        cs.append(_lidar(f"grid_{N if isinstance(N, int) else '%dx%d' % N}", base, keep=keep, edge=_geometry_edge(N, blocks, chunk, empty)))

    # ---- ties at 1280x1920: 93 % of the keys below t, 4 % at t, 3 % above; keep 0.95 cuts the tie class near its middle
    def ties(H, W, seed):
        g = torch.Generator().manual_seed(seed)
        sh = (1, H, W)
        z = torch.randint(2, 80, sh, generator=g).to(F32)
        acc = torch.tensor([0.25, 0.5, 1.0])[torch.randint(0, 3, sh, generator=g)]
        u = torch.rand(sh, generator=g)
        below = torch.randint(-23, 24, sh, generator=g).to(F32) * 0.25  # |q| <= 5.75
        above = torch.randint(25, 41, sh, generator=g).to(F32) * 0.25 * torch.where(torch.rand(sh, generator=g) < 0.5, -1.0, 1.0)
        q = torch.where(u < 0.93, below, torch.where(u < 0.97, torch.where(torch.rand(sh, generator=g) < 0.5, -6.0, 6.0), above))
        lidar = z + q
        mask = torch.rand(sh, generator=g) > 0.1
        return dict(depth=acc * z, acc=acc, lidar=lidar, mask=mask)

    def tie_edge(c, r):
        n = r["key"].size
        blocks, chunk = S64.lidar_grid(n)
        tie = r["valid"] & (r["key"] == r["t"])
        assert S64._f32(torch.tensor([6.0])).view(np.uint32)[0] == r["t"] and r["ties"] > 50_000
        assert 0.2 * r["ties"] < r["take"] < 0.8 * r["ties"], (r["take"], r["ties"])
        nb = NONEMPTY(n, chunk)
        per_block = np.add.reduceat(tie.astype(np.int64), np.arange(0, n, chunk))
        assert (per_block[:nb] > 0).all()
        tiles = np.add.reduceat(tie.astype(np.int64), np.arange(0, n, 256)) > 0
        tiles_per_block = np.add.reduceat(tiles.astype(np.int64), np.arange(0, tiles.size, chunk // 256))
        assert (tiles_per_block[:nb] >= 2).all()
        taken = np.nonzero(tie & r["sel"])[0]
        last_block = int(taken[-1]) // chunk
        assert last_block > 100 and int(np.nonzero(tie)[0][-1]) // chunk > last_block  # the cut lies deep inside the grid
        assert np.array_equal(taken, np.nonzero(tie)[0][:r["take"]])

    cs.append(_lidar("ties_1280x1920", ties(1280, 1920, 21), edge=tie_edge))
    cs.append(_lidar("ties_1279x1921", ties(1279, 1921, 22), weight=-0.7, g_out=0.75, edge=tie_edge))

    # ---- radix edges: where the k-th key t sits in the digits 31..21, 20..10, 9..0
    rng = np.random.default_rng(5)

    def floats_in(lo_bits, hi_bits, n):
        return [_bits(int(b)) for b in rng.integers(lo_bits, hi_bits + 1, n)]

    def radix(name, t_bits, below, above, n_ties=1, take=1, check=None):
        keys = below + [_bits(t_bits)] * n_ties + above
        base = _placed(keys, 6000, seed=t_bits % 10007)
        n = len(keys)
        k = len(below) + take

        def edge(c, r):
            assert r["t"] == t_bits and r["n"] == n and r["k"] == k and r["take"] == take and r["ties"] == n_ties
            if check:
                check(r)
        return _lidar(name, base, keep=_keep_for(k, n), edge=edge)

    B = 0x3F800000  # 1.0: the first key of level-0 bin 0x1FC ([1, 2))
    cs.append(radix("radix_l0_first", B, floats_in(0x3F000000, B - 1, 900) + floats_in(0x3E000000, 0x3EFFFFFF, 300),
                    floats_in(B + 1, B + 0x1FFFFF, 400) + floats_in(0x40000000, 0x40FFFFFF, 200), n_ties=3, take=2,
                    check=lambda r: (r["t"] & 0x1FFFFF) == 0))
    cs.append(radix("radix_l0_last", B | 0x1FFFFF, floats_in(B, (B | 0x1FFFFF) - 1, 900), floats_in(0x40000000, 0x40FFFFFF, 300),
                    n_ties=4, take=4, check=lambda r: (r["t"] & 0x1FFFFF) == 0x1FFFFF))
    T = 0x3FC5A400  # low 10 bits 0, level-1 digit 0x169
    cs.append(radix("radix_l1_first", T, floats_in(0x3FC00000, T - 1, 700), floats_in(T + 1, T + 0x3FF, 300) + floats_in(T + 0x400, 0x3FFFFFFF, 300),
                    n_ties=2, take=1, check=lambda r: (r["t"] & 0x3FF) == 0 and (r["t"] & 0x1FFC00) != 0))
    cs.append(radix("radix_l1_last", T | 0x3FF, floats_in(T, (T | 0x3FF) - 1, 700) + floats_in(0x3FC00000, T - 1, 300),
                    floats_in(T + 0x400, 0x3FFFFFFF, 300), n_ties=5, take=3, check=lambda r: (r["t"] & 0x3FF) == 0x3FF))

    def rank1(r):  # t is the smallest key of its level-0 bin: the level-0 select leaves rank 1
        keys = r["key"][r["valid"]]
        inbin = keys[(keys >> 21) == (r["t"] >> 21)]
        assert inbin.min() == r["t"] and (inbin > r["t"]).sum() > 100 and r["lt"] == int(((keys >> 21) < (r["t"] >> 21)).sum())

    def fullcount(r):  # t is the largest key of its level-0 bin: the rank equals the bin's full count
        keys = r["key"][r["valid"]]
        inbin = keys[(keys >> 21) == (r["t"] >> 21)]
        assert inbin.max() == r["t"] and inbin.size > 100 and r["lt"] + r["take"] == int(((keys >> 21) <= (r["t"] >> 21)).sum())

    T1 = 0x3FA12345
    cs.append(radix("radix_rank1", T1, floats_in(0x3E800000, 0x3F9FFFFF, 800), floats_in(T1 + 1, 0x3FBFFFFF, 400) + floats_in(0x40000000, 0x407FFFFF, 100),
                    check=rank1))
    cs.append(radix("radix_fullcount", T1, floats_in(0x3FA00000, T1 - 1, 800) + floats_in(0x3E800000, 0x3F9FFFFF, 200),
                    floats_in(0x3FC00000, 0x407FFFFF, 300), check=fullcount))
    cs.append(radix("radix_subnormal", 0x00012345, floats_in(1, 0x00012344, 500), floats_in(0x00012346, 0x007FFFFF, 200) + floats_in(0x00800000, 0x3F800000, 200),
                    n_ties=3, take=2, check=lambda r: 0 < r["t"] < 0x00800000))

    # t == 0: e == lidar exactly (acc = 1 makes acc + 1e-10f == 1); sign(0) = 0 leaves those selected pixels without gradient
    def zero_case():
        b = _quantised(4000, seed=8, masked=False)
        z = torch.randint(2, 80, b["depth"].shape, generator=torch.Generator().manual_seed(9)).to(F32)
        pick = torch.rand(b["depth"].shape, generator=torch.Generator().manual_seed(10)) < 0.5
        b["acc"] = torch.where(pick, torch.ones_like(z), b["acc"])
        b["depth"] = torch.where(pick, z, b["depth"])
        b["lidar"] = torch.where(pick, z, b["lidar"])
        return b

    def zero_edge(c, r):
        assert r["t"] == 0 and r["lt"] == 0 and 0 < r["take"] < r["ties"]
        assert not (r["gd"][r["sel"]] != 0).any()
    cs.append(_lidar("radix_zero", zero_case(), keep=0.3, edge=zero_edge))

    # t == +inf, from lidar = +inf (df = -inf) and from acc = -1e-10f (b == 0, e = depth / 0); NaN keys order above +inf
    def inf_case(seed, via):
        b = _quantised(3000, seed=seed, masked=False)
        sh = b["depth"].shape
        pick = torch.rand(sh, generator=torch.Generator().manual_seed(seed + 1)) < 0.2
        if via == "lidar":
            b["lidar"] = torch.where(pick, torch.full(sh, float("inf")), b["lidar"])
            b["depth"] = torch.where(pick, 5.0 * b["acc"], b["depth"])
        else:
            b["acc"] = torch.where(pick, torch.full(sh, -1e-10), b["acc"])
            b["depth"] = torch.where(pick, 3.0, b["depth"])
            b["lidar"] = torch.where(pick, 4.0, b["lidar"])
        nanp = torch.rand(sh, generator=torch.Generator().manual_seed(seed + 2)) < 0.05
        b["depth"] = torch.where(nanp & ~pick, float("nan"), b["depth"])
        b["lidar"] = torch.where(nanp & ~pick, 10.0, b["lidar"])
        return b

    def inf_edge(via):
        def edge(c, r):
            assert r["t"] == 0x7F800000 and 0 < r["take"] < r["ties"]
            nan = r["valid"] & (r["key"] == S64.NAN_KEY)
            assert nan.sum() > 10 and not (nan & r["sel"]).any()
            if via == "acc":
                tie = r["valid"] & (r["key"] == r["t"])
                assert (S64._f32(c["acc"]) + np.float32(1e-10) == 0)[tie].all() and np.isinf(r["gd"][tie & r["sel"]]).all()
        return edge
    cs.append(_lidar("radix_inf_lidar", inf_case(30, "lidar"), keep=0.85, edge=inf_edge("lidar")))
    cs.append(_lidar("radix_inf_acc", inf_case(40, "acc"), keep=0.85, edge=inf_edge("acc")))

    # t == NaN with keep = 1: the value is NaN; NaN pixels get a zero dL/ddepth (dL/dacc is -0 * NaN, NaN as in torch's div backward)
    def nan_case():
        b = _quantised(3000, seed=50, masked=True)
        sh = b["depth"].shape
        p = torch.rand(sh, generator=torch.Generator().manual_seed(51))
        b["depth"] = torch.where(p < 0.03, float("nan"), b["depth"])
        b["lidar"] = torch.where(p < 0.03, 9.0, b["lidar"])
        two = (p >= 0.03) & (p < 0.05)  # e = inf - inf
        b["depth"] = torch.where(two, float("inf"), b["depth"])
        b["acc"] = torch.where(two, 1.0, b["acc"])
        b["lidar"] = torch.where(two, float("inf"), b["lidar"])
        return b

    def nan_edge(c, r):
        nan = r["valid"] & (r["key"] == S64.NAN_KEY)
        assert r["t"] == S64.NAN_KEY and np.isnan(r["value"]) and nan.sum() > 50 and r["k"] == r["n"]
        assert (r["gd"][nan] == 0).all() and np.isnan(r["ga"][nan]).all()
    cs.append(_lidar("radix_nan_keep1", nan_case(), keep=1.0, edge=nan_edge))

    # ---- keep
    def k_edge(kk):
        def edge(c, r):
            assert r["k"] == kk(r), (r["k"], kk(r))
        return edge
    cs.append(_lidar("keep_1", _quantised(5000, 60), keep=1.0, edge=k_edge(lambda r: r["n"])))
    b = _quantised(5000, 61)
    nv = int(((b["lidar"] > 0) & b["mask"]).sum())
    cs.append(_lidar("keep_k1", b, keep=1.5 / nv, edge=k_edge(lambda r: 1)))

    def exact_n(keep, num, den, below):
        """An n with keep n == num n / den mathematically, whose double product is exactly that integer or just below it."""
        for n in range(2000, 2000 + 200 * den, den):
            p = keep * n
            if (p < n * num // den) == below and (below or p == n * num // den):
                return n
        raise AssertionError("no such n")

    for tag, keep, num, den, below in (("exact", 0.95, 19, 20, False), ("below", 0.29, 29, 100, True)):
        n = exact_n(keep, num, den, below)
        keys = [float(x) for x in np.random.default_rng(n).integers(1, 40, n) * 0.25]
        base = _placed(keys, 3 * n, seed=n)

        def edge(c, r, n=n, keep=keep, num=num, den=den, below=below):
            assert r["n"] == n and r["k"] == int(keep * n) == n * num // den - (1 if below else 0)
            assert r["ties"] > 1
        cs.append(_lidar(f"keep_{tag}_{keep}_{n}", base, keep=keep, edge=edge))

    # ---- masks and validity
    cs.append(_lidar("mask_none", _quantised(20000, 70, masked=False), edge=lambda c, r: _require(c["mask"] is None)))
    b = _quantised(20000, 71)
    b["mask"][:] = False
    cs.append(_lidar("mask_all_false", b, edge=lambda c, r: _require(r["n"] == 0 and r["k"] == 0 and np.isnan(r["value"]))))

    def invalid_case():
        b = _quantised(20000, 72)
        sh = b["depth"].shape
        p = torch.rand(sh, generator=torch.Generator().manual_seed(73))
        # e == 0 (depth = 0): were these pixels counted, their keys |lidar| would be among the smallest
        for lo, hi, val in ((0.0, 0.02, -0.25), (0.02, 0.04, -0.0), (0.04, 0.06, float("nan")), (0.06, 0.08, 0.0), (0.08, 0.09, -1e-30)):
            sel = (p >= lo) & (p < hi)
            b["lidar"] = torch.where(sel, torch.full(sh, val), b["lidar"])
            b["depth"] = torch.where(sel, 0.0, b["depth"])
            b["mask"] = b["mask"] | sel
        return b

    def invalid_edge(c, r):
        l = S64._f32(c["lidar"])
        assert (np.signbit(l) & (l == 0)).sum() > 100 and np.isnan(l).sum() > 100 and (l < 0).sum() > 100
        assert not (r["valid"] & ~(l > 0)).any()
    cs.append(_lidar("mask_invalid_lidar", invalid_case(), edge=invalid_edge))

    # ---- autograd paths (the rest run with weight 0.3 and g_out 2.5, both leaves requiring grad)
    cs.append(_lidar("grad_depth_only", _quantised(30000, 80), need=("depth",), weight=1.0, g_out=1.0))
    cs.append(_lidar("grad_acc_only", _quantised(30000, 81), need=("acc",), weight=2.0, g_out=-3.0))
    cs.append(_lidar("grad_none", _quantised((1280, 1920), 82), need=()))
    return cs


# ----------------------------------------------------------------------------------------------- sky / object accumulation losses
LO, HI = S64.ACC_LO, S64.ACC_HI
NEXT_BELOW_LO = float(np.nextafter(np.float32(LO), np.float32(0)))
NEXT_ABOVE_HI = float(np.nextafter(np.float32(HI), np.float32(2)))
EDGE_VALUES = [LO, HI, NEXT_BELOW_LO, NEXT_ABOVE_HI, 0.0, 1.0, float("inf"), float("-inf"), 0.5, float(np.nextafter(np.float32(0.5), np.float32(0))),
               float(np.nextafter(np.float32(0.5), np.float32(1))), 0.4999, 0.5001, 2 * LO, float(np.float32(HI) - np.float32(2 ** -24))]


def _acc(N, seed):
    g = torch.Generator().manual_seed(seed)
    sh = _shape(N)
    acc = torch.rand(sh, generator=g) ** 2
    near1 = torch.rand(sh, generator=g) < 0.01  # 1 - acc down to the clamp
    acc = torch.where(near1, 1.0 - 1e-5 * torch.rand(sh, generator=g), acc)
    flag = torch.rand(sh, generator=g) > 0.5
    return acc, flag


def _acc_case(name, acc, flag, weight=0.1, g_out=3.0, edge=None):
    return dict(name=name, acc=acc, flag=flag, weight=weight, g_out=g_out, edge=edge or (lambda c, r: None))


def acc_cases():
    cs = []
    for N, m in ((270335, 1), (270336, 1), (270337, 2), ((1280, 1920), 10)):
        acc, flag = _acc(N, seed=int(np.prod(_shape(N))) % 7919)

        def edge(c, r, m=m):
            assert r["blocks"] == 1056 and r["terms_per_thread"] == m
        cs.append(_acc_case(f"grid_{N if isinstance(N, int) else '%dx%d' % N}", acc, flag, edge=edge))
    # the clamp edges (gradient on at 1e-6f and 1 - 1e-6f, off one ulp outside), 0, 1, +-inf and the entropy cancellation near 0.5,
    # repeated over a 3000-pixel map with both flags
    vals = torch.tensor(EDGE_VALUES * 100)
    near = 0.5 + (torch.rand(3000, generator=torch.Generator().manual_seed(3)) - 0.5) * 1e-3
    acc = torch.cat([vals, near]).reshape(1, 1, -1)
    flag = (torch.arange(acc.numel()) % 3 == 0).reshape(acc.shape)

    def clamp_edge(c, r):
        a = S64._f32(c["acc"])
        inside = r["inside"].cpu().numpy()
        assert inside[a == LO].all() and inside[a == HI].all() and a[a == LO].size and a[a == HI].size
        assert not inside[a == NEXT_BELOW_LO].any() and not inside[a == NEXT_ABOVE_HI].any() and (a == NEXT_ABOVE_HI).any()
        assert not inside[np.isinf(a) | (a == 0) | (a == 1)].any() and np.isinf(a).sum() == 200
        assert (np.abs(a - 0.5) < 1e-3).sum() > 3000 and np.isfinite(r["value"])
    cs.append(_acc_case("clamp_edges", acc, flag, edge=clamp_edge))
    for on in (True, False):
        acc, _ = _acc(40000, seed=11 + on)
        cs.append(_acc_case(f"flags_all_{'on' if on else 'off'}", acc, torch.full(acc.shape, on), weight=1.5, g_out=-0.5,
                            edge=lambda c, r, on=on: _require(bool((c["flag"] == on).all()))))
    acc, flag = _acc(50000, seed=13)
    acc.reshape(-1)[::997] = float("nan")

    def nan_edge(c, r):
        assert np.isnan(r["value"]) and (r["grad"][torch.isnan(c["acc"].reshape(-1))] == 0).all()
    cs.append(_acc_case("nan", acc, flag, edge=nan_edge))
    return cs
