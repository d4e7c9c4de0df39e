"""CPU pins of the fp64 densification tier: philox_normals64's words against curand's own (tests/golden/curand/philox.npz), densify64
against densify_oracle and the reference's fixture, the edges every builder of tests/densify64_case.py claims, and that the
restatement notices the draw and threshold mistakes it is there to catch."""
import os

import numpy as np
import pytest
import torch

import densify64_case as D
import densify_case as DC
from oracle import densify64 as D64
from oracle import densify_oracle as DO

HERE = os.path.dirname(os.path.abspath(__file__))


def test_philox_words_match_curand():
    z = np.load(os.path.join(HERE, "golden", "curand", "philox.npz"))
    for a, s in enumerate(z["seeds"]):
        assert np.array_equal(D64.philox_words(int(s), z["subsequences"]), z["words"][a]), int(s)


def test_philox_normals_layout_and_bound():
    idx = np.arange(50_000)
    zz, b = D64.philox_normals64(77, idx)
    w = D64.philox_words(77, idx)
    # z[4n] / z[4n+1] from words (x, y) of block n: s(x) sin v(y), s(x) cos v(y)
    u = w[:, 0, 0].astype(np.float32) * np.float32(2.3283064e-10) + np.float32(2.3283064e-10 / 2)
    v = w[:, 0, 1].astype(np.float32) * D64._INV_2PI + D64._INV_2PI / np.float32(2)
    s = np.sqrt(-2 * np.log(u.astype(np.float64)))
    assert np.all(np.abs(zz[:, 0] - s * np.sin(v)) <= b[:, 0]) and np.all(np.abs(zz[:, 1] - s * np.cos(v)) <= b[:, 1])
    assert abs(zz.mean()) < 0.01 and abs(zz.var() - 1) < 0.01 and (b < 2e-5).all()
    # the mistakes the GPU test must see: a neighbouring subsequence, the children's draws swapped
    z1, _ = D64.philox_normals64(77, idx + 1)
    assert (np.abs(z1 - zz) > b).mean() > 0.99
    assert (np.abs(zz[:, 0:3] - zz[:, 3:6]) > b[:, 0:3] + b[:, 3:6]).mean() > 0.99


def test_densify64_matches_oracle_and_fixture():
    models, min_op = DC.load()
    for k, m in enumerate(models):
        kw = DC.oracle_kwargs(m, min_op)
        out, scal, mask, parent, section = DO.densify_model(m["in"], m["kind"], m["draws"], **kw)
        r = D64.densify64(m["in"], m["kind"], m["draws"], **kw)
        assert r["margin"].min() > 1e-5, k   # the fixture has no near-threshold parent
        assert np.array_equal(r["mask"], mask.numpy()) and np.array_equal(r["parent"], parent.numpy())
        assert np.array_equal(r["section"], section.numpy()) and r["scalars"] == scal
        child = r["section"] >= 2
        for a in DC.NAMES:
            ref = m["out"][a].numpy()
            got = r["rows"][a]
            if a in ("xyz", "scaling"):
                assert np.array_equal(got[~child].astype(np.float32), ref[~child])
                # the reference's fp32 values (and the fp32 oracle's) inside the fp64 bound
                assert (np.abs(got[child] - ref[child]) <= r["bound"][a][child]).all(), (k, a)
                assert (np.abs(got[child] - out[a].numpy()[child]) <= r["bound"][a][child]).all(), (k, a)
            else:
                assert np.array_equal(got.astype(np.float32), ref), (k, a)
            for mk in ("exp_avg", "exp_avg_sq"):
                src = m["in"][mk][a].numpy()[r["parent"]]
                src[~r["carries"]] = 0
                assert np.array_equal(src, m["out"][mk][a].numpy()), (k, a, mk)
        # a swapped child draw moves children outside their bound
        sw = m["draws"].clone()
        sw[:, 0:3], sw[:, 3:6] = m["draws"][:, 3:6], m["draws"][:, 0:3]
        r2 = D64.densify64(m["in"], m["kind"], sw, decisions=(np.arange(len(r["mask"])), r["mask"]), **kw)
        c2 = r2["section"] >= 2
        assert (np.abs(r2["rows"]["xyz"][c2] - m["out"]["xyz"].numpy()[c2]) > r["bound"]["xyz"][c2]).any(), k


BUILDERS = {"edge_sizes": D.edge_sizes, "many_40": lambda: D.many_actors(40, 2), "many_70": lambda: D.many_actors(70, 3),
            "tiles": D.tiles, "edges_col0": lambda: D.edges(grad_col_bkgd=0), "edges_col1": lambda: D.edges(grad_col_bkgd=1),
            "edges_M1_fourier5": lambda: D.edges(M=1, S=0, C_act=5), "box_sensitive": D.box_sensitive, "readout": D.readout}


@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_builders_place_their_edges(name):
    models, claims = BUILDERS[name]()
    for c in claims:
        assert D.claim_holds(models, c), c
    if name == "many_70":
        assert len(models) == 71 and sum(m["in"]["xyz"].shape[0] == 0 for m in models) >= 3
    if name.startswith("edges"):
        kinds = {c[0] for c in claims}
        assert len(kinds) >= 17, kinds
    # the restatement decides every designed parent with a known outcome as the claim says
    min_op = 0.005
    for c in claims:
        if len(c) == 4 and c[0] != "tile" and c[3] is not None:
            _, k, l, expect = c
            m = models[k]
            r = D64.densify64(m["in"], m["kind"], m["draws"], **DC.oracle_kwargs(m, min_op))
            assert r["natural"][l] == expect, (c, r["natural"][l])


def test_restatement_notices_a_flipped_threshold_comparison():
    """A '>' for the kernel's '>=' on the gradient threshold flips exactly the parents with g on it: the builders' g-on-threshold
    parents clone under '>=' and would not under '>'."""
    models, claims = D.edges()
    on = [c for c in claims if c[0] in ("g_on_threshold", "neg_g_on_threshold")]
    assert len(on) == 4
    for _, k, l, expect in on:
        m = models[k]
        r = D64.densify64(m["in"], m["kind"], m["draws"], **DC.oracle_kwargs(m, 0.005))
        assert r["natural"][l] == expect == 3 and abs(r["g"][l]) == np.float32(m["grad_threshold"])
        nudged = dict(DC.oracle_kwargs(m, 0.005), grad_threshold=float(np.nextafter(np.float32(m["grad_threshold"]), np.float32(1))))
        assert D64.densify64(m["in"], m["kind"], m["draws"], **nudged)["natural"][l] == 1


def test_reset_opacity64_against_torch_lines():
    o = torch.linspace(-80, 80, 20001)
    r, bound, region = D64.reset_opacity64(o)
    assert not region.any()
    exp = DO.reset_opacity(o).double().numpy()
    assert (np.abs(exp - r) <= bound).all()
    r2, _, region2 = D64.reset_opacity64(torch.tensor([-87.0, -88.0, -100.0, -200.0]))
    assert list(region2) == [False, True, True, True] and np.isneginf(r2[2:]).all()
