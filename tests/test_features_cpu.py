"""CPU: the float64 restatement of the feature operations (tests/feature_oracle.py) against the reference's own outputs and gradients
(tests/golden/callsite/features.npz), the header's declarations of the new C entries against their ctypes prototypes, and the argument
checks of street_gaussians_b200.features and of the C entries that run before anything touches CUDA."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import feature_oracle as FO
import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi

F64 = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "callsite", "features.npz")
MODES = ("logits", "probabilities")
ENTRIES = ("sgr_gaussian_normals_forward", "sgr_gaussian_normals_backward", "sgr_compose_semantics_forward", "sgr_compose_semantics_backward",
           "sgr_finish_features_forward", "sgr_finish_features_backward")


def fixture():
    z = np.load(FIX)
    return {k: torch.from_numpy(z[k]) for k in z.files}


def close(a, b, tol):
    a, b = a.to(F64), b.to(F64)
    return float((a - b).abs().max()) <= tol * (float(b.abs().max()) + 1e-30)


def semantic_inputs(z):
    n_act = len(z["labels"])
    return z["semantic_0"], [z[f"semantic_{k + 1}"] for k in range(n_act)], [int(v) for v in z["labels"]]


@pytest.mark.parametrize("mode", MODES)
def test_semantics_restatement_reproduces_reference(mode):
    z = fixture()
    bg, actors, labels = semantic_inputs(z)
    (out,), gs = FO.grads(lambda b, *a: FO.semantics64(b, a, labels, mode), [bg] + actors, [z[f"sem_{mode}_g"]])
    assert close(out, z[f"sem_{mode}_out"], 2e-7)
    for k, g in enumerate(gs):
        assert close(g, z[f"sem_{mode}_grad_{k}"], 2e-6), k
    # the actors' rows are zero except their class column
    n_bg = bg.shape[0]
    ref = z[f"sem_{mode}_out"]
    for a, lab in enumerate(labels):
        rows = ref[n_bg + a * actors[0].shape[0]: n_bg + (a + 1) * actors[0].shape[0]]
        assert bool((rows[:, [c for c in range(ref.shape[1]) if c != lab]] == 0).all()) and bool((rows[:, lab] != 0).all())


def test_normals_restatement_reproduces_reference():
    z = fixture()
    xyz, sc, c = z["bg_xyz"], z["bg_scaling"], z["camera_center"]

    def fn(rot):
        return FO.normals64(xyz.to(F64), torch.nn.functional.normalize(rot), torch.exp(sc.to(F64)), c.to(F64))["n"]

    (n,), (g,) = FO.grads(fn, [z["bg_rotation"]], [z["normals_g"]])
    assert close(n, z["normals_out"], 1e-6)
    assert close(g, z["normals_grad_rotation"], 1e-5)
    r = FO.normals64(xyz.to(F64), torch.nn.functional.normalize(z["bg_rotation"].to(F64)), torch.exp(sc.to(F64)), c.to(F64))
    assert 0 < int(r["flip"].sum()) < len(r["flip"]) and len(set(r["col"].tolist())) == 3  # both signs, every column


@pytest.mark.parametrize("mode", MODES)
def test_finishing_restatement_reproduces_render_kernel(mode):
    z = fixture()
    feat = z[f"rk_{mode}_feature"]
    (n, s), (g,) = FO.grads(lambda x: FO.finish64(x, 3, mode), [feat], [z[f"rk_{mode}_gn"], z[f"rk_{mode}_gs"]])
    assert close(n, z[f"rk_{mode}_normals"], 1e-6)
    assert close(s, z[f"rk_{mode}_semantic"], 1e-6)
    assert close(g, z[f"rk_{mode}_g_feature"], 1e-5)
    if mode == "logits":
        assert torch.equal(z[f"rk_{mode}_semantic"], feat[3:])


def _declarations():
    text = open(os.path.join(ROOT, "include", "sgr.h")).read()
    out = {}
    for name in ENTRIES:
        m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
        assert m, name
        out[name] = [p.strip() for p in m.group(1).replace("\n", " ").split(",")]
    return out


def test_header_declarations_match_ctypes_prototypes():
    L = _capi.lib()
    for name, params in _declarations().items():
        assert name in _capi.SYMBOLS
        fn = getattr(L, name)
        assert fn.restype is C.c_int, name
        assert len(fn.argtypes) == len(params), (name, len(fn.argtypes), len(params))
        for p, t in zip(params, fn.argtypes):
            if "*" in p:
                assert t is C.c_void_p or issubclass(t, C._Pointer), (name, p, t)
            else:
                assert p.startswith("int32_t") and t is C.c_int32, (name, p, t)
    assert (_capi.SEMANTIC_LOGITS, _capi.SEMANTIC_PROBABILITIES) == (0, 1)
    text = open(os.path.join(ROOT, "include", "sgr.h")).read()
    assert "#define SGR_SEMANTIC_LOGITS 0" in text and "#define SGR_SEMANTIC_PROBABILITIES 1" in text
    assert L.sgr_abi_version() == 7


def test_c_entries_validate_before_touching_cuda():
    L = _capi.lib()
    p = C.c_void_p(16)
    err = lambda: L.sgr_last_error().decode()
    i32 = lambda *v: (C.c_int32 * max(len(v), 1))(*v)
    ptrs = lambda n: (C.c_void_p * n)(*([16] * n))
    assert L.sgr_gaussian_normals_forward(-1, p, p, p, p, p, p, None) == -1 and "bad size" in err()
    assert L.sgr_gaussian_normals_forward(0, None, None, None, None, None, None, None) == 0
    assert L.sgr_gaussian_normals_forward(4, p, p, None, p, p, p, None) == -1 and "NULL" in err()
    assert L.sgr_gaussian_normals_forward(4, p, C.c_void_p(20), p, p, p, p, None) == -1 and "aligned" in err()
    assert L.sgr_gaussian_normals_backward(4, p, None, p, p, None) == -1 and "NULL" in err()
    fwd = lambda K, mode, counts, labels, n_bg=5: L.sgr_compose_semantics_forward(K, mode, n_bg, p, len(counts), i32(*counts), i32(*labels),
                                                                                ptrs(max(len(counts), 1)), p, None)
    assert fwd(0, 0, [], []) == -1 and "at least one class" in err()
    assert fwd(4, 2, [], []) == -1 and "unknown semantic mode" in err()
    assert fwd(4, 0, [3, 2], [1, 4]) == -1 and "class label 4 of actor 1 is outside [0, 4)" in err()
    assert fwd(4, 1, [3], [-1]) == -1 and "class label -1" in err()
    assert fwd(4, 0, [-2], [0]) == -1 and "has -2 rows" in err()
    assert fwd(4, 0, [], [], n_bg=-1) == -1 and "bad sizes" in err()
    assert fwd(4, 0, [0], [0], n_bg=0) == 0  # nothing to compose
    assert L.sgr_compose_semantics_backward(3, 0, 5, 1, i32(2), i32(3), p, p, p, None, None) == -1 and "outside [0, 3)" in err()
    assert L.sgr_compose_semantics_backward(3, 0, 5, 0, None, None, p, None, p, None, None) == -1 and "NULL" in err()
    ff = lambda S, H, W, nc, mode, n=p, s=p: L.sgr_finish_features_forward(S, H, W, nc, mode, p, n, s, None)
    assert ff(0, 4, 4, 0, 0) == -1 and "bad sizes" in err()
    assert ff(3, 0, 4, 3, 0) == -1 and "bad sizes" in err()
    assert ff(5, 4, 4, 2, 0) == -1 and "must be 0 or 3" in err()
    assert ff(2, 4, 4, 3, 0) == -1 and "3 normal channels but S = 2" in err()
    assert ff(5, 4, 4, 3, 7) == -1 and "unknown semantic mode" in err()
    assert ff(5, 4, 4, 3, 0, s=None) == -1 and "NULL" in err()
    assert L.sgr_finish_features_backward(5, 4, 4, 3, 0, p, None, None, None, None) == -1 and "NULL" in err()


def test_wrappers_reject_bad_arguments_without_cuda():
    P = 6
    m, r, s, c = torch.rand(P, 3), torch.rand(P, 4), torch.rand(P, 3), torch.rand(3)
    with pytest.raises(_capi.SgrError, match="no CPU fallback"):
        sgb.gaussian_normals(m, r, s, c)
    with pytest.raises(ValueError, match=r"means3D must be \[P, 3\]"):
        sgb.gaussian_normals(torch.rand(P, 4), r, s, c)
    with pytest.raises(ValueError, match=r"rotations must be \[6, 4\]"):
        sgb.gaussian_normals(m, torch.rand(P, 3), s, c)
    with pytest.raises(ValueError, match="camera_center"):
        sgb.gaussian_normals(m, r, s, torch.rand(4))
    with pytest.raises(ValueError, match="float32"):
        sgb.gaussian_normals(m.double(), r, s, c)
    bg = dict(semantic=torch.rand(5, 4))
    act = dict(semantic=torch.rand(3, 1))
    with pytest.raises(_capi.SgrError, match="no CPU fallback"):
        sgb.compose_semantics([bg, act], [2])
    with pytest.raises(ValueError, match="semantic mode"):
        sgb.compose_semantics([bg, act], [2], mode="softmax")
    with pytest.raises(ValueError, match="class label 4 of actor 0 is outside"):
        sgb.compose_semantics([bg, act], [4])
    with pytest.raises(ValueError, match="1 actors but 0 class labels"):
        sgb.compose_semantics([bg, act], [])
    with pytest.raises(ValueError, match=r"actor 0's _semantic must be \[n, 1\]"):
        sgb.compose_semantics([bg, dict(semantic=torch.rand(3, 4))], [1])
    with pytest.raises(ValueError, match="K >= 1"):
        sgb.compose_semantics([dict(semantic=torch.rand(5, 0))], [])
    with pytest.raises(_capi.SgrError, match="no CPU fallback"):
        sgb.finish_features(torch.rand(5, 4, 4), 3, "logits")
    with pytest.raises(ValueError, match="normal_channels"):
        sgb.finish_features(torch.rand(5, 4, 4), 2, "logits")
    with pytest.raises(ValueError, match=r"\[S, H, W\]"):
        sgb.finish_features(torch.rand(2, 4, 4), 3, "logits")
    with pytest.raises(ValueError, match="semantic mode"):
        sgb.finish_features(torch.rand(5, 4, 4), 3, "log")
