"""GPU: the sky cube map composite (sky.sky_composite over csrc/sky.cu) over the whole sphere, on the views of
tests/sky_sphere_case.py, which put samples on every face, across every face side and on every cube corner.

  * Values: for every view and R of the three families, in both mask modes and with both fills, rgb_out, dL/dacc and dL/dcube within
    tests/sky_oracle.py's per-element bounds of the float64 restatement (sky64), dL/drgb == g bit for bit; the sphere family at R = 16
    also with the seeded jitter.  The coverage each family claims is asserted again on the pixels each frame samples.
  * Marks: the whole frame's backward with blocks= (R = 37, 1000, 1024: several blocks per face, the last one clipped at R = 1000)
    marks between the intersection and the union of tests/test_sky_p2p_gpu.py's _map_bounds, and every block holding a texel of
    nonzero dL/dcube is marked (an unmarked one would be gradient that CubeMapSparseAdam and the peer-memory sum drop).
  * Sparse step: frame after frame of the sphere family, CubeMapSparseAdam equals FusedAdam bit for bit on the marked blocks, which hold
    every texel of nonzero gradient, and leaves the rest untouched.
REPORT collects the largest error / bound per check."""
import pytest
import torch

import sky_oracle as SO
import sky_sphere_case as SC
import street_gaussians_b200 as sgb
from street_gaussians_b200 import sky
from street_gaussians_b200.training import CubeMapSparseAdam
from test_cube_adam_gpu import _fused_step, _texel_blocks, bits
from test_sky_gpu import check
from test_sky_p2p_gpu import _map_bounds

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
F64 = torch.float64
REPORT = {}


def _run(fr, perturb=False, blocks=None):
    rgb, acc, cube = (fr[k].clone().requires_grad_(True) for k in ("rgb", "acc", "cube"))
    out = sgb.sky_composite(rgb, acc, cube, fr["K"], fr["w2c"], sky_mask=fr["mask"], perturb=perturb, white_background=fr["fill"] == 1.0,
                            blocks=blocks)
    out.backward(fr["up"])
    return out.detach(), rgb.grad, acc.grad, cube.grad


def _values(fr, worst, seed=None):
    """One frame through the kernels against sky64; seed: with the jitter drawn from torch.manual_seed(seed)."""
    jx = jy = None
    if seed is not None:
        torch.manual_seed(seed)
    out, drgb, dacc, dcube = _run(fr, perturb=seed is not None)
    if seed is not None:
        torch.manual_seed(seed)  # graphics_utils.py:195-196, as sky_composite draws them
        H, W = fr["rgb"].shape[1:]
        jx, jy = torch.rand(H, W, device=DEV), torch.rand(H, W, device=DEV)
    r = SO.sky64(fr["rgb"], fr["acc"], fr["cube"], fr["K"], fr["w2c"], fr["up"], fr["mask"], jx, jy, fr["fill"])
    assert torch.equal(drgb, fr["up"])
    for k, got in (("out", out), ("dacc", dacc), ("dcube", dcube)):
        worst[k] = max(worst[k], check(got, r[k], r["b_" + k], k, r if k != "dcube" else None))
    return int((dcube != 0).sum())


@pytest.mark.parametrize("mode", SC.MODES)
@pytest.mark.parametrize("family,R", SC.family_cases(), ids=lambda v: str(v))
def test_values_vs_float64(family, R, mode):
    frs = SC.frames(family, R, mode, DEV)
    vs = SC.views(family, R)
    SC.assert_coverage(family, R, SC.union_coverage([SC.coverage(SC.rays64(v, DEV), R, SC.sampled(fr)) for v, fr in zip(vs, frs)]))
    worst = dict(out=0.0, dacc=0.0, dcube=0.0)
    moved = [_values(fr, worst) for fr in frs]
    assert min(moved) > 0
    REPORT[f"{family}_R{R}_{mode}"] = {k: round(x, 4) for k, x in worst.items()}
    print(family, R, mode, REPORT[f"{family}_R{R}_{mode}"])


@pytest.mark.parametrize("mode", SC.MODES)
def test_values_vs_float64_with_jitter(mode):
    R = 16
    worst = dict(out=0.0, dacc=0.0, dcube=0.0)
    for k, fr in enumerate(SC.frames("sphere", R, mode, DEV)):
        _values(fr, worst, seed=SC.seed_of("sphere", R, mode, k))
    REPORT[f"sphere_R{R}_{mode}_jitter"] = {k: round(x, 4) for k, x in worst.items()}
    print("sphere", R, mode, "jitter", REPORT[f"sphere_R{R}_{mode}_jitter"])


MARK_CASES = [("sphere", 37), ("exact", 1000), ("exact", 1024), ("rig", 1024)]


@pytest.mark.parametrize("mode", SC.MODES)
@pytest.mark.parametrize("family,R", MARK_CASES, ids=lambda v: str(v))
def test_marks_cover_every_texel_the_gradient_moves(family, R, mode):
    tb = _texel_blocks(R)
    faces = set()
    for fr in SC.frames(family, R, mode, DEV):
        blocks = sky.block_map(R, DEV)
        _, _, _, dcube = _run(fr, blocks=blocks)
        assert int(blocks.max()) == 1
        marked = set(torch.nonzero(blocks).view(-1).tolist())
        lo, hi = _map_bounds(fr, dict(jx=None, jy=None), torch.ones(fr["rgb"].shape[1], dtype=torch.bool, device=DEV))
        assert lo and lo <= marked <= hi, (len(lo - marked), len(marked - hi))
        moved = tb[dcube.ne(0).any(-1)]
        assert bool(blocks.bool()[moved].all()), sorted(set(moved.unique().tolist()) - marked)[:10]
        faces |= {b // (len(blocks) // 6) for b in marked}
    assert faces == SC.expected(family, R)[0]


def test_sparse_step_is_fused_adam_on_the_marked_blocks():
    R = 37
    vs = SC.views("sphere", R)
    cube = torch.nn.Parameter(SC.cube_of(R, 5, DEV))
    opt = CubeMapSparseAdam([cube], lr=0.01, eps=1e-15)
    blocks = sky.block_map(R, DEV)
    tb = _texel_blocks(R).unsqueeze(-1).expand(6, R, R, 3)
    for it, v in enumerate(vs):
        fr = SC.frame("sphere", v, cube, SC.MODES[it % 2], SC.seed_of("sphere", R, "acc", 50 + it), SC.fill_of(it), DEV)
        cube.grad = None
        out = sgb.sky_composite(fr["rgb"], fr["acc"], cube, fr["K"], fr["w2c"], sky_mask=fr["mask"], white_background=fr["fill"] == 1.0,
                                blocks=blocks)
        out.backward(fr["up"])
        marked = blocks.bool()[tb]
        assert bool(marked[cube.grad != 0].all()) and 0 < int(marked.sum()) < marked.numel()
        p0 = cube.detach().clone()
        st = opt.state[cube]
        m0 = st["exp_avg"].clone() if st else torch.zeros_like(p0)
        v0 = st["exp_avg_sq"].clone() if st else torch.zeros_like(p0)
        want = _fused_step(p0, cube.grad, m0, v0, it + 1, dict(lr=0.01, eps=1e-15))
        opt.step(blocks)
        torch.cuda.synchronize()
        assert opt.state[cube]["step"] == it + 1 and not bool(blocks.any())
        for name, x, w, b in zip(("param", "exp_avg", "exp_avg_sq"), (cube.detach(), opt.state[cube]["exp_avg"], opt.state[cube]["exp_avg_sq"]),
                                 want, (p0, m0, v0)):
            assert torch.equal(bits(x)[marked], bits(w)[marked]), (it, name)
            assert torch.equal(bits(x)[~marked], bits(b)[~marked]), (it, name)
