"""GPU: the sky's lat-long export (sky.cubemap_to_latlong / latlong_u8 / save_latlong_png over sgr_sky_cube_to_latlong) against
tests/sky_oracle.lookup in float64, evaluated at the directions the reference's cubemap_to_latlong (lib/models/sky_cubemap.py:178-191)
forms in fp32 with torch.  Cube sizes R = 16, 100 and 1024, at the (R, 2R) of SkyCubeMap.save_state_dict and at odd sizes; the poles and
the phi = +-pi seam cross every face, and the test asserts that taps past face edges and past cube corners occur.

Bound per pixel: the kernel's direction and torch's differ by at most dd = 16 u |d| + 8 pi u per component (sinf / cosf of the same fp32
angle within 2 ulp each, two products, and one ulp of linspace in the angle); through the face coordinate and the texel coordinate that is
dx (sky_oracle.sky64's propagation), and the lookup moves by at most Lx dx + Ly dy, Lx and Ly its largest slopes over the box, plus its
own rounding 8 u sum w |t|."""
import numpy as np
import pytest
import torch

import sky_oracle as SO
from street_gaussians_b200 import sky

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
U = 2.0 ** -24
F64 = torch.float64


def reference_dirs(H, W):
    """cubemap_to_latlong's reflvec, in fp32 on the GPU, as the reference forms it."""
    gy, gx = torch.meshgrid(torch.linspace(0.0 + 1.0 / H, 1.0 - 1.0 / H, H, device=DEV),
                            torch.linspace(-1.0 + 1.0 / W, 1.0 - 1.0 / W, W, device=DEV), indexing="ij")
    sintheta, costheta = torch.sin(gy * np.pi), torch.cos(gy * np.pi)
    sinphi, cosphi = torch.sin(gx * np.pi), torch.cos(gx * np.pi)
    return torch.stack((sintheta * sinphi, costheta, -sintheta * cosphi), dim=-1)


def oracle(cube, d32):
    """float64 lookup at d32, the per-pixel bound [H, W, 3], and the counts of pixels with a tap past a face edge / a cube corner."""
    R = cube.shape[1]
    c64 = cube.to(F64)
    d = d32.to(F64)
    s = SO.lookup(c64, d)
    face, gx, gy = SO.face_coords(d)
    dd = 16 * U * d.abs() + 8 * np.pi * U
    Nt = torch.tensor(SO.FACE_N, dtype=F64, device=DEV)[face].abs()
    Ut = torch.tensor(SO.FACE_U, dtype=F64, device=DEV)[face].abs()
    Vt = torch.tensor(SO.FACE_V, dtype=F64, device=DEV)[face].abs()
    ma = (d.abs() * Nt).sum(-1)
    dma, dcu, dcv = (dd * Nt).sum(-1), (dd * Ut).sum(-1), (dd * Vt).sum(-1)
    dgx = (dcu + gx.abs() * dma) / ma + 2 * U * gx.abs()
    dgy = (dcv + gy.abs() * dma) / ma + 2 * U * gy.abs()
    dx, dy = R * dgx / 2 + 3 * U * R, R * dgy / 2 + 3 * U * R
    x, y = SO.tex_xy(gx, gy, R)
    flat = c64.reshape(6 * R * R, 3)

    def slopes(xs, ys):
        idx, w = SO.taps(face, xs, ys, R)
        ie, _ = SO.effective(idx, w)
        t = flat[ie.reshape(-1)].reshape(*ie.shape, 3)
        corner = (idx < 0).unsqueeze(-1)
        t = torch.where(corner, (t * ~corner).sum(-2, keepdim=True) / 3, t)
        fx, fy = (xs - torch.floor(xs)).unsqueeze(-1), (ys - torch.floor(ys)).unsqueeze(-1)
        lx = (1 - fy) * (t[..., 1, :] - t[..., 0, :]).abs() + fy * (t[..., 3, :] - t[..., 2, :]).abs()
        ly = (1 - fx) * (t[..., 2, :] - t[..., 0, :]).abs() + fx * (t[..., 3, :] - t[..., 1, :]).abs()
        return lx, ly, idx, w, t

    lx, ly, idx0, w0, t0 = slopes(x, y)
    for sx in (-1, 1):
        for sy in (-1, 1):
            bx, by, *_ = slopes((x + sx * dx).clamp(-0.5, R - 0.5), (y + sy * dy).clamp(-0.5, R - 0.5))
            lx, ly = torch.maximum(lx, bx), torch.maximum(ly, by)
    bound = lx * dx.unsqueeze(-1) + ly * dy.unsqueeze(-1) + 8 * U * (w0.unsqueeze(-1) * t0.abs()).sum(-2) + 1e-30
    past_edge = (x < 0) | (x > R - 1) | (y < 0) | (y > R - 1)  # a tap is read from the adjacent face
    at_corner = ((idx0 < 0) & (w0 > 0)).any(-1)                # a tap past a cube corner carries weight
    return s, bound, int(past_edge.sum()), int(at_corner.sum())


def make_cube(R, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.rand((6, R, R, 3), generator=g, device=DEV) * 1.4 - 0.2).contiguous()  # some texels outside [0, 1]: the u8 clamp


CASES = [(16, None), (16, (7, 13)), (16, (64, 128)), (16, (1, 1)), (16, (2, 3)), (100, None), (100, (37, 91)), (1024, None), (1024, (333, 777))]


@pytest.mark.parametrize("R,res", CASES)
def test_latlong_against_float64_lookup(R, res):
    cube = make_cube(R, R + (0 if res is None else res[0]))
    H, W = (R, 2 * R) if res is None else res
    out = sky.cubemap_to_latlong(cube, (H, W))
    assert out.shape == (H, W, 3) and out.dtype == torch.float32 and out.device == cube.device
    s, bound, n_edge, n_corner = oracle(cube, reference_dirs(H, W))
    err = (out.to(F64) - s).abs()
    bad = err > bound
    assert not bad.any(), (int(bad.sum()), float(err.max()), float((err / bound).max()))
    if (R, res) == (16, (64, 128)):  # dense enough that the grid lands taps past edges and corners
        assert n_edge > 0 and n_corner > 0, (n_edge, n_corner)
    # the uint8 image is the reference's (clamp(0, 1) * 255).astype(uint8) of the fp32 one, formed in the same launch
    u8 = sky.latlong_u8(cube, (H, W))
    want = (out.clamp(0.0, 1.0).cpu().numpy() * 255).astype(np.uint8)
    assert u8.dtype == torch.uint8 and np.array_equal(u8.cpu().numpy(), want)


def test_latlong_default_resolution_and_png(tmp_path):
    from test_sharded_checkpoint_cpu import decode_png
    R = 100
    cube = make_cube(R, 5)
    u8 = sky.latlong_u8(cube)
    assert u8.shape == (R, 2 * R, 3)
    path = tmp_path / "sky_latlong.png"
    sky.save_latlong_png(str(path), cube)
    assert np.array_equal(decode_png(path.read_bytes()), u8.cpu().numpy())
    sky.save_latlong_png(str(path), cube, res=(9, 17))
    assert np.array_equal(decode_png(path.read_bytes()), sky.latlong_u8(cube, (9, 17)).cpu().numpy())


def test_latlong_constant_cube_is_constant():
    # every lookup weight sums to one: a constant cube gives the constant everywhere, seams and corners included
    cube = torch.full((6, 32, 32, 3), 0.25, device=DEV)
    out = sky.cubemap_to_latlong(cube, (64, 128))
    assert torch.allclose(out, torch.full_like(out, 0.25), rtol=0, atol=1e-6)
    assert (sky.latlong_u8(cube, (64, 128)) == 63).all()
