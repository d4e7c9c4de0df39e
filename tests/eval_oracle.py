"""float64 restatement of the evaluation metrics (include/sgr.h, "Evaluation metrics"; street_gaussians_b200/metrics.py), written from the
formulas of lib/utils/loss_utils.py (l1_loss, psnr, ssim) and the PNG round trip of the files metrics.py reads (written by
torchvision.utils.save_image in the visualizers):

    clamp      x -> min(max(x, 0), 1)                                   (fp32, exact)
    quantize8  x -> trunc(clamp(255 x + 0.5, 0, 255)) / 255, every step in fp32 (torchvision.utils.save_image's
               mul(255).add_(0.5).clamp_(0, 255).to(uint8), read back by to_tensor's fp32 divide)
    l1, mse    mean of |x - y| and (x - y)^2 over the masked elements    psnr = 20 log10(1 / sqrt(mse))
    ssim       mean over all elements of ((2 mu1 mu2 + C1)(2 s12 + C2)) / ((mu1^2 + mu2^2 + C1)(s11 + s22 + C2)), mu and the second
               moments 11x11 Gaussian (sigma 1.5) correlations with zero padding, s = E[xy] - mu mu; with ssim_masked both images are
               zeroed outside the mask first.

The window is the reference's fp32 1-D window (torch.Tensor of the 11 exponentials divided by their fp32 sum); its outer product is
applied exactly (separably) in fp64.  `ssim_bound` gives a first-order bound on the error of the fp32 evaluation of the SSIM mean."""
from __future__ import annotations

import numpy as np
from scipy.ndimage import correlate1d

U32 = 2.0 ** -24
C1, C2 = 0.01 ** 2, 0.03 ** 2


def window() -> np.ndarray:
    g = np.array([np.exp(-(k - 5) ** 2 / (2 * 1.5 ** 2)) for k in range(11)], dtype=np.float32)
    return (g / np.float32(np.sum(g.astype(np.float64)))).astype(np.float32)  # torch's sum rounds the exact sum once


def prepare(x: np.ndarray, clamp: bool, quantize8: bool) -> np.ndarray:
    x = np.asarray(x, dtype=np.float32)
    if clamp:
        x = np.where(np.isnan(x), x, np.clip(x, np.float32(0), np.float32(1))).astype(np.float32)
    if quantize8:
        t = (x * np.float32(255)).astype(np.float32) + np.float32(0.5)
        t = np.where(np.isnan(t), t, np.clip(t, np.float32(0), np.float32(255))).astype(np.float32)
        x = (np.trunc(t) / np.float32(255)).astype(np.float32)
    return x


def quant_boundary_values() -> np.ndarray:
    """fp32 inputs at the levels k/255 and at the rounding boundaries (k + 1/2)/255, each with its neighbours one ulp either side."""
    ks = np.arange(0, 256, dtype=np.float64)
    centres = np.concatenate([ks / 255, (ks[:-1] + 0.5) / 255]).astype(np.float32)
    v = np.concatenate([centres, np.nextafter(centres, np.float32(2)), np.nextafter(centres, np.float32(-1))])
    return np.clip(v, np.float32(0), np.float32(1)).astype(np.float32)


def _conv(a: np.ndarray) -> np.ndarray:
    w = window().astype(np.float64)
    a = correlate1d(a, w, axis=-1, mode="constant", cval=0.0)
    return correlate1d(a, w, axis=-2, mode="constant", cval=0.0)


def _moments(x: np.ndarray, y: np.ndarray):
    return _conv(x), _conv(y), _conv(x * x), _conv(y * y), _conv(x * y)


def ssim_map(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    m1, m2, e11, e22, e12 = _moments(x, y)
    a1, a2 = 2 * m1 * m2 + C1, 2 * (e12 - m1 * m2) + C2
    b1, b2 = m1 * m1 + m2 * m2 + C1, (e11 - m1 * m1) + (e22 - m2 * m2) + C2
    return a1 * a2 / (b1 * b2)


def ssim_bound(x: np.ndarray, y: np.ndarray) -> float:
    """Bound on |fp32 SSIM mean - exact SSIM mean| for inputs x, y (fp64 arrays of fp32 values, [C, H, W]).

    Each of the five window sums q = sum w v (v = x, y, x^2, y^2, x y) is two passes of 11 multiply-adds in fp32 and the product v one
    more rounding: |dq| <= e_q = 48 u conv(|v|) (u = 2^-24; 22 roundings a pass, each at most u times the running sum of |terms|, plus
    the rounding of the product).  The map's value S(m1, m2, e11, e22, e12) then moves by at most sum |dS/dq| e_q to first order, plus
    16 u |S| for the ~10 roundings of the formula itself; the factor 2 covers the second-order terms while e_q << the denominators
    (B1 >= C1, and B2 >= C2 up to e_q).  The mean adds the rounding of its sum: per 32 pixels an fp32 warp sum (5 u sum |S|), then fp64."""
    m1, m2, e11, e22, e12 = _moments(x, y)
    a1, a2 = 2 * m1 * m2 + C1, 2 * (e12 - m1 * m2) + C2
    b1, b2 = m1 * m1 + m2 * m2 + C1, (e11 - m1 * m1) + (e22 - m2 * m2) + C2
    S = a1 * a2 / (b1 * b2)
    ax, ay = np.abs(x), np.abs(y)
    e = [48 * U32 * _conv(v) for v in (ax, ay, ax * ax, ay * ay, ax * ay)]
    bb = b1 * b2
    d_m1 = np.abs((2 * m2 * a2 - 2 * m2 * a1) / bb - S * (2 * m1 / b1 - 2 * m1 / b2))
    d_m2 = np.abs((2 * m1 * a2 - 2 * m1 * a1) / bb - S * (2 * m2 / b1 - 2 * m2 / b2))
    d_e11 = d_e22 = np.abs(S / b2)
    d_e12 = np.abs(2 * a1 / bb)
    per_px = 2 * (d_m1 * e[0] + d_m2 * e[1] + d_e11 * e[2] + d_e22 * e[3] + d_e12 * e[4]) + 16 * U32 * np.abs(S)
    return float(per_px.mean() + 6 * U32 * np.abs(S).mean())


def view_metrics(img, gt, mask=None, clamp=True, quantize8=False, ssim_masked=True) -> dict:
    """{psnr, ssim, l1, n} of one view in float64 (img, gt [C, H, W]; mask [H, W] bool or None), and the SSIM bound."""
    x = prepare(img, clamp, quantize8).astype(np.float64)
    y = prepare(gt, clamp, quantize8).astype(np.float64)
    Cn, H, W = x.shape
    m = np.ones((H, W), bool) if mask is None else np.asarray(mask, bool).reshape(H, W)
    d = (x - y)[:, m]
    n = d.size
    with np.errstate(divide="ignore", invalid="ignore"):
        l1 = np.abs(d).sum() / n if n else np.nan
        mse = (d * d).sum() / n if n else np.nan
        p = 20 * np.log10(1.0 / np.sqrt(mse))
    if ssim_masked and mask is not None:
        x, y = np.where(m, x, 0.0), np.where(m, y, 0.0)
    return {"psnr": float(p), "ssim": float(ssim_map(x, y).mean()), "l1": float(l1), "n": n, "ssim_bound": ssim_bound(x, y),
            "sq_diff": float((d * d).sum()), "abs_diff": float(np.abs(d).sum())}
