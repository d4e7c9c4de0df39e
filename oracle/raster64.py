"""float64 torch restatement of the reference rasterizer — TEST INFRASTRUCTURE, not product code (nothing under
street_gaussians_b200/ may import it).  Runs on the CPU or on a CUDA device.  Restates, citing
/root/reference/submodules/diff-gaussian-rasterization/cuda_rasterizer (DGR below):

  auxiliary.h:22-39      SH_C0..SH_C3 (fp32 constants)
  auxiliary.h:41-56      ndc2Pix, getRect (the tile rectangle: fp32 arithmetic, (int) truncation toward zero, clamp)
  auxiliary.h:139-160    in_frustum (near plane 0.2, no lateral cull)
  forward.cu:20-71       computeColorFromSH (+0.5, clamp at 0, clamp bits)
  forward.cu:74-113      computeCov2D (EWA, Jacobian clamp at 1.3 tan(fov), 0.3 dilation)
  forward.cu:118-152     computeCov3D (quaternion NOT normalised, scale_modifier)
  forward.cu:156-256     preprocessCUDA (1/(w + 1e-7), conic, radius = ceil(3 sqrt(lambda_max)), lambda floor 0.1)
  forward.cu:340-467     renderCUDA (power > 0 skip, alpha = min(0.99, o G), alpha < 1/255 skip, T (1 - alpha) < 1e-4 stop)
  backward.cu:144-274    computeCov2DCUDA (1/(den^2 + 1e-7), x/y_grad_mul of the Jacobian clamp)
  backward.cu:278-341    computeCov3D backward (scale gradient taken w.r.t. mod * scale)
  backward.cu:347-412    preprocessCUDA backward (projection, depth and SH paths of dL/dmeans3D)
  backward.cu:415-641    renderCUDA backward (T_final = 1 - alpha image, recurrences, grad2d conventions below)

Two entry points:

  blend64(rec, radii, W, H, bg, ...)   per-Gaussian 2D records -> images (+ per-Gaussian grad2d[P, 12] given upstream image
                                       gradients), in the reference's conventions:
        [0..1] dL/dmean2D in NDC units (the pixel-space derivative times 0.5 W, 0.5 H),
        [2]    sum over pixels of |dL/dx| + |dL/dy| (a statistic, not a gradient),
        [3..5] dL/dconic (xx, xy, yy) with the xy entry -0.5 dx dy dL/dG (half the derivative w.r.t. the symmetric entry),
        [6]    dL/dopacity = sum G dL/dalpha — past the 0.99 cap alpha is capped in value but differentiated as uncapped,
        [7..9] dL/dcolor, [10] dL/ddepth, [11] unused;  background term -T_final / (1 - alpha) bg . dL/dC.
  render64(scene, ...)                 the whole path: preprocess in fp64 with autograd for the per-Gaussian chain rule, then
                                       blend64, then the chain back to every input.

Every output element also comes with its absolute mass (the sum of |term| over the pairs that feed it) and a kappa-weighted
mass; see `blend64` for the derivation of the per-pair factor.  `margins` / `margin_scene` keep scenes away from the discrete
decisions (thresholds, integer rounding, clamps) so that fp32 code and this restatement make the same decision for every pair.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch

F64 = torch.float64
EPS32 = 2.0 ** -24
TILE = 16

# fp32 constants of the reference (auxiliary.h:22-39, forward.cu:420-430); the thresholds are compared in fp64 against
# their fp32 values, the cap is used as a value.
_f = lambda v: float(np.float32(v))
ALPHA_MIN = _f(1.0 / 255.0)
ALPHA_CAP = _f(0.99)
T_STOP = _f(0.0001)
SH_C0 = _f(0.28209479177387814)
SH_C1 = _f(0.4886025119029199)
SH_C2 = [_f(v) for v in (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)]
SH_C3 = [_f(v) for v in (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
                         1.445305721320277, -0.5900435899266435)]


# ----------------------------------------------------------------------------------------------- tiles
def tile_rect(px, py, radii, W, H):
    """getRect (auxiliary.h:46-56) evaluated exactly as the reference does: fp32 (p -+ r) / 16, truncated toward zero, clamped."""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    px32 = torch.as_tensor(px).to(torch.float32)
    py32 = torch.as_tensor(py).to(torch.float32)
    r32 = torch.as_tensor(radii).to(torch.float32)
    t = lambda v, g: torch.clamp(torch.trunc(v).to(torch.int64), 0, g)
    x0 = t((px32 - r32) / TILE, gx)
    y0 = t((py32 - r32) / TILE, gy)
    x1 = t((px32 + r32 + (TILE - 1)) / TILE, gx)
    y1 = t((py32 + r32 + (TILE - 1)) / TILE, gy)
    return x0, y0, x1, y1


def _instances(rec, radii, W, H):
    """(tile, Gaussian) instances of the reference's binning, each tile's list in ascending (view depth, index) order."""
    dev = rec.device
    P = rec.shape[0]
    gx = (W + TILE - 1) // TILE
    x0, y0, x1, y1 = tile_rect(rec[:, 0], rec[:, 1], radii, W, H)
    vis = (torch.as_tensor(radii, device=dev) > 0) & ((x1 - x0) * (y1 - y0) > 0)
    order = torch.argsort(rec[:, 7].to(F64), stable=True)  # depth order, index order among equal depths
    ids, tiles = [], []
    for g in order[vis[order]].tolist():
        ys = torch.arange(int(y0[g]), int(y1[g]), device=dev)
        xs = torch.arange(int(x0[g]), int(x1[g]), device=dev)
        t = (ys[:, None] * gx + xs[None, :]).reshape(-1)
        tiles.append(t)
        ids.append(torch.full_like(t, g))
    if not ids:
        z = torch.zeros(0, dtype=torch.int64, device=dev)
        return z, z, (x0, y0, x1, y1), P
    tiles, ids = torch.cat(tiles), torch.cat(ids)
    srt = torch.argsort(tiles, stable=True)  # stable: keeps depth order within a tile
    return tiles[srt], ids[srt], (x0, y0, x1, y1), P


# ----------------------------------------------------------------------------------------------- blend
def blend64(rec, radii, W: int, H: int, bg, semantics=None, upstream: Optional[Dict] = None, alpha_img=None,
            max_pairs: int = 1 << 21, decisions=None):
    """Blend per-Gaussian records [P, 12] (the GaussRec layout: px, py, conic xx, xy, opacity-free yy ... see below) in fp64.

    rec columns: 0 px, 1 py, 2 conic.xx, 3 conic.xy, 4 conic.yy, 5 opacity, 6 (unused), 7 view depth, 8..10 rgb, 11 clamp bits.
    upstream: dict(color [3,H,W], depth [1,H,W], alpha [1,H,W], semantic [S,H,W]) -> also the backward.
    alpha_img: the alpha image the backward reads T_final = 1 - alpha from (backward.cu:468); default: this forward's.
    decisions: (pix, gid, take) — flat pixel indices, Gaussian indices and bools: those pairs pass (take) or skip the two
      per-pair tests (power > 0, alpha < 1/255) as given instead of as fp64 decides; a forced pass blends alpha =
      min(0.99, o exp(min(power, 0))).  Every other pair, and the T < 1e-4 stop, keep fp64's decision.

    Error model (units of 2^-24, the fp32 unit roundoff).  For a pair i of pixel p the fp32 code computes
      power with absolute error ~ pm_i = 0.5 (|a| dx^2 + |c| dy^2) + |b dx dy| (the terms it sums), so G and alpha carry a relative
      error ~ pm_i + 4 (expf, the product with opacity);  1 - alpha then carries alpha / (1 - alpha) times that;
      T = prod (1 - alpha_j) (forward, or backward by division from T_final) carries the sum of those over the pixel's blended pairs
      plus 2 per factor;  a sum of n terms adds n.
    So every term that involves pair i of pixel p is off by at most  kappa_i = 64 + 2 n_p + pm_i + sum_j alpha_j/(1-alpha_j) (pm_j + 4)
    relative (64 covers the constant-depth steps: reductions, the accurate/approximate exp, the reciprocal).  'kmass' is the sum of
    kappa_i |term|; 'mass' the plain sum of |term|.  The moment form of the geometry gradients (blend_bwd2 sums q dx^k in chunk-local
    integer coordinates and re-centres) is covered by taking |dx| + 16, |dy| + 16 in the masses of [0], [1], [3..5].
    Sums over tiles (one float atomic per tile per component) add tiles_touched(g) x mass: 'ntiles' is returned for that.
    """
    dev = rec.device
    rec = rec.to(F64)
    P = rec.shape[0]
    S = 0 if semantics is None else int(semantics.shape[1])
    sem = None if S == 0 else semantics.to(device=dev, dtype=F64)
    bg = torch.as_tensor(bg, dtype=F64, device=dev).reshape(3)
    HW = H * W
    gx = (W + TILE - 1) // TILE
    tiles, ids, rect, _ = _instances(rec, radii, W, H)

    img = dict(color=torch.zeros(3, HW, dtype=F64, device=dev), depth=torch.zeros(1, HW, dtype=F64, device=dev),
               alpha=torch.zeros(1, HW, dtype=F64, device=dev), semantic=torch.zeros(S, HW, dtype=F64, device=dev))
    imass = {k: torch.zeros_like(v) for k, v in img.items()}
    ikmass = {k: torch.zeros_like(v) for k, v in img.items()}
    n_blend = torch.zeros(HW, dtype=torch.int64, device=dev)
    last_id = torch.full((HW,), -1, dtype=torch.int64, device=dev)
    T_final = torch.ones(HW, dtype=F64, device=dev)
    kap_img = torch.full((HW,), 64.0, dtype=F64, device=dev)
    stopped = torch.zeros(HW, dtype=torch.bool, device=dev)
    n_capped = torch.zeros(HW, dtype=torch.int64, device=dev)
    n_list = torch.zeros(HW, dtype=torch.int64, device=dev)
    bwd = upstream is not None
    if bwd:
        up = {k: torch.as_tensor(upstream[k]).to(device=dev, dtype=F64).reshape(-1, HW) for k in ("color", "depth", "alpha")}
        up["semantic"] = (torch.as_tensor(upstream["semantic"]).to(device=dev, dtype=F64).reshape(S, HW) if S
                          else torch.zeros(0, HW, dtype=F64, device=dev))
        g2d = torch.zeros(P, 12, dtype=F64, device=dev)
        g2m = torch.zeros(P, 12, dtype=F64, device=dev)
        g2k = torch.zeros(P, 12, dtype=F64, device=dev)
        gsem = torch.zeros(P, S, dtype=F64, device=dev)
        gsem_m = torch.zeros(P, S, dtype=F64, device=dev)
        gsem_k = torch.zeros(P, S, dtype=F64, device=dev)
        ntiles = torch.zeros(P, dtype=torch.int64, device=dev)
    # pass 1 (forward) and pass 2 (backward, needs T_final of the given alpha image) share the per-chunk pair evaluation
    if len(tiles):
        ut, counts = torch.unique_consecutive(tiles, return_counts=True)
        starts = torch.cumsum(counts, 0) - counts
        order = torch.argsort(counts)
        chunks, cur, cur_max = [], [], 0
        for i in order.tolist():
            n = int(counts[i])
            if cur and max(cur_max, n) * (len(cur) + 1) * 256 > max_pairs:
                chunks.append(cur); cur, cur_max = [], 0
            cur.append(i); cur_max = max(cur_max, n)
        if cur:
            chunks.append(cur)
    else:
        chunks = []
    lx = torch.arange(256, device=dev) % TILE
    ly = torch.arange(256, device=dev) // TILE
    dec_key = dec_take = None
    if decisions is not None:
        dpix, dgid, dtake = (torch.as_tensor(v, device=dev) for v in decisions)
        dec_key, o_ = torch.sort(dpix.to(torch.int64) * P + dgid.to(torch.int64))
        dec_take = dtake.to(torch.bool)[o_]

    def evaluate(chunk):
        ci = torch.tensor(chunk, device=dev)
        cnt, st, tl = counts[ci], starts[ci], ut[ci]
        L = int(cnt.max())
        slot = torch.arange(L, device=dev)
        present = slot[None, :] < cnt[:, None]
        gid = torch.where(present, ids[(st[:, None] + slot[None, :]).clamp(max=len(ids) - 1)], torch.zeros_like(present, dtype=torch.int64))
        pxi = (tl % gx)[:, None] * TILE + lx[None, :]
        pyi = (tl // gx)[:, None] * TILE + ly[None, :]
        inside = (pxi < W) & (pyi < H)
        pix = torch.where(inside, pyi * W + pxi, torch.zeros_like(pxi))
        r = rec[gid]  # [n, L, 12]
        dx = r[..., 0:1] - pxi[:, None, :].to(F64)
        dy = r[..., 1:2] - pyi[:, None, :].to(F64)
        a, b, c, o = r[..., 2:3], r[..., 3:4], r[..., 4:5], r[..., 5:6]
        power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
        pm = 0.5 * (a.abs() * dx * dx + c.abs() * dy * dy) + (b * dx * dy).abs()
        G = torch.exp(torch.clamp(power, max=0.0))
        alpha = torch.clamp(o * G, max=ALPHA_CAP)
        ok = present[..., None] & inside[:, None, :] & ~(power > 0) & ~(alpha < ALPHA_MIN)
        if dec_key is not None and len(dec_key):
            key = (pix[:, None, :] * P + gid[:, :, None]).reshape(-1)
            pos = torch.searchsorted(dec_key, key).clamp(max=len(dec_key) - 1)
            hit = (dec_key[pos] == key).reshape(ok.shape) & present[..., None] & inside[:, None, :]
            ok = torch.where(hit, dec_take[pos].reshape(ok.shape), ok)
        A = torch.where(ok, alpha, torch.zeros_like(alpha))
        Tincl = torch.cumprod(1 - A, 1)
        keep = ok & ~(Tincl < T_STOP)
        A = torch.where(keep, alpha, torch.zeros_like(alpha))
        Tincl = torch.cumprod(1 - A, 1)
        Tb = torch.cat([torch.ones_like(Tincl[:, :1]), Tincl[:, :-1]], 1)
        w = A * Tb
        npx = keep.sum(1)  # [n, 256]
        amp = torch.where(keep, A / (1 - A) * (pm + 4), torch.zeros_like(A)).sum(1)
        kap = 64.0 + 2.0 * npx[:, None, :].to(F64) + pm + amp[:, None, :]
        kap = torch.where(keep, kap, torch.zeros_like(kap))
        stopped = (ok & ~keep).any(1)
        capped = (keep & (o * G > ALPHA_CAP)).sum(1)
        return dict(gid=gid, pix=pix, inside=inside, dx=dx, dy=dy, a=a, b=b, c=c, o=o, G=G, A=A, keep=keep, Tb=Tb, Tincl=Tincl,
                    stopped=stopped, capped=capped, n_list=cnt,
                    w=w, npx=npx, kap=kap, Tfin=Tincl[:, -1, :], kap_px=64.0 + 2.0 * npx.to(F64) + amp, L=L, slot=slot, r=r)

    cache = []
    for chunk in chunks:
        e = evaluate(chunk)
        ins, pix, w, keep, gid, r = e["inside"], e["pix"], e["w"], e["keep"], e["gid"], e["r"]
        m = ins.reshape(-1)
        p_flat = pix.reshape(-1)[m]

        def put(dst, val, ch):
            dst[ch].index_add_(0, p_flat, val.reshape(-1)[m])

        for ch in range(3):
            put(img["color"], (w * r[..., 8 + ch:9 + ch]).sum(1), ch)
            put(imass["color"], (w * r[..., 8 + ch:9 + ch]).abs().sum(1), ch)
            put(ikmass["color"], (e["kap"] * (w * r[..., 8 + ch:9 + ch]).abs()).sum(1), ch)
        put(img["depth"], (w * r[..., 7:8]).sum(1), 0)
        put(imass["depth"], (w * r[..., 7:8]).abs().sum(1), 0)
        put(ikmass["depth"], (e["kap"] * (w * r[..., 7:8]).abs()).sum(1), 0)
        put(img["alpha"], w.sum(1), 0)
        put(imass["alpha"], w.sum(1), 0)
        put(ikmass["alpha"], (e["kap"] * w).sum(1), 0)
        if S:
            sg = sem[gid]  # [n, L, S]
            ws = torch.einsum("nlp,nls->nsp", w, sg)
            wa = torch.einsum("nlp,nls->nsp", w, sg.abs())
            wk = torch.einsum("nlp,nls->nsp", e["kap"] * w, sg.abs())
            for ch in range(S):
                put(img["semantic"], ws[:, ch], ch)
                put(imass["semantic"], wa[:, ch], ch)
                put(ikmass["semantic"], wk[:, ch], ch)
        T_final[p_flat] = e["Tfin"].reshape(-1)[m]
        n_blend[p_flat] = e["npx"].reshape(-1)[m]
        kap_img[p_flat] = e["kap_px"].reshape(-1)[m]
        stopped[p_flat] = e["stopped"].reshape(-1)[m]
        n_capped[p_flat] = e["capped"].reshape(-1)[m]
        n_list[p_flat] = e["n_list"][:, None].expand_as(pix).reshape(-1)[m]
        kept_slot = torch.where(keep, e["slot"][None, :, None].expand_as(keep), torch.full_like(keep, -1, dtype=torch.int64))
        last = kept_slot.max(1).values  # [n, 256]
        lid = torch.where(last >= 0, torch.gather(gid, 1, last.clamp(min=0)), torch.full_like(last, -1))
        last_id[p_flat] = lid.reshape(-1)[m]
        if bwd:
            cache.append(e)

    # background: colour = sum w c + T_final bg; T_final carries the error of the pixel's T
    out = dict(n_blend=n_blend.reshape(H, W), last_id=last_id.reshape(H, W), T_final=T_final.reshape(H, W), rect=rect,
               stopped=stopped.reshape(H, W), n_capped=n_capped.reshape(H, W), n_list=n_list.reshape(H, W),
               instances=int(len(tiles)), tiles=tiles, ids=ids)
    for ch in range(3):
        img["color"][ch] += T_final * bg[ch]
        imass["color"][ch] += (T_final * bg[ch]).abs()
        ikmass["color"][ch] += kap_img * (T_final * bg[ch]).abs()
    shp = dict(color=(3, H, W), depth=(1, H, W), alpha=(1, H, W), semantic=(S, H, W))
    for k in img:
        out[k] = img[k].reshape(shp[k])
        out["mass_" + k] = imass[k].reshape(shp[k])
        out["kmass_" + k] = ikmass[k].reshape(shp[k])
    if not bwd:
        return out

    Tf_given = (1 - torch.as_tensor(alpha_img).to(device=dev, dtype=F64).reshape(HW)) if alpha_img is not None else out["alpha"].new_ones(HW) - img["alpha"][0]
    kW, kH = 0.5 * W, 0.5 * H
    for e in cache:
        ins, pix, keep, gid, r = e["inside"], e["pix"], e["keep"], e["gid"], e["r"]
        n, L = gid.shape
        pixc = pix  # [n, 256]
        dC = up["color"][:, pixc]  # [3, n, 256]
        dD, dA = up["depth"][0, pixc], up["alpha"][0, pixc]
        dS = up["semantic"][:, pixc]  # [S, n, 256]
        # g_i = value of pair i dotted with this pixel's upstream gradients (colour, features, depth, and 1 for alpha)
        g = (r[..., 8:9] * dC[0][:, None] + r[..., 9:10] * dC[1][:, None] + r[..., 10:11] * dC[2][:, None]
             + r[..., 7:8] * dD[:, None] + dA[:, None])
        gabs = ((r[..., 8:9] * dC[0][:, None]).abs() + (r[..., 9:10] * dC[1][:, None]).abs() + (r[..., 10:11] * dC[2][:, None]).abs()
                + (r[..., 7:8] * dD[:, None]).abs() + dA[:, None].abs())
        if S:
            sg = sem[gid]
            g = g + torch.einsum("nls,snp->nlp", sg, dS)
            gabs = gabs + torch.einsum("nls,snp->nlp", sg.abs(), dS.abs())
        w = e["w"]
        # value behind pair i: sum_{j>i} g_j alpha_j prod_{i<k<j} (1 - alpha_k) = (sum_{j>i} g_j w_j) / Tincl_i
        rc = lambda t: torch.flip(torch.cumsum(torch.flip(t, [1]), 1), [1]) - t
        den = torch.where(keep, e["Tincl"], torch.ones_like(w))
        behind = rc(g * w) / den
        behind_abs = rc(gabs * w) / den
        Tfg = Tf_given[pixc][:, None, :]
        scale = Tfg / e["Tfin"][:, None, :]
        Tbw = e["Tb"] * scale  # T of the backward replay, T_final / prod_{j>=i} (1 - alpha_j)
        A = e["A"]
        oma = torch.where(keep, 1 - A, torch.ones_like(A))
        bgdot = (bg[:, None, None] * dC).sum(0)[:, None, :]
        bgabs = (bg[:, None, None] * dC).abs().sum(0)[:, None, :]
        dLdopa = (g - behind) * Tbw - Tfg / oma * bgdot
        dLdopa_m = (gabs + behind_abs) * Tbw + Tfg / oma * bgabs
        zero = torch.zeros_like(w)
        G, o = e["G"], e["o"]
        q = torch.where(keep, o * G * dLdopa, zero)
        qm = torch.where(keep, (o * G).abs() * dLdopa_m, zero)
        wb = torch.where(keep, A * Tbw, zero)
        dx, dy, a, b, c = e["dx"], e["dy"], e["a"], e["b"], e["c"]
        kap = e["kap"]
        px_, py_ = dx.abs() + 16, dy.abs() + 16
        t0 = -kW * q * (a * dx + b * dy)
        t1 = -kH * q * (c * dy + b * dx)
        terms = [t0, t1, t0.abs() + t1.abs(), -0.5 * q * dx * dx, -0.5 * q * dx * dy, -0.5 * q * dy * dy,
                 torch.where(keep, G * dLdopa, zero),
                 wb * dC[0][:, None], wb * dC[1][:, None], wb * dC[2][:, None], wb * dD[:, None]]
        m0 = kW * qm * (a.abs() * px_ + b.abs() * py_)
        m1 = kH * qm * (c.abs() * py_ + b.abs() * px_)
        masses = [m0, m1, m0 + m1, 0.5 * qm * px_ * px_, 0.5 * qm * px_ * py_, 0.5 * qm * py_ * py_,
                  torch.where(keep, G.abs() * dLdopa_m, zero),
                  (wb * dC[0][:, None]).abs(), (wb * dC[1][:, None]).abs(), (wb * dC[2][:, None]).abs(), (wb * dD[:, None]).abs()]
        flat_g = gid.reshape(-1)
        for k in range(11):
            g2d[:, k].index_add_(0, flat_g, terms[k].sum(2).reshape(-1))
            g2m[:, k].index_add_(0, flat_g, masses[k].sum(2).reshape(-1))
            g2k[:, k].index_add_(0, flat_g, (kap * masses[k]).sum(2).reshape(-1))
        if S:
            gs = torch.einsum("nlp,snp->nls", wb, dS)
            gsm = torch.einsum("nlp,snp->nls", wb, dS.abs())
            gsk = torch.einsum("nlp,snp->nls", kap * wb, dS.abs())
            gsem.index_add_(0, flat_g, gs.reshape(-1, S))
            gsem_m.index_add_(0, flat_g, gsm.reshape(-1, S))
            gsem_k.index_add_(0, flat_g, gsk.reshape(-1, S))
        ntiles.index_add_(0, flat_g, keep.any(2).reshape(-1).to(torch.int64))
    out.update(grad2d=g2d, mass_grad2d=g2m, kmass_grad2d=g2k, grad_semantics=gsem, mass_grad_semantics=gsem_m,
               kmass_grad_semantics=gsem_k, ntiles=ntiles)
    return out


# ----------------------------------------------------------------------------------------------- near-threshold decisions
# Rounding counts (units of 2^-24) of the two values the reference's per-pair tests read (forward.cu:420-430), see power_interval.
EPS_POWER = 8.0
EPS_ALPHA = 8.0


def power_interval(rec, px, py):
    """fp64 power of the pairs (records `rec` [..., 12] against pixel coordinates px, py, broadcast) and a bound `err` with
    |fp32 power - fp64 power| <= err for the reference's expression -0.5 (a dx dx + c dy dy) - b dx dy evaluated in fp32 on the
    same fp32 record, with or without contraction to FMAs.  Returns (power, err, pm).

    Derivation (u = 2^-24, pm = 0.5 (|a| dx^2 + |c| dy^2) + |b dx dy|): dx = x - px rounds once (u |dx|), as does dy.  Each of
    a dx dx, c dy dy, b dx dy then takes two products: 2 u from the rounded coordinates plus 2 roundings, 4 u of its magnitude.
    The sum a dx dx + c dy dy adds one rounding of a value <= |a| dx^2 + |c| dy^2, so -0.5 (...) is off by 5 u of its terms, and the
    final difference adds u |power| <= u pm:  |err| <= 5 u pm + u pm = 6 u pm to first order.  A contracted FMA drops a rounding,
    never adds one.  EPS_POWER = 8 covers the second-order terms."""
    dx = rec[..., 0].to(F64) - px
    dy = rec[..., 1].to(F64) - py
    a, b, c = rec[..., 2].to(F64), rec[..., 3].to(F64), rec[..., 4].to(F64)
    power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
    pm = 0.5 * (a.abs() * dx * dx + c.abs() * dy * dy) + (b * dx * dy).abs()
    return power, EPS_POWER * EPS32 * pm, pm


def pair_decisions(rec, px, py):
    """The reference's blend decision of pairs (power > 0 skips, o exp(power) < 1/255 skips) judged on the interval of
    power_interval and on EPS_ALPHA u of relative error in alpha (expf is within 2 ulp = 4 u, the product with the opacity one
    rounding).  'may': some fp32 evaluation within the bounds blends the pair;  'must': every one does."""
    power, err, pm = power_interval(rec, px, py)
    o = rec[..., 5].to(F64)
    lo, hi = power - err, power + err
    ae = EPS_ALPHA * EPS32
    may = (lo <= 0) & (o * torch.exp(torch.clamp(hi, max=0.0)) * (1 + ae) >= ALPHA_MIN)
    must = (hi <= 0) & (o * torch.exp(torch.clamp(lo, max=0.0)) * (1 - ae) >= ALPHA_MIN)
    return dict(power=power, err=err, pm=pm, may=may, must=must & may)


def instance_pixels(rec, radii, W, H, max_pairs: int = 1 << 22):
    """Yields the (tile, Gaussian) instances of the reference's rectangles in chunks, each with its 256 pixels:
    dict(tile [n], gid [n], pix [n, 256] flat index, inside [n, 256], px, py [n, 256], dec = pair_decisions of every pixel)."""
    tiles, ids, _, _ = _instances(rec, radii, W, H)
    gx = (W + TILE - 1) // TILE
    dev = rec.device
    lx = torch.arange(256, device=dev) % TILE
    ly = torch.arange(256, device=dev) // TILE
    step = max(1, max_pairs // 256)
    for s in range(0, len(tiles), step):
        t, g = tiles[s:s + step], ids[s:s + step]
        pxi = (t % gx)[:, None] * TILE + lx[None, :]
        pyi = (t // gx)[:, None] * TILE + ly[None, :]
        inside = (pxi < W) & (pyi < H)
        pix = torch.where(inside, pyi * W + pxi, torch.zeros_like(pxi))
        dec = pair_decisions(rec[g][:, None, :], pxi.to(F64), pyi.to(F64))
        dec["may"] &= inside
        dec["must"] &= inside
        yield dict(tile=t, gid=g, pix=pix, inside=inside, px=pxi, py=pyi, dec=dec)


def ambiguous_pairs(rec, radii, W, H):
    """(flat pixel, Gaussian) of every pair of the reference's rectangles that may blend but need not: its decision is left to
    fp32 rounding.  Returns dict(pix, gid, power, err) sorted by (pix, gid)."""
    pix, gid, pw, er = [], [], [], []
    for ch in instance_pixels(rec.to(F64), radii, W, H):
        d = ch["dec"]
        amb = d["may"] & ~d["must"]
        n, i = torch.nonzero(amb, as_tuple=True)
        pix.append(ch["pix"][n, i]); gid.append(ch["gid"][n]); pw.append(d["power"][n, i]); er.append(d["err"][n, i])
    if not pix:
        z = torch.zeros(0, dtype=torch.int64, device=rec.device)
        return dict(pix=z, gid=z, power=z.to(F64), err=z.to(F64))
    pix, gid, pw, er = torch.cat(pix), torch.cat(gid), torch.cat(pw), torch.cat(er)
    o = torch.argsort(pix * rec.shape[0] + gid)
    return dict(pix=pix[o], gid=gid[o], power=pw[o], err=er[o])


def bound(kmass, mass=None, ntiles=None, extra: float = 0.0):
    """Per-element bound in absolute units: 2^-24 (kmass + ntiles mass + extra mass) (see blend64 for the derivation)."""
    b = kmass
    if mass is not None and ntiles is not None:
        nt = ntiles.to(kmass.dtype).reshape(-1, *([1] * (kmass.dim() - 1)))
        b = b + nt * mass
    if mass is not None and extra:
        b = b + extra * mass
    return EPS32 * b


# ----------------------------------------------------------------------------------------------- preprocess
class _Conic(torch.autograd.Function):
    """conic = (c, -b, a) / (a c - b^2); its backward uses the reference's 1/(den^2 + 1e-7) (backward.cu:201-212) and takes the
    incoming xy gradient as the reference's half-derivative (grad2d[4])."""

    @staticmethod
    def forward(ctx, a, b, c):
        det = a * c - b * b
        ctx.save_for_backward(a, b, c)
        return c / det, -b / det, a / det

    @staticmethod
    def backward(ctx, gx, gy, gz):
        a, b, c = ctx.saved_tensors
        gy = 0.5 * gy  # the reference's dL_dconic.y is half the derivative w.r.t. the symmetric entry
        den = a * c - b * b
        inv = 1.0 / (den * den + 1e-7)
        da = inv * (-c * c * gx + 2 * b * c * gy + (den - a * c) * gz)
        dc = inv * (-a * a * gz + 2 * a * b * gy + (den - a * c) * gx)
        db = inv * 2 * (b * c * gx - (den + 2 * b * b) * gy + a * b * gz)
        return da, db, dc


def _f32(v) -> float:
    return float(np.float32(v))


def _cam(cam, dev):
    g = lambda k: torch.as_tensor(cam[k]).to(device=dev, dtype=F64)
    W, H = int(cam["image_width"]), int(cam["image_height"])
    tanx, tany = _f32(cam["tanfovx"]), _f32(cam["tanfovy"])
    return dict(W=W, H=H, tanx=tanx, tany=tany, fx=_f32(np.float32(W) / (np.float32(2.0) * np.float32(tanx))),
                fy=_f32(np.float32(H) / (np.float32(2.0) * np.float32(tany))), view=g("viewmatrix"), proj=g("projmatrix"),
                campos=g("campos").reshape(3), bg=g("bg").reshape(3), mod=_f32(cam["scale_modifier"]), D=int(cam["sh_degree"]),
                limx=_f32(np.float32(1.3) * np.float32(tanx)), limy=_f32(np.float32(1.3) * np.float32(tany)))


def _sh_terms(D, dirs, sh):
    """the per-coefficient terms of computeColorFromSH (forward.cu:20-63): list of [P, 3] tensors, summed they give rgb - 0.5."""
    x, y, z = dirs[:, 0:1], dirs[:, 1:2], dirs[:, 2:3]
    t = [SH_C0 * sh[:, 0]]
    if D > 0:
        t += [-SH_C1 * y * sh[:, 1], SH_C1 * z * sh[:, 2], -SH_C1 * x * sh[:, 3]]
        if D > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            t += [SH_C2[0] * xy * sh[:, 4], SH_C2[1] * yz * sh[:, 5], SH_C2[2] * (2.0 * zz - xx - yy) * sh[:, 6],
                  SH_C2[3] * xz * sh[:, 7], SH_C2[4] * (xx - yy) * sh[:, 8]]
            if D > 2:
                t += [SH_C3[0] * y * (3.0 * xx - yy) * sh[:, 9], SH_C3[1] * xy * z * sh[:, 10],
                      SH_C3[2] * y * (4.0 * zz - xx - yy) * sh[:, 11], SH_C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy) * sh[:, 12],
                      SH_C3[4] * x * (4.0 * zz - xx - yy) * sh[:, 13], SH_C3[5] * z * (xx - yy) * sh[:, 14],
                      SH_C3[6] * x * (xx - 3.0 * yy) * sh[:, 15]]
    return t


def preprocess64(scene, device="cpu", requires_grad=False):
    """forward.cu:156-256 in fp64.  Returns the leaves, the records [P, 12] (differentiable columns), radii, and the decision
    quantities that `margins` checks."""
    cam = _cam(scene["cam"], device)
    W, H = cam["W"], cam["H"]
    leaf = lambda k: (scene[k].detach().to(device=device, dtype=F64).clone().requires_grad_(requires_grad)
                      if scene.get(k) is not None else None)
    means = leaf("means3D")
    opac = leaf("opacities")
    shs, colors = leaf("shs"), leaf("colors_precomp")
    cov_pre = leaf("cov3D_precomp")
    scales, rots = (None, None) if cov_pre is not None else (leaf("scales"), leaf("rotations"))
    P = means.shape[0]
    ones = torch.ones(P, 1, dtype=F64, device=device)
    hom = torch.cat([means, ones], 1)
    p_view = hom @ cam["view"]
    p_hom = hom @ cam["proj"]
    p_w = 1.0 / (p_hom[:, 3:4] + 1e-7)
    ndc = p_hom[:, :3] * p_w
    # 3D covariance (forward.cu:118-152): quaternion not normalised, s = mod * scale (its gradient is reported as the scale's)
    s_leaf = None
    if cov_pre is None:
        s_leaf = (cam["mod"] * scales).detach().requires_grad_(requires_grad)
        r, x, y, z = rots[:, 0], rots[:, 1], rots[:, 2], rots[:, 3]
        R = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)], -1),
                         torch.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)], -1),
                         torch.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)], -1)], -2)
        M = s_leaf[:, :, None] * R
        Sig = M.transpose(1, 2) @ M
        cov6 = torch.stack([Sig[:, 0, 0], Sig[:, 0, 1], Sig[:, 0, 2], Sig[:, 1, 1], Sig[:, 1, 2], Sig[:, 2, 2]], -1)
    else:
        cov6 = cov_pre
    V = torch.stack([torch.stack([cov6[:, 0], cov6[:, 1], cov6[:, 2]], -1), torch.stack([cov6[:, 1], cov6[:, 3], cov6[:, 4]], -1),
                     torch.stack([cov6[:, 2], cov6[:, 4], cov6[:, 5]], -1)], -2)
    # 2D covariance (forward.cu:74-113) with the Jacobian clamp; the clamped coordinate carries no gradient (backward.cu:175-176)
    tx, ty, tz = p_view[:, 0], p_view[:, 1], p_view[:, 2]
    txtz, tytz = tx / tz, ty / tz
    clx = (txtz < -cam["limx"]) | (txtz > cam["limx"])
    cly = (tytz < -cam["limy"]) | (tytz > cam["limy"])
    txc = torch.where(clx, (torch.clamp(txtz, -cam["limx"], cam["limx"]) * tz).detach(), tx)
    tyc = torch.where(cly, (torch.clamp(tytz, -cam["limy"], cam["limy"]) * tz).detach(), ty)
    fx, fy = cam["fx"], cam["fy"]
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, zero], -1), torch.stack([zero, fy / tz, zero], -1),
                     torch.stack([-fx * txc / (tz * tz), -fy * tyc / (tz * tz), zero], -1)], -2)
    Wm = cam["view"][:3, :3]
    T = Wm[None] @ J
    cov2 = T.transpose(1, 2) @ V @ T
    a, b, c = cov2[:, 0, 0] + 0.3, cov2[:, 0, 1], cov2[:, 1, 1] + 0.3
    det = a * c - b * b
    ca, cb, cc = _Conic.apply(a, b, c)
    mid = 0.5 * (a + c)
    lam1 = mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
    lam2 = mid - torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
    r3 = 3.0 * torch.sqrt(torch.maximum(lam1, lam2))
    radius = torch.ceil(r3.detach())
    px = ((ndc[:, 0] + 1.0) * W - 1.0) * 0.5
    py = ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5
    # colour (forward.cu:20-71)
    if colors is None:
        dirs = means - cam["campos"][None]
        dirs = dirs / torch.linalg.vector_norm(dirs, dim=1, keepdim=True)
        terms = _sh_terms(cam["D"], dirs, shs)
        raw = sum(terms) + 0.5
        sh_mass = sum(t.abs() for t in terms) + 0.5
        clamped = raw < 0
        rgb = torch.clamp(raw, min=0.0)
    else:
        raw, sh_mass, clamped, rgb = colors, colors.abs(), torch.zeros_like(colors, dtype=torch.bool), colors
    near = ~(tz > 0.2)
    rad_i = torch.where(near | (det == 0), torch.zeros_like(radius), radius).to(torch.int64)
    x0, y0, x1, y1 = tile_rect(px.detach(), py.detach(), rad_i, W, H)
    vis = (rad_i > 0) & ((x1 - x0) * (y1 - y0) > 0)
    rad_i = torch.where(vis, rad_i, torch.zeros_like(rad_i))
    bits = (clamped[:, 0].to(torch.int64) | (clamped[:, 1].to(torch.int64) << 1) | (clamped[:, 2].to(torch.int64) << 2))
    cols = [px, py, ca, cb, cc, opac[:, 0], torch.zeros_like(px), tz, rgb[:, 0], rgb[:, 1], rgb[:, 2], bits.to(F64)]
    recs = torch.stack(cols, 1)
    leaves = dict(means3D=means, opacities=opac, shs=shs, colors_precomp=colors, cov3D_precomp=cov_pre, scales=s_leaf, rotations=rots)
    with torch.no_grad():
        # condition number of the dilated 2D covariance (true eigenvalues, not the radius formula's floored ones)
        lmax = mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.0))
        lmin = det / torch.clamp(lmax, min=1e-300)
        cond = lmax / torch.clamp(lmin, min=1e-300)
        # magnitudes of the terms the fp32 preprocess sums (for the per-element bounds of the records)
        ah = hom.abs()
        ndc_mass = (ah @ cam["proj"].abs())[:, :2] / p_hom[:, 3:4].abs() + ndc[:, :2].abs()
        depth_mass = (ah @ cam["view"].abs())[:, 2]
        Ta = T.abs()
        cov_mass = (Ta.transpose(1, 2) @ V.abs() @ Ta)[:, :2, :2].amax((1, 2)) + 0.3
    return dict(cam=cam, leaves=leaves, cols=cols, rec=recs.detach(), radii=rad_i, vis=vis, tz=tz.detach(), txtz=txtz.detach(),
                tytz=tytz.detach(), r3=r3.detach(), raw_rgb=raw.detach(), sh_mass=sh_mass.detach(), clamped_x=clx, clamped_y=cly,
                cond=cond, lmin=lmin, ndc=ndc, ndc_mass=ndc_mass, depth_mass=depth_mass, cov_mass=cov_mass)


GRAD_COMPONENTS = {0: "ndcx", 1: "ndcy", 3: "ca", 4: "cb", 5: "cc", 6: "opac", 7: "r", 8: "g", 9: "b", 10: "depth"}


def render64(scene, device="cpu", backward=True, alpha_img=None, max_pairs: int = 1 << 21):
    """The whole reference path in fp64.  Returns images, radii, grad2d and the per-input gradients (reference names with a g_
    prefix, as tests/util.run_api) together with their masses:
      mass_g_x   = sum_k |J_k| mass(grad2d_k)                   (the blend's absolute mass carried through the chain rule)
      kmass_g_x  = sum_k |J_k| (kmass(grad2d_k) + ntiles mass(grad2d_k))
      cmass_g_x  = sum_k |J_k grad2d_k| (1 + cond for the conic components) — the chain rule's own terms, summed over the
                   three means3D paths (mean2D, covariance, SH direction) and the depth path.
    J_k is the per-Gaussian derivative of record component k w.r.t. the input element."""
    pre = preprocess64(scene, device, requires_grad=backward)
    cam = pre["cam"]
    W, H = cam["W"], cam["H"]
    sem = scene.get("semantics")
    ups = None
    if backward:
        ups = dict(color=scene["grad_color"], depth=scene["grad_depth"], alpha=scene["grad_alpha"],
                   semantic=scene.get("grad_semantic") if sem is not None else None)
    bl = blend64(pre["rec"], pre["radii"], W, H, cam["bg"], semantics=sem, upstream=ups, alpha_img=alpha_img, max_pairs=max_pairs)
    out = dict(color=bl["color"], depth=bl["depth"], alpha=bl["alpha"], semantic=bl["semantic"], radii=pre["radii"], blend=bl, pre=pre)
    if not backward:
        return out
    vis = pre["vis"].to(F64)[:, None]
    g2d = bl["grad2d"] * vis
    ntiles = bl["ntiles"].to(F64)
    res = dict(out)
    res.update(chain64(pre, g2d, bl["mass_grad2d"] * vis, (bl["kmass_grad2d"] + ntiles[:, None] * bl["mass_grad2d"]) * vis))
    if sem is not None:
        res["g_semantics"] = bl["grad_semantics"]
        res["mass_g_semantics"] = bl["mass_grad_semantics"]
        res["kmass_g_semantics"] = bl["kmass_grad_semantics"] + ntiles[:, None] * bl["mass_grad_semantics"]
        res["cmass_g_semantics"] = torch.zeros_like(bl["grad_semantics"])
    res["grad2d"] = g2d
    return res


# Fixed depth of the fp32 chain rule (backward.cu:144-412): its longest path, dL/dconic -> dL/d(a, b, c) -> dL/dT -> dL/dJ -> dL/dt ->
# dL/dmeans3D, has six levels of sums of at most four products of at most three factors, i.e. at most 6 x (4 + 3) = 42 roundings.
K_CHAIN = 64.0


def chain64(pre, g2d, mass2d=None, kmass2d=None):
    """The per-Gaussian chain rule (backward.cu:144-412) applied to a given grad2d [P, 12], in fp64 (autograd through
    preprocess64's graph).  Returns g_<input> with, per element:
      mass_g_x  = sum_k |J_k| mass2d_k, kmass_g_x = sum_k |J_k| kmass2d_k   (the blend's masses carried through the chain; zero if
                  not given), and cmass_g_x = sum_k |J_k g_k| (1 + cond for the conic components): the chain rule's own terms, summed
                  over the means3D paths (mean2D, covariance, SH direction, depth).  J_k is the per-Gaussian derivative of record
                  component k w.r.t. the input element.  See chain_bound for how these bound the fp32 chain."""
    vis = pre["vis"].to(F64)
    g2d = g2d.to(F64) * vis[:, None]
    mass2d = torch.zeros_like(g2d) if mass2d is None else mass2d.to(F64)
    kmass2d = torch.zeros_like(g2d) if kmass2d is None else kmass2d.to(F64)
    cols = pre["cols"]
    # record component k as a function of the inputs: mean2D in NDC (grad2d[0..1] are NDC gradients), the conic xy entry with
    # twice the stored half-derivative (it appears twice in the quadratic form)
    rec_fn = {0: pre["ndc"][:, 0], 1: pre["ndc"][:, 1], 3: cols[2], 4: cols[3], 5: cols[4], 6: cols[5], 7: cols[8], 8: cols[9],
              9: cols[10], 10: cols[7]}
    factor = {4: 2.0}
    leaves = {k: v for k, v in pre["leaves"].items() if v is not None}
    names = list(leaves)
    grads = {n: torch.zeros_like(leaves[n]) for n in names}
    mass = {n: torch.zeros_like(leaves[n]) for n in names}
    kmass = {n: torch.zeros_like(leaves[n]) for n in names}
    cmass = {n: torch.zeros_like(leaves[n]) for n in names}
    cond = pre["cond"]
    ks = list(rec_fn)
    for i, k in enumerate(ks):
        f = factor.get(k, 1.0)
        Js = torch.autograd.grad(rec_fn[k].sum(), [leaves[n] for n in names], retain_graph=True, allow_unused=True)
        for n, Jn in zip(names, Js):
            if Jn is None:
                continue
            sh = (-1,) + (1,) * (Jn.dim() - 1)
            gk = (f * g2d[:, k]).reshape(sh)
            grads[n] = grads[n] + Jn * gk
            mass[n] = mass[n] + Jn.abs() * (f * mass2d[:, k]).reshape(sh)
            kmass[n] = kmass[n] + Jn.abs() * (f * kmass2d[:, k]).reshape(sh)
            cw = (1.0 + cond).reshape(sh) if k in (3, 4, 5) else 1.0
            cmass[n] = cmass[n] + (Jn * gk).abs() * cw
    name_map = dict(means3D="g_means3D", opacities="g_opacities", shs="g_shs", colors_precomp="g_colors_precomp",
                    cov3D_precomp="g_cov3D_precomp", scales="g_scales", rotations="g_rotations")
    res = {}
    for n in names:
        res[name_map[n]] = grads[n].detach()
        res["mass_" + name_map[n]] = mass[n].detach()
        res["kmass_" + name_map[n]] = kmass[n].detach()
        res["cmass_" + name_map[n]] = cmass[n].detach()
    res["g_means2D"] = g2d[:, 0:3].clone()
    res["mass_g_means2D"] = mass2d[:, 0:3] * vis[:, None]
    res["kmass_g_means2D"] = kmass2d[:, 0:3] * vis[:, None]
    res["cmass_g_means2D"] = torch.zeros_like(res["g_means2D"])
    return res


def chain_bound(res, key):
    """Per-element bound (absolute) of an fp32 evaluation of the chain rule, given fp32-rounding-exact upstream sums:
        2^-24 (kmass + K_CHAIN (cmass + rowmax(cmass)))
    Each of the chain's at most 42 roundings (K_CHAIN) errs by 2^-24 times the value it rounds.  A value on a path to output e is
    either one of e's own terms (bounded by cmass_e) or an intermediate shared by the Gaussian's whole row — dL/d(a, b, c), dL/dT,
    dL/dJ, dL/dt, the SH basis, dL/dM — whose terms are path terms of some element of the same row: at most a few of them, each at
    most rowmax(cmass) (the conic ones already weighted by 1 + cond, the inverse's amplification); the SH basis terms are at most
    4 |dL/drgb| <= 4 / SH_C0 |SH_C0 dL/drgb| < 15 rowmax.  K_CHAIN = 64 covers those factors."""
    cm = res["cmass_" + key]
    rowmax = cm.reshape(cm.shape[0], -1).amax(1).reshape((-1,) + (1,) * (cm.dim() - 1)) if cm.numel() else cm
    return EPS32 * (res["kmass_" + key] + K_CHAIN * (cm + rowmax))


# ----------------------------------------------------------------------------------------------- margins
def margins(rec, radii, W, H, delta: float = 1e-5, pre=None):
    """Indices of the Gaussians that take part in a discrete decision closer than a relative margin delta to its threshold.

    Per pair (only pairs the reference evaluates: inside the rectangle, before the pixel stops):
      alpha vs 1/255 and o G vs the 0.99 cap; T (1 - alpha) vs 1e-4 with a margin delta (1 + k / 8) that grows with the pixel's
      list depth k; power vs 0 relative to pm = 0.5 (|a| dx^2 + |c| dy^2) + |b dx dy|.
    Per Gaussian, when `pre` (preprocess64's output) is given: 3 sqrt(lambda_max) vs an integer; the rectangle edges (p -+ r)/16
    vs an integer; view z vs 0.2; tx/tz, ty/tz vs +-1.3 tan(fov); each SH colour vs 0 relative to its terms' mass."""
    dev = rec.device
    rec = rec.to(F64)
    bad = torch.zeros(rec.shape[0], dtype=torch.bool, device=dev)
    tiles, ids, _, _ = _instances(rec, radii, W, H)
    if len(tiles):
        gx = (W + TILE - 1) // TILE
        ut, counts = torch.unique_consecutive(tiles, return_counts=True)
        starts = torch.cumsum(counts, 0) - counts
        lx = torch.arange(256, device=dev) % TILE
        ly = torch.arange(256, device=dev) // TILE
        for t, st, n in zip(ut.tolist(), starts.tolist(), counts.tolist()):
            gid = ids[st:st + n]
            pxi = (t % gx) * TILE + lx
            pyi = (t // gx) * TILE + ly
            inside = (pxi < W) & (pyi < H)
            r = rec[gid]
            dx = r[:, 0:1] - pxi[None].to(F64)
            dy = r[:, 1:2] - pyi[None].to(F64)
            a, b, c, o = r[:, 2:3], r[:, 3:4], r[:, 4:5], r[:, 5:6]
            power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
            pm = 0.5 * (a.abs() * dx * dx + c.abs() * dy * dy) + (b * dx * dy).abs()
            oG = o * torch.exp(torch.clamp(power, max=0.0))
            alpha = torch.clamp(oG, max=ALPHA_CAP)
            ok = inside[None] & ~(power > 0) & ~(alpha < ALPHA_MIN)
            A = torch.where(ok, alpha, torch.zeros_like(alpha))
            Tb = torch.cat([torch.ones_like(A[:1]), torch.cumprod(1 - A, 0)[:-1]], 0)
            testT = Tb * (1 - A)
            reached = torch.cumsum((ok & (testT < T_STOP)).to(torch.int64), 0)
            evaluated = inside[None] & ((reached - (ok & (testT < T_STOP)).to(torch.int64)) == 0)  # up to and incl. the stopping pair
            near = (power.abs() <= delta * pm) & (pm > 0)
            near |= (power <= 0) & ((alpha - ALPHA_MIN).abs() <= delta * ALPHA_MIN)
            near |= (power <= 0) & ((oG - ALPHA_CAP).abs() <= delta * ALPHA_CAP)
            k = torch.arange(n, device=dev, dtype=F64)[:, None]
            near |= ok & ((testT - T_STOP).abs() <= delta * (1 + k / 8) * T_STOP)
            hit = (near & evaluated).any(1)
            bad[gid[hit]] = True
    if pre is not None:
        cam = pre["cam"]
        r3 = pre["r3"]
        fr = (r3 - torch.round(r3)).abs()
        vis = pre["vis"]
        bad |= vis & (fr <= delta * torch.clamp(r3, min=1.0))
        rad = pre["radii"].to(F64)
        px, py = rec[:, 0], rec[:, 1]
        for v, s in (((px - rad) / TILE, px), ((py - rad) / TILE, py), ((px + rad + TILE - 1) / TILE, px), ((py + rad + TILE - 1) / TILE, py)):
            tol = delta * (1.0 + s.abs() + rad) / TILE
            bad |= vis & ((v - torch.round(v)).abs() <= tol)
        bad |= ((pre["tz"] - 0.2).abs() <= delta * 0.2)
        bad |= ((pre["txtz"].abs() - cam["limx"]).abs() <= delta * cam["limx"])
        bad |= ((pre["tytz"].abs() - cam["limy"]).abs() <= delta * cam["limy"])
        bad |= vis & ((pre["raw_rgb"].abs() <= delta * pre["sh_mass"]).any(1))
    return torch.nonzero(bad).reshape(-1)


_SCENE_PER_GAUSSIAN = ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp", "semantics")


def subset(scene, keep):
    out = dict(scene)
    for k in _SCENE_PER_GAUSSIAN:
        if scene.get(k) is not None:
            out[k] = scene[k][keep].contiguous()
    return out


def margin_scene(scene, delta: float = 1e-5, device="cpu", max_rounds: int = 30):
    """Remove the Gaussians `margins` reports, repeatedly (removing one changes T behind it), until none are left.
    Returns (scene, number removed, kept original indices)."""
    P = scene["means3D"].shape[0]
    keep = torch.arange(P)
    sc = scene
    for _ in range(max_rounds):
        pre = preprocess64(sc, device)
        cam = pre["cam"]
        bad = margins(pre["rec"], pre["radii"], cam["W"], cam["H"], delta, pre=pre).cpu()
        if len(bad) == 0:
            return sc, P - len(keep), keep
        mask = torch.ones(len(keep), dtype=torch.bool)
        mask[bad] = False
        keep = keep[mask]
        sc = subset(scene, keep)
    raise RuntimeError(f"margin_scene did not converge in {max_rounds} rounds")
