// tile_visit.cuh — enumerate the tiles of one Gaussian's 3-sigma rectangle that (a) lie in this process's tile-row
// band and (b) can actually receive a contribution; either count them (preprocess) or emit (tile, gaussian) pairs
// (binning).  Count and emit run the SAME code on the SAME inputs, so counts always match the scanned offsets.
//
// Exact, opacity-aware culling by ROW SPANS.  A pixel contributes only if  q(d) = a dx^2 + 2b dx dy + c dy^2 <= qmax
// (sgr_common.cuh).  For one tile row (a horizontal strip of 16 pixel rows) the set {ellipse ∩ strip} is convex, so the
// tile columns it touches form ONE interval whose ends follow in closed form from the ellipse's x-extent inside the
// strip (two square roots per row).  A tile (full strip height) intersects the convex set iff its x-range intersects
// that interval, so this is exactly the per-tile test, at O(rows) instead of O(rows x cols) cost, with the same
// conservative slack (a tile that is kept needlessly only costs time; a dropped tile receives nothing from any fp32
// evaluation of the reference's `power` within the rounding bound that make_cull's qmax slack covers).
//
// (Tried and removed: an extra 8-bit mask per instance of the tile's eight 8x4-pixel blocks so that the blend warps could
// skip splats that miss their block.  On the BASELINE config-C frame pixels saturate on large near splats, so few
// warp-iterations were skipped, and the per-tile mask math made this kernel several times slower.)
//
// Small rectangles are walked by the owning thread; rectangles above kCoopArea tiles are walked by the whole warp so one
// screen-filling splat cannot serialise 10^4 iterations on one thread (the reference's duplicateWithKeys does,
// rasterizer_impl.cu:70-111).
#pragma once
#include "sgr_common.cuh"

namespace sgr {

constexpr int kCoopArea = 64;

// Approximate (MUFU-based, ~2 ulp) division / square root: this file only decides which tiles are KEPT, with slack
// (0.05 px on the interval ends, 0.02 + 1e-3|tau| on qmax, plus make_cull's term for thin splats) above their error, and count and emit
// evaluate the identical code, so the IEEE versions (10-15 dependent instructions each) buy nothing here.
__device__ __forceinline__ float fast_sqrt(float x) { return x * __frsqrt_rn(fmaxf(x, 1e-30f)); }
__device__ __forceinline__ float fast_div(float x, float y) { return __fdividef(x, y); }

// x-extent [xmin, xmax] (relative to the centre) of {ellipse q <= qmax} ∩ {uy0 <= y <= uy1}; false if empty.
// Requires a finite qmax and a positive-definite conic (make_cull guarantees both when qmax is finite).
struct EllipseAux {
	float det, det_over_a, inv_a, xext, yhi;  // det, det/a, 1/a; extreme |x| of the ellipse, reached at y = -/+ yhi
};
__device__ __forceinline__ EllipseAux ellipse_aux(const CullParams cp) {
	EllipseAux e;
	const float det = cp.a * cp.c - cp.b * cp.b;
	e.det = det;
	e.inv_a = fast_div(1.0f, cp.a);
	e.det_over_a = det * e.inv_a;
	e.xext = fast_sqrt(fast_div(cp.qmax * cp.c, det));
	e.yhi = -cp.b * fast_div(e.xext, cp.c);
	return e;
}
// disc = b^2 y^2 - a (c y^2 - qmax) = a qmax - det y^2, written with ONE rounding of the cancelling part (det is taken once
// from the conic): the expanded form loses O(1) absolute accuracy for thin diagonal splats far from the strip.  Explicit
// fmaf / __fmul_rn so that the count and emit instantiations cannot be contracted differently by nvcc.
__device__ __forceinline__ float strip_disc(const CullParams cp, const EllipseAux ea, float y) {
	return fmaxf(0.f, fmaf(-ea.det, __fmul_rn(y, y), __fmul_rn(cp.a, cp.qmax)));
}
__device__ __forceinline__ bool strip_xrange(const CullParams cp, const EllipseAux ea, float uy0, float uy1, float &xmin, float &xmax) {
	const float yc = fminf(fmaxf(0.f, uy0), uy1);             // strip row closest to the centre
	if (ea.det_over_a * yc * yc > cp.qmax + 1e-3f) return false;  // min_x q(x, yc) = (c - b^2/a) yc^2
	xmax = ea.xext;
	xmin = -ea.xext;
	if (ea.yhi < uy0 || ea.yhi > uy1) {
		const float y = fminf(fmaxf(ea.yhi, uy0), uy1);
		const float disc = strip_disc(cp, ea, y);
		xmax = (-cp.b * y + fast_sqrt(disc)) * ea.inv_a;
	}
	if (-ea.yhi < uy0 || -ea.yhi > uy1) {
		const float y = fminf(fmaxf(-ea.yhi, uy0), uy1);
		const float disc = strip_disc(cp, ea, y);
		xmin = (-cp.b * y - fast_sqrt(disc)) * ea.inv_a;
	}
	return true;
}

// tile columns [xb, xe) of row `ty` (clipped to [x0, x1)) that can receive a contribution
__device__ __forceinline__ void row_span(const CullParams cp, const EllipseAux ea, int ty, int x0, int x1, int &xb, int &xe) {
	xb = x0;
	xe = x1;
	if (!(cp.qmax < __int_as_float(0x7f800000))) return;  // +inf (non-PD / NaN input): keep the whole rectangle row
	const float uy0 = (float)(ty * SGR_TILE) - cp.my;
	float xmin, xmax;
	if (!strip_xrange(cp, ea, uy0, uy0 + (SGR_TILE - 1), xmin, xmax)) {
		xe = xb;
		return;
	}
	// tile tx covers pixel x in [16 tx, 16 tx + 15]; keep it iff that range meets [mx + xmin, mx + xmax] (0.05 px slack)
	const float lo = (cp.mx + xmin - 0.05f - (SGR_TILE - 1)) * (1.0f / SGR_TILE);
	const float hi = (cp.mx + xmax + 0.05f) * (1.0f / SGR_TILE);
	xb = max(x0, (int)ceilf(fmaxf(lo, -1.0f)));
	xe = min(x1, (int)floorf(fminf(hi, 1.0e6f)) + 1);
	if (xe < xb) xe = xb;
}

// Tile predicates of visit_tiles: which of the culled tiles are counted / emitted.  span(ty, xb, xe) = kept tiles among columns
// [xb, xe) of tile row ty, tile(ty, tx) = whether one is kept.
struct KeepAll {  // every tile (one binning pass per frame)
	static constexpr bool kAll = true;
	__device__ __forceinline__ uint32_t span(int, int xb, int xe) const { return (uint32_t)(xe - xb); }
	__device__ __forceinline__ bool tile(int, int) const { return true; }
};
// Far pass of the saturation split (binning.cu): only the tiles the near pass left unsaturated.  sat[y * (gx + 1) + x] = number of
// unsaturated tiles in rows < y and columns < x (unsat_prefix_kernel), so any rectangle of tiles, a row span included, costs four
// loads.
struct KeepUnsaturated {
	static constexpr bool kAll = false;
	const uint32_t *sat;
	int stride;  // gx + 1
	// unsaturated tiles in rows [y0, y1) x columns [x0, x1) (y0 <= y1, x0 <= x1)
	__device__ __forceinline__ uint32_t rect(int y0, int y1, int x0, int x1) const {
		const uint32_t *a = sat + (size_t)y0 * stride, *b = sat + (size_t)y1 * stride;
		return (b[x1] - b[x0]) - (a[x1] - a[x0]);
	}
	__device__ __forceinline__ uint32_t span(int ty, int xb, int xe) const { return xe > xb ? rect(ty, ty + 1, xb, xe) : 0u; }
	__device__ __forceinline__ bool tile(int ty, int tx) const { return rect(ty, ty + 1, tx, tx + 1) != 0u; }
};

template <bool EMIT, typename KeyT = uint32_t, typename Keep = KeepAll>
__device__ __forceinline__ void visit_tiles(bool active, int x0, int y0, int x1, int y1, const CullParams cp, const Band band,
                                            int gx, uint32_t gauss_idx, uint32_t offset, KeyT *__restrict__ keys,
                                            uint32_t *__restrict__ vals, uint32_t &count, KeyT *stage_keys = nullptr,
                                            uint32_t *stage_vals = nullptr, uint32_t stage_cap = 0, uint32_t warp_first = 0,
                                            uint32_t warp_total = 0, uint32_t *big_list = nullptr, uint32_t *big_count = nullptr,
                                            uint32_t big_tag = 0, const Keep keep = Keep()) {
	const unsigned full = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	if (active) {
		y0 = max(y0, band.begin);
		y1 = min(y1, band.end);
		if (y1 <= y0 || cp.qmax < 0.f) active = false;
	}
	// rows of the rectangle this process actually owns: with a cyclic band (row_step = number of ranks) only every step-th row is
	// walked, so a rectangle that is "large" on one GPU is small per rank at N = 8 — without this every rank deferred (and walked
	// warp-cooperatively) every large splat of the frame, and emit_big_kernel did not scale with N at all
	const int w = active ? (x1 - x0) : 0, h = active ? (y1 - y0 + band.step - 1) / band.step : 0;
	const bool coop = w * h > kCoopArea;
	const EllipseAux ea = ellipse_aux(cp);
	count = 0;
	unsigned todo = __ballot_sync(full, coop);
	if (EMIT && big_list != nullptr && todo != 0u) {
		// Defer large rectangles to emit_big_kernel (one warp per Gaussian, spread over the whole GPU).  In depth order the
		// nearest = largest splats sit next to each other; a warp that had to walk 32 of them serially ran for the whole
		// kernel (ncu: busiest SM 492k cycles vs 234k mean) while the rest of the chip idled.
		const uint32_t n_big = (uint32_t)__popc(todo);
		uint32_t base = 0;
		if (lane == 0) base = atomicAdd(big_count, n_big);
		base = __shfl_sync(full, base, 0);
		if (coop) big_list[base + (uint32_t)__popc(todo & ((1u << lane) - 1u))] = big_tag;
		todo = 0u;
	}
	const bool any_coop = __ballot_sync(full, coop) != 0u;
	// Emission of a warp's 32 (depth-consecutive) Gaussians covers ONE contiguous output range.  When it fits the
	// per-warp shared-memory stage (and no lane needs the cooperative path) the lanes scatter into shared memory and the
	// warp then copies the range out with fully coalesced stores; per-thread global scatter (32 sectors per store
	// instruction) is the fallback.
	const bool staged = EMIT && stage_keys != nullptr && !any_coop && warp_total <= stage_cap;
	if (active && !coop) {
		uint32_t off = offset;
		for (int ty = y0; ty < y1; ty++) {
			if (band.step != 1 && !band_owns(band, ty)) continue;
			int xb, xe;
			row_span(cp, ea, ty, x0, x1, xb, xe);
			if (EMIT) {
				if (!Keep::kAll && keep.span(ty, xb, xe) == 0u) continue;
				if (staged) {
					for (int tx = xb; tx < xe; tx++) {
						if (!Keep::kAll && !keep.tile(ty, tx)) continue;
						stage_keys[off - warp_first] = (KeyT)(ty * gx + tx);
						stage_vals[off - warp_first] = gauss_idx;
						off++;
					}
				} else {
					for (int tx = xb; tx < xe; tx++) {
						if (!Keep::kAll && !keep.tile(ty, tx)) continue;
						keys[off] = (KeyT)(ty * gx + tx);
						vals[off] = gauss_idx;
						off++;
					}
				}
			} else {
				off += keep.span(ty, xb, xe);
			}
		}
		count = off - offset;
	}
	if (staged) {
		__syncwarp();
		for (uint32_t i = lane; i < warp_total; i += 32) {
			keys[warp_first + i] = stage_keys[i];
			vals[warp_first + i] = stage_vals[i];
		}
	}
	while (todo) {
		const int src = __ffs(todo) - 1;
		todo &= todo - 1;
		CullParams c2;
		c2.mx = __shfl_sync(full, cp.mx, src); c2.my = __shfl_sync(full, cp.my, src);
		c2.a = __shfl_sync(full, cp.a, src); c2.b = __shfl_sync(full, cp.b, src);
		c2.c = __shfl_sync(full, cp.c, src); c2.qmax = __shfl_sync(full, cp.qmax, src);
		const EllipseAux ea2 = ellipse_aux(c2);
		const int sx0 = __shfl_sync(full, x0, src), sx1 = __shfl_sync(full, x1, src);
		const int sy0 = __shfl_sync(full, y0, src), sy1 = __shfl_sync(full, y1, src);
		const uint32_t sidx = __shfl_sync(full, gauss_idx, src);
		uint32_t base = __shfl_sync(full, offset, src);
		const uint32_t base0 = base;
		for (int r0 = sy0; r0 < sy1; r0 += 32) {  // 32 rows at a time: one row span per lane
			const int ty = r0 + lane;
			int xb = 0, xe = 0;
			if (ty < sy1 && band_owns(band, ty)) row_span(c2, ea2, ty, sx0, sx1, xb, xe);
			const uint32_t n = keep.span(ty, xb, xe);
			uint32_t incl = n;  // inclusive warp scan of the per-row counts
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) {
				const uint32_t t = __shfl_up_sync(full, incl, o);
				if (lane >= o) incl += t;
			}
			if (EMIT) {
				const int nrows = min(32, sy1 - r0);
				for (int r = 0; r < nrows; r++) {  // all lanes write row r together (coalesced)
					const int rxb = __shfl_sync(full, xb, r), rxe = __shfl_sync(full, xe, r);
					const uint32_t rbase = base + __shfl_sync(full, incl - n, r);
					const uint32_t tile0 = (uint32_t)((r0 + r) * gx);
					if (Keep::kAll) {
						for (int tx = rxb + lane; tx < rxe; tx += 32) {
							keys[rbase + (uint32_t)(tx - rxb)] = (KeyT)(tile0 + (uint32_t)tx);
							vals[rbase + (uint32_t)(tx - rxb)] = sidx;
						}
					} else {  // kept tiles of the row, compacted in ascending column order
						uint32_t pos = rbase;
						for (int t0 = rxb; t0 < rxe; t0 += 32) {
							const int tx = t0 + lane;
							const bool k = tx < rxe && keep.tile(r0 + r, tx);
							const unsigned m = __ballot_sync(full, k);
							if (k) {
								const uint32_t q = pos + (uint32_t)__popc(m & ((1u << lane) - 1u));
								keys[q] = (KeyT)(tile0 + (uint32_t)tx);
								vals[q] = sidx;
							}
							pos += (uint32_t)__popc(m);
						}
					}
				}
			}
			base += __shfl_sync(full, incl, 31);
		}
		if (lane == src) count = base - base0;
	}
}

}  // namespace sgr
