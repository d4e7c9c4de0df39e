// blend_bwd2.cu — two-phase backward blend (the S == 0 fast path; blend_bwd.cu remains the path with feature channels).
//
// blend_bwd.cu is issue-bound and spends a large share of its instructions turning 32 per-pixel values into one per-splat sum
// (13 shuffles + 26 selects + 13 adds + the 12 products per (warp, splat)).  This kernel removes the warp reduction:
//
//   phase 1 (thread = pixel, back-to-front over a batch of 32 splats): the reference's per-pixel recurrences
//            (backward.cu:505-614: T, colour/depth/alpha "behind" accumulators, dL/dalpha) produce just TWO numbers per
//            (pixel, splat) pair,  w = alpha*T  and  q = G*dL/dG,  stored to a [32 splats][256 pixels] shared matrix;
//   phase 2 (thread = (splat, 32-pixel chunk)): every sum the reference accumulates with atomics is linear in w or q:
//              colour/depth grads      sum_p w * dL/dpixel_p
//              moments                 sum_p q * {1, dx, dy, dx^2, dx dy, dy^2}   -> mean2D.xy, conic, opacity (= Sq / o)
//              |.| statistic           sum_p |q| (|a dx + b dy| W/2 + |c dy + b dx| H/2)
//            so each thread walks its chunk of the matrix row (padded rows, conflict free) accumulating 11 registers,
//            the 8 chunk-threads of a splat combine with a 3-step butterfly, and 11 global atomics per (tile, splat) leave
//            the SM — exactly one per component, as in blend_bwd.cu.
// No per-pair shuffles, selects or shared-memory partial slabs.  Same math as blend_bwd.cu up to summation order.
//
// Tried and removed: ONE barrier per batch with a double-buffered (w, q) matrix and triple-buffered records, so that phase 2 of
// batch b overlaps phase 1 of batch b+1.  The shared-memory budget forces 16-splat batches (2 x 32 KB), i.e. 16 phase-2 threads
// per splat, a 4-step butterfly and twice the per-splat fixed cost; it was slower than this kernel, as were 8-splat batches
// (4 CTAs/SM) and 32-splat double-buffered batches (1 CTA/SM).  Smaller batches or fewer registers for more resident warps did
// not help either: the kernel is bound by the NUMBER of instructions it issues, not by latency.
// What did pay: cutting instructions.  Phase 2 accumulates the moments in chunk-local integer pixel coordinates
// (compile-time constants of a fully unrolled loop: 3 FMAs per pixel instead of 8, no coordinate loads, no index rotation — the shared
// arrays are padded instead) and re-centres them once per thread; phase 1 takes exp() as ex2.approx, and falls back to the
// forward's expf only for pairs within a few 2^-22 of alpha = 1/255, so that it blends exactly the pairs the forward blended.
#include "sgr_common.cuh"

namespace sgr {

constexpr int kB2 = 32;  // splats per batch
// o G with ex2.approx: at or above kAlphaPass the forward's expf surely gives alpha >= 1/255, below kAlphaSkip surely not
constexpr float kAlphaPass = (1.0f / 255.0f) * (1.0f + 0x1p-16f);
constexpr float kAlphaSkip = (1.0f / 255.0f) * (1.0f - 0x1p-16f);
constexpr uint32_t kRec2 = 48;
// Shared-memory map.  Phase 2 reads pixel i of chunk c (= the 8x4 block of warp c) at a COMPILE-TIME offset, so the 8 chunk-threads
// of a splat (consecutive lanes) must land in different banks by layout, not by rotating the index: each 32-pixel chunk is padded by one
// element (float2 rows: 66 words -> lanes 2 banks apart; float4 pixel gradients: 132 words -> lanes 4 banks apart) and the rows of
// consecutive splats are 528 words = 16 banks apart, so a half-warp (2 splats x 8 chunks) of 8-byte loads and a quarter-warp of 16-byte
// loads are conflict free.
constexpr uint32_t kWQChunk = 33 * 8;                     // bytes per (splat, chunk): 32 x float2 + pad
constexpr uint32_t kWQRow = 8 * kWQChunk;                 // bytes per splat
constexpr uint32_t kPixChunk = 33 * 16;                   // bytes per chunk of float4 pixel gradients + pad
constexpr uint32_t kOffWQ = 0;                            // float2 [kB2][8][33]   (w, q)
constexpr uint32_t kOffPix = kB2 * kWQRow;                // float4 [8][33]        dL/dpixel rgb, dL/dpixel depth
constexpr uint32_t kOffRec = kOffPix + 8 * kPixChunk;     // [2][kB2 * 48]         staged GaussRec
constexpr uint32_t kOffId = kOffRec + 2 * kB2 * kRec2;    // u32 [2][kB2]
constexpr uint32_t kOffMask = kOffId + 2 * kB2 * 4;       // u32 [8]               per-warp "slot has contributions" bits
constexpr uint32_t kSmem2 = kOffMask + 8 * 4;             // 75168 B: 3 CTAs/SM

__device__ __forceinline__ float4 ld4(uint32_t a) {
	float4 v;
	asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
	return v;
}
__device__ __forceinline__ float2 ld2(uint32_t a) {
	float2 v;
	asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a));
	return v;
}
__device__ __forceinline__ uint32_t ldu(uint32_t a) {
	uint32_t v;
	asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
	return v;
}
__device__ __forceinline__ void st4(uint32_t a, float4 v) {
	asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void st2(uint32_t a, float x, float y) { asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory"); }
__device__ __forceinline__ void stu(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

template <bool kFastExp>
__global__ void __launch_bounds__(256, 3) blend_bwd2_kernel(const FrameDev f, const uint2 *__restrict__ ranges,
                                                         const uint32_t *__restrict__ point_list, const GaussRec *__restrict__ rec,
                                                         const uint32_t *__restrict__ n_contrib, const uint32_t *__restrict__ tile_max_contrib,
                                                         const float *__restrict__ alphas, const float *__restrict__ dL_dpixels,
                                                         const float *__restrict__ dL_dpixel_depths, const float *__restrict__ dL_dalphas,
                                                         float *__restrict__ grad2d) {
	extern __shared__ __align__(16) unsigned char smem2[];
	const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
	const int tile_x = blockIdx.x, tile_y = f.band.begin + blockIdx.y * f.band.step;
	const int tile = tile_y * f.gx + tile_x;
	const int n_eff = (int)tile_max_contrib[tile];
	if (n_eff == 0) return;
	const int px = tile_x * SGR_TILE + (warp & 1) * 8 + (lane & 7);
	const int py = tile_y * SGR_TILE + (warp >> 1) * 4 + (lane >> 3);
	const bool inside = px < f.W && py < f.H;
	const size_t HW = (size_t)f.W * f.H;
	const size_t pix_id = (size_t)f.W * py + px;
	const float2 pixf = make_float2((float)px, (float)py);
	const uint32_t list0 = ranges[tile].x;
	const int nb = (n_eff + kB2 - 1) / kB2;
	const uint32_t sb = (uint32_t)__cvta_generic_to_shared(smem2);

	const float T_final = inside ? (1 - alphas[pix_id]) : 0;
	float T = T_final;
	const int last_contributor = inside ? (int)n_contrib[pix_id] : 0;
	float dL_dpixel[3] = {0, 0, 0};
	float behind = 0.f, g_last = 0.f, last_alpha = 0.f;  // scalar form of the reference's accum_rec / last_color family
	float dL_dpixel_depth = 0, dL_dalpha_px = 0;
	if (inside) {
#pragma unroll
		for (int c = 0; c < 3; c++) dL_dpixel[c] = dL_dpixels[c * HW + pix_id];
		dL_dpixel_depth = dL_dpixel_depths[pix_id];
		dL_dalpha_px = dL_dalphas[pix_id];
	}
	float bg_dot_dpixel = 0;
#pragma unroll
	for (int c = 0; c < 3; c++) bg_dot_dpixel += f.bg[c] * dL_dpixel[c];
	const float kW = 0.5f * f.W, kH = 0.5f * f.H;  // d(pixel)/d(NDC), reference backward.cu:501-502
	st4(sb + kOffPix + (uint32_t)warp * kPixChunk + (uint32_t)lane * 16u, make_float4(dL_dpixel[0], dL_dpixel[1], dL_dpixel[2], dL_dpixel_depth));

	// staging: 4 threads per record (q0, q1, q2, id), threads 0..127; slot j of batch b <-> list index (n_eff - b*B) - 1 - j
	const int ld_slot = tid >> 2, ld_part = tid & 3;
	float4 rq = make_float4(0, 0, 0, 0);
	uint32_t rid = 0;
	auto fetch = [&](int b) {
		const int idx = n_eff - b * kB2 - 1 - ld_slot;
		if (ld_slot < kB2 && idx >= 0) {
			rid = point_list[list0 + idx];
			if (ld_part < 3) rq = reinterpret_cast<const float4 *>(rec + rid)[ld_part];
		}
	};
	auto stash = [&](int buf) {
		if (ld_slot < kB2) {
			if (ld_part < 3) st4(sb + kOffRec + (uint32_t)buf * (kB2 * kRec2) + (uint32_t)ld_slot * kRec2 + (uint32_t)ld_part * 16u, rq);
			else stu(sb + kOffId + (uint32_t)(buf * kB2 + ld_slot) * 4u, rid);
		}
	};
	fetch(0);
	stash(0);

	// phase-2 role of this thread
	const int p2_slot = tid >> 3, p2_chunk = tid & 7;
	// pixel (u, v) of chunk c sits at (cx0 + u, cy0 + v), u < 8, v < 4 — the lane order of phase 1
	const float cx0 = (float)(tile_x * SGR_TILE + (p2_chunk & 1) * 8), cy0 = (float)(tile_y * SGR_TILE + (p2_chunk >> 1) * 4);

	for (int b = 0; b < nb; b++) {
		__syncthreads();  // record buffer b&1 published; phase 2 of the previous batch is done with s_wq / s_mask
		if (b + 1 < nb) fetch(b + 1);
		const int buf = b & 1;
		const int hi = n_eff - b * kB2;  // list position (1-based) of slot 0
		const int cnt = min(kB2, hi);
		const uint32_t rbase = sb + kOffRec + (uint32_t)buf * (kB2 * kRec2);

		// ---------------- phase 1: per-pixel recurrences -> (w, q) ----------------
		uint32_t wmask = 0u;
		uint32_t a = rbase;
		uint32_t wq_addr = sb + kOffWQ + (uint32_t)warp * kWQChunk + (uint32_t)lane * 8u;
		for (int j = 0; j < cnt; j++, a += kRec2, wq_addr += kWQRow) {
			const int contributor = hi - 1 - j;
			bool valid = contributor < last_contributor;
			float q = 0.f, w = 0.f;
			if (valid) {
				const float4 q0 = ld4(a);       // pix.x, pix.y, conic.xx, conic.xy
				const float4 q1 = ld4(a + 16);  // conic.yy, opacity, power_min, depth
				const float2 d = make_float2(q0.x - pixf.x, q0.y - pixf.y);
				const float power = -0.5f * (q0.z * d.x * d.x + q1.x * d.y * d.y) - q0.w * d.x * d.y;
				valid = !(power > 0.0f) && !(power < q1.z);
				if (valid) {
					float G;
					if (kFastExp) {
						// ex2.approx of power * log2(e): 2 instructions instead of expf's 10.  Its VALUE is within
						// 2^-21 + |power| 2^-23 relative of the forward's expf (ex2.approx and expf 2^-22 each, the rounded argument
						// and log2(e) |power| 2^-24 each), inside the gradient bounds.  But the forward's DECISION alpha < 1/255
						// must be taken again exactly: a pair the forward blended and this kernel skipped (or the reverse) drops (or
						// invents) its own gradient and puts T off by ~1/255 for every pair in front of it.  So a pair passes at once
						// only when o G clears 1/255 by 2^-16 relative (more than the difference for |power| <= 28, i.e. for any
						// opacity below ~5e9, since |power| = ln(255 o) at the threshold); below that window it is skipped, and
						// inside it G is recomputed with the forward's expf.  The window test costs blend_bwd2 about 3.5 % on config C.
						// (fminf(0.99, .) does not move a decision against 1/255; NaN passes in both kernels.)
						// SGR_BWD2_EXPF=1 selects expf everywhere.
						asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(G) : "f"(power * 1.4426950408889634f));
						valid = !(q1.y * G < kAlphaPass);
						if (!valid && !(q1.y * G < kAlphaSkip)) {
							G = expf(power);
							valid = !(q1.y * G < 1.0f / 255.0f);
						}
					} else {
						G = expf(power);
						valid = !(fminf(0.99f, q1.y * G) < 1.0f / 255.0f);
					}
					if (valid) {
						const float alpha = fminf(0.99f, q1.y * G);
						const float4 q2 = ld4(a + 32);  // r, g, b, clamp bits
						// 1/(1-alpha), alpha <= 0.99: hardware reciprocal + one Newton step (<= 1 ulp) = 3 instructions instead of
						// the ~8 of an IEEE division with its special-case path; serves both T/(1-a) and T_final/(1-a)
						const float oma = 1.f - alpha;  // in [0.01, 1]: no special cases to guard
						float r0;
						asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r0) : "f"(oma));
						const float inv = fmaf(r0, fmaf(-oma, r0, 1.0f), r0);
						T = T * inv;
						w = alpha * T;
						// The reference keeps one "value behind" accumulator per blended quantity (3 colours, depth, the constant 1
						// of the alpha channel), all with the SAME recurrence  acc <- last_alpha*last_q + (1-last_alpha)*acc, and
						// only ever uses them dotted with this pixel's upstream gradients (backward.cu:563-602).  The dot product
						// commutes with the recurrence, so ONE scalar suffices:
						//   g_i = c_i . dL/dC + depth_i * dL/dD + 1 * dL/dA,   A <- last_alpha * g_last + (1-last_alpha) * A,
						//   dL/dalpha_i = (g_i - A) * T_i + bg term.
						const float g = q2.x * dL_dpixel[0] + q2.y * dL_dpixel[1] + q2.z * dL_dpixel[2] + q1.w * dL_dpixel_depth + dL_dalpha_px;
						behind = last_alpha * g_last + (1.f - last_alpha) * behind;
						g_last = g;
						last_alpha = alpha;
						const float dL_dopa = (g - behind) * T + (-T_final * inv) * bg_dot_dpixel;
						q = q1.y * (G * dL_dopa);  // G * dL/dG
					}
				}
			}
			if (__ballot_sync(0xffffffffu, valid) != 0u) {  // warp-uniform
				st2(wq_addr, w, q);
				wmask |= 1u << j;
			}
		}
		if (lane == 0) stu(sb + kOffMask + (uint32_t)warp * 4u, wmask);
		__syncthreads();

		// ---------------- phase 2: per-splat sums over the tile's pixels ----------------
		{
			float Sq = 0.f, Sx = 0.f, Sy = 0.f, Sxx = 0.f, Sxy = 0.f, Syy = 0.f, Sabs = 0.f, Cr = 0.f, Cg = 0.f, Cb = 0.f, Cd = 0.f;
			const bool live = p2_slot < cnt && ((ldu(sb + kOffMask + (uint32_t)p2_chunk * 4u) >> p2_slot) & 1u);
			float4 r0 = make_float4(0, 0, 0, 0), r1 = r0;
			if (live) {
				r0 = ld4(rbase + (uint32_t)p2_slot * kRec2);
				r1 = ld4(rbase + (uint32_t)p2_slot * kRec2 + 16);
				const uint32_t row = sb + kOffWQ + (uint32_t)p2_slot * kWQRow + (uint32_t)p2_chunk * kWQChunk;
				const uint32_t pixb = sb + kOffPix + (uint32_t)p2_chunk * kPixChunk;
				// Moments are accumulated in the chunk's own integer pixel coordinates (u, v) — compile-time constants of the unrolled
				// loops, so a pixel costs 3 FMAs instead of 8 and no coordinate load — and re-centred on the splat once at the end:
				// d = (D - u, E - v) with (D, E) = centre - chunk origin.  |D - dx| <= 7, so the re-centring never cancels catastrophically.
				const float D = r0.x - cx0, E = r0.y - cy0;
				const float ca_ = r0.z, cb_ = r0.w, cc_ = r1.x;
				const float A0 = fmaf(ca_, D, cb_ * E), B0 = fmaf(cc_, E, cb_ * D);  // a dx + b dy and c dy + b dx at (u, v) = (0, 0)
				float M0 = 0.f, Mu = 0.f, Mv = 0.f, Muu = 0.f, Muv = 0.f, Mvv = 0.f;
#pragma unroll
				for (int v = 0; v < 4; v++) {
					float R0 = 0.f, R1 = 0.f, R2 = 0.f;
					const float Av = fmaf(-cb_, (float)v, A0), Bv = fmaf(-cc_, (float)v, B0);
#pragma unroll
					for (int u = 0; u < 8; u++) {
						const uint32_t i = (uint32_t)(v * 8 + u);
						const float2 wq = ld2(row + i * 8u);
						const float4 pg = ld4(pixb + i * 16u);
						R0 += wq.y;
						R1 = fmaf(wq.y, (float)u, R1);
						R2 = fmaf(wq.y, (float)(u * u), R2);
						const float t1 = fmaf(-ca_, (float)u, Av), t2 = fmaf(-cb_, (float)u, Bv);
						Sabs = fmaf(fabsf(wq.y), fmaf(fabsf(t1), kW, fabsf(t2) * kH), Sabs);
						Cr = fmaf(wq.x, pg.x, Cr);
						Cg = fmaf(wq.x, pg.y, Cg);
						Cb = fmaf(wq.x, pg.z, Cb);
						Cd = fmaf(wq.x, pg.w, Cd);
					}
					M0 += R0;
					Mv = fmaf(R0, (float)v, Mv);
					Mvv = fmaf(R0, (float)(v * v), Mvv);
					Mu += R1;
					Muv = fmaf(R1, (float)v, Muv);
					Muu += R2;
				}
				Sq = M0;
				Sx = fmaf(D, M0, -Mu);
				Sy = fmaf(E, M0, -Mv);
				Sxx = fmaf(D, fmaf(D, M0, -2.f * Mu), Muu);
				Syy = fmaf(E, fmaf(E, M0, -2.f * Mv), Mvv);
				Sxy = fmaf(D, fmaf(E, M0, -Mv), fmaf(-E, Mu, Muv));
			}
			// combine the 8 chunk-threads of each splat (consecutive lanes) — all lanes take part
			const unsigned any_live = __ballot_sync(0xffffffffu, live);
			if (any_live) {
#pragma unroll
				for (int o = 1; o < 8; o <<= 1) {
					Sq += __shfl_xor_sync(0xffffffffu, Sq, o); Sx += __shfl_xor_sync(0xffffffffu, Sx, o);
					Sy += __shfl_xor_sync(0xffffffffu, Sy, o); Sxx += __shfl_xor_sync(0xffffffffu, Sxx, o);
					Sxy += __shfl_xor_sync(0xffffffffu, Sxy, o); Syy += __shfl_xor_sync(0xffffffffu, Syy, o);
					Sabs += __shfl_xor_sync(0xffffffffu, Sabs, o); Cr += __shfl_xor_sync(0xffffffffu, Cr, o);
					Cg += __shfl_xor_sync(0xffffffffu, Cg, o); Cb += __shfl_xor_sync(0xffffffffu, Cb, o);
					Cd += __shfl_xor_sync(0xffffffffu, Cd, o);
				}
				// is any chunk of this splat live?  (bits of the 8 lanes of this slot in the ballot)
				const unsigned grp = (any_live >> (lane & 24)) & 0xffu;
				// the conic / opacity of the splat: lanes that were not live did not load the record (all lanes shuffle)
				const int srcl = grp != 0u ? (lane & 24) + (__ffs(grp) - 1) : lane;
				const float ca = __shfl_sync(0xffffffffu, r0.z, srcl), cb = __shfl_sync(0xffffffffu, r0.w, srcl);
				const float cc = __shfl_sync(0xffffffffu, r1.x, srcl), op = __shfl_sync(0xffffffffu, r1.y, srcl);
				if (grp != 0u && p2_slot < cnt) {
					const uint32_t gid = ldu(sb + kOffId + (uint32_t)(buf * kB2 + p2_slot) * 4u);
					float *dst = grad2d + (size_t)gid * 12;
					float o0, o1 = 0.f;
					switch (p2_chunk) {  // lane c of the group writes components c and c + 8
						case 0: o0 = -kW * (ca * Sx + cb * Sy); o1 = Cg; break;
						case 1: o0 = -kH * (cc * Sy + cb * Sx); o1 = Cb; break;
						case 2: o0 = Sabs; o1 = Cd; break;
						case 3: o0 = -0.5f * Sxx; break;
						case 4: o0 = -0.5f * Sxy; break;
						case 5: o0 = -0.5f * Syy; break;
						case 6: o0 = (op != 0.f) ? Sq / op : 0.f; break;
						default: o0 = Cr; break;
					}
					atomicAdd(dst + p2_chunk, o0);
					if (p2_chunk < 3) atomicAdd(dst + 8 + p2_chunk, o1);
				}
			}
		}
		if (b + 1 < nb) stash((b + 1) & 1);
	}
}

cudaError_t launch_blend_bwd2(const FrameDev &f, GeomView g, BinView b, ImgView img, const float *out_alpha, const float *dL_dcolor,
                              const float *dL_ddepth, const float *dL_dalpha, float *grad2d, cudaStream_t st, bool grad2d_zeroed) {
	if (f.P == 0) return cudaSuccess;
	// (grad2d_zeroed: sgr_sharded_forward already cleared the rows this band can touch — see count_tiles_kernel)
	cudaError_t e = grad2d_zeroed ? cudaSuccess : cudaMemsetAsync(grad2d, 0, (size_t)f.P * 12 * sizeof(float), st);
	if (e != cudaSuccess) return e;
	const int rows = band_rows(f.band);
	if (rows <= 0 || f.gx <= 0) return cudaSuccess;
	static const bool fast_exp = [] { const char *v = getenv("SGR_BWD2_EXPF"); return !(v && atoi(v) == 1); }();
	static std::atomic<uint64_t> configured{0}, configured_fast{0};
	count_launch();
	if (fast_exp) {
		if ((e = ensure_dynamic_smem(blend_bwd2_kernel<true>, (int)kSmem2, configured_fast)) != cudaSuccess) return e;
		blend_bwd2_kernel<true><<<dim3(f.gx, rows), 256, kSmem2, st>>>(f, img.ranges, b.vals_out, g.rec, img.n_contrib, img.tile_max_contrib,
		                                                              out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, grad2d);
	} else {
		if ((e = ensure_dynamic_smem(blend_bwd2_kernel<false>, (int)kSmem2, configured)) != cudaSuccess) return e;
		blend_bwd2_kernel<false><<<dim3(f.gx, rows), 256, kSmem2, st>>>(f, img.ranges, b.vals_out, g.rec, img.n_contrib, img.tile_max_contrib,
		                                                               out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, grad2d);
	}
	return cudaGetLastError();
}

}  // namespace sgr
