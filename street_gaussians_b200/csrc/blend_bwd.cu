// blend_bwd.cu — per-tile back-to-front backward blend.
//
// Replaces the reference's BACKWARD::renderCUDA<3,20> (DGR/cuda_rasterizer/backward.cu:415-641).  The per-pixel
// recurrences (T, the "colour behind" accumulators, dL/dalpha) are the reference's; what changes is how the per-Gaussian
// sums are formed and how they leave the SM.  The reference issues 11 scalar atomicAdd per contributing (pixel, splat)
// pair, all 256 threads of a tile hammering the same 44 bytes.  Here:
//   1. MOMENTS instead of products.  With q = G * dL/dG, the six geometry gradients are linear in the pixel moments
//      Sx = sum q dx, Sy = sum q dy, Sxx = sum q dx^2, Sxy = sum q dx dy, Syy = sum q dy^2:
//        dL/dmean2D = -(W/2)(a Sx + b Sy), -(H/2)(c Sy + b Sx);   dL/dconic = -Sxx/2, -Sxy/2, -Syy/2
//      so the conic (a, b, c) is applied ONCE per (tile, splat) in the flush instead of once per pair;
//   2. per splat, each warp (a compact 8x4 pixel block) reduces its 32 lanes with a TRANSPOSED butterfly: the 12 values
//      are reduced with 6+3+2+1+1 = 13 shuffles (instead of 5 per value = 55); warps in which no lane contributes
//      (ballot == 0) skip the reduction altogether;
//   3. the 8 warps park their partial sums in a private shared-memory slab s_part[warp][slot][12] (plain stores, no
//      atomics, no zero-fill: a 64-bit per-warp mask says which slots are live);
//   4. once per 64-splat batch, 4 threads per splat add up the live slabs, apply the conic and issue ONE global atomic
//      per (tile, splat, component): R*11 reductions per frame in total instead of (contributing pairs)*11.
// The list is walked from tile_max_contrib (deepest position any pixel of the tile reached in the forward pass), so the
// unreachable tail of a saturated tile's list is never touched.  The kernel is issue-bound (records and
// lists are L2 hits, DRAM traffic is small): the inner loop uses one running shared address with immediate-offset LDS.128 and one IEEE
// reciprocal shared by the reference's two divisions by (1 - alpha).
#include "sgr_common.cuh"

namespace sgr {

constexpr int kBwdBatch = 64;
constexpr int kNComp = 12;  // 11 used + 1 pad (see sgr.h: grad2d layout)
constexpr uint32_t kRecBytesB = 48;

__device__ __forceinline__ float4 lds128b(uint32_t addr) {
	float4 v;
	asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
	return v;
}
__device__ __forceinline__ void sts128b(uint32_t addr, float4 v) {
	asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void sts32b(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }

// Transposed warp reduction of 12 values per lane (v[11] is the pad): afterwards lane L (bit0 == 0, not (b2 && b1)) holds
// the 32-lane sum of component  6*b4 + 3*b3 + (b2 ? 2 : b1)  in the return value.
__device__ __forceinline__ float warp_reduce12_transposed(const float (&v)[12], const int lane) {
	const unsigned full = 0xffffffffu;
	float a[6], b[3];
	{
		const bool up = lane & 16;
#pragma unroll
		for (int i = 0; i < 6; i++) {
			const float send = up ? v[i] : v[i + 6];
			const float keep = up ? v[i + 6] : v[i];
			a[i] = keep + __shfl_xor_sync(full, send, 16);
		}
	}
	{
		const bool up = lane & 8;
#pragma unroll
		for (int i = 0; i < 3; i++) {
			const float send = up ? a[i] : a[i + 3];
			const float keep = up ? a[i + 3] : a[i];
			b[i] = keep + __shfl_xor_sync(full, send, 8);
		}
	}
	float r0, r1;
	{
		const bool up = lane & 4;  // lower half keeps b[0], b[1]; upper half keeps b[2]
		const float send0 = up ? b[0] : b[2];
		const float keep0 = up ? b[2] : b[0];
		r0 = keep0 + __shfl_xor_sync(full, send0, 4);
		const float send1 = up ? b[1] : 0.f;
		const float keep1 = up ? 0.f : b[1];
		r1 = keep1 + __shfl_xor_sync(full, send1, 4);
	}
	float x;
	{
		const bool up = lane & 2;
		const float send = up ? r0 : r1;
		const float keep = up ? r1 : r0;
		x = keep + __shfl_xor_sync(full, send, 2);
	}
	x += __shfl_xor_sync(full, x, 1);
	return x;
}

template <int SCH>
__global__ void __launch_bounds__(256) blend_bwd_kernel(const FrameDev f, const uint2 *__restrict__ ranges,
                                                        const uint32_t *__restrict__ point_list, const GaussRec *__restrict__ rec,
                                                        const float *__restrict__ semantics, const uint32_t *__restrict__ n_contrib,
                                                        const uint32_t *__restrict__ tile_max_contrib, const float *__restrict__ alphas,
                                                        const float *__restrict__ dL_dpixels, const float *__restrict__ dL_dpixel_depths,
                                                        const float *__restrict__ dL_dalphas, const float *__restrict__ dL_dpixel_sems,
                                                        float *__restrict__ grad2d, float *__restrict__ dL_dsemantics) {
	__shared__ __align__(16) unsigned char s_rec[2][kBwdBatch * kRecBytesB];
	__shared__ uint32_t s_id[2][kBwdBatch];
	__shared__ __align__(16) float s_part[8][kBwdBatch][kNComp];
	__shared__ unsigned long long s_mask[8];

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
	const int nb = (n_eff + kBwdBatch - 1) / kBwdBatch;
	const uint32_t srec = (uint32_t)__cvta_generic_to_shared(&s_rec[0][0]);
	const uint32_t spart = (uint32_t)__cvta_generic_to_shared(&s_part[0][0][0]);
	constexpr uint32_t kBufBytes = kBwdBatch * kRecBytesB;

	const float T_final = inside ? (1 - alphas[pix_id]) : 0;
	float T = T_final;
	const int last_contributor = inside ? (int)n_contrib[pix_id] : 0;
	float accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, dL_dpixel[3] = {0, 0, 0};
	float accum_depth_rec = 0, last_depth = 0, accum_alpha_rec = 0, last_alpha = 0;
	float dL_dpixel_depth = 0, dL_dalpha_px = 0;
	float accum_sem[SCH > 0 ? SCH : 1], last_sem[SCH > 0 ? SCH : 1], dL_dsem_px[SCH > 0 ? SCH : 1];
#pragma unroll
	for (int c = 0; c < (SCH > 0 ? SCH : 1); c++) accum_sem[c] = last_sem[c] = dL_dsem_px[c] = 0.f;
	if (inside) {
#pragma unroll
		for (int c = 0; c < 3; c++) dL_dpixel[c] = dL_dpixels[c * HW + pix_id];
		dL_dpixel_depth = dL_dpixel_depths[pix_id];
		dL_dalpha_px = dL_dalphas[pix_id];
#pragma unroll
		for (int c = 0; c < SCH; c++)
			if (c < f.S) dL_dsem_px[c] = dL_dpixel_sems[c * HW + pix_id];
	}
	float bg_dot_dpixel = 0;
#pragma unroll
	for (int c = 0; c < 3; c++) bg_dot_dpixel += f.bg[c] * dL_dpixel[c];
	const float kW = 0.5f * f.W, kH = 0.5f * f.H;  // d(pixel)/d(NDC), reference backward.cu:501-502

	// which component does this lane hold after the transposed reduction, and where does it park it
	const int comp = ((lane >> 4) & 1) * 6 + ((lane >> 3) & 1) * 3 + ((lane & 4) ? 2 : ((lane >> 1) & 1));
	const bool writer = ((lane & 1) == 0) && !((lane & 4) && (lane & 2));
	const uint32_t part_lane = spart + (uint32_t)(warp * kBwdBatch * kNComp + comp) * 4u;

	// staging: 4 threads per record (q0, q1, q2, id); slot j of batch b <-> list index (n_eff - b*B) - 1 - j
	const int ld_slot = tid >> 2, ld_part = tid & 3;
	float4 rq = make_float4(0, 0, 0, 0);
	uint32_t rid = 0;
	auto fetch = [&](int b) {
		const int idx = n_eff - b * kBwdBatch - 1 - ld_slot;
		if (idx >= 0) {
			rid = point_list[list0 + idx];
			if (ld_part < 3) rq = reinterpret_cast<const float4 *>(rec + rid)[ld_part];
		}
	};
	auto stash = [&](int buf) {
		if (ld_part < 3) sts128b(srec + (uint32_t)buf * kBufBytes + (uint32_t)ld_slot * kRecBytesB + (uint32_t)ld_part * 16u, rq);
		else s_id[buf][ld_slot] = rid;
	};
	fetch(0);
	stash(0);

	for (int b = 0; b < nb; b++) {
		__syncthreads();  // buffer b&1 is published; s_part / s_mask of the previous batch have been consumed
		if (b + 1 < nb) fetch(b + 1);
		const int buf = b & 1;
		const int hi = n_eff - b * kBwdBatch;  // list position (1-based) of slot 0
		const int cnt = min(kBwdBatch, hi);
		unsigned long long wmask = 0ull;
		const uint32_t a0 = srec + (uint32_t)buf * kBufBytes;
		uint32_t a = a0;
		uint32_t pa = part_lane;
		for (int j = 0; j < cnt; j++, a += kRecBytesB, pa += kNComp * 4u) {
			const int contributor = hi - 1 - j;  // 0-based list index of this slot
			bool valid = contributor < last_contributor;
			float q = 0.f, w = 0.f, gdo = 0.f;  // G*dL/dG, alpha*T, G*dL/dalpha — zero on lanes that do not contribute
			float2 d = make_float2(0.f, 0.f);
			float4 q0 = make_float4(0.f, 0.f, 0.f, 0.f), q1 = q0;
			if (valid) {
				q0 = lds128b(a);       // pix.x, pix.y, conic.xx, conic.xy
				q1 = lds128b(a + 16);  // conic.yy, opacity, power_min, depth
				d = make_float2(q0.x - pixf.x, q0.y - pixf.y);
				const float power = -0.5f * (q0.z * d.x * d.x + q1.x * d.y * d.y) - q0.w * d.x * d.y;
				valid = !(power > 0.0f) && !(power < q1.z);  // q1.z: conservative bound below which alpha < 1/255 for sure
				if (valid) {
					const float G = expf(power);
					const float alpha = fminf(0.99f, q1.y * G);
					valid = !(alpha < 1.0f / 255.0f);
					if (valid) {
						const float4 q2 = lds128b(a + 32);  // r, g, b, clamp bits
						const float inv = 1.0f / (1.f - alpha);  // one IEEE division serves T/(1-a) and T_final/(1-a)
						T = T * inv;
						w = alpha * T;
						const float oml = 1.f - last_alpha;
						float dL_dopa = 0.0f;
						const float col[3] = {q2.x, q2.y, q2.z};
#pragma unroll
						for (int ch = 0; ch < 3; ch++) {
							accum_rec[ch] = last_alpha * last_color[ch] + oml * accum_rec[ch];
							last_color[ch] = col[ch];
							dL_dopa += (col[ch] - accum_rec[ch]) * dL_dpixel[ch];
						}
						if (SCH > 0) {
							const float *sp = semantics + (size_t)s_id[buf][j] * f.S;
#pragma unroll
							for (int ch = 0; ch < SCH; ch++)
								if (ch < f.S) {
									const float s = __ldg(sp + ch);
									accum_sem[ch] = last_alpha * last_sem[ch] + oml * accum_sem[ch];
									last_sem[ch] = s;
									dL_dopa += (s - accum_sem[ch]) * dL_dsem_px[ch];
								}
						}
						accum_depth_rec = last_alpha * last_depth + oml * accum_depth_rec;
						last_depth = q1.w;
						dL_dopa += (q1.w - accum_depth_rec) * dL_dpixel_depth;
						accum_alpha_rec = last_alpha + oml * accum_alpha_rec;
						dL_dopa += (1 - accum_alpha_rec) * dL_dalpha_px;
						dL_dopa *= T;
						last_alpha = alpha;
						dL_dopa += (-T_final * inv) * bg_dot_dpixel;
						gdo = G * dL_dopa;
						q = q1.y * gdo;  // G * (opacity * dL/dalpha) = G * dL/dG
					}
				}
			}
			const unsigned any = __ballot_sync(0xffffffffu, valid);
			if (any == 0u) continue;  // warp-uniform
			// lanes that do not contribute carry q = w = gdo = 0, so every value below is an exact zero for them
			const float ca = q0.z, cb = q0.w, cc = q1.x;
			float v[12];
			const float qx = q * d.x, qy = q * d.y;
			v[0] = qx;
			v[1] = qy;
			v[2] = fabsf(q) * (fabsf(ca * d.x + cb * d.y) * kW + fabsf(cc * d.y + cb * d.x) * kH);
			v[3] = qx * d.x;
			v[4] = qx * d.y;
			v[5] = qy * d.y;
			v[6] = gdo;
			v[7] = w * dL_dpixel[0];
			v[8] = w * dL_dpixel[1];
			v[9] = w * dL_dpixel[2];
			v[10] = w * dL_dpixel_depth;
			v[11] = 0.f;
			const float total = warp_reduce12_transposed(v, lane);
			if (writer) sts32b(pa, total);
			wmask |= 1ull << j;
			if (SCH > 0) {
				// feature channels: plain butterfly per channel, one global atomic per (warp, splat, channel)
				const uint32_t gid = s_id[buf][j];
#pragma unroll
				for (int ch = 0; ch < SCH; ch++)
					if (ch < f.S) {
						float t = w * dL_dsem_px[ch];
#pragma unroll
						for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
						if (lane == 0) atomicAdd(dL_dsemantics + (size_t)gid * f.S + ch, t);
					}
			}
		}
		if (lane == 0) s_mask[warp] = wmask;
		__syncthreads();
		// flush: thread -> (slot = tid/4, components 3*(tid%4) .. +2); applies the conic to the moments
		{
			const int slot = tid >> 2, part = tid & 3, c0 = part * 3;
			if (slot < cnt) {
				float s0 = 0.f, s1 = 0.f, s2 = 0.f;
				bool live = false;
#pragma unroll
				for (int wv = 0; wv < 8; wv++)
					if ((s_mask[wv] >> slot) & 1ull) {
						live = true;
						s0 += s_part[wv][slot][c0];
						s1 += s_part[wv][slot][c0 + 1];
						s2 += s_part[wv][slot][c0 + 2];
					}
				if (live) {
					float o0 = s0, o1 = s1, o2 = s2;
					if (part == 0) {  // (Sx, Sy, Sabs) -> dL/dmean2D
						const float4 r0 = lds128b(a0 + (uint32_t)slot * kRecBytesB);
						const float4 r1 = lds128b(a0 + (uint32_t)slot * kRecBytesB + 16);
						o0 = -kW * (r0.z * s0 + r0.w * s1);
						o1 = -kH * (r1.x * s1 + r0.w * s0);
					} else if (part == 1) {  // (Sxx, Sxy, Syy) -> dL/dconic
						o0 = -0.5f * s0; o1 = -0.5f * s1; o2 = -0.5f * s2;
					}
					float *dst = grad2d + (size_t)s_id[buf][slot] * kNComp + c0;
					atomicAdd(dst, o0);
					atomicAdd(dst + 1, o1);
					if (c0 + 2 < 11) atomicAdd(dst + 2, o2);
				}
			}
		}
		if (b + 1 < nb) stash((b + 1) & 1);
	}
}

cudaError_t launch_blend_bwd(const FrameDev &f, GeomView g, BinView b, ImgView img, const float *semantics,
                             const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                             const float *dL_dsem, float *grad2d, float *dL_dsemantics, cudaStream_t st, bool grad2d_zeroed,
                             const uint32_t *reached) {
	if (f.P == 0) return cudaSuccess;
	if (f.S <= 0)  // two-phase fast path
		return launch_blend_bwd2(f, g, b, img, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, grad2d, st, grad2d_zeroed, reached);
	cudaError_t e = cudaMemsetAsync(grad2d, 0, (size_t)f.P * kNComp * sizeof(float), st);
	if (e != cudaSuccess) return e;
	if (f.S > 0 && (e = cudaMemsetAsync(dL_dsemantics, 0, (size_t)f.P * f.S * sizeof(float), st)) != cudaSuccess) return e;
	const int rows = band_rows(f.band);
	if (rows <= 0 || f.gx <= 0) return cudaSuccess;
	const dim3 grid(f.gx, rows);
	count_launch();
#define SGR_LAUNCH_BWD(SCH)                                                                                                      \
	blend_bwd_kernel<SCH><<<grid, 256, 0, st>>>(f, img.ranges, b.vals_out, g.rec, semantics, img.n_contrib, img.tile_max_contrib, \
	                                            out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, dL_dsem, grad2d, dL_dsemantics)
	if (f.S <= 0)
		SGR_LAUNCH_BWD(0);
	else if (f.S <= 4)
		SGR_LAUNCH_BWD(4);
	else if (f.S <= 8)
		SGR_LAUNCH_BWD(8);
	else if (f.S <= 16)
		SGR_LAUNCH_BWD(16);
	else
		SGR_LAUNCH_BWD(32);
#undef SGR_LAUNCH_BWD
	return cudaGetLastError();
}

}  // namespace sgr
