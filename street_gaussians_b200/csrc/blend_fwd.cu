// blend_fwd.cu — per-tile front-to-back alpha blend (forward).
//
// Replaces the reference's renderCUDA<3> (DGR/cuda_rasterizer/forward.cu:340-467).  Same per-(pixel, splat) arithmetic
// (expression shapes kept so `power`, `alpha` and the three hard thresholds flip on exactly the same pairs), different
// machinery:
//   * one CTA per OWNED tile (tile-row band), 8 warps, each warp owns a compact 8x4 pixel block;
//   * the tile's splat list is staged through shared memory from the packed 48-B GaussRec (3 x 16-B gathers per
//     instance instead of id + float2 + float4 + per-contribution global re-gathers of colour and depth);
//   * double-buffered staging with register prefetch: the gathers of batch k+1 are in flight while batch k is blended,
//     one __syncthreads_count per batch (it doubles as the "whole tile saturated" vote);
//   * the kernel is ISSUE-bound (records and lists are L2 hits, DRAM traffic is small), so the inner loop is written for
//     instruction count: one running 32-bit shared address, three LDS.128 with immediate offsets per splat
//     (explicit ld.shared — indexing the arrays through C++ made nvcc rebuild a cluster-window address with
//     S2R/LEA every iteration, 12 of 76 instructions), and a conservative `power` bound from the record that skips
//     expf for pairs that cannot reach alpha >= 1/255;
//   * semantics are accumulated in registers and written once (the reference does a global read-modify-write per
//     contribution, forward.cu:442-444).
// Saturation split (binning.cu): PASS = kBlendNear blends the near lists; a tile whose inside pixels all saturated is final, any
// other one parks its per-pixel state (C and weight / depth sums in the output images, last contributor in n_contrib, T with the
// `done` bit as its sign in blend_T) and marks itself by the top bit of tile_max_contrib over its near count.  PASS = kBlendResume
// runs on those tiles only, over the final list from that position on.  The state round-trips bit for bit and the per-pixel loop
// does not depend on where batches start, so every output equals the one-pass blend's.
#include "sgr_common.cuh"

namespace sgr {

constexpr int kFwdBatch = 256;
constexpr uint32_t kRecBytes = 48;

__device__ __forceinline__ float4 lds128(uint32_t addr) {
	float4 v;
	asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
	return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, float4 v) {
	asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

template <int SCH, int PASS = kBlendFull>
__global__ void __launch_bounds__(256) blend_fwd_kernel(const FrameDev f, const uint2 *__restrict__ ranges,
                                                        const uint32_t *__restrict__ point_list, const GaussRec *__restrict__ rec,
                                                        const float *__restrict__ semantics, uint32_t *__restrict__ n_contrib,
                                                        uint32_t *__restrict__ tile_max_contrib, float *__restrict__ out_color,
                                                        float *__restrict__ out_depth, float *__restrict__ out_alpha,
                                                        float *__restrict__ out_sem, const int sem_ch0, const int sem_only,
                                                        float *__restrict__ blend_T) {
	static_assert(PASS == kBlendFull || SCH == 0, "the split passes carry no semantic channels");
	__shared__ __align__(16) unsigned char s_rec[2][kFwdBatch * kRecBytes];  // 2 x 12 KB: GaussRec per list slot
	__shared__ uint32_t s_id[SCH > 0 ? 2 : 1][SCH > 0 ? kFwdBatch : 1];
	__shared__ uint32_t s_max;

	const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
	const int tile_x = blockIdx.x, tile_y = f.band.begin + blockIdx.y * f.band.step;
	const int tile = tile_y * f.gx + tile_x;
	const int px = tile_x * SGR_TILE + (warp & 1) * 8 + (lane & 7);
	const int py = tile_y * SGR_TILE + (warp >> 1) * 4 + (lane >> 3);
	const bool inside = px < f.W && py < f.H;
	const size_t HW = (size_t)f.W * f.H;
	const size_t pix_id = (size_t)f.W * py + px;
	const float2 pixf = make_float2((float)px, (float)py);

	uint32_t start = 0u;  // first list position blended here (kBlendResume: the tile's near count)
	if (PASS == kBlendResume) {
		const uint32_t w = tile_max_contrib[tile];
		if (!(w >> 31)) return;  // saturated in the near pass: its outputs are final
		start = w & 0x7fffffffu;
	}
	const uint2 range = ranges[tile];
	const int n = (int)(range.y - range.x - start);
	const int nb = (n + kFwdBatch - 1) / kFwdBatch;
	if (tid == 0) s_max = 0;
	__syncthreads();
	const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(&s_rec[0][0]);
	constexpr uint32_t kBufBytes = kFwdBatch * kRecBytes;

	bool done = !inside;
	float T = 1.0f;
	float C0 = 0.f, C1 = 0.f, C2 = 0.f, weight = 0.f, Dacc = 0.f;
	float sem[SCH > 0 ? SCH : 1];
#pragma unroll
	for (int c = 0; c < (SCH > 0 ? SCH : 1); c++) sem[c] = 0.f;
	const int nsem = SCH > 0 ? min(SCH, f.S - sem_ch0) : 0;
	uint32_t last_contributor = 0;
	if (PASS == kBlendResume && inside) {
		const uint32_t tb = __float_as_uint(blend_T[pix_id]);
		done = (tb >> 31) != 0u;
		T = __uint_as_float(tb & 0x7fffffffu);
		C0 = out_color[pix_id]; C1 = out_color[HW + pix_id]; C2 = out_color[2 * HW + pix_id];
		weight = out_alpha[pix_id];
		Dacc = out_depth[pix_id];
		last_contributor = n_contrib[pix_id];
	}

	float4 r0 = make_float4(0, 0, 0, 0), r1 = r0, r2 = r0;
	uint32_t rid = 0;
	auto fetch = [&](int b) {
		const int k = b * kFwdBatch + tid;
		if (k < n) {
			rid = point_list[range.x + start + k];
			const GaussRec *p = rec + rid;
			r0 = p->q0; r1 = p->q1; r2 = p->q2;
		}
	};
	auto stash = [&](int buf) {
		const uint32_t a = sbase + (uint32_t)buf * kBufBytes + (uint32_t)tid * kRecBytes;
		sts128(a, r0); sts128(a + 16, r1); sts128(a + 32, r2);
		if (SCH > 0) s_id[buf][tid] = rid;
	};
	if (nb > 0) { fetch(0); stash(0); }

	for (int b = 0; b < nb; b++) {
		// barrier: publishes buffer b&1 and votes on "every pixel of the tile is saturated"
		const int num_done = __syncthreads_count(done);
		if (num_done == SGR_TILE_PIX) break;
		if (b + 1 < nb) fetch(b + 1);
		const int buf = b & 1;
		const int cnt = min(kFwdBatch, n - b * kFwdBatch);
		const uint32_t a0 = sbase + (uint32_t)buf * kBufBytes;
		const uint32_t a_end = a0 + (uint32_t)cnt * kRecBytes;
		uint32_t a_last = 0xffffffffu;
		for (uint32_t a = a0; !done && a < a_end; a += kRecBytes) {
			const float4 q0 = lds128(a);       // pix.x, pix.y, conic.xx, conic.xy
			const float4 q1 = lds128(a + 16);  // conic.yy, opacity, power_min, depth
			const float2 d = make_float2(q0.x - pixf.x, q0.y - pixf.y);
			const float power = -0.5f * (q0.z * d.x * d.x + q1.x * d.y * d.y) - q0.w * d.x * d.y;
			if (power > 0.0f) continue;
			if (power < q1.z) continue;  // conservative: alpha < 1/255 for sure, skip the expf (exact test still below)
			const float alpha = fminf(0.99f, q1.y * expf(power));
			if (alpha < 1.0f / 255.0f) continue;
			const float test_T = T * (1 - alpha);
			if (test_T < 0.0001f) {
				done = true;
				continue;
			}
			const float4 q2 = lds128(a + 32);  // r, g, b, clamp bits
			C0 += q2.x * alpha * T;
			C1 += q2.y * alpha * T;
			C2 += q2.z * alpha * T;
			if (SCH > 0) {
				const uint32_t j = (a - a0) / kRecBytes;
				const float *sp = semantics + (size_t)s_id[buf][j] * f.S + sem_ch0;
#pragma unroll
				for (int c = 0; c < SCH; c++)
					if (c < nsem) sem[c] += __ldg(sp + c) * alpha * T;
			}
			weight += alpha * T;
			Dacc += q1.w * alpha * T;
			T = test_T;
			a_last = a;
		}
		if (a_last != 0xffffffffu) last_contributor = start + (uint32_t)(b * kFwdBatch) + (a_last - a0) / kRecBytes + 1u;
		if (b + 1 < nb) stash((b + 1) & 1);
	}

	if (PASS == kBlendNear && __syncthreads_count(done) != SGR_TILE_PIX) {  // unsaturated: park the state for kBlendResume
		if (inside) {
			n_contrib[pix_id] = last_contributor;
			out_color[pix_id] = C0;
			out_color[HW + pix_id] = C1;
			out_color[2 * HW + pix_id] = C2;
			out_alpha[pix_id] = weight;
			out_depth[pix_id] = Dacc;
			blend_T[pix_id] = __uint_as_float(__float_as_uint(T) | (done ? 0x80000000u : 0u));
		}
		if (tid == 0) tile_max_contrib[tile] = 0x80000000u | (uint32_t)n;
		return;
	}
	if (inside) {
		if (!sem_only) {
			n_contrib[pix_id] = last_contributor;
			out_color[pix_id] = C0 + T * f.bg[0];
			out_color[HW + pix_id] = C1 + T * f.bg[1];
			out_color[2 * HW + pix_id] = C2 + T * f.bg[2];
			out_alpha[pix_id] = weight;
			out_depth[pix_id] = Dacc;
		}
		if (SCH > 0) {
#pragma unroll
			for (int c = 0; c < SCH; c++)
				if (c < nsem) out_sem[(size_t)(sem_ch0 + c) * HW + pix_id] = sem[c];
		}
	}
	if (!sem_only) {
		// deepest list position any pixel of this tile reached: lets the backward pass skip the tail of the list
		const uint32_t wmax = __reduce_max_sync(0xffffffffu, inside ? last_contributor : 0u);
		if (lane == 0) atomicMax(&s_max, wmax);
		__syncthreads();
		if (tid == 0) tile_max_contrib[tile] = s_max;
	}
}

cudaError_t launch_blend_fwd(const FrameDev &f, GeomView g, BinView b, ImgView img, const float *semantics, float *out_color,
                             float *out_depth, float *out_alpha, float *out_sem, cudaStream_t st, BlendPass pass) {
	const int rows = band_rows(f.band);
	if (rows <= 0 || f.gx <= 0) return cudaSuccess;
	const dim3 grid(f.gx, rows);
	count_launch();
	if (pass != kBlendFull && f.S > 0) return cudaErrorInvalidValue;
	if (pass == kBlendNear || pass == kBlendResume) {
		if (pass == kBlendNear)
			blend_fwd_kernel<0, kBlendNear><<<grid, 256, 0, st>>>(f, img.ranges, b.vals_out, g.rec, nullptr, img.n_contrib, img.tile_max_contrib,
			                                                      out_color, out_depth, out_alpha, nullptr, 0, 0, img.blend_T);
		else
			blend_fwd_kernel<0, kBlendResume><<<grid, 256, 0, st>>>(f, img.ranges, b.vals_out, g.rec, nullptr, img.n_contrib, img.tile_max_contrib,
			                                                        out_color, out_depth, out_alpha, nullptr, 0, 0, img.blend_T);
		return cudaGetLastError();
	}
#define SGR_LAUNCH_FWD(SCH, ch0, only)                                                                                        \
	blend_fwd_kernel<SCH><<<grid, 256, 0, st>>>(f, img.ranges, b.vals_out, g.rec, semantics, img.n_contrib,                     \
	                                            img.tile_max_contrib, out_color, out_depth, out_alpha, out_sem, ch0, only, nullptr)
	if (f.S <= 0)
		SGR_LAUNCH_FWD(0, 0, 0);
	else if (f.S <= 4)
		SGR_LAUNCH_FWD(4, 0, 0);
	else if (f.S <= 8)
		SGR_LAUNCH_FWD(8, 0, 0);
	else if (f.S <= 16)
		SGR_LAUNCH_FWD(16, 0, 0);
	else {
		SGR_LAUNCH_FWD(32, 0, 0);
		for (int ch0 = 32; ch0 < f.S; ch0 += 32) {  // further channel chunks: semantics only
			count_launch();
			SGR_LAUNCH_FWD(32, ch0, 1);
		}
	}
#undef SGR_LAUNCH_FWD
	return cudaGetLastError();
}

}  // namespace sgr
