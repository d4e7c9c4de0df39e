// corrections.cu — the per-camera colour correction of street_gaussians (lib/models/color_correction.py:129-140) as fused kernels.
//
// The reference applies a learned 3x4 affine to every rendered image, einsum('ij,jhw->ihw', A[:3,:3], rgb) + A[:3,3], and adds the
// regularisation mean(|A - I| + |A_sky - I|) to the loss (train.py:134-138).  Forward and backward are single HBM streams over the
// 3 x H x W image; the 12 gradient sums of the backward are reduced in a fixed order (per-block partials, then one finishing
// block), so repeated calls give bit-identical dL/dA, and every grid size depends on H x W only (the calls capture in a CUDA graph).
// The band forms (multi-GPU, DESIGN.md §8) run the same kernels over the pixels of a tile-row band; their backward accumulates the 12
// sums in double, so the ranks' summed partials round once to the frame's dL/dA whatever the split of the rows.
#include <initializer_list>
#include <type_traits>

#include "sgr_common.cuh"

namespace sgr {

constexpr int kCcThreads = 256;
constexpr int kCcMaxBlocks = 4 * (int)kNumSMs;

// One output channel: the three products in einsum's order (a GEMM over k = 0, 1, 2 that starts from a product), then the bias.
__device__ __forceinline__ float cc_row(const float a0, const float a1, const float a2, const float x0, const float x1, const float x2) {
	return __fmaf_rn(a2, x2, __fmaf_rn(a1, x1, __fmul_rn(a0, x0)));
}

// Work items: 4 consecutive pixels when VEC (N % 4 == 0 and 16-byte aligned rows), else one pixel.  With kBand the kernels loop over
// the M items of the band's tile rows (band_pixel, `strip` items per tile row) and skip those past the image; else M = items.
static int cc_blocks(int64_t items) {
	const int64_t b = (items + kCcThreads - 1) / kCcThreads;
	return (int)(b < kCcMaxBlocks ? (b > 0 ? b : 1) : kCcMaxBlocks);
}

template <bool VEC, bool kBand>
__global__ void __launch_bounds__(kCcThreads) color_correct_fwd_kernel(const int64_t N, const int64_t M, const Band band, const int64_t strip,
                                                                       const float *__restrict__ img, const float *__restrict__ A,
                                                                       float *__restrict__ out) {
	float a[12];
#pragma unroll
	for (int k = 0; k < 12; k++) a[k] = __ldg(A + k);
	const int64_t items = VEC ? N / 4 : N;
	const int64_t stride = (int64_t)gridDim.x * blockDim.x;
	for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < M; t += stride) {
		const int64_t it = kBand ? band_pixel(t, band, strip) : t;
		if (kBand && it >= items) continue;
		if (VEC) {
			const float4 x0 = __ldg(reinterpret_cast<const float4 *>(img) + it), x1 = __ldg(reinterpret_cast<const float4 *>(img + N) + it),
			             x2 = __ldg(reinterpret_cast<const float4 *>(img + 2 * N) + it);
#pragma unroll
			for (int i = 0; i < 3; i++) {
				const float *r = a + 4 * i;
				float4 o;
				o.x = __fadd_rn(cc_row(r[0], r[1], r[2], x0.x, x1.x, x2.x), r[3]);
				o.y = __fadd_rn(cc_row(r[0], r[1], r[2], x0.y, x1.y, x2.y), r[3]);
				o.z = __fadd_rn(cc_row(r[0], r[1], r[2], x0.z, x1.z, x2.z), r[3]);
				o.w = __fadd_rn(cc_row(r[0], r[1], r[2], x0.w, x1.w, x2.w), r[3]);
				reinterpret_cast<float4 *>(out + i * N)[it] = o;
			}
		} else {
			const float x0 = __ldg(img + it), x1 = __ldg(img + N + it), x2 = __ldg(img + 2 * N + it);
#pragma unroll
			for (int i = 0; i < 3; i++) out[i * N + it] = __fadd_rn(cc_row(a[4 * i], a[4 * i + 1], a[4 * i + 2], x0, x1, x2), a[4 * i + 3]);
		}
	}
}

// The sums' accumulation: fp32 for the whole frame; double for a band (the products of two floats are exact in double).
__device__ __forceinline__ float cc_fma(const float g, const float x, const float s) { return __fmaf_rn(g, x, s); }
__device__ __forceinline__ double cc_fma(const float g, const float x, const double s) { return __fma_rn((double)g, (double)x, s); }
__device__ __forceinline__ float cc_add(const float s, const float g) { return __fadd_rn(s, g); }
__device__ __forceinline__ double cc_add(const double s, const float g) { return __dadd_rn(s, (double)g); }

// One pixel of the backward: dL/dimage = A^T g (einsum's backward is the same GEMM form), and the 12 sums g_i [x_j, 1].
template <typename Acc>
__device__ __forceinline__ void cc_bwd_pixel(const float *a, const float x0, const float x1, const float x2, const float g0, const float g1,
                                             const float g2, Acc *s, float &d0, float &d1, float &d2) {
	d0 = cc_row(a[0], a[4], a[8], g0, g1, g2);
	d1 = cc_row(a[1], a[5], a[9], g0, g1, g2);
	d2 = cc_row(a[2], a[6], a[10], g0, g1, g2);
	const float g[3] = {g0, g1, g2};
#pragma unroll
	for (int i = 0; i < 3; i++) {
		s[4 * i] = cc_fma(g[i], x0, s[4 * i]);
		s[4 * i + 1] = cc_fma(g[i], x1, s[4 * i + 1]);
		s[4 * i + 2] = cc_fma(g[i], x2, s[4 * i + 2]);
		s[4 * i + 3] = cc_add(s[4 * i + 3], g[i]);
	}
}

template <bool VEC, bool kBand, typename Acc = std::conditional_t<kBand, double, float>>
__global__ void __launch_bounds__(kCcThreads) color_correct_bwd_kernel(const int64_t N, const int64_t M, const Band band, const int64_t strip,
                                                                       const float *__restrict__ img, const float *__restrict__ A,
                                                                       const float *__restrict__ gout, float *__restrict__ gimg,
                                                                       Acc *__restrict__ partials) {
	__shared__ Acc warp_sums[kCcThreads / 32][12];
	float a[12];
	Acc s[12];
#pragma unroll
	for (int k = 0; k < 12; k++) { a[k] = __ldg(A + k); s[k] = 0; }
	const int64_t items = VEC ? N / 4 : N;
	const int64_t stride = (int64_t)gridDim.x * blockDim.x;
	for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < M; t += stride) {
		const int64_t it = kBand ? band_pixel(t, band, strip) : t;
		if (kBand && it >= items) continue;
		if (VEC) {
			const float4 x0 = __ldg(reinterpret_cast<const float4 *>(img) + it), x1 = __ldg(reinterpret_cast<const float4 *>(img + N) + it),
			             x2 = __ldg(reinterpret_cast<const float4 *>(img + 2 * N) + it);
			const float4 g0 = __ldg(reinterpret_cast<const float4 *>(gout) + it), g1 = __ldg(reinterpret_cast<const float4 *>(gout + N) + it),
			             g2 = __ldg(reinterpret_cast<const float4 *>(gout + 2 * N) + it);
			float4 d0, d1, d2;
			cc_bwd_pixel(a, x0.x, x1.x, x2.x, g0.x, g1.x, g2.x, s, d0.x, d1.x, d2.x);
			cc_bwd_pixel(a, x0.y, x1.y, x2.y, g0.y, g1.y, g2.y, s, d0.y, d1.y, d2.y);
			cc_bwd_pixel(a, x0.z, x1.z, x2.z, g0.z, g1.z, g2.z, s, d0.z, d1.z, d2.z);
			cc_bwd_pixel(a, x0.w, x1.w, x2.w, g0.w, g1.w, g2.w, s, d0.w, d1.w, d2.w);
			if (gimg) {
				reinterpret_cast<float4 *>(gimg)[it] = d0;
				reinterpret_cast<float4 *>(gimg + N)[it] = d1;
				reinterpret_cast<float4 *>(gimg + 2 * N)[it] = d2;
			}
		} else {
			float d0, d1, d2;
			cc_bwd_pixel(a, __ldg(img + it), __ldg(img + N + it), __ldg(img + 2 * N + it), __ldg(gout + it), __ldg(gout + N + it),
			             __ldg(gout + 2 * N + it), s, d0, d1, d2);
			if (gimg) { gimg[it] = d0; gimg[N + it] = d1; gimg[2 * N + it] = d2; }
		}
	}
	// fixed-order block reduction: a butterfly per warp, then warp 0 adds the warps' sums in warp order
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
	for (int k = 0; k < 12; k++) {
		Acc v = s[k];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
		if (lane == 0) warp_sums[warp][k] = v;
	}
	__syncthreads();
	if (threadIdx.x < 12) {
		Acc v = warp_sums[0][threadIdx.x];
		for (int w = 1; w < kCcThreads / 32; w++) v += warp_sums[w][threadIdx.x];
		partials[(size_t)blockIdx.x * 12 + threadIdx.x] = v;
	}
}

// One block, warp k = component k: lane l adds the partials of blocks l, l + 32, ... in double, then a butterfly over the lanes.
// Out: the fp32 dL/dA (whole frame) or the band's 12 double sums.
template <typename P, typename O>
__global__ void color_correct_finish_kernel(const int nblocks, const P *__restrict__ partials, O *__restrict__ gA) {
	const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
	double v = 0.0;
	for (int b = lane; b < nblocks; b += 32) v += (double)partials[(size_t)b * 12 + k];
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	if (lane == 0) gA[k] = (O)v;
}

// dL/dA from the 12 sums the ranks added up.
__global__ void color_correct_affine_grad_kernel(const double *__restrict__ sums, float *__restrict__ gA) {
	if (threadIdx.x < 12) gA[threadIdx.x] = (float)sums[threadIdx.x];
}

// mean(|A - I| + |A_sky - I|) over the 12 entries (color_correction.py:134-140) times weight, and its gradients
// weight / 12 * sign(A - I) with sign(0) = 0 (torch's abs backward).  One warp; the lanes' terms are added in a fixed butterfly.
__global__ void color_correction_reg_kernel(const float *__restrict__ A, const float *__restrict__ S, const float weight, float *__restrict__ value,
                                            float *__restrict__ gA, float *__restrict__ gS) {
	const int k = threadIdx.x;
	const float eye = (k < 12 && k % 4 == k / 4) ? 1.f : 0.f;
	const float dA = k < 12 ? A[k] - eye : 0.f, dS = (k < 12 && S) ? S[k] - eye : 0.f;
	float v = fabsf(dA) + fabsf(dS);
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	const float gw = weight / 12.f;
	const auto sgn = [](float d) { return d > 0.f ? 1.f : (d < 0.f ? -1.f : (d == d ? 0.f : d)); };  // NaN stays NaN, like torch.sign
	if (k < 12) {
		if (gA) gA[k] = sgn(dA) * gw;
		if (gS) gS[k] = sgn(dS) * gw;
	}
	if (k == 0) *value = weight * (v / 12.f);
}

static bool cc_vec(int64_t N, std::initializer_list<const void *> ptrs) {
	if (N % 4 != 0) return false;
	for (const void *p : ptrs)
		if (p && (reinterpret_cast<uintptr_t>(p) & 15u)) return false;
	return true;
}

cudaError_t launch_color_correct_fwd(int64_t N, const float *image, const float *affine, float *out, cudaStream_t st) {
	const bool vec = cc_vec(N, {image, out});
	count_launch();
	if (vec) color_correct_fwd_kernel<true, false><<<cc_blocks(N / 4), kCcThreads, 0, st>>>(N, N / 4, Band{0, 1, 1}, 1, image, affine, out);
	else color_correct_fwd_kernel<false, false><<<cc_blocks(N), kCcThreads, 0, st>>>(N, N, Band{0, 1, 1}, 1, image, affine, out);
	return cudaGetLastError();
}

size_t color_correct_scratch_bytes(int64_t N) { return (size_t)cc_blocks(N) * 12 * sizeof(float); }

cudaError_t launch_color_correct_bwd(int64_t N, const float *image, const float *affine, const float *g_out, float *g_image, float *g_affine,
                                     void *scratch, cudaStream_t st) {
	const bool vec = cc_vec(N, {image, g_out, g_image});
	const int blocks = vec ? cc_blocks(N / 4) : cc_blocks(N);
	float *partials = static_cast<float *>(scratch);
	count_launch(2);
	if (vec) color_correct_bwd_kernel<true, false><<<blocks, kCcThreads, 0, st>>>(N, N / 4, Band{0, 1, 1}, 1, image, affine, g_out, g_image, partials);
	else color_correct_bwd_kernel<false, false><<<blocks, kCcThreads, 0, st>>>(N, N, Band{0, 1, 1}, 1, image, affine, g_out, g_image, partials);
	color_correct_finish_kernel<float, float><<<1, 12 * 32, 0, st>>>(blocks, partials, g_affine);
	return cudaGetLastError();
}

// The band's items: the band's tile rows of 16 W pixels (4 W float4 items when VEC; a tile row starts at a multiple of 64 bytes).
cudaError_t launch_color_correct_fwd(int H, int W, Band band, const float *image, const float *affine, float *out, cudaStream_t st) {
	const int64_t N = (int64_t)H * W, strip = (int64_t)kBandTileRows * W, M = band_rows(band) * strip;
	if (M == 0) return cudaSuccess;
	const bool vec = cc_vec(N, {image, out});
	count_launch();
	if (vec) color_correct_fwd_kernel<true, true><<<cc_blocks(M / 4), kCcThreads, 0, st>>>(N, M / 4, band, strip / 4, image, affine, out);
	else color_correct_fwd_kernel<false, true><<<cc_blocks(M), kCcThreads, 0, st>>>(N, M, band, strip, image, affine, out);
	return cudaGetLastError();
}

size_t color_correct_band_scratch_bytes(int H, int W) {
	return (size_t)cc_blocks((int64_t)((H + kBandTileRows - 1) / kBandTileRows) * kBandTileRows * W) * 12 * sizeof(double);
}

cudaError_t launch_color_correct_bwd(int H, int W, Band band, const float *image, const float *affine, const float *g_out, float *g_image,
                                     double *sums, void *scratch, cudaStream_t st) {
	const int64_t N = (int64_t)H * W, strip = (int64_t)kBandTileRows * W, M = band_rows(band) * strip;
	const bool vec = cc_vec(N, {image, g_out, g_image});
	const int blocks = M == 0 ? 0 : (vec ? cc_blocks(M / 4) : cc_blocks(M));
	double *partials = static_cast<double *>(scratch);
	if (blocks > 0) {
		count_launch();
		if (vec) color_correct_bwd_kernel<true, true><<<blocks, kCcThreads, 0, st>>>(N, M / 4, band, strip / 4, image, affine, g_out, g_image, partials);
		else color_correct_bwd_kernel<false, true><<<blocks, kCcThreads, 0, st>>>(N, M, band, strip, image, affine, g_out, g_image, partials);
	}
	count_launch();
	color_correct_finish_kernel<double, double><<<1, 12 * 32, 0, st>>>(blocks, partials, sums);  // an empty band: zeros
	return cudaGetLastError();
}

cudaError_t launch_color_correct_affine_grad(const double *sums, float *g_affine, cudaStream_t st) {
	count_launch();
	color_correct_affine_grad_kernel<<<1, 32, 0, st>>>(sums, g_affine);
	return cudaGetLastError();
}

cudaError_t launch_color_correction_reg(const float *affine, const float *affine_sky, float weight, float *value, float *g_affine,
                                        float *g_affine_sky, cudaStream_t st) {
	count_launch();
	color_correction_reg_kernel<<<1, 32, 0, st>>>(affine, affine_sky, weight, value, g_affine, g_affine_sky);
	return cudaGetLastError();
}

}  // namespace sgr
