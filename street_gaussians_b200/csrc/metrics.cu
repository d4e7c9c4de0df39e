// metrics.cu — scoring rendered views: masked L1, PSNR and SSIM per view, value only (include/sgr.h, "Evaluation metrics").
//
// The reference scores views with torch lines: training_report (train.py:274-303) sums l1_loss and psnr (lib/utils/loss_utils.py:21-37,
// 61-78) of the clamped render per view, and metrics.py:76-81 takes ssim and psnr of the PNGs torchvision's save_image wrote.  Here one
// view costs three kernels and no host synchronisation:
//   eval_tile_kernel          one block per (view, channel, 16x16 tile): the SSIM map of the tile (ssim_tile.cuh, the image loss's
//                             arithmetic) and the tile's partial sums {SSIM, |x - y|, (x - y)^2, masked elements}, written to its own
//                             scratch slot (no atomics);
//   eval_reduce_kernel<false> kReduceChunk tile partials per block, summed in a fixed order in fp64;
//   eval_reduce_kernel<true>  one block per view: the chunk sums in order, added to the view's SgrEvalSums.
// eval_finish_kernel turns the sums into {psnr, ssim, l1, n} per view and their means.  The grids depend on V, C, H, W and the band only,
// so a scoring loop can be captured in a CUDA graph, and two identical calls give the same bits.
#include "ssim_tile.cuh"

namespace sgr {

namespace {

constexpr int kTile = kSsimTile, kHalo = kSsimHalo, kExt = kSsimExt;  // 16, 5, 26
constexpr unsigned kReduceChunk = 2048;                                // tile partials per first-level reduction block

struct TilePartial {
	double ssim, abs_diff, sq_diff;
	unsigned long long masked;
};

// Clamp to [0, 1] (NaN stays NaN, as torch.clamp keeps it), then the round trip of a PNG written by torchvision.utils.save_image and
// read back by to_tensor: mul(255).add_(0.5).clamp_(0, 255).to(uint8) in fp32 (round to the nearest level, halves up), then / 255 in fp32.
__device__ __forceinline__ float eval_input(float v, int flags) {
	if (flags & SGR_EVAL_CLAMP) v = v != v ? v : fminf(fmaxf(v, 0.f), 1.f);
	if (flags & SGR_EVAL_QUANT8) {
		const float t = __fadd_rn(__fmul_rn(v, 255.f), 0.5f);
		v = __fdiv_rn(truncf(t != t ? t : fminf(fmaxf(t, 0.f), 255.f)), 255.f);
	}
	return v;
}

// The four sums of a 256-thread block in a fixed order (a warp butterfly, then the 8 warps in order); the result is thread 0's.
// kSsimF32: the SSIM sum runs in fp32 within a warp, as ssim_stats_kernel forms its block sums.
template <bool kSsimF32>
__device__ __forceinline__ TilePartial block_sum(double ssim, double a, double q, unsigned long long n) {
	__shared__ double red[3][8];
	__shared__ unsigned long long red_n[8];
	float s32 = (float)ssim;
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		if (kSsimF32)
			s32 += __shfl_xor_sync(0xffffffffu, s32, o);
		else
			ssim += __shfl_xor_sync(0xffffffffu, ssim, o);
		a += __shfl_xor_sync(0xffffffffu, a, o);
		q += __shfl_xor_sync(0xffffffffu, q, o);
		n += __shfl_xor_sync(0xffffffffu, n, o);
	}
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	if (lane == 0) { red[0][warp] = kSsimF32 ? (double)s32 : ssim; red[1][warp] = a; red[2][warp] = q; red_n[warp] = n; }
	__syncthreads();
	TilePartial p{0.0, 0.0, 0.0, 0ull};
	if (threadIdx.x == 0)
		for (int k = 0; k < 8; k++) { p.ssim += red[0][k]; p.abs_diff += red[1][k]; p.sq_diff += red[2][k]; p.masked += red_n[k]; }
	return p;
}

// Block (x, y, v C + c): tile x of the band's y-th tile row, channel c of view v.  Its SSIM block sum is formed as ssim_stats_kernel's
// (fp32 within a warp, fp64 over the 8 warps), so a tile gives the same SSIM partial as the image loss's block for that tile.
__global__ void __launch_bounds__(256) eval_tile_kernel(const int C, const int H, const int W, const Band band, const int flags, const GaussWin win,
                                                       const float *__restrict__ img, const float *__restrict__ gt,
                                                       const uint8_t *__restrict__ mask, TilePartial *__restrict__ part) {
	__shared__ float sx[kExt][kExt + 1], sy[kExt][kExt + 1];
	__shared__ float h[5][kExt][kTile + 1];
	const int v = blockIdx.z / C, c = blockIdx.z - v * C;
	const int tile_y = band.begin + (int)blockIdx.y * band.step;
	const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
	const int x0 = blockIdx.x * kTile - kHalo, y0 = tile_y * kTile - kHalo;
	const size_t plane = (size_t)H * W;
	const float *ip = img + ((size_t)v * C + c) * plane, *gp = gt + ((size_t)v * C + c) * plane;
	const uint8_t *mp = mask ? mask + (size_t)v * plane : nullptr;
	const bool with_ssim = !(flags & SGR_EVAL_NO_SSIM);  // block-uniform
	if (with_ssim) {
		const uint8_t *zero_mask = (flags & SGR_EVAL_SSIM_MASKED) ? mp : nullptr;  // ssim(mask=) zeroes both images outside the mask
		for (int e = threadIdx.x; e < kExt * kExt; e += 256) {
			const int r = e / kExt, q = e - r * kExt, yy = y0 + r, xx = x0 + q;
			float a = 0.f, b = 0.f;
			if (yy >= 0 && yy < H && xx >= 0 && xx < W && (zero_mask == nullptr || zero_mask[(size_t)yy * W + xx])) {
				a = eval_input(ip[(size_t)yy * W + xx], flags);
				b = eval_input(gp[(size_t)yy * W + xx], flags);
			}
			sx[r][q] = a;
			sy[r][q] = b;
		}
		__syncthreads();
		ssim_tile_horizontal(sx, sy, h, win);
		__syncthreads();
	}
	const int px = blockIdx.x * kTile + tx, py = tile_y * kTile + ty;
	float v_ssim = 0.f;
	double v_abs = 0.0, v_sq = 0.0;
	unsigned long long v_n = 0;
	if (px < W && py < H) {
		if (with_ssim) v_ssim = ssim_terms(ssim_tile_vertical(h, win, tx, ty)).S;
		const size_t o = (size_t)py * W + px;
		if (mp == nullptr || mp[o]) {
			// the difference of two fp32 values and its square are exact in fp64: the sums carry only their own rounding
			const double d = (double)eval_input(ip[o], flags) - (double)eval_input(gp[o], flags);
			v_abs = fabs(d);
			v_sq = d * d;
			v_n = 1;
		}
	}
	const TilePartial p = block_sum<true>(v_ssim, v_abs, v_sq, v_n);
	if (threadIdx.x == 0) part[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = p;
}

// Block (x, v): the n inputs of view v (in[v n .. v n + n)) in chunks of `chunk`, thread t summing items t, t + 256, ... of chunk x.
// First level: writes the chunk's sum to out[v gridDim.x + x].  kFinal (one chunk per view): adds it to sums[v] with `elements`.
template <bool kFinal>
__global__ void __launch_bounds__(256) eval_reduce_kernel(const unsigned n, const unsigned chunk, const TilePartial *__restrict__ in,
                                                         TilePartial *__restrict__ out, const double elements, SgrEvalSums *__restrict__ sums) {
	const TilePartial *p = in + (size_t)blockIdx.y * n;
	const unsigned lo = blockIdx.x * chunk, hi = min(n, lo + chunk);
	double s = 0.0, a = 0.0, q = 0.0;
	unsigned long long m = 0;
	for (unsigned b = lo + threadIdx.x; b < hi; b += 256) {
		const TilePartial t = p[b];
		s += t.ssim; a += t.abs_diff; q += t.sq_diff; m += t.masked;
	}
	const TilePartial t = block_sum<false>(s, a, q, m);
	if (threadIdx.x != 0) return;
	if (!kFinal) {
		out[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = t;
		return;
	}
	SgrEvalSums &o = sums[blockIdx.y];
	o.abs_diff += t.abs_diff;
	o.sq_diff += t.sq_diff;
	o.ssim += t.ssim;
	o.masked += (double)t.masked;
	o.elements += elements;
}

// out[v] = {psnr, ssim, l1, n} of view v; out[V] = {mean psnr, mean ssim, mean l1, V}, the means of the fp32 per-view values summed in
// fp64 (as training_report sums .double() values).  IEEE arithmetic keeps the reference's edge results: mse = 0 gives psnr = +inf,
// an empty mask 0 / 0 = NaN for psnr and l1 (and a view scored without SSIM 0 / 0 = NaN for ssim).
__global__ void __launch_bounds__(256) eval_finish_kernel(const int V, const SgrEvalSums *__restrict__ sums, float *__restrict__ out) {
	for (int v = threadIdx.x; v < V; v += 256) {
		const SgrEvalSums s = sums[v];
		const double mse = s.sq_diff / s.masked;
		out[4 * v + 0] = (float)(20.0 * log10(1.0 / sqrt(mse)));
		out[4 * v + 1] = (float)(s.ssim / s.elements);
		out[4 * v + 2] = (float)(s.abs_diff / s.masked);
		out[4 * v + 3] = (float)s.masked;
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		double m[3] = {0.0, 0.0, 0.0};
		for (int v = 0; v < V; v++)
			for (int k = 0; k < 3; k++) m[k] += (double)out[4 * v + k];
		for (int k = 0; k < 3; k++) out[4 * V + k] = (float)(m[k] / V);
		out[4 * V + 3] = (float)V;
	}
}

inline unsigned tiles_x(int W) { return (unsigned)((W + kTile - 1) / kTile); }
inline size_t tiles_of(int C, int H, int W) { return (size_t)C * tiles_x(W) * ((H + kTile - 1) / kTile); }
inline size_t chunks_of(size_t n) { return (n + kReduceChunk - 1) / kReduceChunk; }

}  // namespace

// the tile partials [V][tiles] and the first-level chunk sums [V][chunks], both sized for the whole frame
size_t eval_metrics_scratch_bytes(int V, int C, int H, int W) {
	const size_t n = tiles_of(C, H, W);
	return align_up((size_t)V * n * sizeof(TilePartial)) + align_up((size_t)V * chunks_of(n) * sizeof(TilePartial));
}

cudaError_t launch_eval_metrics(int V, int C, int H, int W, Band band, int flags, const float *img, const float *gt, const uint8_t *mask,
                                SgrEvalSums *sums, void *scratch, cudaStream_t st) {
	const unsigned rows = (unsigned)band_rows(band);
	if (rows == 0) return cudaSuccess;
	TilePartial *part = reinterpret_cast<TilePartial *>(scratch);
	TilePartial *mid = reinterpret_cast<TilePartial *>(reinterpret_cast<char *>(scratch) + align_up((size_t)V * tiles_of(C, H, W) * sizeof(TilePartial)));
	// elements of the band: C W times the image rows of its tile rows (the last tile row may be partial); none without the SSIM
	const int last = band.begin + (int)(rows - 1) * band.step;
	const int64_t px_rows = (int64_t)(rows - 1) * kTile + min(kTile, H - kTile * last);
	const double elements = (flags & SGR_EVAL_NO_SSIM) ? 0.0 : (double)C * (double)W * (double)px_rows;
	const unsigned n = tiles_x(W) * rows * C, chunks = (unsigned)chunks_of(n);
	count_launch(3);
	eval_tile_kernel<<<dim3(tiles_x(W), rows, V * C), 256, 0, st>>>(C, H, W, band, flags, ssim_window(), img, gt, mask, part);
	eval_reduce_kernel<false><<<dim3(chunks, V), 256, 0, st>>>(n, kReduceChunk, part, mid, 0.0, nullptr);
	eval_reduce_kernel<true><<<dim3(1, V), 256, 0, st>>>(chunks, chunks, mid, nullptr, elements, sums);
	return cudaGetLastError();
}

cudaError_t launch_eval_metrics_finish(int V, const SgrEvalSums *sums, float *out, cudaStream_t st) {
	count_launch(1);
	eval_finish_kernel<<<1, 256, 0, st>>>(V, sums, out);
	return cudaGetLastError();
}

}  // namespace sgr
