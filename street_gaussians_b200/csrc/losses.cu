// losses.cu — the image-space training losses of street_gaussians, value AND gradient in two kernels (SURVEY.md §8 row f2).
//
// The reference builds  loss = (1 - l) * l1w * L1(image, gt, mask) + l * (1 - SSIM(image, gt, mask))  (train.py:101-104) out of
// lib/utils/loss_utils.py:21-37 (l1_loss) and :91-126 (ssim: five 11x11 Gaussian convolutions per image pair as grouped
// F.conv2d calls, plus ~15 elementwise kernels), then autograd replays all of it backwards to obtain dL/dimage — the tensor
// the rasterizer's backward consumes.  Here:
//   kernel 1 (ssim_stats_kernel): per 16x16 tile with a 5-pixel halo, separable 11-tap convolution of (x, y, x^2, y^2, xy) in
//            shared memory -> the SSIM map value, its three partial derivatives w.r.t. (mu_x, E[x^2], E[xy]) and the tile's
//            partial sums of SSIM, |x - y| over the mask and the mask count;
//   kernel 2 (ssim_grad_kernel): convolves the three derivative maps with the same window (the zero-padded Gaussian window
//            is symmetric, hence self-adjoint) and combines them with x, y, the L1 sign term and the mask into dL/dimage;
//            block (0,0,0) also finalises the scalars.
// Semantics follow the reference exactly: with a mask both images are ZEROED outside it before SSIM (loss_utils.py:95-97) and
// the SSIM mean runs over all pixels, while L1 averages over the masked pixels only (:31-35).
#include "ssim_tile.cuh"

namespace sgr {

constexpr int kWin = kSsimWin, kHalo = kSsimHalo, kTileL = kSsimTile, kExt = kSsimExt;  // 26

// The tiles ssim_stats_kernel covers for a band: its own tile rows and the neighbours above and below them.  With step <= 2 they form
// one run of tile rows; otherwise block row y is neighbour y % 3 - 1 of the (y / 3)-th owned tile row, -1 when that lies outside
// the image.  The whole image is every tile row once, in order.
static unsigned stats_tiles(const Band b, int rows) {
	const int n = band_rows(b);
	if (n == 0) return 0;
	if (b.step > 2) return 3u * n;
	const int last = b.begin + (n - 1) * b.step;
	return (unsigned)(min(rows, last + 2) - max(0, b.begin - 1));
}
__device__ __forceinline__ int stats_tile(const Band b, int y, int rows) {
	if (b.step <= 2) return max(0, b.begin - 1) + y;
	const int t = b.begin + (y / 3) * b.step + y % 3 - 1;
	return t >= 0 && t < rows ? t : -1;
}

// loss_utils.py:84-86: exp(-(x - 5)^2 / (2 * 1.5^2)) normalised (float32, like torch.Tensor([...]) / sum).  The sum is the fp32
// rounding of the exact sum, as torch's sum gives for these 11 values; a sequential fp32 sum is one ulp low and would move 9 of the
// 11 weights by one ulp.
static GaussWin make_window() {
	GaussWin g;
	double s = 0.0;
	for (int k = 0; k < kWin; k++) {
		g.w[k] = (float)exp(-(double)((k - kWin / 2) * (k - kWin / 2)) / (2.0 * 1.5 * 1.5));
		s += (double)g.w[k];
	}
	const float sf = (float)s;
	for (int k = 0; k < kWin; k++) g.w[k] /= sf;
	return g;
}

// acc: [0] sum of the SSIM map, [1] sum |x - y| over masked elements, [2] number of masked PIXELS (counted on channel 0), over the
// pixels of the band's tile rows.  The blocks are the tiles of band_stats_tile(): the band's own tile rows and their neighbours, whose
// rows within kHalo of an owned row are where ssim_grad_kernel reads the derivative maps.  The whole image is every tile row.
__global__ void __launch_bounds__(256) ssim_stats_kernel(const int C, const int H, const int W, const Band band, const GaussWin win,
                                                        const float *__restrict__ img, const float *__restrict__ gt,
                                                        const uint8_t *__restrict__ mask, float *__restrict__ d_mu, float *__restrict__ d_xx,
                                                        float *__restrict__ d_xy, double *__restrict__ acc) {
	__shared__ float sx[kExt][kExt + 1], sy[kExt][kExt + 1];
	__shared__ float h[5][kExt][kTileL + 1];
	__shared__ float red[3][8];
	const int tile_y = stats_tile(band, blockIdx.y, (H + kTileL - 1) / kTileL);
	if (tile_y < 0) return;  // a neighbour above the first or below the last tile row
	const int c = blockIdx.z, tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
	const int x0 = blockIdx.x * kTileL - kHalo, y0 = tile_y * kTileL - kHalo;
	const bool owned = band_owns(band, tile_y);
	// rows of a neighbour tile that no owned pixel's window reaches are not needed (their inputs may be foreign rows)
	const bool needed = owned || (ty < kHalo && band_owns(band, tile_y - 1)) || (ty >= kTileL - kHalo && band_owns(band, tile_y + 1));
	const size_t plane = (size_t)H * W;
	const float *ip = img + (size_t)c * plane, *gp = gt + (size_t)c * plane;
	for (int e = threadIdx.x; e < kExt * kExt; e += 256) {
		const int r = e / kExt, q = e - r * kExt, yy = y0 + r, xx = x0 + q;
		float a = 0.f, b = 0.f;
		if (yy >= 0 && yy < H && xx >= 0 && xx < W && (mask == nullptr || mask[(size_t)yy * W + xx])) {
			a = ip[(size_t)yy * W + xx];
			b = gp[(size_t)yy * W + xx];
		}
		sx[r][q] = a;
		sy[r][q] = b;
	}
	__syncthreads();
	ssim_tile_horizontal(sx, sy, h, win);
	__syncthreads();
	const int px = blockIdx.x * kTileL + tx, py = tile_y * kTileL + ty;
	float v_ssim = 0.f, v_l1 = 0.f, v_cnt = 0.f;
	if (px < W && py < H && needed) {
		const SsimSums q = ssim_tile_vertical(h, win, tx, ty);
		const float m1 = q.m1, m2 = q.m2;
		const SsimTerms t = ssim_terms(q);
		const float A1 = t.A1, A2 = t.A2, B1 = t.B1, B2 = t.B2, inv = t.inv, S = t.S;
		v_ssim = owned ? S : 0.f;
		const size_t o = (size_t)c * plane + (size_t)py * W + px;
		// S = A1 A2 / (B1 B2);  dA1/dmu1 = 2 mu2, dA2/dmu1 = -2 mu2, dB1/dmu1 = 2 mu1, dB2/dmu1 = -2 mu1, dB2/ds11 = 1, dA2/ds12 = 2
		d_mu[o] = 2.f * m2 * (A2 - A1) * inv - S * 2.f * m1 * (1.0f / B1 - 1.0f / B2);
		d_xx[o] = -S / B2;
		d_xy[o] = 2.f * A1 * inv;
		const bool on = owned && (mask == nullptr || mask[(size_t)py * W + px]);
		if (on) {
			v_l1 = fabsf(ip[(size_t)py * W + px] - gp[(size_t)py * W + px]);
			v_cnt = c == 0 ? 1.f : 0.f;
		}
	}
	// block reduction of the three partial sums
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		v_ssim += __shfl_xor_sync(0xffffffffu, v_ssim, o);
		v_l1 += __shfl_xor_sync(0xffffffffu, v_l1, o);
		v_cnt += __shfl_xor_sync(0xffffffffu, v_cnt, o);
	}
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	if (lane == 0) { red[0][warp] = v_ssim; red[1][warp] = v_l1; red[2][warp] = v_cnt; }
	__syncthreads();
	if (threadIdx.x < 3) {
		double s = 0.0;
		for (int k = 0; k < 8; k++) s += (double)red[threadIdx.x][k];
		atomicAdd(acc + threadIdx.x, s);
	}
}

// dL/dimage = w_ssim/(C H W) * [ conv(d_mu) + 2 x conv(d_xx) + y conv(d_xy) ] + w_l1/(n_mask C) * sign(x - y), zero outside the mask.
// scalars: [0] w_l1 * L1 + w_ssim * SSIM, [1] L1, [2] SSIM, [3] masked pixel count
// One block row per owned tile row (blockIdx.y = its index in the band); acc holds the sums of every band of the frame.
__global__ void __launch_bounds__(256) ssim_grad_kernel(const int C, const int H, const int W, const Band band, const GaussWin win,
                                                       const float *__restrict__ img, const float *__restrict__ gt,
                                                       const uint8_t *__restrict__ mask, const float *__restrict__ d_mu,
                                                       const float *__restrict__ d_xx, const float *__restrict__ d_xy,
                                                       const double *__restrict__ acc, const float w_l1, const float w_ssim,
                                                       float *__restrict__ grad, float *__restrict__ scalars) {
	__shared__ float s[3][kExt][kExt + 1];
	__shared__ float h[3][kExt][kTileL + 1];
	const int tile_y = band.begin + (int)blockIdx.y * band.step;
	const int c = blockIdx.z, tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
	const int x0 = blockIdx.x * kTileL - kHalo, y0 = tile_y * kTileL - kHalo;
	const size_t plane = (size_t)H * W;
	const double n_el = (double)C * (double)plane, n_l1 = acc[2] * (double)C;
	if (blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 0 && scalars != nullptr) {
		const double l1 = n_l1 > 0.0 ? acc[1] / n_l1 : 0.0 / 0.0;  // (an empty mask is a NaN mean in the reference as well)
		const double ss = acc[0] / n_el;
		// a term with weight 0 is absent, not 0 * NaN: ssim() under an empty mask is 1, as in the reference
		scalars[0] = (float)((w_l1 != 0.f ? (double)w_l1 * l1 : 0.0) + (double)w_ssim * ss);
		scalars[1] = (float)l1;
		scalars[2] = (float)ss;
		scalars[3] = (float)acc[2];
	}
	if (grad == nullptr || tile_y >= band.end) return;  // (an empty band launches one block for the scalars)
	const size_t cbase = (size_t)c * plane;
	for (int e = threadIdx.x; e < kExt * kExt; e += 256) {
		const int r = e / kExt, q = e - r * kExt, yy = y0 + r, xx = x0 + q;
		const bool in = yy >= 0 && yy < H && xx >= 0 && xx < W;
		const size_t o = cbase + (size_t)yy * W + xx;
		s[0][r][q] = in ? d_mu[o] : 0.f;
		s[1][r][q] = in ? d_xx[o] : 0.f;
		s[2][r][q] = in ? d_xy[o] : 0.f;
	}
	__syncthreads();
	for (int e = threadIdx.x; e < kExt * kTileL; e += 256) {
		const int r = e / kTileL, q = e - r * kTileL;
		float a = 0.f, b = 0.f, d = 0.f;
#pragma unroll
		for (int k = 0; k < kWin; k++) {
			const float w = win.w[k];
			a += w * s[0][r][q + k]; b += w * s[1][r][q + k]; d += w * s[2][r][q + k];
		}
		h[0][r][q] = a; h[1][r][q] = b; h[2][r][q] = d;
	}
	__syncthreads();
	const int px = blockIdx.x * kTileL + tx, py = tile_y * kTileL + ty;
	if (px >= W || py >= H) return;
	const size_t o = cbase + (size_t)py * W + px;
	const bool on = mask == nullptr || mask[(size_t)py * W + px];
	float g = 0.f;
	if (on) {
		float a = 0.f, b = 0.f, d = 0.f;
#pragma unroll
		for (int k = 0; k < kWin; k++) {
			const float w = win.w[k];
			a += w * h[0][ty + k][tx]; b += w * h[1][ty + k][tx]; d += w * h[2][ty + k][tx];
		}
		const float x = img[o], y = gt[o];
		g = (float)((double)w_ssim / n_el) * (a + 2.f * x * b + y * d);
		const float df = x - y;
		const float sgn = df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f);  // torch.abs backward: sign(0) = 0
		if (n_l1 > 0.0) g += (float)((double)w_l1 / n_l1) * sgn;
	}
	grad[o] = g;
}

// Per-pixel losses of an accumulation map clamped to [1e-6, 1 - 1e-6], selected per pixel by a uint8 flag.
// sky (train.py:107-108):          sky ? -log(1 - acc) : -log(acc)
struct SkyForm {
	static __device__ __forceinline__ float value(float ac, bool s) { return s ? -logf(1.f - ac) : -logf(ac); }
	static __device__ __forceinline__ float deriv(float ac, bool s) { return s ? 1.f / (1.f - ac) : -1.f / ac; }
};
// object accumulation (train.py:117-120): obj_bound ? -(acc log acc + (1 - acc) log(1 - acc)) : -log(1 - acc)
struct ObjForm {
	static __device__ __forceinline__ float value(float ac, bool b) {
		const float om = 1.f - ac;
		return b ? -__fadd_rn(__fmul_rn(ac, logf(ac)), __fmul_rn(om, logf(om))) : -logf(om);  // two roundings, as torch does them
	}
	static __device__ __forceinline__ float deriv(float ac, bool b) {
		const float om = 1.f - ac;
		return b ? logf(om) - logf(ac) : 1.f / om;
	}
};

// out[0] += sum of Form::value; grad = weight / N * d/dacc (zero where the clamp is active, like torch.clamp's backward).
// A NaN acc stays NaN through the clamp, as in torch.clamp (fmaxf alone would turn it into 1e-6): the value reports the diverged
// render, and the pixel's gradient is 0 since `inside` is false for NaN.
// kBand: the loop runs over the M = band_rows * strip pixels of the band's tile rows (strip = 16 W pixels per tile row), the rows past
// the image's last one skipped; N stays the pixel count of the whole frame.
template <class Form, bool kBand>
__global__ void __launch_bounds__(256) acc_loss_kernel(const size_t N, const size_t M, const Band band, const size_t strip,
                                                      const float *__restrict__ accm, const uint8_t *__restrict__ flag, const float weight,
                                                      float *__restrict__ grad, double *__restrict__ out) {
	__shared__ float red[8];
	float v = 0.f;
	for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < M; j += (size_t)gridDim.x * blockDim.x) {
		const size_t i = kBand ? (size_t)(band.begin + (int)(j / strip) * band.step) * strip + j % strip : j;
		if (kBand && i >= N) continue;
		const float a = accm[i];
		const float ac = a != a ? a : fminf(fmaxf(a, 1e-6f), 1.f - 1e-6f);
		const bool inside = a >= 1e-6f && a <= 1.f - 1e-6f;
		const bool s = flag[i] != 0;
		v += Form::value(ac, s);
		if (grad) grad[i] = inside ? (weight / (float)N) * Form::deriv(ac, s) : 0.f;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
	__syncthreads();
	if (threadIdx.x == 0) {
		double s = 0.0;
		for (int k = 0; k < 8; k++) s += (double)red[k];
		atomicAdd(out, s);
	}
}
__global__ void acc_loss_finalize_kernel(const size_t N, const float weight, const double *__restrict__ sum, float *__restrict__ scalars) {
	scalars[0] = (float)((double)weight * (*sum / (double)N));
	scalars[1] = (float)(*sum / (double)N);
}

size_t image_loss_scratch_bytes(int C, int H, int W) { return align_up((size_t)3 * C * H * W * sizeof(float)) + 256; }

const GaussWin &ssim_window() {
	static const GaussWin win = make_window();
	return win;
}

cudaError_t launch_image_loss_stats(int C, int H, int W, Band band, const float *img, const float *gt, const uint8_t *mask, double *acc,
                                    void *scratch, cudaStream_t st) {
	const size_t n = (size_t)C * H * W;
	float *d_mu = reinterpret_cast<float *>(scratch), *d_xx = d_mu + n, *d_xy = d_xx + n;
	cudaError_t e = cudaMemsetAsync(acc, 0, 3 * sizeof(double), st);
	if (e != cudaSuccess) return e;
	const unsigned tiles = stats_tiles(band, (H + kTileL - 1) / kTileL);
	if (tiles == 0) return cudaSuccess;
	count_launch(1);
	ssim_stats_kernel<<<dim3((W + kTileL - 1) / kTileL, tiles, C), 256, 0, st>>>(C, H, W, band, ssim_window(), img, gt, mask, d_mu, d_xx, d_xy, acc);
	return cudaGetLastError();
}

cudaError_t launch_image_loss_grad(int C, int H, int W, Band band, const float *img, const float *gt, const uint8_t *mask, const double *acc,
                                   float w_l1, float w_ssim, float *grad, float *scalars, void *scratch, cudaStream_t st) {
	const size_t n = (size_t)C * H * W;
	const float *d_mu = reinterpret_cast<float *>(scratch), *d_xx = d_mu + n, *d_xy = d_xx + n;
	const unsigned rows = band_rows(band);
	count_launch(1);
	ssim_grad_kernel<<<grad && rows ? dim3((W + kTileL - 1) / kTileL, rows, C) : dim3(1, 1, 1), 256, 0, st>>>(
	    C, H, W, band, ssim_window(), img, gt, mask, d_mu, d_xx, d_xy, acc, w_l1, w_ssim, grad, scalars);
	return cudaGetLastError();
}

cudaError_t launch_image_loss(int C, int H, int W, const float *img, const float *gt, const uint8_t *mask, float w_l1, float w_ssim, float *grad,
                              float *scalars, void *scratch, cudaStream_t st) {
	const size_t n = (size_t)C * H * W;
	double *acc = reinterpret_cast<double *>(reinterpret_cast<char *>(scratch) + align_up(3 * n * sizeof(float)));
	const Band whole{0, (H + kTileL - 1) / kTileL, 1};
	cudaError_t e = launch_image_loss_stats(C, H, W, whole, img, gt, mask, acc, scratch, st);
	if (e != cudaSuccess) return e;
	return launch_image_loss_grad(C, H, W, whole, img, gt, mask, acc, w_l1, w_ssim, grad, scalars, scratch, st);
}

static unsigned acc_loss_blocks(size_t M) { return (unsigned)((M + 255) / 256 < kNumSMs * 8 ? (M + 255) / 256 : kNumSMs * 8); }

template <class Form>
static cudaError_t launch_acc_loss(size_t N, const float *accm, const uint8_t *flag, float weight, float *grad, float *scalars, void *scratch,
                                   cudaStream_t st) {
	double *sum = reinterpret_cast<double *>(scratch);
	cudaError_t e = cudaMemsetAsync(sum, 0, sizeof(double), st);
	if (e != cudaSuccess) return e;
	const unsigned nblk = acc_loss_blocks(N);
	count_launch(2);
	acc_loss_kernel<Form, false><<<nblk ? nblk : 1, 256, 0, st>>>(N, N, Band{0, 1, 1}, N, accm, flag, weight, grad, sum);
	acc_loss_finalize_kernel<<<1, 1, 0, st>>>(N, weight, sum, scalars);
	return cudaGetLastError();
}

cudaError_t launch_sky_loss(size_t N, const float *accm, const uint8_t *sky, float weight, float *grad, float *scalars, void *scratch, cudaStream_t st) {
	return launch_acc_loss<SkyForm>(N, accm, sky, weight, grad, scalars, scratch, st);
}

cudaError_t launch_obj_acc_loss(size_t N, const float *accm, const uint8_t *obj_bound, float weight, float *grad, float *scalars, void *scratch,
                                cudaStream_t st) {
	return launch_acc_loss<ObjForm>(N, accm, obj_bound, weight, grad, scalars, scratch, st);
}

template <class Form>
static cudaError_t launch_acc_loss_band(int H, int W, Band band, const float *accm, const uint8_t *flag, float weight, float *grad, double *sum,
                                        cudaStream_t st) {
	cudaError_t e = cudaMemsetAsync(sum, 0, sizeof(double), st);
	if (e != cudaSuccess) return e;
	const size_t N = (size_t)H * W, strip = (size_t)kTileL * W, M = (size_t)band_rows(band) * strip;
	if (M == 0) return cudaSuccess;
	count_launch(1);
	acc_loss_kernel<Form, true><<<acc_loss_blocks(M), 256, 0, st>>>(N, M, band, strip, accm, flag, weight, grad, sum);
	return cudaGetLastError();
}

cudaError_t launch_acc_loss_band(int form, int H, int W, Band band, const float *accm, const uint8_t *flag, float weight, float *grad, double *sum,
                                 cudaStream_t st) {
	return form == 0 ? launch_acc_loss_band<SkyForm>(H, W, band, accm, flag, weight, grad, sum, st)
	                 : launch_acc_loss_band<ObjForm>(H, W, band, accm, flag, weight, grad, sum, st);
}

cudaError_t launch_acc_loss_value(size_t N, float weight, const double *sum, float *scalars, cudaStream_t st) {
	count_launch(1);
	acc_loss_finalize_kernel<<<1, 1, 0, st>>>(N, weight, sum, scalars);
	return cudaGetLastError();
}

// ---- LiDAR depth loss (train.py:124-132) ----
// Radix digits of the 32-bit keys: bits 31..21, 20..10, 9..0.  Valid errors are >= 0 (NaN included, |x| clears the sign), so the
// unsigned order of their bit patterns is the float order with NaN above +inf, as torch.topk orders it.
// The select state is SgrLidarState (include/sgr.h):
//   n       valid pixels
//   k       int(keep * n)
//   prefix  digits selected so far; after the last level the k-th smallest key t
//   rank    1-based rank of the k-th smallest key among the keys carrying `prefix`; in the end the number of ties taken
//   sum_lt  sum of the errors whose key is < t (single-GPU call; a band writes its partial sums to the caller's `sums` instead)
//   hist    the three levels' histograms
constexpr int kLidarBins = SGR_LIDAR_BINS;
using LidarState = SgrLidarState;
// Every pass splits the image into the same lidar_grid(N) blocks of contiguous pixel ranges (the grid depends on N only, so the call
// can be captured in a CUDA graph); the k smallest errors are found by an exact radix select on their fp32 bit patterns.
struct LidarGrid {
	unsigned blocks;
	size_t chunk;  // pixels per block, a multiple of 256
};
// The pixels of the passes: block (x, y) covers [row0 + x chunk, +chunk) clipped to [row0, row0 + row_px) and to N, with
// row0 = (begin + y step) row_px.  The single-GPU call is one row of N pixels (y = 0); a band has one row of 16 W pixels (a tile row)
// per owned tile row, so each block's pixels lie in one tile row.
struct PixelRows {
	size_t row_px;
	int begin, step;
	__device__ __forceinline__ int tile() const { return begin + (int)blockIdx.y * step; }
	__device__ __forceinline__ void range(size_t N, size_t chunk, size_t &lo, size_t &hi) const {
		const size_t row0 = (size_t)tile() * row_px, end = row0 + row_px < N ? row0 + row_px : N;
		lo = row0 + (size_t)blockIdx.x * chunk;
		hi = lo + chunk < end ? lo + chunk : end;
	}
};
static LidarGrid lidar_grid(size_t N) {
	const size_t tiles = (N + 255) / 256;
	const size_t blocks = tiles < kNumSMs * 4 ? tiles : kNumSMs * 4;
	return LidarGrid{(unsigned)(blocks ? blocks : 1), ((tiles + blocks - 1) / (blocks ? blocks : 1)) * 256};
}

size_t lidar_depth_loss_scratch_bytes(size_t N) {
	return align_up(sizeof(LidarState)) + align_up((size_t)lidar_grid(N).blocks * sizeof(uint32_t)) + align_up(N * sizeof(uint32_t));
}

// pass 1: e = depth / (acc + 1e-10), key = bits of |e - lidar| on valid pixels (0xFFFFFFFF elsewhere), n, histogram of key >> 21
__global__ void __launch_bounds__(256) lidar_key_kernel(const size_t N, const size_t chunk, const PixelRows px, const float *__restrict__ depth,
                                                       const float *__restrict__ acc, const float *__restrict__ lidar,
                                                       const uint8_t *__restrict__ mask, uint32_t *__restrict__ keys, LidarState *__restrict__ s) {
	__shared__ uint32_t hist[kLidarBins];
	__shared__ uint32_t nblk;
	for (int b = threadIdx.x; b < kLidarBins; b += 256) hist[b] = 0;
	if (threadIdx.x == 0) nblk = 0;
	__syncthreads();
	size_t lo, hi;
	px.range(N, chunk, lo, hi);
	uint32_t cnt = 0;
	for (size_t i = lo + threadIdx.x; i < hi; i += 256) {
		const float l = lidar[i];
		uint32_t key = 0xFFFFFFFFu;
		if (l > 0.f && (mask == nullptr || mask[i])) {
			const float e = __fdiv_rn(depth[i], __fadd_rn(acc[i], 1e-10f));
			key = __float_as_uint(fabsf(__fsub_rn(e, l)));
			atomicAdd(&hist[key >> 21], 1u);
			cnt++;
		}
		keys[i] = key;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
	if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&nblk, cnt);
	__syncthreads();
	for (int b = threadIdx.x; b < kLidarBins; b += 256)
		if (hist[b]) atomicAdd(&s->hist[0][b], hist[b]);
	if (threadIdx.x == 0 && nblk) atomicAdd(&s->n, nblk);
}

// passes 2 and 3: histogram of the next digit of the keys that carry the prefix selected so far
//   level 1: keys with key >> 21 == prefix, digit (key >> 10) & 2047;  level 2: key >> 10 == prefix, digit key & 1023
__global__ void __launch_bounds__(256) lidar_hist_kernel(const size_t N, const size_t chunk, const PixelRows px, const int level,
                                                        const uint32_t *__restrict__ keys,
                                                        LidarState *__restrict__ s) {
	__shared__ uint32_t hist[kLidarBins];
	if (s->k == 0) return;
	for (int b = threadIdx.x; b < kLidarBins; b += 256) hist[b] = 0;
	__syncthreads();
	const uint32_t prefix = s->prefix;
	const int shift = level == 1 ? 21 : 10, dshift = level == 1 ? 10 : 0;
	const uint32_t dmask = level == 1 ? 2047u : 1023u;
	size_t lo, hi;
	px.range(N, chunk, lo, hi);
	for (size_t i = lo + threadIdx.x; i < hi; i += 256) {
		const uint32_t key = keys[i];
		if (key != 0xFFFFFFFFu && (key >> shift) == prefix) atomicAdd(&hist[(key >> dshift) & dmask], 1u);
	}
	__syncthreads();
	for (int b = threadIdx.x; b < kLidarBins; b += 256)
		if (hist[b]) atomicAdd(&s->hist[level][b], hist[b]);
}

// One block of 1024 threads: finds the digit of the level's histogram that holds the rank-th smallest key and narrows the prefix and the
// rank to that bin.  Level 0 first forms k = int(keep * n) in fp64, exactly Python's int(0.95 * n).
__global__ void __launch_bounds__(1024) lidar_select_kernel(const int level, const double keep, LidarState *__restrict__ s) {
	__shared__ uint32_t warp_sum[32];
	__shared__ uint32_t k_sh;
	if (threadIdx.x == 0) {
		if (level == 0) s->k = (uint32_t)(keep * (double)s->n);
		k_sh = s->k;
	}
	__syncthreads();
	if (k_sh == 0) return;
	const uint32_t rank = level == 0 ? k_sh : s->rank;  // 1-based rank among the keys that carry the prefix
	constexpr int kPer = kLidarBins / 1024;
	const uint32_t *h = s->hist[level];
	uint32_t c[kPer], own = 0;
#pragma unroll
	for (int j = 0; j < kPer; j++) own += (c[j] = h[threadIdx.x * kPer + j]);
	// block inclusive scan of `own`
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t inc = own;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
		if (lane >= o) inc += t;
	}
	if (lane == 31) warp_sum[warp] = inc;
	__syncthreads();
	if (warp == 0) {
		uint32_t w = warp_sum[lane];
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, w, o);
			if (lane >= o) w += t;
		}
		warp_sum[lane] = w;
	}
	__syncthreads();
	if (warp > 0) inc += warp_sum[warp - 1];
	const uint32_t exc = inc - own;
	if (own == 0 || rank <= exc || rank > inc) return;  // exactly one thread holds the rank
	static_assert(kPer == 2, "two bins per thread");
	uint32_t below = exc, d = 0;
	if (rank > below + c[0]) {  // then the rank lies in the second bin, since rank <= inc
		below += c[0];
		d = 1;
	}
	const uint32_t digit = threadIdx.x * kPer + d;
	const int bits = level == 2 ? 10 : 11;
	s->prefix = level == 0 ? digit : ((s->prefix << bits) | digit);
	s->rank = rank - below;
}

// pass 4: t = prefix (the k-th smallest key).  sum of err over keys < t (fp64, into *sum_lt) and the number of keys == t in each block
// (and, for a band, in each tile row: row_ties, fp64 counts)
__global__ void __launch_bounds__(256) lidar_sum_kernel(const size_t N, const size_t chunk, const PixelRows px, const uint32_t *__restrict__ keys,
                                                       const LidarState *__restrict__ s, double *__restrict__ sum_lt,
                                                       uint32_t *__restrict__ block_ties, double *__restrict__ row_ties) {
	__shared__ double red_s[8];
	__shared__ uint32_t red_t[8];
	if (s->k == 0) return;
	const uint32_t t = s->prefix;
	size_t lo, hi;
	px.range(N, chunk, lo, hi);
	double sum = 0.0;
	uint32_t ties = 0;
	for (size_t i = lo + threadIdx.x; i < hi; i += 256) {
		const uint32_t key = keys[i];
		if (key < t) sum += (double)__uint_as_float(key);
		ties += key == t;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		sum += __shfl_xor_sync(0xffffffffu, sum, o);
		ties += __shfl_xor_sync(0xffffffffu, ties, o);
	}
	if ((threadIdx.x & 31) == 0) { red_s[threadIdx.x >> 5] = sum; red_t[threadIdx.x >> 5] = ties; }
	__syncthreads();
	if (threadIdx.x == 0) {
		double bs = 0.0;
		uint32_t bt = 0;
		for (int w = 0; w < 8; w++) { bs += red_s[w]; bt += red_t[w]; }
		if (bs != 0.0) atomicAdd(sum_lt, bs);
		block_ties[blockIdx.y * gridDim.x + blockIdx.x] = bt;
		if (row_ties != nullptr && bt) atomicAdd(row_ties + px.tile(), (double)bt);
	}
}

// pass 5: the k selected pixels (keys < t, plus the s->rank tied pixels of lowest flat index) get g = weight * sign(e - lidar) / k,
//   dL/ddepth = g / (acc + 1e-10), dL/dacc = -g * (e / (acc + 1e-10)) (torch's div backward); every other pixel 0.
//   Block 0 writes scalars {weight * mean, mean, n, k}; k == 0 gives NaN and all-zero gradients, like the mean of an empty top-k.
//   The ties before a block are those of the blocks before it in its row and, for a band, those of every rank's tile rows above
//   its own (row_ties: the per-tile-row counts summed over the ranks).
__global__ void __launch_bounds__(256) lidar_grad_kernel(const size_t N, const size_t chunk, const PixelRows px, const float *__restrict__ depth,
                                                        const float *__restrict__ acc, const float *__restrict__ lidar,
                                                        const uint32_t *__restrict__ keys, const LidarState *__restrict__ s,
                                                        const double *__restrict__ sum_lt, const uint32_t *__restrict__ block_ties,
                                                        const double *__restrict__ row_ties, const float weight, float *__restrict__ dL_ddepth,
                                                        float *__restrict__ dL_dacc, float *__restrict__ scalars) {
	__shared__ uint32_t warp_cnt[8];
	__shared__ uint32_t base_sh;
	const uint32_t k = s->k, t = s->prefix, take = s->rank;
	if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
		const double mean = k ? (*sum_lt + (double)take * (double)__uint_as_float(t)) / (double)k : 0.0 / 0.0;
		scalars[0] = (float)((double)weight * mean);
		scalars[1] = (float)mean;
		scalars[2] = (float)s->n;
		scalars[3] = (float)k;
	}
	if (dL_ddepth == nullptr && dL_dacc == nullptr) return;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	// ties in the blocks before this one
	uint32_t before = 0;
	if (k) {
		for (unsigned b = threadIdx.x; b < blockIdx.x; b += 256) before += block_ties[blockIdx.y * gridDim.x + b];
		if (row_ties != nullptr)
			for (int r = threadIdx.x; r < px.tile(); r += 256) before += (uint32_t)row_ties[r];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
		if (lane == 0) warp_cnt[warp] = before;
		__syncthreads();
		if (threadIdx.x == 0) {
			uint32_t b = 0;
			for (int w = 0; w < 8; w++) b += warp_cnt[w];
			base_sh = b;
		}
		__syncthreads();
		before = base_sh;
	}
	const float gk = k ? weight / (float)k : 0.f;
	size_t lo, hi;
	px.range(N, chunk, lo, hi);
	for (size_t i0 = lo; i0 < hi; i0 += 256) {  // block-uniform trip count: the tie scan below needs every thread
		const size_t i = i0 + threadIdx.x;
		const uint32_t key = (k && i < hi) ? keys[i] : 0xFFFFFFFFu;
		const bool tie = k && key == t;
		const unsigned ballot = __ballot_sync(0xffffffffu, tie);
		__syncthreads();  // warp_cnt of the previous tile has been read
		if (lane == 0) warp_cnt[warp] = __popc(ballot);
		__syncthreads();
		uint32_t rank = before + __popc(ballot & ((1u << lane) - 1u));
		for (int w = 0; w < warp; w++) rank += warp_cnt[w];
		for (int w = 0; w < 8; w++) before += warp_cnt[w];
		if (i >= hi) continue;
		float gd = 0.f, ga = 0.f;
		if (key < t || (tie && rank < take)) {
			const float l = lidar[i], b = __fadd_rn(acc[i], 1e-10f);
			const float e = __fdiv_rn(depth[i], b), df = __fsub_rn(e, l);
			const float g = (df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f)) * gk;  // torch.abs backward: sign(0) = sign(NaN) = 0
			gd = __fdiv_rn(g, b);
			ga = -g * __fdiv_rn(e, b);
		}
		if (dL_ddepth) dL_ddepth[i] = gd;
		if (dL_dacc) dL_dacc[i] = ga;
	}
}

cudaError_t launch_lidar_depth_loss(size_t N, const float *depth, const float *acc, const float *lidar, const uint8_t *mask, double keep, float weight,
                                    float *dL_ddepth, float *dL_dacc, float *scalars, void *scratch, cudaStream_t st) {
	const LidarGrid G = lidar_grid(N);
	char *p = reinterpret_cast<char *>(scratch);
	LidarState *s = reinterpret_cast<LidarState *>(p);
	uint32_t *block_ties = reinterpret_cast<uint32_t *>(p + align_up(sizeof(LidarState)));
	uint32_t *keys = reinterpret_cast<uint32_t *>(p + align_up(sizeof(LidarState)) + align_up((size_t)G.blocks * sizeof(uint32_t)));
	cudaError_t e = cudaMemsetAsync(s, 0, sizeof(LidarState), st);
	if (e != cudaSuccess) return e;
	const PixelRows px{N, 0, 0};
	count_launch(8);
	lidar_key_kernel<<<G.blocks, 256, 0, st>>>(N, G.chunk, px, depth, acc, lidar, mask, keys, s);
	lidar_select_kernel<<<1, 1024, 0, st>>>(0, keep, s);
	lidar_hist_kernel<<<G.blocks, 256, 0, st>>>(N, G.chunk, px, 1, keys, s);
	lidar_select_kernel<<<1, 1024, 0, st>>>(1, keep, s);
	lidar_hist_kernel<<<G.blocks, 256, 0, st>>>(N, G.chunk, px, 2, keys, s);
	lidar_select_kernel<<<1, 1024, 0, st>>>(2, keep, s);
	lidar_sum_kernel<<<G.blocks, 256, 0, st>>>(N, G.chunk, px, keys, s, &s->sum_lt, block_ties, nullptr);
	lidar_grad_kernel<<<(dL_ddepth || dL_dacc) ? G.blocks : 1, 256, 0, st>>>(N, G.chunk, px, depth, acc, lidar, keys, s, &s->sum_lt, block_ties,
	                                                                        nullptr, weight, dL_ddepth, dL_dacc, scalars);
	return cudaGetLastError();
}

// ---- LiDAR depth loss on a band: the same passes over the band's tile rows, a block row per owned tile row of kBandChunks blocks.  The
// caller sums the state's level-l histogram over the ranks before select level l, so every rank selects the same n, k and t; then it
// sums `sums` = {sum of err < t, keys == t per tile row}, from which each rank takes the ties above its own rows.
constexpr size_t kBandChunk = 2048;  // pixels per block, a multiple of 256
static dim3 lidar_band_grid(int W, Band band) {
	const size_t row_px = (size_t)kTileL * W;
	return dim3((unsigned)((row_px + kBandChunk - 1) / kBandChunk), (unsigned)band_rows(band), 1);
}

size_t lidar_band_scratch_bytes(int H, int W) {
	const Band whole{0, (H + kTileL - 1) / kTileL, 1};
	const dim3 g = lidar_band_grid(W, whole);
	return align_up((size_t)H * W * sizeof(uint32_t)) + align_up((size_t)g.x * g.y * sizeof(uint32_t));
}

static uint32_t *band_keys(void *scratch) { return reinterpret_cast<uint32_t *>(scratch); }
static uint32_t *band_block_ties(int H, int W, void *scratch) {
	return reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(scratch) + align_up((size_t)H * W * sizeof(uint32_t)));
}

cudaError_t launch_lidar_band_keys(int H, int W, Band band, const float *depth, const float *acc, const float *lidar, const uint8_t *mask,
                                   LidarState *s, void *scratch, cudaStream_t st) {
	cudaError_t e = cudaMemsetAsync(s, 0, sizeof(LidarState), st);
	if (e != cudaSuccess) return e;
	const dim3 g = lidar_band_grid(W, band);
	if (g.y == 0) return cudaSuccess;
	count_launch(1);
	lidar_key_kernel<<<g, 256, 0, st>>>((size_t)H * W, kBandChunk, PixelRows{(size_t)kTileL * W, band.begin, band.step}, depth, acc, lidar, mask,
	                                    band_keys(scratch), s);
	return cudaGetLastError();
}

cudaError_t launch_lidar_band_select(int level, double keep, int H, int W, Band band, LidarState *s, double *sums, void *scratch, cudaStream_t st) {
	const dim3 g = lidar_band_grid(W, band);
	const size_t N = (size_t)H * W;
	const PixelRows px{(size_t)kTileL * W, band.begin, band.step};
	count_launch(1);
	lidar_select_kernel<<<1, 1024, 0, st>>>(level - 1, keep, s);
	if (level == 3) {
		cudaError_t e = cudaMemsetAsync(sums, 0, (1 + (size_t)(H + kTileL - 1) / kTileL) * sizeof(double), st);
		if (e != cudaSuccess) return e;
	}
	if (g.y > 0) {
		count_launch(1);
		if (level < 3)
			lidar_hist_kernel<<<g, 256, 0, st>>>(N, kBandChunk, px, level, band_keys(scratch), s);
		else
			lidar_sum_kernel<<<g, 256, 0, st>>>(N, kBandChunk, px, band_keys(scratch), s, sums, band_block_ties(H, W, scratch), sums + 1);
	}
	return cudaGetLastError();
}

cudaError_t launch_lidar_band_grad(int H, int W, Band band, const float *depth, const float *acc, const float *lidar, float weight, const LidarState *s,
                                   const double *sums, float *dL_ddepth, float *dL_dacc, float *scalars, void *scratch, cudaStream_t st) {
	dim3 g = lidar_band_grid(W, band);
	if (g.y == 0 || !(dL_ddepth || dL_dacc)) {
		g = dim3(1, 1, 1);
		dL_ddepth = dL_dacc = nullptr;
	}
	count_launch(1);
	lidar_grad_kernel<<<g, 256, 0, st>>>((size_t)H * W, kBandChunk, PixelRows{(size_t)kTileL * W, band.begin, band.step}, depth, acc, lidar,
	                                     band_keys(scratch), s, sums, band_block_ties(H, W, scratch), sums + 1, weight, dL_ddepth, dL_dacc,
	                                     scalars);
	return cudaGetLastError();
}

}  // namespace sgr

namespace sgr {

// ---- Halo of a band for the photometric loss: the image rows within kBandHalo of its tile rows that other ranks own.  A message is a
// list of strips of kBandHalo rows, strip i at pixel row 16 (first + i step) + offset, the last one clipped at H:
//   send up    the first rows of each owned tile row t >= 1 whose row above is foreign       (for the owner of t - 1)
//   send down  the last rows of each owned tile row t < rows - 1 whose row below is foreign  (for the owner of t + 1)
//   recv up    the rows above the tile rows of "send up", from the owner of t - 1 (its "send down")
//   recv down  the rows below the tile rows of "send down", from the owner of t + 1 (its "send up")
// With step >= 2 (the cyclic layout) no two owned tile rows touch, so every owned tile row has both; with step 1 only the band's
// first and last tile rows do.
HaloStrips halo_strips(int H, Band b, int side) {
	const int rows = (H + kTileL - 1) / kTileL, n = band_rows(b);
	HaloStrips h{0, 0, b.step, 0};
	if (n == 0) return h;
	const int last = b.begin + (n - 1) * b.step;
	const bool up = side == SGR_HALO_SEND_UP || side == SGR_HALO_RECV_UP;
	if (up) {
		h.first = b.begin == 0 ? b.begin + b.step : b.begin;
		h.count = b.step == 1 ? (b.begin >= 1 ? 1 : 0) : n - (b.begin == 0 ? 1 : 0);
	} else {
		h.first = b.step == 1 ? last : b.begin;
		h.count = b.step == 1 ? (last + 1 < rows ? 1 : 0) : n - (last + 1 >= rows ? 1 : 0);
	}
	h.offset = side == SGR_HALO_SEND_UP ? 0 : side == SGR_HALO_SEND_DOWN ? kTileL - kBandHalo : side == SGR_HALO_RECV_UP ? -kBandHalo : kTileL;
	return h;
}

int64_t halo_rows(int H, const HaloStrips &h) {
	if (h.count == 0) return 0;
	const int base = kTileL * (h.first + (h.count - 1) * h.step) + h.offset;
	return (int64_t)kBandHalo * (h.count - 1) + min(kBandHalo, H - base);
}

// buffer [C][rows][W]; kPack: image -> buffer, else buffer -> image
template <bool kPack>
__global__ void __launch_bounds__(256) halo_copy_kernel(const int H, const int W, const HaloStrips h, const size_t rows, const size_t total,
                                                       float *__restrict__ image, float *__restrict__ buf) {
	for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
		const size_t plane = rows * W, c = e / plane, rem = e - c * plane, j = rem / W, x = rem - j * W;
		const int row = kTileL * (h.first + (int)(j / kBandHalo) * h.step) + h.offset + (int)(j % kBandHalo);
		float *px = image + c * (size_t)H * W + (size_t)row * W + x;
		if (kPack)
			buf[e] = *px;
		else
			*px = buf[e];
	}
}

cudaError_t launch_halo_copy(bool pack, int C, int H, int W, Band band, int side, float *image, float *buf, cudaStream_t st) {
	const HaloStrips h = halo_strips(H, band, side);
	const size_t rows = (size_t)halo_rows(H, h), total = (size_t)C * rows * W;
	if (total == 0) return cudaSuccess;
	const unsigned nblk = (unsigned)((total + 255) / 256 < kNumSMs * 8 ? (total + 255) / 256 : kNumSMs * 8);
	count_launch(1);
	if (pack)
		halo_copy_kernel<true><<<nblk, 256, 0, st>>>(H, W, h, rows, total, image, buf);
	else
		halo_copy_kernel<false><<<nblk, 256, 0, st>>>(H, W, h, rows, total, image, buf);
	return cudaGetLastError();
}

}  // namespace sgr
