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
#include "sgr_common.cuh"

namespace sgr {

constexpr int kWin = 11, kHalo = 5, kTileL = 16, kExt = kTileL + 2 * kHalo;  // 26

struct GaussWin {
	float w[kWin];
};
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

// acc: [0] sum of the SSIM map, [1] sum |x - y| over masked elements, [2] number of masked PIXELS (counted on channel 0)
__global__ void __launch_bounds__(256) ssim_stats_kernel(const int C, const int H, const int W, const GaussWin win, const float *__restrict__ img,
                                                        const float *__restrict__ gt, const uint8_t *__restrict__ mask,
                                                        float *__restrict__ d_mu, float *__restrict__ d_xx, float *__restrict__ d_xy,
                                                        double *__restrict__ acc) {
	__shared__ float sx[kExt][kExt + 1], sy[kExt][kExt + 1];
	__shared__ float h[5][kExt][kTileL + 1];
	__shared__ float red[3][8];
	const int c = blockIdx.z, tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
	const int x0 = blockIdx.x * kTileL - kHalo, y0 = blockIdx.y * kTileL - kHalo;
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
	// horizontal pass: 26 rows x 16 columns x 5 quantities
	for (int e = threadIdx.x; e < kExt * kTileL; e += 256) {
		const int r = e / kTileL, q = e - r * kTileL;
		float m1 = 0.f, m2 = 0.f, s11 = 0.f, s22 = 0.f, s12 = 0.f;
#pragma unroll
		for (int k = 0; k < kWin; k++) {
			const float a = sx[r][q + k], b = sy[r][q + k], w = win.w[k];
			m1 += w * a; m2 += w * b; s11 += w * a * a; s22 += w * b * b; s12 += w * a * b;
		}
		h[0][r][q] = m1; h[1][r][q] = m2; h[2][r][q] = s11; h[3][r][q] = s22; h[4][r][q] = s12;
	}
	__syncthreads();
	const int px = blockIdx.x * kTileL + tx, py = blockIdx.y * kTileL + ty;
	float v_ssim = 0.f, v_l1 = 0.f, v_cnt = 0.f;
	if (px < W && py < H) {
		float m1 = 0.f, m2 = 0.f, s11 = 0.f, s22 = 0.f, s12 = 0.f;
#pragma unroll
		for (int k = 0; k < kWin; k++) {
			const float w = win.w[k];
			m1 += w * h[0][ty + k][tx]; m2 += w * h[1][ty + k][tx]; s11 += w * h[2][ty + k][tx]; s22 += w * h[3][ty + k][tx];
			s12 += w * h[4][ty + k][tx];
		}
		const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
		const float mu1_sq = m1 * m1, mu2_sq = m2 * m2, mu12 = m1 * m2;
		const float sig1 = s11 - mu1_sq, sig2 = s22 - mu2_sq, sig12 = s12 - mu12;
		const float A1 = 2.f * mu12 + C1, A2 = 2.f * sig12 + C2, B1 = mu1_sq + mu2_sq + C1, B2 = sig1 + sig2 + C2;
		const float inv = 1.0f / (B1 * B2);
		const float S = A1 * A2 * inv;
		v_ssim = S;
		const size_t o = (size_t)c * plane + (size_t)py * W + px;
		// S = A1 A2 / (B1 B2);  dA1/dmu1 = 2 mu2, dA2/dmu1 = -2 mu2, dB1/dmu1 = 2 mu1, dB2/dmu1 = -2 mu1, dB2/ds11 = 1, dA2/ds12 = 2
		d_mu[o] = 2.f * m2 * (A2 - A1) * inv - S * 2.f * m1 * (1.0f / B1 - 1.0f / B2);
		d_xx[o] = -S / B2;
		d_xy[o] = 2.f * A1 * inv;
		const bool on = mask == nullptr || mask[(size_t)py * W + px];
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
__global__ void __launch_bounds__(256) ssim_grad_kernel(const int C, const int H, const int W, const GaussWin win, const float *__restrict__ img,
                                                       const float *__restrict__ gt, const uint8_t *__restrict__ mask,
                                                       const float *__restrict__ d_mu, const float *__restrict__ d_xx,
                                                       const float *__restrict__ d_xy, const double *__restrict__ acc, const float w_l1,
                                                       const float w_ssim, float *__restrict__ grad, float *__restrict__ scalars) {
	__shared__ float s[3][kExt][kExt + 1];
	__shared__ float h[3][kExt][kTileL + 1];
	const int c = blockIdx.z, tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
	const int x0 = blockIdx.x * kTileL - kHalo, y0 = blockIdx.y * kTileL - kHalo;
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
	if (grad == nullptr) return;
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
	const int px = blockIdx.x * kTileL + tx, py = blockIdx.y * kTileL + ty;
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
template <class Form>
__global__ void __launch_bounds__(256) acc_loss_kernel(const size_t N, const float *__restrict__ accm, const uint8_t *__restrict__ flag, const float weight,
                                                      float *__restrict__ grad, double *__restrict__ out) {
	__shared__ float red[8];
	float v = 0.f;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (size_t)gridDim.x * blockDim.x) {
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

cudaError_t launch_image_loss(int C, int H, int W, const float *img, const float *gt, const uint8_t *mask, float w_l1, float w_ssim, float *grad,
                              float *scalars, void *scratch, cudaStream_t st) {
	static const GaussWin win = make_window();
	const size_t n = (size_t)C * H * W;
	float *d_mu = reinterpret_cast<float *>(scratch), *d_xx = d_mu + n, *d_xy = d_xx + n;
	double *acc = reinterpret_cast<double *>(reinterpret_cast<char *>(scratch) + align_up(3 * n * sizeof(float)));
	cudaError_t e = cudaMemsetAsync(acc, 0, 4 * sizeof(double), st);
	if (e != cudaSuccess) return e;
	const dim3 grid((W + kTileL - 1) / kTileL, (H + kTileL - 1) / kTileL, C);
	count_launch(2);
	ssim_stats_kernel<<<grid, 256, 0, st>>>(C, H, W, win, img, gt, mask, d_mu, d_xx, d_xy, acc);
	ssim_grad_kernel<<<grad ? grid : dim3(1, 1, 1), 256, 0, st>>>(C, H, W, win, img, gt, mask, d_mu, d_xx, d_xy, acc, w_l1, w_ssim, grad, scalars);
	return cudaGetLastError();
}

template <class Form>
static cudaError_t launch_acc_loss(size_t N, const float *accm, const uint8_t *flag, float weight, float *grad, float *scalars, void *scratch,
                                   cudaStream_t st) {
	double *sum = reinterpret_cast<double *>(scratch);
	cudaError_t e = cudaMemsetAsync(sum, 0, sizeof(double), st);
	if (e != cudaSuccess) return e;
	const unsigned nblk = (unsigned)((N + 255) / 256 < kNumSMs * 8 ? (N + 255) / 256 : kNumSMs * 8);
	count_launch(2);
	acc_loss_kernel<Form><<<nblk ? nblk : 1, 256, 0, st>>>(N, accm, flag, weight, grad, sum);
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

// ---- LiDAR depth loss (train.py:124-132) ----
// Radix digits of the 32-bit keys: bits 31..21, 20..10, 9..0.  Valid errors are >= 0 (NaN included, |x| clears the sign), so the
// unsigned order of their bit patterns is the float order with NaN above +inf, as torch.topk orders it.
constexpr int kLidarBins = 2048;
struct LidarState {
	uint32_t n;       // valid pixels
	uint32_t k;       // int(keep * n)
	uint32_t prefix;  // digits selected so far; after the last level the k-th smallest key t
	uint32_t rank;    // 1-based rank of the k-th smallest key among the keys carrying `prefix`; in the end the number of ties taken
	double sum_lt;    // sum of the errors whose key is < t
	uint32_t hist[3][kLidarBins];
};
// Every pass splits the image into the same lidar_grid(N) blocks of contiguous pixel ranges (the grid depends on N only, so the call
// can be captured in a CUDA graph); the k smallest errors are found by an exact radix select on their fp32 bit patterns.
struct LidarGrid {
	unsigned blocks;
	size_t chunk;  // pixels per block, a multiple of 256
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
__global__ void __launch_bounds__(256) lidar_key_kernel(const size_t N, const size_t chunk, const float *__restrict__ depth,
                                                       const float *__restrict__ acc, const float *__restrict__ lidar,
                                                       const uint8_t *__restrict__ mask, uint32_t *__restrict__ keys, LidarState *__restrict__ s) {
	__shared__ uint32_t hist[kLidarBins];
	__shared__ uint32_t nblk;
	for (int b = threadIdx.x; b < kLidarBins; b += 256) hist[b] = 0;
	if (threadIdx.x == 0) nblk = 0;
	__syncthreads();
	const size_t lo = (size_t)blockIdx.x * chunk, hi = lo + chunk < N ? lo + chunk : N;
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
__global__ void __launch_bounds__(256) lidar_hist_kernel(const size_t N, const size_t chunk, const int level, const uint32_t *__restrict__ keys,
                                                        LidarState *__restrict__ s) {
	__shared__ uint32_t hist[kLidarBins];
	if (s->k == 0) return;
	for (int b = threadIdx.x; b < kLidarBins; b += 256) hist[b] = 0;
	__syncthreads();
	const uint32_t prefix = s->prefix;
	const int shift = level == 1 ? 21 : 10, dshift = level == 1 ? 10 : 0;
	const uint32_t dmask = level == 1 ? 2047u : 1023u;
	const size_t lo = (size_t)blockIdx.x * chunk, hi = lo + chunk < N ? lo + chunk : N;
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

// pass 4: t = prefix (the k-th smallest key).  sum of err over keys < t (fp64) and the number of keys == t in each block
__global__ void __launch_bounds__(256) lidar_sum_kernel(const size_t N, const size_t chunk, const uint32_t *__restrict__ keys,
                                                       LidarState *__restrict__ s, uint32_t *__restrict__ block_ties) {
	__shared__ double red_s[8];
	__shared__ uint32_t red_t[8];
	if (s->k == 0) return;
	const uint32_t t = s->prefix;
	const size_t lo = (size_t)blockIdx.x * chunk, hi = lo + chunk < N ? lo + chunk : N;
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
		if (bs != 0.0) atomicAdd(&s->sum_lt, bs);
		block_ties[blockIdx.x] = bt;
	}
}

// pass 5: the k selected pixels (keys < t, plus the s->rank tied pixels of lowest flat index) get g = weight * sign(e - lidar) / k,
//   dL/ddepth = g / (acc + 1e-10), dL/dacc = -g * (e / (acc + 1e-10)) (torch's div backward); every other pixel 0.
//   Block 0 writes scalars {weight * mean, mean, n, k}; k == 0 gives NaN and all-zero gradients, like the mean of an empty top-k.
__global__ void __launch_bounds__(256) lidar_grad_kernel(const size_t N, const size_t chunk, const float *__restrict__ depth,
                                                        const float *__restrict__ acc, const float *__restrict__ lidar,
                                                        const uint32_t *__restrict__ keys, const LidarState *__restrict__ s,
                                                        const uint32_t *__restrict__ block_ties, const float weight, float *__restrict__ dL_ddepth,
                                                        float *__restrict__ dL_dacc, float *__restrict__ scalars) {
	__shared__ uint32_t warp_cnt[8];
	__shared__ uint32_t base_sh;
	const uint32_t k = s->k, t = s->prefix, take = s->rank;
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		const double mean = k ? (s->sum_lt + (double)take * (double)__uint_as_float(t)) / (double)k : 0.0 / 0.0;
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
		for (unsigned b = threadIdx.x; b < blockIdx.x; b += 256) before += block_ties[b];
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
	const size_t lo = (size_t)blockIdx.x * chunk, hi = lo + chunk < N ? lo + chunk : N;
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
	count_launch(8);
	lidar_key_kernel<<<G.blocks, 256, 0, st>>>(N, G.chunk, depth, acc, lidar, mask, keys, s);
	lidar_select_kernel<<<1, 1024, 0, st>>>(0, keep, s);
	lidar_hist_kernel<<<G.blocks, 256, 0, st>>>(N, G.chunk, 1, keys, s);
	lidar_select_kernel<<<1, 1024, 0, st>>>(1, keep, s);
	lidar_hist_kernel<<<G.blocks, 256, 0, st>>>(N, G.chunk, 2, keys, s);
	lidar_select_kernel<<<1, 1024, 0, st>>>(2, keep, s);
	lidar_sum_kernel<<<G.blocks, 256, 0, st>>>(N, G.chunk, keys, s, block_ties);
	lidar_grad_kernel<<<(dL_ddepth || dL_dacc) ? G.blocks : 1, 256, 0, st>>>(N, G.chunk, depth, acc, lidar, keys, s, block_ties, weight, dL_ddepth,
	                                                                        dL_dacc, scalars);
	return cudaGetLastError();
}

}  // namespace sgr
