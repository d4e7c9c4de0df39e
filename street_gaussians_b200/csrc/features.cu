// features.cu — the feature channels of street_gaussians' renderer (street_gaussian_renderer.py:206-264, cfg.render.render_normal and
// cfg.data.use_semantic) as fused kernels: the per-Gaussian normals (GaussianModel.get_normals, gaussian_model.py:256-269), the
// composed semantics (GaussianModel / GaussianModelActor.get_semantic, gaussian_model.py:243-247, gaussian_model_actor.py:62-69) and
// the finishing of the rendered maps (F.normalize of the normals, the probabilities' log).
//
// All three are streams: one thread per Gaussian row (normals, background semantics), per output element (actor semantics) or per
// pixel (finishing).  Grids depend on the sizes only and nothing is read back to the host.  The normals' forward keeps one byte per
// Gaussian (argmin column, sign) that its backward applies, so the backward takes the forward's decisions on every row.  Arithmetic
// that the reference fixes (the quaternion's matrix, the sign test) is written with explicit _rn intrinsics so nvcc contracts
// nothing into an FMA.
#include "sgr_common.cuh"

namespace sgr {

constexpr int kFeatThreads = 256;
constexpr int kSemSeg = SGR_MAX_SEGMENTS_PER_LAUNCH;
constexpr uint8_t kNormalFlip = 4;  // decision byte: bits 0-1 the argmin column, bit 2 set where the normal is negated

static int feat_blocks(int64_t n) { return (int)((n + kFeatThreads - 1) / kFeatThreads); }

// ---- gaussian normals -----------------------------------------------------------------------------------------------------------

// Column k of quaternion_to_matrix(q) (general_utils.py:125-146): its own normalisation by sqrt(q.q), then the entries in the
// reference's operation order.
__device__ __forceinline__ void rot_column(const float4 r, const int k, float n[3]) {
	const float nn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r.x, r.x), __fmul_rn(r.y, r.y)), __fmul_rn(r.z, r.z)), __fmul_rn(r.w, r.w)));
	const float w = __fdiv_rn(r.x, nn), x = __fdiv_rn(r.y, nn), y = __fdiv_rn(r.z, nn), z = __fdiv_rn(r.w, nn);
	const auto one_minus = [](float a, float b) { return __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(a, b))); };
	const auto two_plus = [](float a, float b) { return __fmul_rn(2.f, __fadd_rn(a, b)); };
	const auto two_minus = [](float a, float b) { return __fmul_rn(2.f, __fsub_rn(a, b)); };
	const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
	const float xy = __fmul_rn(x, y), xz = __fmul_rn(x, z), yz = __fmul_rn(y, z);
	const float wx = __fmul_rn(w, x), wy = __fmul_rn(w, y), wz = __fmul_rn(w, z);
	if (k == 0) {
		n[0] = one_minus(yy, zz); n[1] = two_plus(xy, wz); n[2] = two_minus(xz, wy);
	} else if (k == 1) {
		n[0] = two_minus(xy, wz); n[1] = one_minus(xx, zz); n[2] = two_plus(yz, wx);
	} else {
		n[0] = two_plus(xz, wy); n[1] = two_minus(yz, wx); n[2] = one_minus(xx, yy);
	}
}

// torch.argmin over three values: the first minimum, and a NaN counts as smaller than everything (the first NaN wins).
__device__ __forceinline__ int argmin3(const float s0, const float s1, const float s2) {
	int k = 0;
	float best = s0;
	if (!(best != best) && (s1 < best || s1 != s1)) { k = 1; best = s1; }
	if (!(best != best) && (s2 < best || s2 != s2)) k = 2;
	return k;
}

__global__ void __launch_bounds__(kFeatThreads) gaussian_normals_fwd_kernel(const int P, const float *__restrict__ means, const float4 *__restrict__ rots,
                                                                             const float *__restrict__ scales, const float *__restrict__ center,
                                                                             float *__restrict__ normals, uint8_t *__restrict__ decision) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const int k = argmin3(__ldg(scales + 3 * i), __ldg(scales + 3 * i + 1), __ldg(scales + 3 * i + 2));
	float n[3];
	rot_column(__ldg(rots + i), k, n);
	// dir_pp / |dir_pp| (gaussian_model.py:264-265), then sum(-d * n) >= 0 keeps n; a NaN (a Gaussian at the camera centre) takes -n
	const float dx = __fsub_rn(__ldg(means + 3 * i), __ldg(center)), dy = __fsub_rn(__ldg(means + 3 * i + 1), __ldg(center + 1));
	const float dz = __fsub_rn(__ldg(means + 3 * i + 2), __ldg(center + 2));
	const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
	const float ux = __fdiv_rn(dx, len), uy = __fdiv_rn(dy, len), uz = __fdiv_rn(dz, len);
	const float dot = __fadd_rn(__fadd_rn(__fmul_rn(-ux, n[0]), __fmul_rn(-uy, n[1])), __fmul_rn(-uz, n[2]));
	const bool keep = dot >= 0.f;
	const float s = keep ? 1.f : -1.f;
	normals[3 * i] = s * n[0];
	normals[3 * i + 1] = s * n[1];
	normals[3 * i + 2] = s * n[2];
	decision[i] = (uint8_t)(k | (keep ? 0 : kNormalFlip));
}

// dL/dr through n = s R(r / |r|)[:, k]: g_q = s J_k^T g (J_k the column's derivative in the normalised quaternion q = (w, x, y, z)),
// then dL/dr = (g_q - q (q . g_q)) / |r|.  The column and the sign are the forward's, read from its decision byte.
__global__ void __launch_bounds__(kFeatThreads) gaussian_normals_bwd_kernel(const int P, const float4 *__restrict__ rots,
                                                                             const uint8_t *__restrict__ decision, const float *__restrict__ gn,
                                                                             float4 *__restrict__ grot) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const float4 r = __ldg(rots + i);
	const uint8_t dec = __ldg(decision + i);
	const int k = dec & 3;
	const float s = (dec & kNormalFlip) ? -1.f : 1.f;
	const float g0 = s * __ldg(gn + 3 * i), g1 = s * __ldg(gn + 3 * i + 1), g2 = s * __ldg(gn + 3 * i + 2);
	const float nn = sqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
	const float w = r.x / nn, x = r.y / nn, y = r.z / nn, z = r.w / nn;
	float gw, gx, gy, gz;
	if (k == 0) {  // (1 - 2(y^2 + z^2), 2(xy + wz), 2(xz - wy))
		gw = 2.f * (z * g1 - y * g2);
		gx = 2.f * (y * g1 + z * g2);
		gy = -4.f * y * g0 + 2.f * (x * g1 - w * g2);
		gz = -4.f * z * g0 + 2.f * (w * g1 + x * g2);
	} else if (k == 1) {  // (2(xy - wz), 1 - 2(x^2 + z^2), 2(yz + wx))
		gw = 2.f * (x * g2 - z * g0);
		gx = 2.f * (y * g0 + w * g2) - 4.f * x * g1;
		gy = 2.f * (x * g0 + z * g2);
		gz = 2.f * (y * g2 - w * g0) - 4.f * z * g1;
	} else {  // (2(xz + wy), 2(yz - wx), 1 - 2(x^2 + y^2))
		gw = 2.f * (y * g0 - x * g1);
		gx = 2.f * (z * g0 - w * g1) - 4.f * x * g2;
		gy = 2.f * (w * g0 + z * g1) - 4.f * y * g2;
		gz = 2.f * (x * g0 + y * g1);
	}
	const float qg = w * gw + x * gx + y * gy + z * gz;
	grot[i] = make_float4((gw - w * qg) / nn, (gx - x * qg) / nn, (gy - y * qg) / nn, (gz - z * qg) / nn);
}

cudaError_t launch_gaussian_normals_fwd(int P, const float *means, const float *rots, const float *scales, const float *center, float *normals,
                                        uint8_t *decision, cudaStream_t st) {
	count_launch();
	gaussian_normals_fwd_kernel<<<feat_blocks(P), kFeatThreads, 0, st>>>(P, means, reinterpret_cast<const float4 *>(rots), scales, center, normals,
	                                                                      decision);
	return cudaGetLastError();
}

cudaError_t launch_gaussian_normals_bwd(int P, const float *rots, const uint8_t *decision, const float *g_normals, float *g_rots, cudaStream_t st) {
	count_launch();
	gaussian_normals_bwd_kernel<<<feat_blocks(P), kFeatThreads, 0, st>>>(P, reinterpret_cast<const float4 *>(rots), decision, g_normals,
	                                                                      reinterpret_cast<float4 *>(g_rots));
	return cudaGetLastError();
}

// ---- composed semantics ---------------------------------------------------------------------------------------------------------

struct SemTable {
	int n;                   // actor segments in this launch
	int start[kSemSeg + 1];  // composed row of each segment's first Gaussian; start[n] = end
	int label[kSemSeg];
	const float *src[kSemSeg];
	float *grad[kSemSeg];
};

__device__ __forceinline__ int sem_segment(const SemTable &t, int row) {
	int lo = 0, hi = t.n - 1;  // largest s with start[s] <= row
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (t.start[mid] <= row) lo = mid; else hi = mid - 1;
	}
	return lo;
}

__device__ __forceinline__ float sigmoid_ref(float v) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-v))); }

// Background rows in 'probabilities' mode: softmax over the row (max, sum of exp(x - max), exp(x - max) / sum).
__global__ void __launch_bounds__(kFeatThreads) semantic_softmax_fwd_kernel(const int n, const int K, const float *__restrict__ src,
                                                                            float *__restrict__ out) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float *x = src + (int64_t)i * K;
	float *y = out + (int64_t)i * K;
	float m = __ldg(x);
	for (int c = 1; c < K; c++) {
		const float v = __ldg(x + c);
		m = (v > m || v != v) ? v : m;
	}
	float sum = 0.f;
	for (int c = 0; c < K; c++) sum = __fadd_rn(sum, expf(__fsub_rn(__ldg(x + c), m)));
	for (int c = 0; c < K; c++) y[c] = __fdiv_rn(expf(__fsub_rn(__ldg(x + c), m)), sum);
}

// softmax backward: dL/dx = y (g - sum_c g_c y_c), with y the forward's output rows.
__global__ void __launch_bounds__(kFeatThreads) semantic_softmax_bwd_kernel(const int n, const int K, const float *__restrict__ y,
                                                                            const float *__restrict__ g, float *__restrict__ gx) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float *yr = y + (int64_t)i * K;
	const float *gr = g + (int64_t)i * K;
	float dot = 0.f;
	for (int c = 0; c < K; c++) dot = fmaf(__ldg(gr + c), __ldg(yr + c), dot);
	float *o = gx + (int64_t)i * K;
	for (int c = 0; c < K; c++) o[c] = __ldg(yr + c) * (__ldg(gr + c) - dot);
}

// Actor rows: one thread per output element; column `label` holds _semantic[:, 0] (logits) or its sigmoid, the rest are 0.
__global__ void __launch_bounds__(kFeatThreads) semantic_actor_fwd_kernel(const SemTable t, const int K, const int mode, float *__restrict__ out) {
	const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	const int64_t base = (int64_t)t.start[0] * K;
	if (e >= (int64_t)t.start[t.n] * K - base) return;
	const int row = (int)((base + e) / K), col = (int)((base + e) - (int64_t)row * K);
	const int s = sem_segment(t, row);
	float v = 0.f;
	if (col == t.label[s]) {
		v = __ldg(t.src[s] + (row - t.start[s]));
		if (mode == SGR_SEMANTIC_PROBABILITIES) v = sigmoid_ref(v);
	}
	out[base + e] = v;
}

// dL/d_semantic[:, 0] = g[:, label] (logits) or g[:, label] (1 - y) y with y the forward's sigmoid (torch's sigmoid_backward).
__global__ void __launch_bounds__(kFeatThreads) semantic_actor_bwd_kernel(const SemTable t, const int K, const int mode, const float *__restrict__ y,
                                                                          const float *__restrict__ g) {
	const int row = t.start[0] + blockIdx.x * blockDim.x + threadIdx.x;
	if (row >= t.start[t.n]) return;
	const int s = sem_segment(t, row);
	const int64_t at = (int64_t)row * K + t.label[s];
	float v = __ldg(g + at);
	if (mode == SGR_SEMANTIC_PROBABILITIES) {
		const float yy = __ldg(y + at);
		v = __fmul_rn(__fmul_rn(v, __fsub_rn(1.f, yy)), yy);
	}
	t.grad[s][row - t.start[s]] = v;
}

template <typename F>
static cudaError_t for_actor_groups(int n_act, const int32_t *start, const int32_t *label, F &&launch) {
	for (int first = 0; first < n_act; first += kSemSeg) {
		SemTable t;
		t.n = n_act - first < kSemSeg ? n_act - first : kSemSeg;
		for (int k = 0; k <= t.n; k++) t.start[k] = start[first + k];
		for (int k = 0; k < t.n; k++) t.label[k] = label[first + k];
		if (t.start[t.n] == t.start[0]) continue;
		if (cudaError_t e = launch(t, first)) return e;
	}
	return cudaSuccess;
}

cudaError_t launch_compose_semantics_fwd(int n_bg, int K, int mode, const float *bg, int n_act, const int32_t *start, const int32_t *label,
                                         const float *const *actor, float *out, cudaStream_t st) {
	if (n_bg > 0) {
		if (mode == SGR_SEMANTIC_LOGITS) {
			if (cudaError_t e = cudaMemcpyAsync(out, bg, (size_t)n_bg * K * sizeof(float), cudaMemcpyDeviceToDevice, st)) return e;
		} else {
			count_launch();
			semantic_softmax_fwd_kernel<<<feat_blocks(n_bg), kFeatThreads, 0, st>>>(n_bg, K, bg, out);
			if (cudaError_t e = cudaGetLastError()) return e;
		}
	}
	return for_actor_groups(n_act, start, label, [&](SemTable &t, int first) {
		for (int k = 0; k < t.n; k++) t.src[k] = actor[first + k], t.grad[k] = nullptr;
		count_launch();
		semantic_actor_fwd_kernel<<<feat_blocks((int64_t)(t.start[t.n] - t.start[0]) * K), kFeatThreads, 0, st>>>(t, K, mode, out);
		return cudaGetLastError();
	});
}

cudaError_t launch_compose_semantics_bwd(int n_bg, int K, int mode, const float *out, const float *g, float *g_bg, int n_act, const int32_t *start,
                                         const int32_t *label, float *const *g_actor, cudaStream_t st) {
	if (n_bg > 0 && g_bg) {
		if (mode == SGR_SEMANTIC_LOGITS) {
			if (cudaError_t e = cudaMemcpyAsync(g_bg, g, (size_t)n_bg * K * sizeof(float), cudaMemcpyDeviceToDevice, st)) return e;
		} else {
			count_launch();
			semantic_softmax_bwd_kernel<<<feat_blocks(n_bg), kFeatThreads, 0, st>>>(n_bg, K, out, g, g_bg);
			if (cudaError_t e = cudaGetLastError()) return e;
		}
	}
	if (!g_actor) return cudaSuccess;
	return for_actor_groups(n_act, start, label, [&](SemTable &t, int first) {
		for (int k = 0; k < t.n; k++) t.src[k] = nullptr, t.grad[k] = g_actor[first + k];
		count_launch();
		semantic_actor_bwd_kernel<<<feat_blocks(t.start[t.n] - t.start[0]), kFeatThreads, 0, st>>>(t, K, mode, out, g);
		return cudaGetLastError();
	});
}

// ---- finishing of the rendered feature maps -------------------------------------------------------------------------------------

constexpr float kNormalEps = 1e-12f;  // F.normalize's eps
constexpr float kProbEps = 1e-8f;     // street_gaussian_renderer.py:261-262

// One thread per pixel.  Channels [0, nc) are the normals (nc = 3) or absent (nc = 0); channels [nc, S) the semantics.
//   normals:  x / max(|x|, eps)
//   semantic: 'probabilities'  log(x / (sum_c x_c + 1e-8) + 1e-8);  'logits'  x
// Work item t is pixel t of the frame, or with kBand pixel band_pixel(t) of the band's M = band_rows * 16 W pixels (those past the
// image's last row do nothing).  Either way a pixel keeps its frame index p, so a band's rows equal the whole frame's bit for bit.
// The whole-frame instantiation ignores the trailing band arguments, so its instructions do not depend on them.
template <bool kBand>
__global__ void __launch_bounds__(kFeatThreads) finish_features_fwd_kernel(const int64_t N, const int S, const int nc, const int mode,
                                                                           const float *__restrict__ in, float *__restrict__ nout,
                                                                           float *__restrict__ sout, const int64_t M, const Band band,
                                                                           const int64_t strip) {
	const int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (item >= (kBand ? M : N)) return;
	const int64_t p = kBand ? band_pixel(item, band, strip) : item;
	if (kBand && p >= N) return;
	if (nc == 3) {
		const float x0 = __ldg(in + p), x1 = __ldg(in + N + p), x2 = __ldg(in + 2 * N + p);
		const float d = fmaxf(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x0, x0), __fmul_rn(x1, x1)), __fmul_rn(x2, x2))), kNormalEps);
		nout[p] = __fdiv_rn(x0, d);
		nout[N + p] = __fdiv_rn(x1, d);
		nout[2 * N + p] = __fdiv_rn(x2, d);
	}
	const int K = S - nc;
	const float *x = in + (int64_t)nc * N + p;
	if (mode == SGR_SEMANTIC_LOGITS) {
		for (int c = 0; c < K; c++) sout[c * N + p] = __ldg(x + c * N);
		return;
	}
	float t = 0.f;
	for (int c = 0; c < K; c++) t = __fadd_rn(t, __ldg(x + c * N));
	t = __fadd_rn(t, kProbEps);
	for (int c = 0; c < K; c++) sout[c * N + p] = logf(__fadd_rn(__fdiv_rn(__ldg(x + c * N), t), kProbEps));
}

// Fused backward of both.  normals: dL/dx = g / d - [|x| >= eps] (g . x) / d^2 x / |x| (the clamp passes no gradient below eps).
// 'probabilities': with t = sum x + 1e-8, p = x / t, h = g / (p + 1e-8): dL/dx = (h - sum_c h_c p_c) / t.  A NULL gradient is 0.
// The pixels as in the forward.
template <bool kBand>
__global__ void __launch_bounds__(kFeatThreads) finish_features_bwd_kernel(const int64_t N, const int S, const int nc, const int mode,
                                                                           const float *__restrict__ in, const float *__restrict__ gn,
                                                                           const float *__restrict__ gs, float *__restrict__ gin,
                                                                           const int64_t M, const Band band, const int64_t strip) {
	const int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (item >= (kBand ? M : N)) return;
	const int64_t p = kBand ? band_pixel(item, band, strip) : item;
	if (kBand && p >= N) return;
	if (nc == 3) {
		if (gn) {
			const float x0 = __ldg(in + p), x1 = __ldg(in + N + p), x2 = __ldg(in + 2 * N + p);
			const float g0 = __ldg(gn + p), g1 = __ldg(gn + N + p), g2 = __ldg(gn + 2 * N + p);
			const float len = sqrtf(x0 * x0 + x1 * x1 + x2 * x2);
			const float d = fmaxf(len, kNormalEps);
			const float c = len >= kNormalEps ? (g0 * x0 + g1 * x1 + g2 * x2) / (d * d) / len : 0.f;
			gin[p] = g0 / d - c * x0;
			gin[N + p] = g1 / d - c * x1;
			gin[2 * N + p] = g2 / d - c * x2;
		} else {
			gin[p] = gin[N + p] = gin[2 * N + p] = 0.f;
		}
	}
	const int K = S - nc;
	const float *x = in + (int64_t)nc * N + p;
	float *gx = gin + (int64_t)nc * N + p;
	if (!gs) {
		for (int c = 0; c < K; c++) gx[c * N] = 0.f;
		return;
	}
	const float *g = gs + p;
	if (mode == SGR_SEMANTIC_LOGITS) {
		for (int c = 0; c < K; c++) gx[c * N] = __ldg(g + c * N);
		return;
	}
	float t = 0.f;
	for (int c = 0; c < K; c++) t = __fadd_rn(t, __ldg(x + c * N));
	t = __fadd_rn(t, kProbEps);
	float hp = 0.f;
	for (int c = 0; c < K; c++) {
		const float pc = __fdiv_rn(__ldg(x + c * N), t);
		hp = fmaf(__ldg(g + c * N) / (pc + kProbEps), pc, hp);
	}
	for (int c = 0; c < K; c++) {
		const float pc = __fdiv_rn(__ldg(x + c * N), t);
		gx[c * N] = (__ldg(g + c * N) / (pc + kProbEps) - hp) / t;
	}
}

cudaError_t launch_finish_features_fwd(int S, int H, int W, int nc, int mode, const float *in, float *nout, float *sout, cudaStream_t st) {
	const int64_t N = (int64_t)H * W;
	count_launch();
	finish_features_fwd_kernel<false><<<feat_blocks(N), kFeatThreads, 0, st>>>(N, S, nc, mode, in, nout, sout, N, Band{0, 1, 1}, 1);
	return cudaGetLastError();
}

cudaError_t launch_finish_features_bwd(int S, int H, int W, int nc, int mode, const float *in, const float *gn, const float *gs, float *gin,
                                       cudaStream_t st) {
	const int64_t N = (int64_t)H * W;
	count_launch();
	finish_features_bwd_kernel<false><<<feat_blocks(N), kFeatThreads, 0, st>>>(N, S, nc, mode, in, gn, gs, gin, N, Band{0, 1, 1}, 1);
	return cudaGetLastError();
}

// The band's pixels: band_rows(band) tile rows of 16 W pixels each; an empty band launches nothing.  The grid depends on the band and
// the image size only.
cudaError_t launch_finish_features_fwd(int S, int H, int W, Band band, int nc, int mode, const float *in, float *nout, float *sout, cudaStream_t st) {
	const int64_t N = (int64_t)H * W, strip = (int64_t)kBandTileRows * W, M = band_rows(band) * strip;
	if (M == 0) return cudaSuccess;
	count_launch();
	finish_features_fwd_kernel<true><<<feat_blocks(M), kFeatThreads, 0, st>>>(N, S, nc, mode, in, nout, sout, M, band, strip);
	return cudaGetLastError();
}

cudaError_t launch_finish_features_bwd(int S, int H, int W, Band band, int nc, int mode, const float *in, const float *gn, const float *gs,
                                       float *gin, cudaStream_t st) {
	const int64_t N = (int64_t)H * W, strip = (int64_t)kBandTileRows * W, M = band_rows(band) * strip;
	if (M == 0) return cudaSuccess;
	count_launch();
	finish_features_bwd_kernel<true><<<feat_blocks(M), kFeatThreads, 0, st>>>(N, S, nc, mode, in, gn, gs, gin, M, band, strip);
	return cudaGetLastError();
}

}  // namespace sgr
