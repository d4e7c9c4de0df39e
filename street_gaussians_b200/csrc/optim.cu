// optim.cu — what runs right after the rasterizer's backward in every training iteration (SURVEY.md §8 row f3):
//
//  * densification statistics (lib/models/street_gaussian_model.py:551-571): per sub-model, for the Gaussians that were visible
//    (radii > 0):  max_radii2D = max(max_radii2D, radii),  xyz_gradient_accum[:,0] += |grad2D.xy|,  [:,1] += |grad2D.z|,  denom += 1.
//    The reference slices the composed arrays per model and runs ~8 indexed PyTorch kernels per model per iteration; here ONE
//    kernel walks the composed index space with the same segment table the composer uses.
//  * the optimiser step (lib/models/gaussian_model.py:316-318 -> torch.optim.Adam(lr per group, eps = 1e-15), :300-303): one
//    multi-tensor Adam kernel over every parameter tensor of every sub-model (the reference: 6 groups x (1 + #actors) models,
//    each a handful of foreach kernels), same arithmetic as torch.optim.Adam without weight decay / amsgrad:
//        m <- m + (g - m)(1 - b1);  v <- b2 v + (1 - b2) g^2;  p <- p - (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
//  * an opt-in visibility-masked Adam (no reference counterpart): the same update, only on the rows of the Gaussians with radii > 0,
//    walking the composed index space tile by tile like the densification statistics.
#include "sgr_common.cuh"

namespace sgr {

constexpr int kStatSeg = SGR_MAX_SEGMENTS_PER_LAUNCH;
struct StatTable {
	int n;
	int start[kStatSeg + 1];
	float *max_radii2D[kStatSeg];
	float *grad_accum[kStatSeg];  // [count, 2]
	float *denom[kStatSeg];       // [count, 1]
};

__global__ void __launch_bounds__(256) densify_stats_kernel(const StatTable t, const int32_t *__restrict__ radii,
                                                           const float *__restrict__ grad2d /* viewspace_points.grad [P,3] */) {
	const int i = t.start[0] + blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= t.start[t.n]) return;
	const int r = radii[i];
	if (r <= 0) return;  // visibility_filter = radii > 0 (street_gaussian_renderer.py:274)
	int lo = 0, hi = t.n - 1;
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (t.start[mid] <= i) lo = mid; else hi = mid - 1;
	}
	const size_t l = (size_t)(i - t.start[lo]);
	float *mr = t.max_radii2D[lo] + l;
	*mr = fmaxf(*mr, (float)r);
	const float gx = grad2d[3 * (size_t)i], gy = grad2d[3 * (size_t)i + 1], gz = grad2d[3 * (size_t)i + 2];
	t.grad_accum[lo][2 * l] += sqrtf(gx * gx + gy * gy);  // torch.norm(grad[:, :2], dim=-1)
	t.grad_accum[lo][2 * l + 1] += fabsf(gz);             // torch.norm(grad[:, 2:], dim=-1) of one column
	t.denom[lo][l] += 1.f;
}

cudaError_t launch_densify_stats(const SgrStatSegment *segs, int nseg, const int32_t *radii, const float *grad2d, cudaStream_t st) {
	for (int first = 0; first < nseg; first += kStatSeg) {
		StatTable t;
		const int n = nseg - first < kStatSeg ? nseg - first : kStatSeg;
		t.n = n;
		for (int k = 0; k < n; k++) {
			const SgrStatSegment &s = segs[first + k];
			t.start[k] = s.start;
			t.max_radii2D[k] = s.max_radii2D; t.grad_accum[k] = s.xyz_gradient_accum; t.denom[k] = s.denom;
		}
		t.start[n] = segs[first + n - 1].start + segs[first + n - 1].count;
		const int count = t.start[n] - t.start[0];
		if (count <= 0) continue;
		count_launch();
		densify_stats_kernel<<<(count + 255) / 256, 256, 0, st>>>(t, radii, grad2d);
	}
	return cudaGetLastError();
}

// ---- multi-tensor Adam ----
constexpr int kAdamTensors = 48;         // tensors per launch (kernel-parameter table)
constexpr int kAdamChunk = 256 * 4 * 8;  // elements per block
struct AdamTable {
	int n;
	float *p[kAdamTensors];
	const float *g[kAdamTensors];
	float *m[kAdamTensors], *v[kAdamTensors];
	long long numel[kAdamTensors];
	float step_size[kAdamTensors];   // lr / (1 - b1^t)
	float inv_sqrt_bc2[kAdamTensors];  // 1 / sqrt(1 - b2^t)
	int block_start[kAdamTensors + 1];  // first block of each tensor
};

// The per-element Adam update of element i, shared by the dense and the visibility-masked kernel so that both round identically.
// omb1 = fl(1 - beta1), omb2 = fl(1 - beta2) formed in double on the host, exactly the scalars torch hands to lerp_ / addcmul_
__device__ __forceinline__ void adam_update(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m, float *__restrict__ v,
                                            size_t i, float omb1, float b2, float omb2, float eps, float ss, float ibc2) {
	const float gi = g[i];
	const float mi = m[i] + (gi - m[i]) * omb1;              // exp_avg.lerp_(grad, 1 - beta1)
	const float vi = v[i] * b2 + omb2 * gi * gi;             // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value = 1 - beta2)
	m[i] = mi;
	v[i] = vi;
	p[i] = p[i] - ss * (mi / (sqrtf(vi) * ibc2 + eps));      // param.addcdiv_(exp_avg, sqrt(v)/sqrt(bc2) + eps, value = -step_size)
}

// step_size = lr / (1 - b1^t) and 1 / sqrt(1 - b2^t), formed in double and rounded once, for both kernels
static void adam_scalars(float lr, int step, double beta1, double beta2, float *step_size, float *inv_sqrt_bc2) {
	const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
	*step_size = (float)((double)lr / bc1);
	*inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
}

__global__ void __launch_bounds__(256) adam_kernel(const AdamTable t, const float omb1, const float b2, const float omb2, const float eps) {
	int k = 0;  // tensor of this block (linear search: <= 48 entries, warp-uniform)
	while (k + 1 < t.n && (int)blockIdx.x >= t.block_start[k + 1]) k++;
	const long long base = (long long)(blockIdx.x - t.block_start[k]) * kAdamChunk;
	const long long n = t.numel[k];
	const float ss = t.step_size[k], ibc2 = t.inv_sqrt_bc2[k];
	for (long long i = base + threadIdx.x; i < base + kAdamChunk && i < n; i += 256)
		adam_update(t.p[k], t.g[k], t.m[k], t.v[k], (size_t)i, omb1, b2, omb2, eps, ss, ibc2);
}

cudaError_t launch_adam(const SgrAdamTensor *ts, int n_tensors, double beta1, double beta2, double eps, cudaStream_t st) {
	for (int first = 0; first < n_tensors; first += kAdamTensors) {
		AdamTable t;
		const int n = n_tensors - first < kAdamTensors ? n_tensors - first : kAdamTensors;
		t.n = n;
		int blocks = 0;
		for (int k = 0; k < n; k++) {
			const SgrAdamTensor &a = ts[first + k];
			t.p[k] = a.param; t.g[k] = a.grad; t.m[k] = a.exp_avg; t.v[k] = a.exp_avg_sq; t.numel[k] = a.numel;
			adam_scalars(a.lr, a.step, beta1, beta2, &t.step_size[k], &t.inv_sqrt_bc2[k]);
			t.block_start[k] = blocks;
			blocks += (int)((a.numel + kAdamChunk - 1) / kAdamChunk);
		}
		t.block_start[n] = blocks;
		if (blocks == 0) continue;
		count_launch();
		adam_kernel<<<blocks, 256, 0, st>>>(t, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps);
	}
	return cudaGetLastError();
}

// ---- visibility-masked Adam ----
// One block per 256-row tile of one segment.  The tile's radii are read once; a tile with no visible row returns before touching any
// tensor.  Otherwise each tensor's flat span [r0 w, (r0 + 256) w) is walked coalesced and only elements of visible rows are loaded and
// stored, so the traffic is 4 B per row of radii plus 28 B per element of a visible row (up to 32-B sector granularity).
constexpr int kSparseTile = 256;
constexpr int kSparseSeg = SGR_MAX_SEGMENTS_PER_LAUNCH;
constexpr int kSparseTensors = SGR_DENSIFY_TENSORS;
struct SparseAdamTable {  // ~10 KB of kernel parameters (CUDA 12.1+ allows 32 KB)
	int n;
	int start[kSparseSeg + 1];        // composed index of each segment's first row; start[n] = end of the last one
	int block_start[kSparseSeg + 1];  // first block of each segment
	float *p[kSparseSeg][kSparseTensors];
	const float *g[kSparseSeg][kSparseTensors];
	float *m[kSparseSeg][kSparseTensors], *v[kSparseSeg][kSparseTensors];
	int width[kSparseSeg][kSparseTensors];  // 0: tensor not updated
	float step_size[kSparseSeg][kSparseTensors], inv_sqrt_bc2[kSparseSeg][kSparseTensors];
};

__global__ void __launch_bounds__(kSparseTile) sparse_adam_kernel(const SparseAdamTable t, const int32_t *__restrict__ radii, const float omb1,
                                                                 const float b2, const float omb2, const float eps) {
	__shared__ unsigned vis[kSparseTile / 32];
	int lo = 0, hi = t.n - 1;  // segment of this block
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (t.block_start[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
	}
	const int k = lo;
	const int r0 = ((int)blockIdx.x - t.block_start[k]) * kSparseTile;  // first row of the tile, local to the segment
	const int nrows = min(kSparseTile, t.start[k + 1] - t.start[k] - r0);
	const bool mine = (int)threadIdx.x < nrows && radii[t.start[k] + r0 + threadIdx.x] > 0;  // visibility_filter = radii > 0
	const unsigned ballot = __ballot_sync(0xffffffffu, mine);
	if ((threadIdx.x & 31) == 0) vis[threadIdx.x >> 5] = ballot;
	if (!__syncthreads_or(mine)) return;
	for (int a = 0; a < kSparseTensors; a++) {
		const int w = t.width[k][a];
		if (w == 0) continue;
		const size_t base = (size_t)r0 * w;
		const int n = nrows * w;  // <= 256 * SGR_SPARSE_ADAM_MAX_WIDTH < 2^31
		const float ss = t.step_size[k][a], ibc2 = t.inv_sqrt_bc2[k][a];
		for (int e = threadIdx.x; e < n; e += kSparseTile) {
			const int rl = e / w;
			if ((vis[rl >> 5] >> (rl & 31)) & 1u) adam_update(t.p[k][a], t.g[k][a], t.m[k][a], t.v[k][a], base + e, omb1, b2, omb2, eps, ss, ibc2);
		}
	}
}

cudaError_t launch_sparse_adam(const SgrSparseAdamSegment *segs, int nseg, const int32_t *radii, double beta1, double beta2, double eps,
                               cudaStream_t st) {
	for (int first = 0; first < nseg; first += kSparseSeg) {
		SparseAdamTable t;
		const int n = nseg - first < kSparseSeg ? nseg - first : kSparseSeg;
		t.n = n;
		int blocks = 0;
		bool any = false;
		for (int k = 0; k < n; k++) {
			const SgrSparseAdamSegment &s = segs[first + k];
			t.start[k] = s.start;
			t.block_start[k] = blocks;
			blocks += (s.count + kSparseTile - 1) / kSparseTile;
			for (int a = 0; a < kSparseTensors; a++) {
				t.p[k][a] = s.param[a]; t.g[k][a] = s.grad[a]; t.m[k][a] = s.exp_avg[a]; t.v[k][a] = s.exp_avg_sq[a];
				t.width[k][a] = s.width[a];
				t.step_size[k][a] = t.inv_sqrt_bc2[k][a] = 0.f;
				if (s.width[a] > 0) adam_scalars(s.lr[a], s.step[a], beta1, beta2, &t.step_size[k][a], &t.inv_sqrt_bc2[k][a]);
				any |= s.count > 0 && s.width[a] > 0;
			}
		}
		t.start[n] = segs[first + n - 1].start + segs[first + n - 1].count;
		t.block_start[n] = blocks;
		if (!any) continue;
		count_launch();
		sparse_adam_kernel<<<blocks, kSparseTile, 0, st>>>(t, radii, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps);
	}
	return cudaGetLastError();
}

// ---- block-masked Adam of the sky cube map ----
// One CTA per kSkyBlock x kSkyBlock block of the cube [6, R, R, 3] (the blocks sgr_sky_grad_blocks numbers), so the grid depends on R
// only.  Thread 0 reads the block's map byte and clears it; a block whose byte was 0 returns before touching any tensor.  A marked block
// walks its texel rows one warp per row (3 x its width contiguous floats), each float through adam_update, so the traffic is 1 B per
// block plus 28 B per float of a marked block.
constexpr int kCubeAdamThreads = 256;

__global__ void __launch_bounds__(kCubeAdamThreads) cube_sparse_adam_kernel(const int R, float *__restrict__ p, const float *__restrict__ g,
                                                                           float *__restrict__ m, float *__restrict__ v,
                                                                           uint8_t *__restrict__ map, const float omb1, const float b2,
                                                                           const float omb2, const float eps, const float ss, const float ibc2) {
	const int b = blockIdx.x;
	if (!__syncthreads_or(threadIdx.x == 0 && map[b] != 0)) return;
	if (threadIdx.x == 0) map[b] = 0;  // only thread 0 read it, before the barrier
	const int nb = sky_blocks_per_side(R), f = b / (nb * nb), br = (b / nb) % nb, bc = b % nb;
	const int r0 = br * kSkyBlock, r1 = min(R, r0 + kSkyBlock), c0 = bc * kSkyBlock, len = (min(R, c0 + kSkyBlock) - c0) * 3;
	const int lane = threadIdx.x & 31;
	for (int r = r0 + (int)(threadIdx.x >> 5); r < r1; r += kCubeAdamThreads / 32) {
		const size_t s = ((size_t)(f * R + r) * R + c0) * 3;
		for (int e = lane; e < len; e += 32) adam_update(p, g, m, v, s + e, omb1, b2, omb2, eps, ss, ibc2);
	}
}

cudaError_t launch_cube_sparse_adam(int R, const SgrAdamTensor &a, uint8_t *map, double beta1, double beta2, double eps, cudaStream_t st) {
	float ss, ibc2;
	adam_scalars(a.lr, a.step, beta1, beta2, &ss, &ibc2);
	count_launch();
	cube_sparse_adam_kernel<<<(unsigned)sky_block_count(R), kCubeAdamThreads, 0, st>>>(R, a.param, a.grad, a.exp_avg, a.exp_avg_sq, map,
	                                                                                  (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2),
	                                                                                  (float)eps, ss, ibc2);
	return cudaGetLastError();
}

}  // namespace sgr
