// densify.cu — densification of every sub-model in one pass (SURVEY.md §8 row f3): clone / split / prune with the Adam moments
// resized together with the parameters, and the opacity reset.  Reference: GaussianModelBkgd / GaussianModelActor.densify_and_prune
// (lib/models/gaussian_model_bkgd.py:74-114, lib/models/gaussian_model_actor.py:204-261) over GaussianModel.densify_and_clone / _split /
// prune_points / densification_postfix (lib/models/gaussian_model.py:416-520).  The reference does ~6 .item() syncs and dozens of
// boolean-index / torch.cat kernels per sub-model; here:
//   1. plan kernel   — one thread per parent over the composed index space: clone / split decision, the survival of each of its (at
//                      most two) output rows, a 4-bit section mask {self, clone, child 0, child 1}, and the reported counts;
//   2. one exclusive scan of the masks with component-wise uint4 sums: the output row of every kept row, per section;
//   3. one device-to-host copy of the per-segment sizes and counts (the only host sync; the caller allocates the outputs);
//   4. apply kernel  — per tile of 256 parents of one segment, every output row is written once: the rows of one section that come
//                      from one tile are contiguous in the output, so each tensor is copied as a flat span (coalesced stores, loads
//                      coalesced along runs of kept parents).  Children's xyz / scaling come from the same draws the plan used.
#include "sgr_common.cuh"

#include <cub/cub.cuh>
#include <curand_kernel.h>
#include <thrust/iterator/transform_iterator.h>

#include <vector>

namespace sgr {

namespace {

constexpr int kTile = 256;       // parents per apply block (= threads)
constexpr int kDraws = SGR_DENSIFY_DRAWS;

__device__ __forceinline__ int row_width(const SgrDensifySegment &s, int a) {
	switch (a) {
	case 1: return s.dc_width;
	case 2: return s.rest_width;
	case 6: return s.semantic_width;
	case 3: return 1;
	case 5: return 4;
	default: return 3;  // xyz, scaling
	}
}

// segment of composed index i (start[] ascending, start[n] = P)
__device__ __forceinline__ int find_segment(const int32_t *start, int n, int i) {
	int lo = 0, hi = n - 1;
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (start[mid] <= i) lo = mid; else hi = mid - 1;
	}
	return lo;
}

// The 18 normal draws of parent i: the caller's [P,18] table (test seam) or Philox keyed by (seed, composed parent index).
template <bool kGiven>
__device__ __forceinline__ void load_draws(const float *__restrict__ draws, unsigned long long seed, int i, float z[20]) {
	if constexpr (kGiven) {
		const float *d = draws + (size_t)i * kDraws;
#pragma unroll
		for (int k = 0; k < kDraws; k++) z[k] = d[k];
		z[18] = z[19] = 0.f;
	} else {
		curandStatePhilox4_32_10_t st;
		curand_init(seed, (unsigned long long)i, 0ULL, &st);
#pragma unroll
		for (int k = 0; k < 20; k += 4) {
			const float4 v = curand_normal4(&st);
			z[k] = v.x; z[k + 1] = v.y; z[k + 2] = v.z; z[k + 3] = v.w;
		}
	}
}

// quaternion_to_matrix (lib/utils/general_utils.py:125-146): normalises q first.  twice: the actor's box test feeds it get_rotation,
// which is F.normalize(_rotation) (x / max(||x||, 1e-12)) already.
__device__ __forceinline__ void quat_to_matrix(const float *q, bool twice, float R[9]) {
	float w = q[0], x = q[1], y = q[2], z = q[3];
	if (twice) {
		const float n = fmaxf(sqrtf(w * w + x * x + y * y + z * z), 1e-12f);
		w /= n; x /= n; y /= n; z /= n;
	}
	const float n = sqrtf(w * w + x * x + y * y + z * z);
	w /= n; x /= n; y /= n; z /= n;
	R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - w * z);       R[2] = 2.f * (x * z + w * y);
	R[3] = 2.f * (x * y + w * z);       R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - w * x);
	R[6] = 2.f * (x * z - w * y);       R[7] = 2.f * (y * z + w * x);       R[8] = 1.f - 2.f * (x * x + y * y);
}

// R (z (*) s) + x  — the split child's position (torch.bmm(rots, samples) + xyz) and the actor's box samples
__device__ __forceinline__ void sample_point(const float R[9], const float *z, const float s[3], const float x[3], float out[3]) {
	const float v0 = z[0] * s[0], v1 = z[1] * s[1], v2 = z[2] * s[2];
#pragma unroll
	for (int r = 0; r < 3; r++) out[r] = (R[3 * r] * v0 + R[3 * r + 1] * v1 + R[3 * r + 2] * v2) + x[r];
}

// child c of a split parent: xyz from draws z[3c..3c+3), raw scaling log(exp(s) / (0.8 * N)) with N = 2
__device__ __forceinline__ void make_child(const float R[9], const float *zc, const float s[3], const float x[3], float cx[3], float cs_raw[3]) {
	sample_point(R, zc, s, x, cx);
#pragma unroll
	for (int r = 0; r < 3; r++) cs_raw[r] = logf(s[r] / 1.6f);
}

struct Parent {  // what the plan and the apply kernel both read of one parent
	float x[3], s[3], q[4], sig;
	bool clone, split;
};

__device__ __forceinline__ Parent read_parent(const SgrDensifySegment &sg, size_t l) {
	Parent p;
	const float *xyz = sg.param[0] + 3 * l, *sc = sg.param[4] + 3 * l, *rot = sg.param[5] + 4 * l;
#pragma unroll
	for (int r = 0; r < 3; r++) { p.x[r] = xyz[r]; p.s[r] = expf(sc[r]); }
#pragma unroll
	for (int r = 0; r < 4; r++) p.q[r] = rot[r];
	p.sig = 1.f / (1.f + expf(-sg.param[3][l]));
	float g = sg.xyz_gradient_accum[2 * l + sg.grad_col] / sg.denom[l];
	if (isnan(g)) g = 0.f;  // grads[grads.isnan()] = 0.0
	const float ms = fmaxf(fmaxf(p.s[0], p.s[1]), p.s[2]);
	p.clone = fabsf(g) >= sg.grad_threshold && ms <= sg.dense_threshold;  // torch.norm of a one-column tensor
	p.split = g >= sg.grad_threshold && ms > sg.dense_threshold;
	return p;
}

// ---- 1. plan ----
template <bool kGiven>
__global__ void __launch_bounds__(256) densify_plan_kernel(const SgrDensifySegment *__restrict__ segs, const int32_t *__restrict__ start, int nseg,
                                                           unsigned long long seed, const float *__restrict__ draws, uint8_t *__restrict__ mask,
                                                           unsigned *__restrict__ counters) {
	const int P = start[nseg];
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	int k = -1;
	unsigned c_clone = 0, c_split = 0, c_below = 0, c_big = 0, c_pruned = 0;
	if (i < P) {
		k = find_segment(start, nseg, i);
		const SgrDensifySegment &sg = segs[k];
		const size_t l = (size_t)(i - start[k]);
		const Parent p = read_parent(sg, l);
		const bool actor = sg.kind == SGR_DENSIFY_ACTOR;
		const bool box = actor && sg.prune_big;
		float z[20];
		if (p.split || box) load_draws<kGiven>(draws, seed, i, z);
		float Rbox[9];
		if (box) quat_to_matrix(p.q, true, Rbox);
		// survival of one row after clone + split (gaussian_model_bkgd.py:90-105, gaussian_model_actor.py:222-252)
		auto survives = [&](const float x[3], const float s[3], int slot) {
			const bool below = p.sig < sg.min_opacity;
			bool big = false, outside = false;
			if (sg.prune_big) {
				big = fmaxf(fmaxf(s[0], s[1]), s[2]) > sg.big_threshold;
				if (!actor) {
					const float dx = x[0] - sg.sphere_center[0], dy = x[1] - sg.sphere_center[1], dz = x[2] - sg.sphere_center[2];
					if (sqrtf(dx * dx + dy * dy + dz * dz) > sg.sphere_diameter) big = false;
				} else {
#pragma unroll
					for (int j = 0; j < 2; j++) {
						float y[3];
						sample_point(Rbox, z + 6 + 3 * (2 * slot + j), s, x, y);
#pragma unroll
						for (int r = 0; r < 3; r++) outside |= !(y[r] >= sg.min_xyz[r] && y[r] <= sg.max_xyz[r]);
					}
				}
			}
			const bool pruned = below || big || outside;
			c_below += below; c_big += big; c_pruned += pruned;
			return !pruned;
		};
		unsigned m = 0;
		if (!p.split) {
			m |= survives(p.x, p.s, 0) ? 1u : 0u;
			if (p.clone) m |= survives(p.x, p.s, 1) ? 2u : 0u;
		} else {
			float R[9];
			quat_to_matrix(p.q, false, R);
#pragma unroll
			for (int c = 0; c < 2; c++) {
				float cx[3], cr[3], cs[3];
				make_child(R, z + 3 * c, p.s, p.x, cx, cr);
#pragma unroll
				for (int r = 0; r < 3; r++) cs[r] = expf(cr[r]);  // get_scaling of the child: exp(log(exp(s) / 1.6))
				m |= survives(cx, cs, c) ? (4u << c) : 0u;
			}
		}
		c_clone = p.clone; c_split = p.split;
		mask[i] = (uint8_t)m;
	} else if (i == P) {
		mask[P] = 0;  // the exclusive scan's element P is the total
	}
	// per-segment counts: one atomic per (warp, segment) group
	const unsigned grp = __match_any_sync(0xffffffffu, k);
	const bool leader = (threadIdx.x & 31) == __ffs(grp) - 1;
	const unsigned v[5] = {c_clone, c_split, c_below, c_big, c_pruned};
#pragma unroll
	for (int q = 0; q < 5; q++) {
		const unsigned t = __reduce_add_sync(grp, v[q]);
		if (leader && k >= 0 && t) atomicAdd(&counters[8 * k + q], t);
	}
}

struct MaskToU4 {
	__host__ __device__ uint4 operator()(uint8_t m) const { return make_uint4(m & 1u, (m >> 1) & 1u, (m >> 2) & 1u, (m >> 3) & 1u); }
};
struct U4Sum {
	__host__ __device__ uint4 operator()(const uint4 &a, const uint4 &b) const { return make_uint4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
};
using MaskIt = thrust::transform_iterator<MaskToU4, const uint8_t *, uint4>;

__device__ __forceinline__ unsigned comp(const uint4 &v, int t) { return t == 0 ? v.x : t == 1 ? v.y : t == 2 ? v.z : v.w; }

__global__ void densify_result_kernel(const int32_t *__restrict__ start, int nseg, const uint4 *__restrict__ prefix,
                                      const unsigned *__restrict__ counters, long long *__restrict__ result) {
	for (int k = threadIdx.x; k < nseg; k += blockDim.x) {
		const uint4 a = prefix[start[k]], b = prefix[start[k + 1]];
		long long *r = result + SGR_DENSIFY_RESULT * k;
		r[0] = (long long)(b.x - a.x) + (b.y - a.y) + (b.z - a.z) + (b.w - a.w);
		r[1] = start[k + 1] - start[k];
		for (int q = 0; q < 5; q++) r[2 + q] = counters[8 * k + q];
		r[7] = 0;
	}
}

// ---- 4. apply ----
template <bool kGiven>
__global__ void __launch_bounds__(kTile) densify_apply_kernel(const SgrDensifySegment *__restrict__ segs, const SgrDensifyOutput *__restrict__ outs,
                                                              const int32_t *__restrict__ start, const int32_t *__restrict__ block_start, int nseg,
                                                              unsigned long long seed, const float *__restrict__ draws,
                                                              const uint8_t *__restrict__ mask, const uint4 *__restrict__ prefix) {
	__shared__ uint16_t src[4][kTile];          // local parent of the tile's j-th output row of each section
	__shared__ float child[2][6][kTile];        // children's xyz (0..2) and raw scaling (3..5)
	__shared__ long long row0[4];               // first output row of the tile's rows of each section
	__shared__ int nrows[4];
	const int k = find_segment(block_start, nseg, blockIdx.x);
	const SgrDensifySegment &sg = segs[k];
	const SgrDensifyOutput &out = outs[k];
	const int s0 = start[k], s1 = start[k + 1];
	const int p0 = s0 + (blockIdx.x - block_start[k]) * kTile;
	const int pend = min(p0 + kTile, s1);
	const uint4 base = prefix[p0];
	if (threadIdx.x < 4) {
		const int t = threadIdx.x;
		const uint4 a = prefix[s0], b = prefix[s1], e = prefix[pend];
		long long sec = 0;
		for (int u = 0; u < t; u++) sec += comp(b, u) - comp(a, u);
		row0[t] = sec + (comp(base, t) - comp(a, t));
		nrows[t] = (int)(comp(e, t) - comp(base, t));
	}
	const int i = p0 + threadIdx.x;
	if (i < pend) {
		const unsigned m = mask[i];
		const uint4 pr = prefix[i];
#pragma unroll
		for (int t = 0; t < 4; t++)
			if (m & (1u << t)) src[t][comp(pr, t) - comp(base, t)] = (uint16_t)threadIdx.x;
		if (m & 12u) {  // a split parent with a surviving child: recompute both children from the plan's draws
			const Parent p = read_parent(sg, (size_t)(i - s0));
			float z[20], R[9];
			load_draws<kGiven>(draws, seed, i, z);
			quat_to_matrix(p.q, false, R);
#pragma unroll
			for (int c = 0; c < 2; c++) {
				float cx[3], cr[3];
				make_child(R, z + 3 * c, p.s, p.x, cx, cr);
#pragma unroll
				for (int r = 0; r < 3; r++) { child[c][r][threadIdx.x] = cx[r]; child[c][3 + r][threadIdx.x] = cr[r]; }
			}
		}
	}
	__syncthreads();
	const long long lim = out.count;
	for (int t = 0; t < 4; t++) {
		const int nr = nrows[t];
		if (nr == 0) continue;
		const long long r0 = row0[t];
		if (r0 + nr > lim) return;  // outputs smaller than the plan's result: write nothing past them
		for (int a = 0; a < SGR_DENSIFY_TENSORS; a++) {
			const int w = row_width(sg, a);
			if (w == 0) continue;
			const int n = nr * w;  // < 2^31: at most kTile rows per section and tile
			const float *pin = sg.param[a], *min_ = sg.exp_avg[a], *vin = sg.exp_avg_sq[a];
			float *pout = out.param[a] + r0 * w, *mout = out.exp_avg[a], *vout = out.exp_avg_sq[a];
			if (mout) mout += r0 * w;
			if (vout) vout += r0 * w;
			const bool computed = t >= 2 && (a == 0 || a == 4);
			for (int e = threadIdx.x; e < n; e += kTile) {
				const int rl = e / w, col = e - rl * w;
				const int lp = src[t][rl];
				const size_t at = (size_t)(p0 - s0 + lp) * w + col;
				pout[e] = computed ? child[t - 2][(a == 4 ? 3 : 0) + col][lp] : pin[at];
				if (mout) {  // kept originals carry their moments; clones and children start at zero
					mout[e] = t == 0 ? min_[at] : 0.f;
					vout[e] = t == 0 ? vin[at] : 0.f;
				}
			}
		}
		for (int e = threadIdx.x; e < nr; e += kTile) {  // statistics restart at zero for every row
			out.max_radii2D[r0 + e] = 0.f;
			out.denom[r0 + e] = 0.f;
			out.xyz_gradient_accum[2 * (r0 + e)] = 0.f;
			out.xyz_gradient_accum[2 * (r0 + e) + 1] = 0.f;
		}
	}
}

// ---- opacity reset ----
constexpr int kResetSeg = SGR_MAX_SEGMENTS_PER_LAUNCH;
struct ResetTable {
	int n;
	int start[kResetSeg + 1];
	float *opacity[kResetSeg], *m[kResetSeg], *v[kResetSeg];
};

__global__ void __launch_bounds__(256) reset_opacity_kernel(const ResetTable t) {
	const int i = t.start[0] + blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= t.start[t.n]) return;
	const int k = find_segment(t.start, t.n, i);
	const size_t l = (size_t)(i - t.start[k]);
	const float p = fminf(1.f / (1.f + expf(-t.opacity[k][l])), 0.01f);  // torch.min(get_opacity, ones * 0.01)
	t.opacity[k][l] = logf(p / (1.f - p));                              // inverse_sigmoid
	if (t.m[k]) t.m[k][l] = 0.f;
	if (t.v[k]) t.v[k][l] = 0.f;
}

// scratch layout (every piece 256-B aligned)
struct Scratch {
	SgrDensifySegment *segs;
	SgrDensifyOutput *outs;
	int32_t *start, *block_start;
	uint8_t *mask;
	uint4 *prefix;
	unsigned *counters;
	long long *result;
	void *temp;
	size_t temp_bytes, total;
};

Scratch carve(void *base, int nseg, long long P) {
	Scratch s;
	size_t o = 0;
	char *b = reinterpret_cast<char *>(base);
	auto take = [&](size_t bytes) { char *r = b + o; o += align_up(bytes); return r; };
	s.segs = reinterpret_cast<SgrDensifySegment *>(take(sizeof(SgrDensifySegment) * nseg));
	s.outs = reinterpret_cast<SgrDensifyOutput *>(take(sizeof(SgrDensifyOutput) * nseg));
	s.start = reinterpret_cast<int32_t *>(take(sizeof(int32_t) * (nseg + 1)));
	s.block_start = reinterpret_cast<int32_t *>(take(sizeof(int32_t) * (nseg + 1)));
	s.mask = reinterpret_cast<uint8_t *>(take(P + 1));
	s.prefix = reinterpret_cast<uint4 *>(take(sizeof(uint4) * (P + 1)));
	s.counters = reinterpret_cast<unsigned *>(take(sizeof(unsigned) * 8 * nseg));
	s.result = reinterpret_cast<long long *>(take(sizeof(long long) * SGR_DENSIFY_RESULT * nseg));
	s.temp_bytes = 0;
	cub::DeviceScan::ExclusiveScan(nullptr, s.temp_bytes, MaskIt(nullptr, MaskToU4()), (uint4 *)nullptr, U4Sum(), make_uint4(0, 0, 0, 0),
	                               (int)(P + 1));
	s.temp = take(s.temp_bytes);
	s.total = o;
	return s;
}

// host staging of the tables + start / block_start, copied to the device in one transfer
cudaError_t upload_tables(const Scratch &s, const SgrDensifySegment *segs, const SgrDensifyOutput *outs, int nseg, cudaStream_t st) {
	const size_t bs = (char *)s.outs - (char *)s.segs, bo = (char *)s.start - (char *)s.outs, bst = (char *)s.block_start - (char *)s.start;
	std::vector<char> h((char *)s.mask - (char *)s.segs, 0);
	memcpy(h.data(), segs, sizeof(SgrDensifySegment) * nseg);
	if (outs) memcpy(h.data() + bs, outs, sizeof(SgrDensifyOutput) * nseg);
	int32_t *start = reinterpret_cast<int32_t *>(h.data() + bs + bo), *bstart = reinterpret_cast<int32_t *>(h.data() + bs + bo + bst);
	int at = 0, blocks = 0;
	for (int k = 0; k < nseg; k++) {
		start[k] = at; bstart[k] = blocks;
		at += segs[k].count;
		blocks += (segs[k].count + kTile - 1) / kTile;
	}
	start[nseg] = at; bstart[nseg] = blocks;
	return cudaMemcpyAsync(s.segs, h.data(), h.size(), cudaMemcpyHostToDevice, st);
}

long long total_count(const SgrDensifySegment *segs, int nseg) {
	long long P = 0;
	for (int k = 0; k < nseg; k++) P += segs[k].count;
	return P;
}

}  // namespace

size_t densify_scratch_bytes(int nseg, long long P) { return carve(nullptr, nseg, P).total; }

cudaError_t launch_densify_plan(const SgrDensifySegment *segs, int nseg, unsigned long long seed, const float *draws, void *scratch,
                                long long *result_host, cudaStream_t st) {
	const long long P = total_count(segs, nseg);
	const Scratch s = carve(scratch, nseg, P);
	cudaError_t e = upload_tables(s, segs, nullptr, nseg, st);
	if (e != cudaSuccess) return e;
	if ((e = cudaMemsetAsync(s.counters, 0, sizeof(unsigned) * 8 * nseg, st)) != cudaSuccess) return e;
	const int blocks = (int)((P + 1 + 255) / 256);
	count_launch();
	if (draws) densify_plan_kernel<true><<<blocks, 256, 0, st>>>(s.segs, s.start, nseg, seed, draws, s.mask, s.counters);
	else densify_plan_kernel<false><<<blocks, 256, 0, st>>>(s.segs, s.start, nseg, seed, nullptr, s.mask, s.counters);
	if ((e = cudaGetLastError()) != cudaSuccess) return e;
	size_t tb = s.temp_bytes;
	e = cub::DeviceScan::ExclusiveScan(s.temp, tb, MaskIt(s.mask, MaskToU4()), s.prefix, U4Sum(), make_uint4(0, 0, 0, 0), (int)(P + 1), st);
	if (e != cudaSuccess) return e;
	count_launch();
	densify_result_kernel<<<1, 128, 0, st>>>(s.start, nseg, s.prefix, s.counters, s.result);
	if ((e = cudaGetLastError()) != cudaSuccess) return e;
	if ((e = cudaMemcpyAsync(result_host, s.result, sizeof(long long) * SGR_DENSIFY_RESULT * nseg, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
	return cudaStreamSynchronize(st);
}

cudaError_t launch_densify_apply(const SgrDensifySegment *segs, const SgrDensifyOutput *outs, int nseg, unsigned long long seed, const float *draws,
                                 void *scratch, cudaStream_t st) {
	const long long P = total_count(segs, nseg);
	const Scratch s = carve(scratch, nseg, P);
	cudaError_t e = upload_tables(s, segs, outs, nseg, st);
	if (e != cudaSuccess) return e;
	int blocks = 0;
	for (int k = 0; k < nseg; k++) blocks += (segs[k].count + kTile - 1) / kTile;
	if (blocks == 0) return cudaSuccess;
	count_launch();
	if (draws) densify_apply_kernel<true><<<blocks, kTile, 0, st>>>(s.segs, s.outs, s.start, s.block_start, nseg, seed, draws, s.mask, s.prefix);
	else densify_apply_kernel<false><<<blocks, kTile, 0, st>>>(s.segs, s.outs, s.start, s.block_start, nseg, seed, nullptr, s.mask, s.prefix);
	return cudaGetLastError();
}

cudaError_t launch_reset_opacity(const SgrDensifySegment *segs, int nseg, cudaStream_t st) {
	int at = 0;
	for (int first = 0; first < nseg; first += kResetSeg) {
		ResetTable t;
		const int n = nseg - first < kResetSeg ? nseg - first : kResetSeg;
		t.n = n;
		for (int k = 0; k < n; k++) {
			const SgrDensifySegment &s = segs[first + k];
			t.start[k] = at;
			t.opacity[k] = s.param[3]; t.m[k] = s.exp_avg[3]; t.v[k] = s.exp_avg_sq[3];
			at += s.count;
		}
		t.start[n] = at;
		const int count = t.start[n] - t.start[0];
		if (count <= 0) continue;
		count_launch();
		reset_opacity_kernel<<<(count + 255) / 256, 256, 0, st>>>(t);
	}
	return cudaGetLastError();
}

}  // namespace sgr
