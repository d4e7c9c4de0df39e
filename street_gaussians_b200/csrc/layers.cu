// layers.cu — render layers (row ranges of the call's Gaussians) in the same rasterizer call as the full frame.
//
// A layer [begin, end) is what a separate call on the sliced tensors would render (the reference's render_object /
// render_background, street_gaussian_renderer.py:13-40).  Preprocessing and the exact tile cull are per Gaussian, emission follows
// the stable (depth, index) pre-sort and the tile sort is stable, so the separate call's list of every tile is exactly the
// subsequence of the main call's list whose ids lie in the range.  The kernels below compact those subsequences out of the main
// lists; the unmodified blend kernels then run on them with the main call's records, so the layer images are bit-identical to a
// separate call by construction and nothing is projected or sorted again.
//
//   layer_count_kernel    one CTA per tile: entries of the main list with ids in [begin, end) -> ranges[t].y
//   layer_scan_kernel     one CTA: exclusive scan of the counts -> ranges[t] = [start, start + count)
//   layer_compact_kernel  one CTA per tile: stable compaction of the matching entries into the layer's list
// Grids depend on the tile count only (never on a read-back instance count), so a layered bounded-mode step captures in a CUDA graph.
//
// Backward: blend_bwd2 runs on the layer's list into the layer's own rows (a row-offset base: the list holds ids in [begin, end) only),
// then the chain rule runs ONCE on main + layer sums (it is linear in the 12 screen-space sums), while dL/dmeans2D keeps the main sums
// only (the densification statistics read it):
//   layer_stash_kernel    copy grad2d[:, 0:3] of the rows the layers cover to a scratch
//   layer_merge_kernel    add every layer's rows into the main grad2d, write each layer's [0:3] to its dL/dmeans2D sink
//   preprocess_bwd        unchanged
//   layer_restore_kernel  dL/dmeans2D of the covered rows <- the stashed main sums (what preprocess_bwd writes from unmerged rows)
#include "sgr_common.cuh"

namespace sgr {

constexpr int kLayerThreads = 256;

__global__ void __launch_bounds__(kLayerThreads) layer_count_kernel(const uint2 *__restrict__ ranges, const uint32_t *__restrict__ list,
                                                                    const uint32_t begin, const uint32_t end, uint2 *__restrict__ out_ranges) {
	__shared__ uint32_t s_warp[kLayerThreads / 32];
	const int tile = blockIdx.x;
	const uint2 r = ranges[tile];
	uint32_t n = 0;
	for (uint32_t k = r.x + threadIdx.x; k < r.y; k += kLayerThreads) {
		const uint32_t id = list[k];
		n += (id >= begin && id < end) ? 1u : 0u;
	}
	n = __reduce_add_sync(0xffffffffu, n);
	if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = n;
	__syncthreads();
	if (threadIdx.x == 0) {
		uint32_t t = 0;
#pragma unroll
		for (int w = 0; w < kLayerThreads / 32; w++) t += s_warp[w];
		out_ranges[tile] = make_uint2(0u, t);
	}
}

// one block of 1024 threads walks the tile counts in chunks of 1024 (a few thousand tiles per frame)
__global__ void __launch_bounds__(1024) layer_scan_kernel(uint2 *__restrict__ ranges, const uint32_t ntile) {
	__shared__ uint32_t s_warp[32];
	__shared__ uint32_t s_carry;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	if (threadIdx.x == 0) s_carry = 0u;
	__syncthreads();
	for (uint32_t base = 0; base < ntile; base += 1024u) {
		const uint32_t t = base + threadIdx.x;
		const uint32_t v = t < ntile ? ranges[t].y : 0u;
		uint32_t incl = v;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= o) incl += u;
		}
		if (lane == 31) s_warp[warp] = incl;
		__syncthreads();
		if (warp == 0) {
			uint32_t w = s_warp[lane];
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) {
				const uint32_t u = __shfl_up_sync(0xffffffffu, w, o);
				if (lane >= o) w += u;
			}
			s_warp[lane] = w;
		}
		__syncthreads();
		const uint32_t carry = s_carry;
		const uint32_t excl = carry + (warp ? s_warp[warp - 1] : 0u) + incl - v;
		if (t < ntile) ranges[t] = make_uint2(excl, excl + v);
		__syncthreads();
		if (threadIdx.x == 1023) s_carry = carry + s_warp[31];
		__syncthreads();
	}
}

// stable: within a chunk of 256 entries the output position is the number of matching entries before it (warp ballots + warp prefix)
__global__ void __launch_bounds__(kLayerThreads) layer_compact_kernel(const uint2 *__restrict__ ranges, const uint32_t *__restrict__ list,
                                                                      const uint32_t begin, const uint32_t end,
                                                                      const uint2 *__restrict__ out_ranges, uint32_t *__restrict__ out_list) {
	__shared__ uint32_t s_warp[kLayerThreads / 32];
	const int tile = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint2 r = ranges[tile];
	uint32_t at = out_ranges[tile].x;
	for (uint32_t k0 = r.x; k0 < r.y; k0 += kLayerThreads) {
		const uint32_t k = k0 + threadIdx.x;
		uint32_t id = 0;
		bool hit = false;
		if (k < r.y) {
			id = list[k];
			hit = id >= begin && id < end;
		}
		const unsigned b = __ballot_sync(0xffffffffu, hit);
		if (lane == 0) s_warp[warp] = (uint32_t)__popc(b);
		__syncthreads();
		uint32_t before = 0, total = 0;
#pragma unroll
		for (int w = 0; w < kLayerThreads / 32; w++) {
			const uint32_t c = s_warp[w];
			before += w < warp ? c : 0u;
			total += c;
		}
		if (hit) out_list[at + before + (uint32_t)__popc(b & ((1u << lane) - 1u))] = id;
		at += total;
		__syncthreads();  // s_warp is rewritten by the next chunk
	}
}

// a layer with an empty range: colour bg, depth and alpha zero (what the blend writes for a pixel no Gaussian reaches)
__global__ void __launch_bounds__(kLayerThreads) layer_fill_kernel(const size_t HW, const float *__restrict__ bg, float *__restrict__ color,
                                                                   float *__restrict__ depth, float *__restrict__ alpha) {
	const float b0 = bg[0], b1 = bg[1], b2 = bg[2];
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (size_t)gridDim.x * blockDim.x) {
		color[i] = b0;
		color[HW + i] = b1;
		color[2 * HW + i] = b2;
		depth[i] = 0.f;
		alpha[i] = 0.f;
	}
}

cudaError_t launch_layer_lists(const FrameDev &f, ImgView main_img, BinView main_bin, int begin, int end, ImgView layer_img, uint32_t *layer_list,
                               cudaStream_t st) {
	const int ntile = f.gx * f.gy;
	if (ntile <= 0) return cudaSuccess;
	count_launch(3);
	layer_count_kernel<<<ntile, kLayerThreads, 0, st>>>(main_img.ranges, main_bin.vals_out, (uint32_t)begin, (uint32_t)end, layer_img.ranges);
	layer_scan_kernel<<<1, 1024, 0, st>>>(layer_img.ranges, (uint32_t)ntile);
	layer_compact_kernel<<<ntile, kLayerThreads, 0, st>>>(main_img.ranges, main_bin.vals_out, (uint32_t)begin, (uint32_t)end, layer_img.ranges,
	                                                      layer_list);
	return cudaGetLastError();
}

cudaError_t launch_layer_fill(const FrameDev &f, const float *bg, float *color, float *depth, float *alpha, cudaStream_t st) {
	const size_t HW = (size_t)f.W * f.H;
	const size_t want = (HW + kLayerThreads - 1) / kLayerThreads;
	const unsigned blocks = (unsigned)(want < kNumSMs * 8 ? want : kNumSMs * 8);
	count_launch();
	layer_fill_kernel<<<blocks > 0 ? blocks : 1, kLayerThreads, 0, st>>>(HW, bg, color, depth, alpha);
	return cudaGetLastError();
}

// ---- backward merge ----
constexpr int kMergeLayers = 8;  // layers per merge launch; more layers take further launches (in table order)
struct MergeTable {
	int n;
	int begin[kMergeLayers], end[kMergeLayers];
	const float *grad2d[kMergeLayers];  // [end-begin, 12]
	float *sink[kMergeLayers];          // [end-begin, 3] or NULL
};

// rows [lo, hi): stash[i - lo] = grad2d[i, 0:3]
__global__ void __launch_bounds__(kLayerThreads) layer_stash_kernel(const float *__restrict__ grad2d, const int lo, const int hi,
                                                                    float *__restrict__ stash, const int restore, float *__restrict__ dL_dmeans2D) {
	const int i = lo + (int)(blockIdx.x * blockDim.x + threadIdx.x);
	if (i >= hi) return;
	const size_t j = (size_t)(i - lo);
	if (restore) {
		dL_dmeans2D[3 * (size_t)i] = stash[3 * j];
		dL_dmeans2D[3 * (size_t)i + 1] = stash[3 * j + 1];
		dL_dmeans2D[3 * (size_t)i + 2] = stash[3 * j + 2];
	} else {
		stash[3 * j] = grad2d[12 * (size_t)i];
		stash[3 * j + 1] = grad2d[12 * (size_t)i + 1];
		stash[3 * j + 2] = grad2d[12 * (size_t)i + 2];
	}
}

// thread = row i of [lo, hi): grad2d[i] += every covering layer's row (table order); sinks get the layer's [0:3]
__global__ void __launch_bounds__(kLayerThreads) layer_merge_kernel(float *__restrict__ grad2d, const int lo, const int hi, const MergeTable t) {
	const int i = lo + (int)(blockIdx.x * blockDim.x + threadIdx.x);
	if (i >= hi) return;
	float4 *row = reinterpret_cast<float4 *>(grad2d) + 3 * (size_t)i;
	float4 a = row[0], b = row[1], c = row[2];
	bool touched = false;
	for (int k = 0; k < t.n; k++) {
		if (i < t.begin[k] || i >= t.end[k]) continue;
		const size_t r = (size_t)(i - t.begin[k]);
		const float4 *src = reinterpret_cast<const float4 *>(t.grad2d[k]) + 3 * r;
		const float4 x = src[0], y = src[1], z = src[2];
		a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w;
		b.x += y.x; b.y += y.y; b.z += y.z; b.w += y.w;
		c.x += z.x; c.y += z.y; c.z += z.z; c.w += z.w;
		touched = true;
		if (t.sink[k]) {
			t.sink[k][3 * r] = x.x;
			t.sink[k][3 * r + 1] = x.y;
			t.sink[k][3 * r + 2] = x.z;
		}
	}
	if (touched) {
		row[0] = a; row[1] = b; row[2] = c;
	}
}

cudaError_t launch_layer_stash(const float *grad2d, int lo, int hi, float *stash, bool restore, float *dL_dmeans2D, cudaStream_t st) {
	if (hi <= lo) return cudaSuccess;
	count_launch();
	layer_stash_kernel<<<(unsigned)((hi - lo + kLayerThreads - 1) / kLayerThreads), kLayerThreads, 0, st>>>(grad2d, lo, hi, stash, restore ? 1 : 0,
	                                                                                                        dL_dmeans2D);
	return cudaGetLastError();
}

cudaError_t launch_layer_merge(float *grad2d, const SgrLayerGrad *layers, int n, cudaStream_t st) {
	for (int k0 = 0; k0 < n;) {
		MergeTable t = {};
		int lo = 0x7fffffff, hi = 0;
		for (; k0 < n && t.n < kMergeLayers; k0++) {
			const SgrLayerGrad &l = layers[k0];
			if (!l.grad2d || l.end <= l.begin) continue;
			t.begin[t.n] = l.begin; t.end[t.n] = l.end; t.grad2d[t.n] = l.grad2d; t.sink[t.n] = l.dL_dmeans2D;
			t.n++;
			lo = l.begin < lo ? l.begin : lo;
			hi = l.end > hi ? l.end : hi;
		}
		if (t.n == 0) continue;
		count_launch();
		layer_merge_kernel<<<(unsigned)((hi - lo + kLayerThreads - 1) / kLayerThreads), kLayerThreads, 0, st>>>(grad2d, lo, hi, t);
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess) return e;
	}
	return cudaSuccess;
}

}  // namespace sgr
