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
//
// The fused Gaussian-sharded step (sgr_sharded_*_layers) lists slots, not ids: the *_masked passes keep the slots whose delivered layer
// byte has the layer's bit, layer_zero_rows_kernel clears the layer rows of the slots delivered to a rank, and layer_gather_kernel sums
// an owner's main and layer rows from the ranks that rendered them before preprocess_bwd runs once on the sum.
#include "sgr_common.cuh"

namespace sgr {

constexpr int kLayerThreads = 256;

// which entries of the main list a layer keeps: one GPU, ids in [begin, end); the fused Gaussian-sharded step, slots whose delivered
// layer byte has the layer's bit (the lists hold slots, which do not give back an owner's row)
struct InRange {
	uint32_t begin, end;
	__device__ __forceinline__ bool operator()(uint32_t id) const { return id >= begin && id < end; }
};
struct MaskBit {
	const uint8_t *mask;
	uint32_t bit;
	__device__ __forceinline__ bool operator()(uint32_t id) const { return (mask[id] >> bit) & 1u; }
};

template <typename Keep>
__device__ __forceinline__ void layer_count(const uint2 *__restrict__ ranges, const uint32_t *__restrict__ list, const Keep keep,
                                            uint2 *__restrict__ out_ranges) {
	__shared__ uint32_t s_warp[kLayerThreads / 32];
	const int tile = blockIdx.x;
	const uint2 r = ranges[tile];
	uint32_t n = 0;
	for (uint32_t k = r.x + threadIdx.x; k < r.y; k += kLayerThreads) {
		const uint32_t id = list[k];
		n += keep(id) ? 1u : 0u;
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
template <typename Keep>
__device__ __forceinline__ void layer_compact(const uint2 *__restrict__ ranges, const uint32_t *__restrict__ list, const Keep keep,
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
			hit = keep(id);
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

__global__ void __launch_bounds__(kLayerThreads) layer_count_kernel(const uint2 *__restrict__ ranges, const uint32_t *__restrict__ list,
                                                                    const uint32_t begin, const uint32_t end, uint2 *__restrict__ out_ranges) {
	layer_count(ranges, list, InRange{begin, end}, out_ranges);
}
__global__ void __launch_bounds__(kLayerThreads) layer_compact_kernel(const uint2 *__restrict__ ranges, const uint32_t *__restrict__ list,
                                                                      const uint32_t begin, const uint32_t end,
                                                                      const uint2 *__restrict__ out_ranges, uint32_t *__restrict__ out_list) {
	layer_compact(ranges, list, InRange{begin, end}, out_ranges, out_list);
}
__global__ void __launch_bounds__(kLayerThreads) layer_count_masked_kernel(const uint2 *__restrict__ ranges, const uint32_t *__restrict__ list,
                                                                           const uint8_t *__restrict__ mask, const uint32_t bit,
                                                                           uint2 *__restrict__ out_ranges) {
	layer_count(ranges, list, MaskBit{mask, bit}, out_ranges);
}
__global__ void __launch_bounds__(kLayerThreads) layer_compact_masked_kernel(const uint2 *__restrict__ ranges, const uint32_t *__restrict__ list,
                                                                             const uint8_t *__restrict__ mask, const uint32_t bit,
                                                                             const uint2 *__restrict__ out_ranges, uint32_t *__restrict__ out_list) {
	layer_compact(ranges, list, MaskBit{mask, bit}, out_ranges, out_list);
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
// the same three passes keeping the slots whose delivered layer byte has bit `bit` (the fused Gaussian-sharded step)
cudaError_t launch_layer_lists_masked(const FrameDev &f, ImgView main_img, BinView main_bin, const uint8_t *mask, int bit, ImgView layer_img,
                                      uint32_t *layer_list, cudaStream_t st) {
	const int ntile = f.gx * f.gy;
	if (ntile <= 0) return cudaSuccess;
	count_launch(3);
	layer_count_masked_kernel<<<ntile, kLayerThreads, 0, st>>>(main_img.ranges, main_bin.vals_out, mask, (uint32_t)bit, layer_img.ranges);
	layer_scan_kernel<<<1, 1024, 0, st>>>(layer_img.ranges, (uint32_t)ntile);
	layer_compact_masked_kernel<<<ntile, kLayerThreads, 0, st>>>(main_img.ranges, main_bin.vals_out, mask, (uint32_t)bit, layer_img.ranges,
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

// ---- the fused Gaussian-sharded step (sgr_sharded_forward_layers / sgr_sharded_backward_layers) ----
// The rows of a rank's layer sections that its owners read back are those of every slot delivered to the rank, but its layer blends
// write only the slots of their lists.  So, like count_runs_kernel for the main rows, the forward clears the layer rows of the delivered
// slots: thread j = j-th delivered Gaussian (cval, in ascending slot order), j < the delivered count on the device (status[4]) and the
// depth-order slots n of the call.
__global__ void __launch_bounds__(kLayerThreads) layer_zero_rows_kernel(const uint32_t *__restrict__ cval, const uint32_t *__restrict__ status,
                                                                        const uint32_t n, const LayerRows t) {
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= n || j >= status[4]) return;
	const size_t g = cval[j];
	const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
	for (int k = 0; k < kMaxShardedLayers; k++) {
		if (k >= t.n) break;
		float4 *row = reinterpret_cast<float4 *>(t.rows[k]) + 3 * g;
		row[0] = z; row[1] = z; row[2] = z;
	}
}
cudaError_t launch_layer_zero_rows(GeomView g, int n, const LayerRows &t, cudaStream_t st) {
	if (n <= 0 || t.n == 0) return cudaSuccess;
	count_launch();
	layer_zero_rows_kernel<<<(unsigned)((n + kLayerThreads - 1) / kLayerThreads), kLayerThreads, 0, st>>>(g.cval, g.big_count, (uint32_t)n, t);
	return cudaGetLastError();
}

// Owner side of the layered backward: every block fetches the rows of its 256 Gaussians from the ranks that rendered them, the main
// section and then each live layer's (gather_runs: the same runs, ascending rank order, from 0), and writes
//   out[i]         = main + every covering live layer in table order (what layer_merge_kernel makes of them on one GPU),
//   dL_dmeans2D[i] = main[0:3]             (the densification statistics read the main sums only),
//   sink_k[i - b]  = layer k's [0:3].
// Rows of Gaussians without a destination are zero (their mask is 0).
__global__ void __launch_bounds__(kRunBlock) layer_gather_kernel(const int P, const PeerTable pt, const LayerGatherTable t,
                                                                 const int32_t *__restrict__ radii, const uint32_t *__restrict__ masks,
                                                                 float *__restrict__ out, float *__restrict__ dL_dmeans2D) {
	__shared__ RunScratch rs;
	__shared__ float4 s_g[3 * kRunBlock];
	const int idx = blockIdx.x * kRunBlock + threadIdx.x;
	const bool in_range = idx < P;
	const uint32_t mask = in_range && radii[idx] > 0 ? masks[idx] : 0u;
	float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a, c = a;
	gather_runs(pt, mask, rs, s_g, a, b, c);
	if (in_range) {
		dL_dmeans2D[3 * (size_t)idx] = a.x; dL_dmeans2D[3 * (size_t)idx + 1] = a.y; dL_dmeans2D[3 * (size_t)idx + 2] = a.z;
	}
#pragma unroll
	for (int k = 0; k < kMaxShardedLayers; k++) {
		if (k >= t.n) break;  // (uniform over the block: gather_runs is collective)
		__syncthreads();      // the previous gather's last readers of rs are done
		float4 x = make_float4(0.f, 0.f, 0.f, 0.f), y = x, z = x;
		gather_runs(t.sec[k], mask, rs, s_g, x, y, z);
		if (in_range && idx >= t.begin[k] && idx < t.end[k]) {
			a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w;
			b.x += y.x; b.y += y.y; b.z += y.z; b.w += y.w;
			c.x += z.x; c.y += z.y; c.z += z.z; c.w += z.w;
			if (t.sink[k]) {
				const size_t r = (size_t)(idx - t.begin[k]);
				t.sink[k][3 * r] = x.x; t.sink[k][3 * r + 1] = x.y; t.sink[k][3 * r + 2] = x.z;
			}
		}
	}
	if (in_range) {
		float4 *dst = reinterpret_cast<float4 *>(out) + 3 * (size_t)idx;
		dst[0] = a; dst[1] = b; dst[2] = c;
	}
}
cudaError_t launch_layer_gather(int P, const PeerTable &pt, const LayerGatherTable &t, const int32_t *radii, const uint32_t *masks, float *out,
                                float *dL_dmeans2D, cudaStream_t st) {
	if (P == 0) return cudaSuccess;
	count_launch();
	layer_gather_kernel<<<(unsigned)((P + kRunBlock - 1) / kRunBlock), kRunBlock, 0, st>>>(P, pt, t, radii, masks, out, dL_dmeans2D);
	return cudaGetLastError();
}

}  // namespace sgr
