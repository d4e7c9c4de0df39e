// binning.cu — depth pre-sort, instance offsets, (tile, gaussian) pair emission, stable tile bucketing, per-tile ranges.
//
// Replaces the reference's cub InclusiveSum + duplicateWithKeys + 64-bit cub SortPairs + identifyTileRanges
// (DGR/cuda_rasterizer/rasterizer_impl.cu:278-321, 70-138).  The reference sorts all R instances on a 46-bit
// (tile << 32 | depth bits) key: 6 onesweep passes x 24 B per instance.  Here the two halves of that key are sorted
// where they are cheapest:
//   1. the P Gaussians are sorted ONCE by their 32-bit depth bits (stable radix sort, ties keep ascending index);
//   2. instances are emitted in that order, so the unsorted list is already depth-ordered;
//   3. a STABLE sort on the tile id alone then yields exactly the reference's order: ascending tile, within a tile ascending
//      depth bits, ties by ascending Gaussian index.  Frames of at most kBucketMaxTiles tiles bucket the emitted instances
//      (launch_bucketing: two 7-bit digit passes, ranges from the tile histogram); larger ones take a cub radix sort over the
//      whole list and find the ranges in the sorted keys.
// Integer / bit work: the resulting per-tile lists equal the reference's lists minus the instances removed by the
// exact cull (tile_visit.cuh); tests/test_parity_gpu.py checks images bit-for-bit / to 1e-6 against the reference.
#include <cub/block/block_radix_rank.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include "sgr_common.cuh"
#include "tile_visit.cuh"

namespace sgr {

struct GatherCount {
	const uint32_t *tiles_touched, *perm, *depth_sorted;
	// entries whose sorted key is 0xFFFFFFFF emit nothing: Gaussians without instances (uncompacted order) or the padding
	// behind the selected ones (compacted order, where perm is meaningless) — a real view depth > 0.2 never has those bits
	__host__ __device__ __forceinline__ uint32_t operator()(int t) const {
		return depth_sorted[t] == 0xffffffffu ? 0u : tiles_touched[perm[t]];
	}
};
using CountIter = cub::TransformInputIterator<uint32_t, GatherCount, cub::CountingInputIterator<int>>;

// Frames of up to this many tiles bucket their instances by tile (launch_bucketing below): the per-tile histogram and cursors
// live in shared memory (64 KB).  Larger frames take the tile radix sort.
constexpr int kBucketMaxTiles = 16384;

size_t geom_temp_bytes(int P) {
	const int n = P > 0 ? P : 1;
	size_t a = 0, b = 0;
	CountIter it(cub::CountingInputIterator<int>(0), GatherCount{nullptr, nullptr, nullptr});
	cub::DeviceScan::InclusiveSum(nullptr, a, it, (uint32_t *)nullptr, n);
	size_t d = 0;  // the far pass of the saturation split scans a plain count array
	cub::DeviceScan::InclusiveSum(nullptr, d, (const uint32_t *)nullptr, (uint32_t *)nullptr, n);
	a = a > d ? a : d;
	cub::DeviceRadixSort::SortPairs(nullptr, b, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, n);
	return a > b ? a : b;
}
size_t sort_temp_bytes(int64_t R) {
	size_t a = 0, b = 0;
	const int64_t n = R > 0 ? R : 1;
	cub::DeviceRadixSort::SortPairs(nullptr, a, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, n);
	cub::DeviceRadixSort::SortPairs(nullptr, b, (uint16_t *)nullptr, (uint16_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, n);
	return a > b ? a : b;
}

// A Gaussian's footprint on the tile grid, from its record and radius: the 3-sigma tile rectangle [x0, x1) x [y0, y1) and the
// parameters of the exact cull.  The default (empty) footprint is what a thread without a Gaussian hands to visit_tiles.
struct Footprint {
	int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
	CullParams cp = {};
};
__device__ __forceinline__ Footprint rec_footprint(const FrameDev &f, const GaussRec &rec, int radius) {
	const float4 q0 = rec.q0, q1 = rec.q1;
	Footprint fp;
	tile_rect(q0.x, q0.y, radius, f.gx, f.gy, fp.x0, fp.y0, fp.x1, fp.y1);
	fp.cp = make_cull(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y);
	return fp;
}
// clears row i of a grad2d[P, 12] (nullable)
__device__ __forceinline__ void zero_grad2d_row(float4 *__restrict__ rows, size_t i) {
	if (!rows) return;
	const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
	rows[3 * i] = z; rows[3 * i + 1] = z; rows[3 * i + 2] = z;
}

// Gaussian-sharded mode (include/sgr.h, sgr_forward_records): the records were projected on other ranks and gathered, so
// the tail of preprocess_fwd_kernel — instance count against THIS rank's tile-row band, depth sort key, identity
// permutation — runs here from the 48-B record + radius.  Same rec_footprint / visit_tiles as the emission
// kernels below, so counts and emitted ranges agree by construction.
// zero_rows (nullable): this rank's partial grad2d[P,12].  The rows of the Gaussians delivered to this rank (radius != 0 <=>
// rectangle meets the band) are the only ones its blend_bwd can touch and the only ones their owners read back, so they are
// zeroed here — 48 B x (Gaussians in the band) instead of a 48 B x P_total memset in front of every backward.
// reached: every Gaussian with a radius starts reached — the inputs of its chain rule were projected elsewhere and are not checked here.
__global__ void __launch_bounds__(256) count_tiles_kernel(const FrameDev f, const GaussRec *__restrict__ rec,
                                                         const int32_t *__restrict__ radii, uint32_t *__restrict__ tiles_touched,
                                                         uint32_t *__restrict__ depth_key, uint32_t *__restrict__ iota,
                                                         uint32_t *__restrict__ reached, float4 *__restrict__ zero_rows) {
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const bool in_range = idx < f.P;
	bool ok = false;
	Footprint fp;
	float depth = 0.f;
	if (in_range) {
		const int r = radii[idx];
		if (r > 0) {
			fp = rec_footprint(f, rec[idx], r);
			depth = rec[idx].q1.w;
			ok = true;
			zero_grad2d_row(zero_rows, idx);
		}
	}
	uint32_t count = 0;
	visit_tiles<false, uint32_t>(ok, fp.x0, fp.y0, fp.x1, fp.y1, fp.cp, f.band, f.gx, 0u, 0u, nullptr, nullptr, count);
	if (in_range) {
		tiles_touched[idx] = count;
		depth_key[idx] = count > 0 ? __float_as_uint(depth) : 0xffffffffu;
		iota[idx] = (uint32_t)idx;
		reached[idx] = ok ? 1u : 0u;
	}
}
cudaError_t launch_count_tiles(const FrameDev &f, GeomView g, const int32_t *radii, cudaStream_t st, float *zero_rows) {
	if (f.P == 0) return cudaSuccess;
	count_launch();
	count_tiles_kernel<<<(f.P + 255) / 256, 256, 0, st>>>(f, g.rec, radii, g.tiles_touched, g.depth_key, g.iota, g.reached,
	                                                      reinterpret_cast<float4 *>(zero_rows));
	return cudaGetLastError();
}

// n (depth key, Gaussian) pairs sorted into g.depth_sorted / g.perm, then the inclusive scan of the Gaussians' instance counts
// (g.tiles_touched) in that order into g.offsets
static cudaError_t sort_and_scan_depth(GeomView g, const uint32_t *keys, const uint32_t *vals, int n, cudaStream_t st) {
	size_t bytes = g.temp_bytes;
	cudaError_t e = cub::DeviceRadixSort::SortPairs(g.temp, bytes, keys, g.depth_sorted, vals, g.perm, n, 0, 32, st);
	if (e != cudaSuccess) return e;
	CountIter it(cub::CountingInputIterator<int>(0), GatherCount{g.tiles_touched, g.perm, g.depth_sorted});
	bytes = g.temp_bytes;
	return cub::DeviceScan::InclusiveSum(g.temp, bytes, it, g.offsets, n, st);
}

// depth order of the Gaussians + inclusive scan of their instance counts in that order (uncompacted: all f.P Gaussians take part,
// those without instances carry the key 0xFFFFFFFF and sort to the end).  tiles_touched / depth_key / iota come from
// preprocess_fwd_kernel<COUNT> or count_tiles_kernel.
cudaError_t launch_depth_order(const FrameDev &f, GeomView g, cudaStream_t st) {
	if (f.P == 0) return cudaSuccess;
	return sort_and_scan_depth(g, g.depth_key, g.iota, f.P, st);
}

// ---- fused Gaussian-sharded forward: the delivered runs (sgr_common.cuh "block-run exchange") -> compact depth-sort input ----
// cnt[s * nblk + b] = number of records block b of owner s delivered to this rank (written by the owners' projection kernels before the
// barrier).  One block turns the table into an exclusive prefix (entry e = first compact position of run e) and the total (status[4]).
__global__ void __launch_bounds__(1024) run_prefix_kernel(const uint32_t *__restrict__ cnt, uint32_t *__restrict__ pre, const uint32_t entries,
                                                          uint32_t *__restrict__ status) {
	__shared__ uint32_t s_warp[32];
	__shared__ uint32_t s_carry;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	if (threadIdx.x == 0) s_carry = 0u;
	__syncthreads();
	for (uint32_t base = 0; base < entries; base += 1024u) {
		const uint32_t e = base + threadIdx.x;
		const uint32_t v = e < entries ? cnt[e] : 0u;
		uint32_t incl = v;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= o) incl += t;
		}
		if (lane == 31) s_warp[warp] = incl;
		__syncthreads();
		if (warp == 0) {
			uint32_t w = s_warp[lane];
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) {
				const uint32_t t = __shfl_up_sync(0xffffffffu, w, o);
				if (lane >= o) w += t;
			}
			s_warp[lane] = w;  // inclusive prefix of the warp totals
		}
		__syncthreads();
		const uint32_t carry = s_carry;
		const uint32_t excl = carry + (warp ? s_warp[warp - 1] : 0u) + incl - v;
		if (e < entries) pre[e] = excl;
		__syncthreads();
		if (threadIdx.x == 1023) s_carry = carry + s_warp[31];
		__syncthreads();
	}
	if (threadIdx.x == 0) status[4] = s_carry;
}

// thread j = j-th delivered Gaussian in ascending slot order (= ascending global id): locate its run by binary search in the prefix table,
// take the radius out of the record, count its tiles against this rank's band, write the depth-sort input and clear its grad2d row.
__global__ void __launch_bounds__(256) count_runs_kernel(const FrameDev f, const GaussRec *__restrict__ rec, int32_t *__restrict__ radii,
                                                        const uint32_t *__restrict__ pre, const uint32_t entries, const uint32_t nblk,
                                                        const long long chunk, uint32_t *__restrict__ status, const uint32_t cap_v,
                                                        uint32_t *__restrict__ tiles_touched, uint32_t *__restrict__ ckey,
                                                        uint32_t *__restrict__ cval, float4 *__restrict__ zero_rows) {
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t n_act = status[4];
	if (j == 0 && n_act > cap_v) atomicOr(&status[2], 2u);
	const bool live = j < n_act && j < cap_v;
	bool ok = false;
	Footprint fp;
	float depth = 0.f;
	uint32_t gidx = 0u;
	if (live) {
		uint32_t lo = 0u, hi = entries;  // largest e with pre[e] <= j  (pre[0] = 0 <= j)
		while (hi - lo > 1u) {
			const uint32_t mid = (lo + hi) >> 1;
			if (pre[mid] <= j) lo = mid; else hi = mid;
		}
		const uint32_t s = lo / nblk, b = lo - s * nblk;
		gidx = (uint32_t)((long long)s * chunk + (long long)b * kRunBlock) + (j - pre[lo]);
		const int r = packed_radius(rec[gidx].q2.w);
		radii[gidx] = r;  // emit_pairs / emit_big read the radius from here
		fp = rec_footprint(f, rec[gidx], r);
		depth = rec[gidx].q1.w;
		ok = true;
		zero_grad2d_row(zero_rows, gidx);
	}
	uint32_t count = 0;
	visit_tiles<false, uint32_t>(ok, fp.x0, fp.y0, fp.x1, fp.y1, fp.cp, f.band, f.gx, 0u, 0u, nullptr, nullptr, count);
	if (j < cap_v) {
		ckey[j] = (live && count > 0u) ? __float_as_uint(depth) : 0xffffffffu;
		cval[j] = gidx;
		if (live) tiles_touched[gidx] = count;
	}
}

// g.iota = count table (filled by the owners), g.perm = its prefix (dead before the sort writes g.perm), cap_v < 0 -> all f.P slots
cudaError_t launch_count_and_order_runs(const FrameDev &f, GeomView g, int32_t *radii, int world, long long chunk, cudaStream_t st, int64_t cap_v,
                                        float *zero_rows, int *n_order) {
	if (n_order) *n_order = f.P;
	if (f.P == 0) return cudaSuccess;
	const int n = (int)(cap_v < 0 ? (int64_t)f.P : (cap_v < 1 ? 1 : (cap_v > f.P ? f.P : cap_v)));
	const uint32_t nblk = (uint32_t)((chunk + kRunBlock - 1) / kRunBlock);
	const uint32_t entries = (uint32_t)world * nblk;
	// the prefix table lives in g.offsets until the count kernel has consumed it (the scan below then overwrites it)
	uint32_t *pre = g.offsets;
	count_launch();
	run_prefix_kernel<<<1, 1024, 0, st>>>(g.iota, pre, entries, g.big_count);
	count_launch();
	count_runs_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(f, g.rec, radii, pre, entries, nblk, chunk, g.big_count, (uint32_t)n, g.tiles_touched,
	                                                               g.ckey, g.cval, reinterpret_cast<float4 *>(zero_rows));
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return e;
	if (n_order) *n_order = n;
	return sort_and_scan_depth(g, g.ckey, g.cval, n, st);
}

constexpr uint32_t kEmitStage = 512;  // instances staged per warp (2 x 2 KB of shared memory per warp)

// thread t handles the t-th Gaussian in depth order.  KeyT = uint16_t whenever the image has at most 65,536 tiles (up to
// 4096 x 4096 px): the tile sort then moves 6 instead of 8 bytes per pair per pass.
// Saturation split (launch_near_binning / launch_far_binning): the near pass passes dev_cap -> its end of the emitted sequence, so
// only the Gaussians before the split emit; the far pass passes its own offsets, dev_cap -> the end of the emitted sequence,
// dev_floor -> the near pass's end (the Gaussians before the split then have empty ranges there) and the KeepUnsaturated predicate.
// A pass whose device-side cap does not exceed its floor (0 without one) has nothing to emit: the whole grid returns.
// reached (nullable): set for every Gaussian with a non-empty range in this pass — the Gaussians the per-tile lists can hold, so the only
// ones a blend backward can add to (the ranges already exclude what the bounded mode drops and, in the far pass, the saturated tiles).
template <typename KeyT, typename Keep = KeepAll>
__global__ void __launch_bounds__(256) emit_pairs_kernel(const FrameDev f, const GaussRec *__restrict__ rec, const int32_t *__restrict__ radii,
                                                        const uint32_t *__restrict__ perm, const uint32_t *__restrict__ offsets, KeyT *__restrict__ keys,
                                                        uint32_t *__restrict__ vals, uint32_t *__restrict__ big_list,
                                                        uint32_t *__restrict__ big_count, uint32_t *__restrict__ reached, uint32_t cap, const int n_order,
                                                        const uint32_t *__restrict__ dev_cap = nullptr,
                                                        const uint32_t *__restrict__ dev_floor = nullptr, const Keep keep = Keep()) {
	if (dev_cap && *dev_cap <= (dev_floor ? *dev_floor : 0u)) return;
	__shared__ KeyT s_keys[8][kEmitStage];
	__shared__ uint32_t s_vals[8][kEmitStage];
	const int warp = threadIdx.x >> 5;
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	bool active = false;
	Footprint fp;
	uint32_t gidx = 0;
	// [off, end) = this Gaussian's output range (offsets = inclusive scan in depth order); lanes past P get an empty range
	const int tc = min(t, n_order - 1);  // n_order = depth-order slots: f.P, or the Gaussian capacity of the compacted mode
	uint32_t end = offsets[tc];
	uint32_t off = tc == 0 ? 0u : offsets[tc - 1];
	if (t >= n_order) off = end;
	if (dev_cap) cap = min(cap, *dev_cap);
	if (dev_floor) {
		const uint32_t fl = *dev_floor;
		off = max(off, fl);
		end = max(end, fl);
	}
	// bounded mode: a Gaussian whose range does not fit the caller's capacity emits nothing.  BOTH ends are clamped so that
	// warp_first / warp_last (taken from lanes 0 / 31 below) never address past `cap`, even when every lane of the warp
	// overflows: the staged flush then covers at most [warp_first, cap), and pad_keys_kernel rewrites [emitted, cap).
	if (end > cap) {
		off = min(off, cap);
		end = off;
	}
	if (t < n_order) {
		if (end > off) {
			gidx = perm[t];  // (padding slots of the compacted order have end == off and a meaningless perm)
			fp = rec_footprint(f, rec[gidx], radii[gidx]);
			active = true;
			if (reached) reached[gidx] = 1u;
		}
	}
	const uint32_t warp_first = __shfl_sync(0xffffffffu, off, 0);
	const uint32_t warp_last = __shfl_sync(0xffffffffu, end, 31);
	const uint32_t warp_total = warp_last >= warp_first ? warp_last - warp_first : 0xffffffffu;  // (overflow tail: no staging)
	uint32_t count;
	visit_tiles<true, KeyT, Keep>(active, fp.x0, fp.y0, fp.x1, fp.y1, fp.cp, f.band, f.gx, gidx, off, keys, vals, count, s_keys[warp], s_vals[warp],
	                              kEmitStage, warp_first, warp_total, big_list, big_count, (uint32_t)t, keep);
}

// One warp per deferred (large-rectangle) Gaussian, grid-strided over the device-side list: no host round trip for the count.
template <typename KeyT, typename Keep = KeepAll>
__global__ void __launch_bounds__(256) emit_big_kernel(const FrameDev f, const GaussRec *__restrict__ rec, const int32_t *__restrict__ radii,
                                                      const uint32_t *__restrict__ perm, const uint32_t *__restrict__ offsets,
                                                      KeyT *__restrict__ keys, uint32_t *__restrict__ vals,
                                                      const uint32_t *__restrict__ big_list, const uint32_t *__restrict__ big_count,
                                                      const uint32_t cap, const Keep keep = Keep()) {
	const uint32_t n = *big_count;
	const uint32_t nwarps = gridDim.x * 8u;
	const int lane = threadIdx.x & 31;
	for (uint32_t i = blockIdx.x * 8u + (threadIdx.x >> 5); i < n; i += nwarps) {
		const uint32_t t = big_list[i];
		const uint32_t gidx = perm[t];
		const Footprint fp = rec_footprint(f, rec[gidx], radii[gidx]);
		const uint32_t off = t == 0 ? 0u : offsets[t - 1];
		if (offsets[t] > cap) continue;  // bounded mode overflow (never deferred in practice: emit_pairs already skipped it)
		// lane 0 carries the Gaussian through the cooperative path of visit_tiles (all other lanes inactive)
		uint32_t count;
		visit_tiles<true, KeyT, Keep>(lane == 0, fp.x0, fp.y0, fp.x1, fp.y1, fp.cp, f.band, f.gx, gidx, off, keys, vals, count, nullptr, nullptr, 0u, 0u, 0u,
		                              nullptr, nullptr, 0u, keep);
	}
}

// the emission of one pass: the instances of depth-order slot t go to [offsets[t - 1], offsets[t]) of (b.keys_in, b.vals_in);
// status = the status block whose word 0 counts the deferred Gaussians.  dev_cap, dev_floor, keep: see emit_pairs_kernel.
template <typename KeyT, typename Keep = KeepAll>
static cudaError_t launch_emit(const FrameDev &f, GeomView g, const int32_t *radii, const BinView &b, const uint32_t *offsets, uint32_t *status,
                               uint32_t cap32, int n_order, cudaStream_t st, const uint32_t *dev_cap = nullptr,
                               const uint32_t *dev_floor = nullptr, const Keep keep = Keep()) {
	KeyT *keys = reinterpret_cast<KeyT *>(b.keys_in);
	count_launch(2);
	emit_pairs_kernel<KeyT, Keep><<<(unsigned)((n_order + 255) / 256), 256, 0, st>>>(f, g.rec, radii, g.perm, offsets, keys, b.vals_in,
	                                                                               g.big_list, status, g.reached, cap32, n_order, dev_cap, dev_floor,
	                                                                               keep);
	// persistent-style grid for the deferred large rectangles
	emit_big_kernel<KeyT, Keep><<<kNumSMs * 4, 256, 0, st>>>(f, g.rec, radii, g.perm, offsets, keys, b.vals_in, g.big_list, status, cap32, keep);
	return cudaGetLastError();
}

// One thread per sorted instance: a tile's range starts / ends where the tile id changes
// (reference identifyTileRanges, rasterizer_impl.cu:116-138).  ranges must be zero-initialised.
constexpr int kRangeKeysPerThread = 8;
template <typename KeyT>
__global__ void __launch_bounds__(256) tile_ranges_kernel(int64_t L, const KeyT *__restrict__ keys, uint2 *__restrict__ ranges, const uint32_t ntile) {
	// 8 consecutive keys per thread (one 16-B load for 16-bit tile ids): the one-key-per-thread version was far from the bandwidth bound.
	const int64_t base = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * kRangeKeysPerThread;
	if (base >= L) return;
	uint32_t k[kRangeKeysPerThread];
	if (base + kRangeKeysPerThread <= L) {
		if (sizeof(KeyT) == 2) {
			const uint4 v = *reinterpret_cast<const uint4 *>(keys + base);  // base is a multiple of 8 -> 16-B aligned
			k[0] = v.x & 0xffffu; k[1] = v.x >> 16; k[2] = v.y & 0xffffu; k[3] = v.y >> 16;
			k[4] = v.z & 0xffffu; k[5] = v.z >> 16; k[6] = v.w & 0xffffu; k[7] = v.w >> 16;
		} else {
			const uint4 a = reinterpret_cast<const uint4 *>(keys + base)[0], b = reinterpret_cast<const uint4 *>(keys + base)[1];
			k[0] = a.x; k[1] = a.y; k[2] = a.z; k[3] = a.w; k[4] = b.x; k[5] = b.y; k[6] = b.z; k[7] = b.w;
		}
	} else {
#pragma unroll
		for (int i = 0; i < kRangeKeysPerThread; i++) k[i] = base + i < L ? (uint32_t)keys[base + i] : 0xffffffffu;
	}
	// keys >= ntile are the padding of the bounded mode (they sort behind every real tile)
	uint32_t prev = base == 0 ? 0xffffffffu : (uint32_t)keys[base - 1];
#pragma unroll
	for (int i = 0; i < kRangeKeysPerThread; i++) {
		const int64_t idx = base + i;
		if (idx >= L) break;
		const uint32_t cur = k[i];
		if (cur != prev || idx == 0) {
			if (idx != 0 && prev < ntile) ranges[prev].y = (uint32_t)idx;
			if (cur < ntile) ranges[cur].x = (uint32_t)idx;
		}
		if (idx == L - 1 && cur < ntile) ranges[cur].y = (uint32_t)L;
		prev = cur;
	}
}

// number of leading depth-order slots whose inclusive offset is <= limit (offsets ascend)
__device__ __forceinline__ int slots_within(const uint32_t *__restrict__ offsets, int n, uint32_t limit) {
	int lo = 0, hi = n;  // first index with offsets[i] > limit
	while (lo < hi) {
		const int mid = (lo + hi) >> 1;
		if (offsets[mid] > limit) hi = mid; else lo = mid + 1;
	}
	return lo;
}

// status words: [1] = R (true instance count), [2] = overflow flag, [3] = instances actually emitted (<= cap)
__global__ void count_status_kernel(const uint32_t *__restrict__ offsets, int P, uint32_t cap, uint32_t *__restrict__ status) {
	const uint32_t R = offsets[P - 1];
	uint32_t emitted = R;
	if (R > cap) {  // largest scanned offset that still fits: Gaussians are emitted in depth order, the tail is dropped
		const int lo = slots_within(offsets, P, cap);
		emitted = lo == 0 ? 0u : offsets[lo - 1];
	}
	status[1] = R;
	status[2] |= R > cap ? 1u : 0u;  // (bit 1 = Gaussian-capacity overflow of the compacted depth order; the words are zeroed per forward)
	status[3] = emitted;
}
// grid-stride over [emitted, cap): the number of padding slots is only known on the device, and one thread per slot of the whole
// capacity spends its time retiring tens of thousands of empty blocks
template <typename KeyT>
__global__ void __launch_bounds__(256) pad_keys_kernel(KeyT *__restrict__ keys, uint32_t *__restrict__ vals, uint32_t cap,
                                                      const uint32_t *__restrict__ status) {
	const uint32_t stride = gridDim.x * blockDim.x;
	for (uint32_t i = status[3] + blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += stride) {
		keys[i] = (KeyT)~(KeyT)0;
		vals[i] = 0u;
	}
}

static int bits_for(uint32_t n) {  // smallest b with (1 << b) >= n, i.e. enough bits for tile ids 0..n-1
	int b = 0;
	while (b < 32 && (1ull << b) < (unsigned long long)n) b++;
	return b > 0 ? b : 1;
}

// the per-tile lists of a frame that does not bucket: a stable radix sort of the R emitted slots by tile id, then the ranges.  The
// bounded mode (R = its capacity) first pads [emitted, R) with the largest key, so every sort bit of KeyT takes part; the exact mode
// sorts on the bits the tile ids use.
template <typename KeyT>
static cudaError_t launch_tile_sort(const BinView &b, ImgView img, const uint32_t *status, int ntile, int64_t R, bool bounded, cudaStream_t st) {
	KeyT *kin = reinterpret_cast<KeyT *>(b.keys_in), *kout = reinterpret_cast<KeyT *>(b.keys_out);
	cudaError_t e;
	if (bounded) {
		count_launch();
		pad_keys_kernel<KeyT><<<(unsigned)std::min<int64_t>(R / 256 + 1, kNumSMs * 8), 256, 0, st>>>(kin, b.vals_in, (uint32_t)R, status);
		if ((e = cudaGetLastError()) != cudaSuccess) return e;
	}
	const int sort_bits = bounded ? 8 * (int)sizeof(KeyT) : bits_for(ntile);
	size_t bytes = b.sort_temp_bytes;
	if ((e = cub::DeviceRadixSort::SortPairs(b.sort_temp, bytes, kin, kout, b.vals_in, b.vals_out, R, 0, sort_bits, st)) != cudaSuccess) return e;
	count_launch();
	tile_ranges_kernel<KeyT><<<(unsigned)((R + 256 * kRangeKeysPerThread - 1) / (256 * kRangeKeysPerThread)), 256, 0, st>>>(R, kout, img.ranges,
	                                                                                                                  (uint32_t)ntile);
	return cudaGetLastError();
}

// ---- tile bucketing: the per-tile lists as a stable LSD radix sort of the EMITTED instances [0, E) on two 7-bit digits ----
// Emission already writes the instances in their final within-tile order (ascending depth bits, ties by ascending index), so a
// stable bucketing by tile id gives exactly the list the tile radix sort gives, over E instead of the whole capacity and without
// padding.  A single ranked scatter straight into the ~10^4 tile buckets writes isolated words (a partition holds ~3 instances of
// a tile); on config C it took 0.40 ms on an H100, more than the radix sort it replaces.  Two passes over 128 buckets write runs.
//   1. bucket_count<TILES>:  [0, E) is cut into partitions of bucket_part(E) instances; CTA p counts its partition's tile ids in a
//                            shared-memory histogram, adds its non-zero bins into the tile totals (ranges[t].y, zeroed first) and
//                            writes row p of the (partition x low digit) matrix;
//   2. bucket_columns:       per digit, the total over the partitions and the exclusive prefix over the partitions, in place;
//   3. bucket_ranges:        one CTA scans the tile totals into `ranges` ((0, 0) for a tile without instances);
//   4. bucket_pass<false>:   CTA p walks its partition in rounds; a stable match-based block rank of the round on the low digit
//                            gives every instance its position among equal digits, added to the digit's running cursor in shared
//                            memory; the Gaussian index with the high digit in its top 7 bits goes to the digit-ordered
//                            intermediate array (frames of at most 2^25 Gaussians; larger ones take the radix sort);
//   5. bucket_count<false>, bucket_columns, bucket_pass<true>: the same on the high digit of the intermediate array, writing the
//                            Gaussian indices into vals_out.
// Positions come from ranks and prefix sums only, never from the order of atomics (the tile totals are integer sums, which do not
// depend on it).  E is read on the device (*n_inst: status word 3, or the far pass's count) and the grids are sized for the most partitions any E up to the capacity
// can give, so the bounded mode stays free of host synchronisation.
constexpr int kBucketThreads = 512;  // histogram CTAs
constexpr int kPassThreads = 256;    // rank-and-scatter CTAs: 72 registers, 3 CTAs per SM
constexpr int kDigitBits = 7, kDigits = 1 << kDigitBits;
constexpr int kPassItems = 8;
constexpr uint32_t kPassRound = kPassThreads * kPassItems;
// Partition size: about E / kBucketTargetParts instances in whole rounds, at least one round and at most kBucketMaxPart.  With a
// fixed 32768 a frame of 1.4 M instances (config C's saturation split) had 43 partitions for 132 SMs, each walking 16 rounds behind
// three barriers per round; the target was chosen by a sweep on config C (DESIGN.md §7).  SGR_BUCKET_TARGET_PARTS exists for that
// sweep (tools/saturation_split_ab.py --sweep-parts builds one library per value).
#ifndef SGR_BUCKET_TARGET_PARTS
#define SGR_BUCKET_TARGET_PARTS 396
#endif
constexpr uint32_t kBucketTargetParts = SGR_BUCKET_TARGET_PARTS;
constexpr uint32_t kBucketMaxPart = 32768;
static_assert(kBucketTargetParts > 0 && kBucketMaxPart % kPassRound == 0, "partitions are whole rounds");
static_assert(kBucketThreads % kDigits == 0, "a histogram thread's tiles share one low digit");
__host__ __device__ __forceinline__ uint32_t bucket_part(uint32_t E) {
	const uint32_t per = E / kBucketTargetParts + (E % kBucketTargetParts != 0u);
	const uint32_t whole = (per + kPassRound - 1u) / kPassRound * kPassRound;
	return min(max(whole, kPassRound), kBucketMaxPart);
}
// Partitions of any E <= slots: bucket_part(E) >= ceil(E / kBucketTargetParts) unless capped, so at most kBucketTargetParts of them, or
// ceil(slots / kBucketMaxPart) when capped; and never more than ceil(slots / kPassRound).  CTAs past the last partition return.
static unsigned bucket_grid(int64_t slots) {
	const int64_t n = slots > 0 ? slots : 1;
	const int64_t most = std::max<int64_t>(kBucketTargetParts, (n + kBucketMaxPart - 1) / kBucketMaxPart);
	return (unsigned)std::min<int64_t>(most, (n + kPassRound - 1) / kPassRound);
}
static_assert(kBucketMaxTiles <= (1 << (2 * kDigitBits)), "two digits cover every tile id of a bucketed frame");
constexpr uint32_t kNoGaussian = 0xffffffffu;  // value of the slots of the last round past E
// the intermediate words carry the high digit in their top 7 bits, so a bucketed frame has at most 2^25 Gaussians
constexpr int kPackShift = 32 - kDigitBits;
constexpr uint32_t kPackMask = (1u << kPackShift) - 1u;
// whether a frame's instances are bucketed (16-bit tile ids) rather than taking the tile radix sort
static bool bucketable(const FrameDev &f) { return f.gx * f.gy <= kBucketMaxTiles && (uint32_t)f.P <= kPackMask + 1u; }

// the bucketing scratch behind the cub temp of the binning state (carve_bin): the two (partition x digit) count matrices and the
// digit totals.
struct BucketScratch {
	uint32_t *digit_counts[2], *digit_totals[2];
	size_t bytes;
};
static BucketScratch carve_bucket(void *base, int64_t slots) {
	BucketScratch s;
	char *p = reinterpret_cast<char *>(base);
	const size_t nparts = bucket_grid(slots);
	auto take = [&](size_t bytes) { char *r = p; p += align_up(bytes); return r; };
	for (int i = 0; i < 2; i++) s.digit_counts[i] = reinterpret_cast<uint32_t *>(take(nparts * kDigits * sizeof(uint32_t)));
	for (int i = 0; i < 2; i++) s.digit_totals[i] = reinterpret_cast<uint32_t *>(take(kDigits * sizeof(uint32_t)));
	s.bytes = (size_t)(p - reinterpret_cast<char *>(base));
	return s;
}
size_t bucket_scratch_bytes(int64_t slots) { return carve_bucket(nullptr, slots).bytes; }

// The slots [first, last) a bucketing pass covers (first = 0 unless the far pass of the saturation split buckets its instances
// behind the near ones).  Its partitions of bucket_part(last - base) slots start at base = first rounded down to a multiple of 8, so
// that the 16-B loads of 8 tile ids stay aligned; the slots before `first` take no part.  last - base <= the capacity, so the
// grids of bucket_grid(capacity) CTAs cover every partition.
struct BucketSpan {
	uint32_t first, base, end, part;
	__device__ __forceinline__ BucketSpan(const uint32_t *first_p, const uint32_t *last_p) {
		first = first_p ? *first_p : 0u;
		base = first & ~7u;
		end = *last_p;
		part = bucket_part(end - base);
	}
	__device__ __forceinline__ uint32_t parts() const { return (end - base) / part + ((end - base) % part != 0u); }
};

// TILES: tile_totals[2 t] += this partition's instances of tile t (ranges[t].y, zeroed by the caller)
template <bool TILES>
__global__ void __launch_bounds__(kBucketThreads) bucket_count_kernel(const uint16_t *__restrict__ keys, const uint32_t *__restrict__ first_p,
                                                                    const uint32_t *__restrict__ last_p, const uint32_t ntile,
                                                                    uint32_t *__restrict__ tile_totals, uint32_t *__restrict__ digit_counts) {
	extern __shared__ uint32_t s_hist[];  // TILES: per tile id of keys_in; else per high digit of the intermediate words
	__shared__ uint32_t s_digit[kDigits];
	const BucketSpan sp(first_p, last_p);
	const uint32_t begin = sp.base + blockIdx.x * sp.part;
	if (begin >= sp.end) return;  // (rows past the last partition are never read)
	const uint32_t end = min(begin + sp.part, sp.end), first = sp.first;
	const uint32_t nbin = TILES ? ntile : (uint32_t)kDigits;
	for (uint32_t t = threadIdx.x; t < nbin; t += kBucketThreads) s_hist[t] = 0u;
	if (TILES && threadIdx.x < kDigits) s_digit[threadIdx.x] = 0u;
	__syncthreads();
	if (!TILES) {
		const uint32_t *words = reinterpret_cast<const uint32_t *>(keys);
		for (uint32_t i = begin + threadIdx.x * 4u; i < end; i += kBucketThreads * 4u) {
			if (i >= first && i + 4u <= end) {
				const uint4 v = *reinterpret_cast<const uint4 *>(words + i);
				atomicAdd(&s_hist[v.x >> kPackShift], 1u); atomicAdd(&s_hist[v.y >> kPackShift], 1u);
				atomicAdd(&s_hist[v.z >> kPackShift], 1u); atomicAdd(&s_hist[v.w >> kPackShift], 1u);
			} else {
				for (uint32_t j = max(i, first); j < min(i + 4u, end); j++) atomicAdd(&s_hist[words[j] >> kPackShift], 1u);
			}
		}
	} else
	for (uint32_t i = begin + threadIdx.x * 8u; i < end; i += kBucketThreads * 8u) {
		if (i >= first && i + 8u <= end) {  // begin is a multiple of 8 and keys is 256-B aligned: one 16-B load of 8 tile ids
			const uint4 v = *reinterpret_cast<const uint4 *>(keys + i);
			atomicAdd(&s_hist[v.x & 0xffffu], 1u); atomicAdd(&s_hist[v.x >> 16], 1u);
			atomicAdd(&s_hist[v.y & 0xffffu], 1u); atomicAdd(&s_hist[v.y >> 16], 1u);
			atomicAdd(&s_hist[v.z & 0xffffu], 1u); atomicAdd(&s_hist[v.z >> 16], 1u);
			atomicAdd(&s_hist[v.w & 0xffffu], 1u); atomicAdd(&s_hist[v.w >> 16], 1u);
		} else {
			for (uint32_t j = max(i, first); j < min(i + 8u, end); j++) atomicAdd(&s_hist[keys[j]], 1u);
		}
	}
	__syncthreads();
	uint32_t *drow = digit_counts + (size_t)blockIdx.x * kDigits;
	if (TILES) {
		// thread i visits the tiles i + 512 k, which all have the low digit (tile id mod 128) i mod 128
		uint32_t dsum = 0u;
		for (uint32_t t = threadIdx.x; t < ntile; t += kBucketThreads) {
			const uint32_t c = s_hist[t];
			if (c) atomicAdd(&tile_totals[2 * (size_t)t], c);
			dsum += c;
		}
		atomicAdd(&s_digit[threadIdx.x & (kDigits - 1)], dsum);
		__syncthreads();
		if (threadIdx.x < kDigits) drow[threadIdx.x] = s_digit[threadIdx.x];
	} else {
		for (uint32_t d = threadIdx.x; d < (uint32_t)kDigits; d += kBucketThreads) drow[d] = s_hist[d];
	}
}

// The (partition x digit) matrix: 32 digits per CTA (one per lane: coalesced rows), the partitions split into 32 contiguous slices
// (one per warp).  Each warp sums its slice and the slice totals are scanned across the warps in shared memory: totals[d] = the
// digit's total, and the slice is rewritten as the exclusive prefix over the partitions.
__global__ void __launch_bounds__(1024) bucket_columns_kernel(uint32_t *__restrict__ counts, const uint32_t *__restrict__ first_p,
                                                             const uint32_t *__restrict__ last_p, uint32_t *__restrict__ totals) {
	__shared__ uint32_t s_tot[32][33];
	const uint32_t nparts = BucketSpan(first_p, last_p).parts();
	const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
	const uint32_t c = blockIdx.x * 32u + lane;
	const uint32_t per = (nparts + 31u) / 32u;
	const uint32_t p0 = min(w * per, nparts), p1 = min(p0 + per, nparts);
	uint32_t sum = 0u;
#pragma unroll 4
	for (uint32_t p = p0; p < p1; p++) sum += counts[(size_t)p * kDigits + c];
	s_tot[w][lane] = sum;
	__syncthreads();
	uint32_t run = 0u;
	for (uint32_t v = 0; v < w; v++) run += s_tot[v][lane];
	if (w == 31u) totals[c] = run + sum;
	for (uint32_t p = p0; p < p1; p++) {
		const uint32_t x = counts[(size_t)p * kDigits + c];
		counts[(size_t)p * kDigits + c] = run;
		run += x;
	}
}

// one CTA of 1024 threads: out[t] = (start, start + total(t)) from the exclusive scan of the tile totals, (0, 0) for a tile without
// instances.  Warp w owns tiles [512 w, 512 w + 512), read and written 32 consecutive tiles at a time; every total is read before
// any range is written, so `out` may be where the totals come from.
constexpr int kRangesPerLane = kBucketMaxTiles / (32 * 32);
template <typename Total>
__device__ __forceinline__ void scan_tile_ranges(const Total total, uint2 *out, const uint32_t ntile) {
	__shared__ uint32_t s_warp[32];
	const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
	const uint32_t seg = w * 32u * kRangesPerLane;
	uint32_t tot[kRangesPerLane], excl[kRangesPerLane];
#pragma unroll
	for (int j = 0; j < kRangesPerLane; j++) {
		const uint32_t t = seg + j * 32u + lane;
		tot[j] = t < ntile ? total(t) : 0u;
	}
	uint32_t carry = 0u;
#pragma unroll
	for (int j = 0; j < kRangesPerLane; j++) {
		uint32_t inc = tot[j];
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
			if (lane >= (uint32_t)o) inc += y;
		}
		excl[j] = carry + inc - tot[j];
		carry += __shfl_sync(0xffffffffu, inc, 31);
	}
	if (lane == 0) s_warp[w] = carry;
	__syncthreads();
	if (w == 0) {
		const uint32_t x = s_warp[lane];
		uint32_t inc = x;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
			if (lane >= (uint32_t)o) inc += y;
		}
		s_warp[lane] = inc - x;
	}
	__syncthreads();
	const uint32_t base = s_warp[w];
#pragma unroll
	for (int j = 0; j < kRangesPerLane; j++) {
		const uint32_t t = seg + j * 32u + lane;
		if (t < ntile) out[t] = tot[j] ? make_uint2(base + excl[j], base + excl[j] + tot[j]) : make_uint2(0u, 0u);
	}
}
// ranges[t] = its range, from the tile totals the histogram pass accumulated in ranges[t].y
struct BucketTotal {
	const uint2 *ranges;
	__device__ __forceinline__ uint32_t operator()(uint32_t t) const { return ranges[t].y; }
};
__global__ void __launch_bounds__(1024) bucket_ranges_kernel(uint2 *ranges, const uint32_t ntile) {
	scan_tile_ranges(BucketTotal{ranges}, ranges, ntile);
}

struct TileDigit {
	int shift;
	__device__ __forceinline__ uint32_t Digit(uint32_t key) const { return (key >> shift) & (kDigits - 1); }
};

// HIGH = false: (keys, vals) -> out by the low digit, out = Gaussian | high digit << 25; HIGH = true: (-, vals = those words) -> out
// = Gaussian by the high digit.
// prefix[p * 128 + d] = instances of digit d in the partitions before p; totals[d] = instances of digit d.
// A round is held warp-striped (warp w: instances base + 256 w + 32 j + lane), the order in which the match-based block rank
// counts, so the ranks are stable; the round is then staged in shared memory in digit order and written out in runs.
template <bool HIGH>
__global__ void __launch_bounds__(kPassThreads) bucket_pass_kernel(const uint16_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                                   const uint32_t *__restrict__ first_p, const uint32_t *__restrict__ last_p,
                                                                   const uint32_t *__restrict__ prefix,
                                                                   const uint32_t *__restrict__ totals, uint32_t *__restrict__ out) {
	constexpr int kShift = HIGH ? kDigitBits : 0;
	using Rank = cub::BlockRadixRankMatch<kPassThreads, kDigitBits, false>;
	__shared__ typename Rank::TempStorage tmp;
	__shared__ uint32_t s_vals[kPassRound];
	__shared__ uint16_t s_keys[kPassRound];
	__shared__ uint32_t s_cursor[kDigits];  // per digit: output position of the first instance of this round
	__shared__ uint32_t s_pref[kDigits];    // per digit: its first position in the round's digit order
	// The rounds start at the partition's first slot in [first, last): a slot loaded but not bucketed still takes a rank among its
	// digit and moves that digit's cursor, which is harmless only behind the last instance.
	const BucketSpan sp(HIGH ? nullptr : first_p, last_p);  // (the intermediate words start at 0)
	const uint32_t part_begin = sp.base + blockIdx.x * sp.part;
	const uint32_t begin = max(part_begin, sp.first);
	if (begin >= sp.end) return;
	const uint32_t end = min(part_begin + sp.part, sp.end);
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	if (threadIdx.x < 32) {  // digit starts (exclusive scan of the totals, 4 digits per lane) + this partition's prefix
		const uint4 t4 = reinterpret_cast<const uint4 *>(totals)[lane];
		const uint32_t sum = t4.x + t4.y + t4.z + t4.w;
		uint32_t inc = sum;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
			if (lane >= (uint32_t)o) inc += y;
		}
		const uint4 p4 = reinterpret_cast<const uint4 *>(prefix + (size_t)blockIdx.x * kDigits)[lane];
		uint32_t x = inc - sum;
		s_cursor[4 * lane + 0] = x + p4.x; x += t4.x;
		s_cursor[4 * lane + 1] = x + p4.y; x += t4.y;
		s_cursor[4 * lane + 2] = x + p4.z; x += t4.z;
		s_cursor[4 * lane + 3] = x + p4.w;
	}
	uint32_t k[kPassItems], v[kPassItems];
	// the round's instances, warp-striped; called for the next round as soon as this one is staged in shared memory, so that the
	// loads overlap the stores
	auto load = [&](const uint32_t base) {
#pragma unroll
		for (int j = 0; j < kPassItems; j++) {
			const uint32_t i = base + warp * (32u * kPassItems) + j * 32u + lane;
			const bool in = i < end;  // slots past the end: the largest digit, behind every real instance of it, written nowhere
			if (HIGH) {
				const uint32_t x = in ? vals[i] : 0u;
				k[j] = in ? (x >> kPackShift) << kDigitBits : 0xffffu;
				v[j] = in ? x & kPackMask : kNoGaussian;
			} else {
				k[j] = in ? (uint32_t)keys[i] : 0xffffu;
				v[j] = in ? vals[i] : kNoGaussian;
			}
		}
	};
	load(begin);
	for (uint32_t base = begin; base < end; base += kPassRound) {
		int rank[kPassItems];
		int pref[Rank::BINS_TRACKED_PER_THREAD];
		Rank(tmp).RankKeys(k, rank, TileDigit{kShift}, pref);
		if (threadIdx.x < kDigits) s_pref[threadIdx.x] = (uint32_t)pref[0];
#pragma unroll
		for (int j = 0; j < kPassItems; j++) {
			s_vals[rank[j]] = v[j];
			s_keys[rank[j]] = (uint16_t)k[j];
		}
		if (base + kPassRound < end) load(base + kPassRound);
		__syncthreads();
		// position q of the round's digit order holds the (q - pref[d])-th instance of digit d in this round
#pragma unroll
		for (int j = 0; j < kPassItems; j++) {
			const uint32_t q = j * kPassThreads + threadIdx.x;
			const uint32_t val = s_vals[q];
			if (val == kNoGaussian) continue;
			const uint32_t key = s_keys[q], d = (key >> kShift) & (kDigits - 1);
			const uint32_t pos = s_cursor[d] + q - s_pref[d];
			out[pos] = HIGH ? val : val | (key >> kDigitBits) << kPackShift;
		}
		__syncthreads();
		if (threadIdx.x < kDigits)
			s_cursor[threadIdx.x] += (threadIdx.x + 1 < kDigits ? s_pref[threadIdx.x + 1] : kPassRound) - s_pref[threadIdx.x];
		__syncthreads();
	}
}

// 16-bit tile ids, at most kBucketMaxTiles tiles and 2^25 Gaussians.  Buckets the instances [*first, *last) of (b.keys_in, b.vals_in)
// (first = nullptr: from 0) into b.vals_out[0, *last - *first) and `ranges`; n_mid = the number of instances, *last - *first, on the
// device.  The intermediate words live in keys_out, the count matrices and totals in the bucketing scratch.
static cudaError_t launch_bucketing(const BinView &b, uint2 *ranges, const uint32_t *first, const uint32_t *last, const uint32_t *n_mid,
                                   int ntile, int64_t slots, cudaStream_t st) {
	static std::atomic<uint64_t> smem_count{0};
	cudaError_t e;
	if ((e = ensure_dynamic_smem(bucket_count_kernel<true>, kBucketMaxTiles * sizeof(uint32_t), smem_count)) != cudaSuccess) return e;
	const BucketScratch sc = carve_bucket(b.bucket, slots);
	const unsigned nparts = bucket_grid(slots);
	const uint16_t *keys = reinterpret_cast<const uint16_t *>(b.keys_in);
	// the tile totals accumulate in ranges[t].y
	if ((e = cudaMemsetAsync(ranges, 0, (size_t)ntile * sizeof(uint2), st)) != cudaSuccess) return e;
	count_launch(7);
	bucket_count_kernel<true><<<nparts, kBucketThreads, (size_t)ntile * sizeof(uint32_t), st>>>(
		keys, first, last, (uint32_t)ntile, reinterpret_cast<uint32_t *>(ranges) + 1, sc.digit_counts[0]);
	bucket_ranges_kernel<<<1, 1024, 0, st>>>(ranges, (uint32_t)ntile);
	bucket_columns_kernel<<<kDigits / 32, 1024, 0, st>>>(sc.digit_counts[0], first, last, sc.digit_totals[0]);
	uint32_t *mid = b.keys_out;
	bucket_pass_kernel<false><<<nparts, kPassThreads, 0, st>>>(keys, b.vals_in, first, last, sc.digit_counts[0], sc.digit_totals[0], mid);
	bucket_count_kernel<false><<<nparts, kBucketThreads, kDigits * sizeof(uint32_t), st>>>(reinterpret_cast<const uint16_t *>(mid), nullptr,
	                                                                                     n_mid, 0u, nullptr, sc.digit_counts[1]);
	bucket_columns_kernel<<<kDigits / 32, 1024, 0, st>>>(sc.digit_counts[1], nullptr, n_mid, sc.digit_totals[1]);
	bucket_pass_kernel<true><<<nparts, kPassThreads, 0, st>>>(nullptr, mid, nullptr, n_mid, sc.digit_counts[1], sc.digit_totals[1], b.vals_out);
	return cudaGetLastError();
}

cudaError_t launch_binning(const FrameDev &f, GeomView g, const int32_t *radii, BinView b, ImgView img, int64_t R, cudaStream_t st,
                           int64_t cap, int n_order) {
	if (n_order < 0) n_order = f.P;
	const int ntile = f.gx * f.gy;
	const bool bounded = cap >= 0;
	cudaError_t e = cudaMemsetAsync(img.ranges, 0, (size_t)ntile * sizeof(uint2), st);
	if (e != cudaSuccess) return e;
	if (f.P == 0) return cudaSuccess;
	const uint32_t cap32 = bounded ? (uint32_t)cap : 0xffffffffu;
	count_launch();
	count_status_kernel<<<1, 1, 0, st>>>(g.offsets, n_order, cap32, g.big_count);
	if ((e = cudaGetLastError()) != cudaSuccess) return e;
	if (bounded) R = cap;  // every pass below runs over the caller's capacity; the padding carries the largest key
	if (R == 0) return cudaSuccess;
	if ((e = cudaMemsetAsync(g.big_count, 0, sizeof(uint32_t), st)) != cudaSuccess) return e;
	if (tile_key_bytes(ntile, bounded) == 2) {
		if ((e = launch_emit<uint16_t>(f, g, radii, b, g.offsets, g.big_count, cap32, n_order, st)) != cudaSuccess) return e;
		if (bucketable(f)) return launch_bucketing(b, img.ranges, nullptr, g.big_count + 3, g.big_count + 3, ntile, R, st);
		return launch_tile_sort<uint16_t>(b, img, g.big_count, ntile, R, bounded, st);
	}
	if ((e = launch_emit<uint32_t>(f, g, radii, b, g.offsets, g.big_count, cap32, n_order, st)) != cudaSuccess) return e;
	return launch_tile_sort<uint32_t>(b, img, g.big_count, ntile, R, bounded, st);
}

// ---- saturation split: near pass, blend, far pass (include/sgr.h sgr_set_near_budget, DESIGN.md §7) ----
// Most instances of a frame lie behind the point where every pixel of their tile has saturated (T < 1e-4): the blend never reads
// them.  The split emits and buckets the nearest Gaussians first (those whose depth-order offsets stay within the budget B), blends
// those lists (blend_fwd.cu, kBlendNear), and emits the remaining Gaussians only into the tiles that pass left unsaturated.  The
// emitted sequence is near ++ far, both in depth order, and the bucketing is stable, so a tile's list is its near list followed by
// its far list: the far pass buckets the far instances alone and splices each tile's two lists.  Every unsaturated tile then has
// exactly the list of the unsplit binning and every saturated tile its near part; kBlendResume finishes the unsaturated tiles from
// the stored per-pixel state.  Images, n_contrib and tile_max_contrib do not depend on B.
// Buffers: the emitted sequence is [0, E) of (keys_in, vals_in), as in the unsplit binning.  The near lists are bucketed through
// vals_out into keys_out (split_near_lists), the far lists through vals_out into sort_temp (a bucketed frame never sorts, and
// carve_bin sizes it for that), and the splice writes vals_out.

// one thread: the split.  fit = Gaussians whose whole instance counts fit the capacity (all unless the bounded mode can overflow);
// B = the budget (budget < 0: R / kNearBudgetDivisor), clamped to what fits; K = Gaussians whose inclusive offset is <= B.  The near
// block's word 3 = its end in the emitted sequence, as the bucketing reads it.  Words 2 and 3 are settled by split_total_kernel.
__global__ void split_status_kernel(const uint32_t *__restrict__ offsets, int n, uint32_t cap, long long budget, uint32_t *__restrict__ status) {
	const uint32_t R = offsets[n - 1];
	const int fit = R > cap ? slots_within(offsets, n, cap) : n;
	const uint32_t fit_end = fit == 0 ? 0u : offsets[fit - 1];
	uint32_t B = budget < 0 ? R / kNearBudgetDivisor : (uint32_t)min(budget, 0xffffffffll);
	B = min(B, fit_end);
	const int K = slots_within(offsets, fit, B);
	status[1] = R;
	status[kStatusNear] = 0u;
	status[kStatusNear + 3] = K == 0 ? 0u : offsets[K - 1];
	status[kStatusSplitK] = (uint32_t)K;
	status[kStatusSplitFit] = (uint32_t)fit;
}

// thread t = t-th Gaussian in depth order: its instance count in the emitted sequence.  Near Gaussians keep their scanned count;
// a far one counts the tiles of its rectangle that the near blend left unsaturated, by the code emit_pairs / emit_big run.  Every
// row span of that walk lies inside the rectangle, so a rectangle without an unsaturated tile (four table loads) counts 0 without it:
// on config C almost every tile saturates in the near slab, and most far Gaussians stop there.  When no tile is left unsaturated
// (the table's last entry is 0), no far Gaussian is gathered at all.
__global__ void __launch_bounds__(256) far_count_kernel(const FrameDev f, const GaussRec *__restrict__ rec, const int32_t *__restrict__ radii,
                                                       const uint32_t *__restrict__ perm, const uint32_t *__restrict__ offsets,
                                                       const uint32_t *__restrict__ status, const int n_order,
                                                       const KeepUnsaturated keep, uint32_t *__restrict__ cnt) {
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	const int K = (int)status[kStatusSplitK];
	const bool any = keep.sat[(size_t)f.gy * keep.stride + f.gx] != 0u;
	bool active = false;
	int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
	CullParams cp = {};
	uint32_t c = 0u;
	if (t < n_order) {
		const uint32_t off = t == 0 ? 0u : offsets[t - 1], end = offsets[t];
		if (t < K) {
			c = end - off;
		} else if (any && end > off) {
			const uint32_t gidx = perm[t];
			const float4 q0 = rec[gidx].q0;
			tile_rect(q0.x, q0.y, radii[gidx], f.gx, f.gy, x0, y0, x1, y1);
			if (x1 > x0 && y1 > y0 && keep.rect(y0, y1, x0, x1) != 0u) {
				const float4 q1 = rec[gidx].q1;
				cp = make_cull(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y);
				active = true;
			}
		}
	}
	uint32_t count = 0u;
	visit_tiles<false, uint16_t, KeepUnsaturated>(active, x0, y0, x1, y1, cp, f.band, f.gx, 0u, 0u, nullptr, nullptr, count, nullptr, nullptr,
	                                              0u, 0u, 0u, nullptr, nullptr, 0u, keep);
	if (t < n_order) cnt[t] = active ? count : c;
}

// one CTA, after the near blend: the table of KeepUnsaturated, sat[y * (gx + 1) + x] = unsaturated tiles (top bit of
// tile_max_contrib) in rows < y and columns < x.  The warps prefix the tile rows, then the threads the columns.  sat lives in the img
// state's split table: (gx + 1)(gy + 1) <= 2 gx gy + 2 words.
constexpr int kSatBatch = 16;  // rows loaded ahead by each column thread
__global__ void __launch_bounds__(1024) unsat_prefix_kernel(const uint32_t *__restrict__ tile_word, const int gx, const int gy, uint32_t *sat) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int stride = gx + 1;
	for (int x = threadIdx.x; x < stride; x += blockDim.x) sat[x] = 0u;
	for (int ty = warp; ty < gy; ty += 32) {
		uint32_t *row = sat + (size_t)(ty + 1) * stride;
		if (lane == 0) row[0] = 0u;
		uint32_t carry = 0u;
		for (int t0 = 0; t0 < gx; t0 += 32) {
			const int tx = t0 + lane;
			const bool u = tx < gx && (tile_word[(size_t)ty * gx + tx] >> 31) != 0u;
			const unsigned m = __ballot_sync(0xffffffffu, u);
			if (tx < gx) row[tx + 1] = carry + (uint32_t)__popc(m & (0xffffffffu >> (31 - lane)));
			carry += (uint32_t)__popc(m);
		}
	}
	__syncthreads();  // (also orders the rows' global stores before the column pass reads them)
	for (int x = threadIdx.x; x < stride; x += blockDim.x) {
		uint32_t run = 0u;
		for (int y0 = 1; y0 <= gy; y0 += kSatBatch) {
			uint32_t v[kSatBatch];
#pragma unroll
			for (int j = 0; j < kSatBatch; j++) v[j] = y0 + j <= gy ? sat[(size_t)(y0 + j) * stride + x] : 0u;
#pragma unroll
			for (int j = 0; j < kSatBatch; j++) {
				run += v[j];
				if (y0 + j <= gy) sat[(size_t)(y0 + j) * stride + x] = run;
			}
		}
	}
}

// one thread, after the scan of far_count_kernel's counts: E = the instances emitted, E_far = E - E_near.  A bounded frame overflows
// only if the emitted sequence exceeds the capacity; it then keeps the Gaussians whose whole instance counts fit (split_status_kernel's
// `fit`), as the one-pass binning does, so that an overflowing frame is the same whatever the budget.  The far emission reads E as its
// cap; the far bucketing covers [E_near, E) and its second digit pass the E_far words of the first.
__global__ void split_total_kernel(const uint32_t *__restrict__ offsets, int n, uint32_t cap, uint32_t *__restrict__ status) {
	const uint32_t total = offsets[n - 1];
	uint32_t E = total;
	if (total > cap) {
		const int fit = (int)status[kStatusSplitFit];
		E = fit == 0 ? 0u : offsets[fit - 1];
		status[2] |= 1u;
	}
	status[3] = E;
	status[kStatusFarEnd] = E - status[kStatusNear + 3];
}

// a tile's spliced list: its near list followed by its far list
struct SplicedTotal {
	const uint2 *near, *far;
	__device__ __forceinline__ uint32_t operator()(uint32_t t) const {
		const uint2 a = near[t], b = far[t];
		return (a.y - a.x) + (b.y - b.x);
	}
};
__global__ void __launch_bounds__(1024) splice_ranges_kernel(const uint2 *__restrict__ near, const uint2 *__restrict__ far, uint2 *__restrict__ out,
                                                            const uint32_t ntile) {
	scan_tile_ranges(SplicedTotal{near, far}, out, ntile);
}
// one warp per tile: its near list, then its far list, copied to the spliced range; the spliced range then replaces the near one
constexpr int kSpliceWarps = 8;
__global__ void __launch_bounds__(32 * kSpliceWarps) splice_lists_kernel(uint2 *ranges, const uint2 *__restrict__ far_ranges,
                                                                         const uint2 *__restrict__ spliced, const uint32_t *__restrict__ near_lists,
                                                                         const uint32_t *__restrict__ far_lists, uint32_t *__restrict__ out,
                                                                         const uint32_t ntile) {
	const uint32_t t = blockIdx.x * kSpliceWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
	if (t >= ntile) return;
	const uint2 nr = ranges[t], fr = far_ranges[t], sr = spliced[t];
	const uint32_t nn = nr.y - nr.x, nf = fr.y - fr.x;
	for (uint32_t i = lane; i < nn; i += 32u) out[sr.x + i] = near_lists[nr.x + i];
	for (uint32_t i = lane; i < nf; i += 32u) out[sr.x + nn + i] = far_lists[fr.x + i];
	__syncwarp();  // (every lane has read ranges[t])
	if (lane == 0) ranges[t] = sr;
}

bool split_applies(const FrameDev &f, int64_t R, int64_t budget, bool from_records) {
	const bool whole_image = f.band.begin == 0 && f.band.end == f.gy && f.band.step == 1;
	return !from_records && f.P > 0 && R > 0 && (budget < 0 || budget < R) && f.S == 0 && whole_image && bucketable(f);
}

// near pass: split, emit the Gaussians before it into [0, E_near), bucket them into keys_out (split_near_lists) / ranges.
// slots = binning capacity.
cudaError_t launch_near_binning(const FrameDev &f, GeomView g, const int32_t *radii, BinView b, ImgView img, int64_t slots, cudaStream_t st,
                                int64_t cap, int n_order, int64_t budget) {
	const uint32_t cap32 = cap >= 0 ? (uint32_t)cap : 0xffffffffu;
	uint32_t *near = g.big_count + kStatusNear;
	count_launch();
	split_status_kernel<<<1, 1, 0, st>>>(g.offsets, n_order, cap32, (long long)budget, g.big_count);
	cudaError_t e = launch_emit<uint16_t>(f, g, radii, b, g.offsets, near, cap32, n_order, st, near + 3);
	if (e != cudaSuccess) return e;
	BinView nb = split_near_lists(b);
	nb.keys_out = b.vals_out;  // (the intermediate words)
	return launch_bucketing(nb, img.ranges, nullptr, near + 3, near + 3, f.gx * f.gy, slots, st);
}

// far pass, after the near blend marked the unsaturated tiles: count, scan (into g.ckey; g.iota holds the counts — both are dead
// after the depth sort of this forward), emit behind the near instances, bucket [E_near, E) alone into sort_temp / img.far_ranges,
// and splice the near and far lists into vals_out / ranges.
cudaError_t launch_far_binning(const FrameDev &f, GeomView g, const int32_t *radii, BinView b, ImgView img, int64_t slots, cudaStream_t st,
                               int64_t cap, int n_order) {
	const uint32_t cap32 = cap >= 0 ? (uint32_t)cap : 0xffffffffu;
	const int ntile = f.gx * f.gy;
	const unsigned nblk = (unsigned)((n_order + 255) / 256);
	uint32_t *sat = reinterpret_cast<uint32_t *>(img.split);  // (gx + 1)(gy + 1) <= 2 (ntile + 1) words
	const KeepUnsaturated keep{sat, f.gx + 1};
	uint32_t *far_offsets = g.ckey;
	uint32_t *status = g.big_count, *near_end = g.big_count + kStatusNear + 3;
	count_launch(2);
	unsat_prefix_kernel<<<1, 1024, 0, st>>>(img.tile_max_contrib, f.gx, f.gy, sat);
	far_count_kernel<<<nblk, 256, 0, st>>>(f, g.rec, radii, g.perm, g.offsets, status, n_order, keep, g.iota);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return e;
	size_t bytes = g.temp_bytes;
	if ((e = cub::DeviceScan::InclusiveSum(g.temp, bytes, g.iota, far_offsets, n_order, st)) != cudaSuccess) return e;
	if ((e = cudaMemsetAsync(status, 0, sizeof(uint32_t), st)) != cudaSuccess) return e;
	count_launch();
	split_total_kernel<<<1, 1, 0, st>>>(far_offsets, n_order, cap32, status);
	if ((e = launch_emit<uint16_t>(f, g, radii, b, far_offsets, status, cap32, n_order, st, status + 3, near_end, keep)) != cudaSuccess) return e;
	BinView fb = b;
	fb.keys_out = b.vals_out;  // (the intermediate words)
	fb.vals_out = reinterpret_cast<uint32_t *>(b.sort_temp);
	if ((e = launch_bucketing(fb, img.far_ranges, near_end, status + 3, status + kStatusFarEnd, ntile, slots, st)) != cudaSuccess) return e;
	count_launch(2);
	splice_ranges_kernel<<<1, 1024, 0, st>>>(img.ranges, img.far_ranges, img.split, (uint32_t)ntile);
	splice_lists_kernel<<<(unsigned)((ntile + kSpliceWarps - 1) / kSpliceWarps), 32 * kSpliceWarps, 0, st>>>(
		img.ranges, img.far_ranges, img.split, split_near_lists(b).vals_out, fb.vals_out, b.vals_out, (uint32_t)ntile);
	return cudaGetLastError();
}

}  // namespace sgr
