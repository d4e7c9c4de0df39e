// sgr_common.cuh — shared device helpers, state layout and the exact tile-cull test.
//
// The caller-owned states (include/sgr.h) are carved by carve_geom / carve_img / carve_bin (capi.cu) into the views below;
// sgr_state_layout reports the carved offsets.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include "../../include/sgr.h"

#define SGR_TILE 16            // tile edge in pixels (reference BLOCK_X = BLOCK_Y = 16, DGR/cuda_rasterizer/config.h:17-18)
#define SGR_TILE_PIX 256
#define SGR_ALIGN 256

namespace sgr {

// Streaming multiprocessors of the target GPU (H100 SXM: 132); sizes the persistent-style grids of grid-stride kernels.
constexpr unsigned kNumSMs = 132;

// 48-byte per-Gaussian record written by preprocess_fwd and gathered by both blend passes.
//   q0 = (pix.x, pix.y, conic.xx, conic.xy)   q1 = (conic.yy, opacity, power_min, view depth)   q2 = (r, g, b, bits(clamped))
// power_min = -qmax/2 (conservative): a pair with power < power_min cannot reach alpha >= 1/255, so the blend loops skip
// it before evaluating expf; pairs that pass still take the reference's exact alpha test.
struct __align__(16) GaussRec {
	float4 q0, q1, q2;
};

struct GeomView {
	GaussRec *rec;
	uint32_t *tiles_touched;  // per Gaussian (original order): number of (tile) instances it emits
	uint32_t *depth_key;      // per Gaussian: float bits of the view depth, 0xFFFFFFFF if it emits nothing
	uint32_t *iota;           // 0..P-1 (values fed to the depth sort)
	uint32_t *depth_sorted;   // sorted depth keys (scratch)
	uint32_t *perm;           // Gaussian indices in ascending (depth, index) order
	uint32_t *offsets;        // inclusive scan of tiles_touched[perm[.]]  (depth order)
	uint32_t *big_list;       // depth-order positions of Gaussians whose rectangle is emitted by a whole warp (emit_big_kernel)
	uint32_t *big_count;      // status words, zeroed per forward: [0] number of entries in big_list (device counter)
	                          // [1] instance count R, [2] overflow bits (1 = instance capacity, 2 = Gaussian capacity of the compacted
	                          // depth order), [3] instances actually emitted (bounded mode), [4] Gaussians with instances (compacted mode)
	                          // [8..14] saturation split (kStatusNear ...); include/sgr.h names them SGR_STATUS_*
	float4 *jac;              // per Gaussian with SH colour: 3 float4, d colour / d view direction + clamp bits (gaussian_geom.cuh)
	uint32_t *ckey, *cval;    // compacted depth-sort input (keys / Gaussian indices), Gaussian-sharded forward only; the saturation
	                          // split's far offsets live in ckey (and its far counts in iota, dead after the depth sort)
	void *temp;               // cub temp storage: max(scan, depth sort)
	size_t temp_bytes;
	size_t total_bytes;
};
struct ImgView {
	uint2 *ranges;
	uint32_t *n_contrib;
	uint32_t *tile_max_contrib;
	float *blend_T;  // saturation split: T of each pixel of an unsaturated tile between the near blend and its resumption (sign = done)
	// saturation split (forward img states only, like blend_T; ntile + 1 entries each): far_ranges = the per-tile ranges of the far
	// lists; split = the unsaturated-tile table of the far pass (KeepUnsaturated), then the spliced ranges until they replace `ranges`
	uint2 *far_ranges, *split;
	size_t total_bytes;
};

// Saturation split (binning.cu launch_near_binning / launch_far_binning, blend_fwd.cu kBlendNear / kBlendResume): status words
// kStatusNear.. = the near pass's block as the emission and bucketing read it ([+0] its big-list counter, [+3] its end E_near in the
// emitted sequence); kStatusSplitK = Gaussians of the near pass (depth order), kStatusSplitFit = Gaussians that fit the capacity;
// kStatusFarEnd = instances the far pass emitted (the emitted sequence is E_near + that).
constexpr int kStatusNear = SGR_STATUS_NEAR, kStatusSplitK = SGR_STATUS_SPLIT_K, kStatusSplitFit = SGR_STATUS_SPLIT_FIT,
              kStatusFarEnd = SGR_STATUS_FAR_END;
// the near budget when the caller sets none: R / kNearBudgetDivisor instances (DESIGN.md §7, sweep on config C)
constexpr uint32_t kNearBudgetDivisor = 8;
enum BlendPass { kBlendFull = 0, kBlendNear = 1, kBlendResume = 2 };
struct BinView {
	uint32_t *keys_in, *keys_out;  // tile ids
	uint32_t *vals_in, *vals_out;  // Gaussian indices; vals_out is the tile-ordered, depth-sorted point list
	void *sort_temp;  // cub temp of the tile radix sort; in a bucketed frame the far lists of the saturation split (>= 4 B per slot)
	size_t sort_temp_bytes;
	void *bucket;  // tile-bucketing scratch (binning.cu carve_bucket): count matrices, digit totals
	size_t bucket_bytes;
	size_t total_bytes;
};
// The near pass of the saturation split leaves its per-tile lists in keys_out (vals_out receives the spliced lists of the far pass):
// the view the near blend reads them through.
static inline BinView split_near_lists(BinView b) {
	b.vals_out = b.keys_out;
	return b;
}

static inline size_t align_up(size_t v, size_t a = SGR_ALIGN) { return (v + a - 1) / a * a; }
// Bytes per tile id in keys_in: 16-bit ids whenever every tile id fits below the bounded mode's padding key 0xFFFF (or, in the exact
// mode, which pads nothing, fits at all); the key arrays are allocated for 32-bit ids either way.
static inline int tile_key_bytes(int ntile, bool bounded) { return ntile <= 65535 || (!bounded && ntile <= 65536) ? 2 : 4; }

// Number of kernels of THIS library enqueued so far by the process (cub's internal kernels are not counted); read through
// sgr_launch_count() — bench.py reports the delta over its timed region as `gpu_launches`.
extern std::atomic<uint64_t> g_kernel_launches;
static inline void count_launch(unsigned n = 1) { g_kernel_launches.fetch_add(n, std::memory_order_relaxed); }

// cudaFuncAttributeMaxDynamicSharedMemorySize is per (function, device).  `done` holds one bit per device ordinal; the
// check-then-set is idempotent (two threads racing both set the same attribute to the same value), and the bit is published
// with release/acquire ordering, so the library stays thread-safe without a lock.
template <typename K>
static inline cudaError_t ensure_dynamic_smem(K kernel, int bytes, std::atomic<uint64_t> &done) {
	int dev = 0;
	cudaError_t e = cudaGetDevice(&dev);
	if (e != cudaSuccess) return e;
	const bool tracked = dev >= 0 && dev < 64;
	if (tracked && ((done.load(std::memory_order_acquire) >> dev) & 1ull)) return cudaSuccess;
	e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
	if (e == cudaSuccess && tracked) done.fetch_or(1ull << dev, std::memory_order_release);
	return e;
}

// Column-major 3x3 (m[c][r]) with the product written as a left-associated sum of three products.  The reference
// uses glm::mat3, whose operator* has this exact algebraic form; keeping the form lets nvcc contract mul+add
// pairs identically so that depth / conic / radius come out bit-equal to the reference's (SURVEY.md §7
// "Bit-level parity traps").
struct M3 {
	float m[3][3];
};
__device__ __forceinline__ M3 m3_mul(const M3 &a, const M3 &b) {
	M3 r;
#pragma unroll
	for (int c = 0; c < 3; c++)
#pragma unroll
		for (int i = 0; i < 3; i++) r.m[c][i] = a.m[0][i] * b.m[c][0] + a.m[1][i] * b.m[c][1] + a.m[2][i] * b.m[c][2];
	return r;
}
// Rotation matrix of the raw (not normalised) quaternion q = (r, x, y, z), column-major like the reference's glm::mat3
// (forward.cu:130-134 / backward.cu).  Which product of each two-product sum is fused into the add and which is rounded first
// is spelled out: the reference's build fuses x*y, x*x, y*z and r*y and rounds the other product, and leaving that choice to
// ptxas does not reproduce it on every architecture (sm_90 fused x*z instead of r*y), which moved the conic of near-degenerate
// splats by hundreds of ulps.  The forward and the backward share this so that the backward's recomputed cov3D is the forward's.
__device__ __forceinline__ M3 quat_rot_colmajor(const float4 q) {
	const float r = q.x, x = q.y, y = q.z, z = q.w;
	M3 R;
	R.m[0][0] = 1.f - 2.f * __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z));
	R.m[0][1] = 2.f * __fmaf_rn(x, y, -__fmul_rn(r, z));
	R.m[0][2] = 2.f * __fmaf_rn(r, y, __fmul_rn(x, z));
	R.m[1][0] = 2.f * __fmaf_rn(x, y, __fmul_rn(r, z));
	R.m[1][1] = 1.f - 2.f * __fmaf_rn(x, x, __fmul_rn(z, z));
	R.m[1][2] = 2.f * __fmaf_rn(y, z, -__fmul_rn(r, x));
	R.m[2][0] = 2.f * __fmaf_rn(-r, y, __fmul_rn(x, z));
	R.m[2][1] = 2.f * __fmaf_rn(y, z, __fmul_rn(r, x));
	R.m[2][2] = 1.f - 2.f * __fmaf_rn(x, x, __fmul_rn(y, y));
	return R;
}
__device__ __forceinline__ M3 m3_t(const M3 &a) {
	M3 r;
#pragma unroll
	for (int c = 0; c < 3; c++)
#pragma unroll
		for (int i = 0; i < 3; i++) r.m[c][i] = a.m[i][c];
	return r;
}

// Column-major affine / projective point transforms (reference: transformPoint4x3 / 4x4, auxiliary.h:58-77).
__device__ __forceinline__ float3 xform4x3(const float3 p, const float *__restrict__ m) {
	return make_float3(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12], m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
	                   m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14]);
}
__device__ __forceinline__ float4 xform4x4(const float3 p, const float *__restrict__ m) {
	return make_float4(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12], m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
	                   m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14], m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15]);
}

// NDC -> pixel.  The reference writes the constants as double literals (auxiliary.h:41-44), i.e. fp64 arithmetic.
__device__ __forceinline__ float ndc2pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

// 3-sigma tile rectangle, truncating toward zero before the clamp exactly like auxiliary.h:46-56.
__device__ __forceinline__ void tile_rect(float px, float py, int radius, int gx, int gy, int &x0, int &y0, int &x1, int &y1) {
	x0 = min(gx, max(0, (int)((px - radius) / SGR_TILE)));
	y0 = min(gy, max(0, (int)((py - radius) / SGR_TILE)));
	x1 = min(gx, max(0, (int)((px + radius + SGR_TILE - 1) / SGR_TILE)));
	y1 = min(gy, max(0, (int)((py + radius + SGR_TILE - 1) / SGR_TILE)));
}

// Which tile rows does this process own (multi-GPU tile-row sharding)?
struct Band {
	int begin, end, step;
};
__host__ __device__ __forceinline__ bool band_owns(const Band b, int row) {
	return row >= b.begin && row < b.end && ((row - b.begin) % b.step) == 0;
}
// dense index of an owned row within the band (used to launch one CTA per owned tile)
__host__ __device__ __forceinline__ int band_rows(const Band b) { return b.end > b.begin ? (b.end - b.begin + b.step - 1) / b.step : 0; }
// Item t of the band's pixels in a [H, W] plane, the band_rows(b) * strip items of its tile rows in order (strip = the items of one
// 16-row tile row): its index in the frame.  Items of the last tile row past the image's last row map to indices >= H W.
constexpr int kBandTileRows = 16;
__host__ __device__ __forceinline__ int64_t band_pixel(const int64_t t, const Band b, const int64_t strip) {
	const int64_t k = t / strip;
	return (int64_t)(b.begin + (int)k * b.step) * strip + (t - k * strip);
}

// ---- TMA bulk copies (cp.async.bulk, 1-D) + mbarrier: the Hopper (sm_90) way to move a contiguous row block between HBM and
// shared memory without a register round trip.  SASS: UBLKCP (copy), SYNCS.ARRIVE.TRANS64 (expect_tx), SYNCS.PHASECHK (try_wait).
// Size and both addresses must be multiples of 16 bytes.
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
	asm volatile(
	    "{\n"
	    ".reg .pred p;\n"
	    "WAIT_%=:\n"
	    "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
	    "@p bra DONE_%=;\n"
	    "bra WAIT_%=;\n"
	    "DONE_%=:\n"
	    "}\n" ::"r"(bar),
	    "r"(parity)
	    : "memory");
}
// generic-proxy writes to shared memory (mbarrier.init, st.shared) must be made visible to the async proxy (TMA) and vice versa
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void *src_gmem, uint32_t bytes, uint32_t bar) {
	asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem), "l"(src_gmem), "r"(bytes),
	             "r"(bar)
	             : "memory");
}
__device__ __forceinline__ void bulk_s2g(void *dst_gmem, uint32_t src_smem, uint32_t bytes) {
	asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(src_smem), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// ---- exact, opacity-aware tile culling -------------------------------------------------------------------------
// A (Gaussian, tile) pair of the reference's 3-sigma rectangle can be dropped without changing ANY output iff no pixel
// of the tile passes the reference's two per-pixel tests (forward.cu:420-430):  power <= 0  and  o*exp(power) >= 1/255.
// With q(d) = a dx^2 + 2b dx dy + c dy^2 = -2*power this is  q <= 2*ln(255*o) =: qmax, i.e. the pixel lies inside an
// ellipse.  tile_visit.cuh intersects that ellipse with each tile row in closed form.  Everything is evaluated
// conservatively ("keep" on NaN / non-PD input), with two slacks on qmax:
//   0.02 + 1e-3 |tau|        the approximate log and the culling's own fast division / square root;
//   2^-17 (a c / det) |2 tau| the fp32 rounding of `power` itself.  The reference sums terms of magnitude up to
//                            |a| dx^2 + |c| dy^2 + 2 |b dx dy| <= 4 (a c / det) q on the ellipse, with ~6 roundings, and det = a c - b^2
//                            cancels by the same ratio.  For a thin diagonal splat (conic condition number kappa, a c / det ~ kappa / 4)
//                            that error is ~1e-2 q at kappa = 1e5 and comparable to q at kappa = 1e6, far above the constant slack:
//                            without this term tiles holding pairs the reference blends were dropped.  Round or axis-aligned splats
//                            (a c / det ~ 1) are not affected.
// So a dropped tile receives nothing from any fp32 evaluation of the reference's expression within those rounding bounds.
struct CullParams {
	float mx, my, a, b, c, qmax;  // qmax < 0 => nothing can pass; qmax = +inf => keep all of the rectangle
};
__device__ __forceinline__ CullParams make_cull(float mx, float my, float a, float b, float c, float opacity) {
	CullParams cp{mx, my, a, b, c, __int_as_float(0x7f800000)};
	const float det = a * c - b * b;
	const bool pd = (a > 0.f) && (c > 0.f) && (det > 0.f);
	const float tau = __logf(255.0f * opacity);  // (approximate log: the slack below dwarfs its error) NaN for negative / NaN opacity -> keep
	if (pd && tau == tau) {
		const float ratio = __fdividef(a * c, det);  // >= 1
		cp.qmax = 2.0f * tau + (0.02f + 1e-3f * fabsf(tau)) + 0x1p-17f * ratio * fabsf(2.0f * tau);
	}
	return cp;
}
// state carving (host) — implemented in capi.cu
GeomView carve_geom(void *base, int P);
ImgView carve_img(void *base, int W, int H, bool blend_state = true);
BinView carve_bin(void *base, int64_t R);

// kernel launchers (host) — one per translation unit
struct FrameDev {  // SgrFrame + derived values, passed by value to kernels
	int P, D, M, S, W, H, gx, gy;
	float tanx, tany, fx, fy, mod;
	Band band;
	const float *bg, *view, *proj, *campos;
};

cudaError_t launch_preprocess_fwd(const FrameDev &f, const float *means3D, const float *shs, const float *colors_precomp,
                                  const float *opacities, const float *scales, const float *rotations,
                                  const float *cov3D_precomp, int32_t *radii, GeomView g, cudaStream_t st);
// records + radii only (no tile counts): step 1 of the Gaussian-sharded forward
cudaError_t launch_project(const FrameDev &f, const float *means3D, const float *shs, const float *colors_precomp,
                           const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp,
                           int32_t *radii, GaussRec *rec, float4 *jac, cudaStream_t st);
cudaError_t launch_filter(const FrameDev &f, const float *means3D, const float *scales, const float *rotations,
                          const float *cov3D_precomp, int32_t *radii, float *means2D, cudaStream_t st);
cudaError_t launch_mark_visible(int P, const float *means3D, const float *view, uint8_t *present, cudaStream_t st);
cudaError_t launch_depth_order(const FrameDev &f, GeomView g, cudaStream_t st);
// fused Gaussian-sharded forward: tile counts + depth order of the runs delivered to this rank (binning.cu)
cudaError_t launch_count_and_order_runs(const FrameDev &f, GeomView g, int32_t *radii, int world, long long chunk, cudaStream_t st, int64_t cap_v,
                                        float *zero_rows, int *n_order);
// Gaussian-sharded exchange over peer memory (peer_exchange.cu); device copy of include/sgr.h's SgrPeers
constexpr int kMaxPeers = 16;
struct PeerTable {
	int world, rank;
	long long chunk;
	GaussRec *rec[kMaxPeers];
	int32_t *radii[kMaxPeers];
	const float *grad2d[kMaxPeers];
	uint32_t *flags[kMaxPeers];  // rank p's barrier pad: u32[kMaxPeers], slot q = last epoch at which rank q arrived
};
// ranks whose cyclic band (row r -> rank r % world) meets tile rows [y0, y1)
__device__ __forceinline__ uint32_t touched_ranks(int y0, int y1, int world) {
	if (y1 <= y0) return 0u;
	if (y1 - y0 >= world) return world >= 32 ? 0xffffffffu : ((1u << world) - 1u);
	uint32_t m = 0u;
	for (int y = y0; y < y1; y++) m |= 1u << (y % world);
	return m;
}
// ---- block-run exchange of the fused Gaussian-sharded step (sgr_sharded_forward / sgr_sharded_backward) -------------------------------
// The 256 consecutive Gaussians of one thread block that go to rank d are delivered as ONE contiguous run: block b of owner s owns the
// 256 slots [s*chunk + b*256, +256) of every rank's gathered arrays and fills the first c(s, b, d) of them on rank d, in ascending
// Gaussian order.  Ascending slot order therefore equals ascending global-id order (the tie order of the depth sort on one GPU), the
// records of a run leave the SM as whole 128-B lines (48-B records stored one by one fill only part of an NVLink packet
// each, and the barrier after them waits for those posted writes to drain), and in the backward the owner reads its rows back as the same runs.
// The radius travels in the record (q2.w = radius << 3 | colour-clamp bits); no per-Gaussian array is indexed by the global id.
constexpr int kRunBlock = 256;
__device__ __forceinline__ float pack_radius_clamp(int radius, uint32_t clamp_bits) { return __uint_as_float(((uint32_t)radius << 3) | (clamp_bits & 7u)); }
__device__ __forceinline__ int packed_radius(float w) { return (int)(__float_as_uint(w) >> 3); }
struct RunScratch {
	uint32_t wcnt[8][kMaxPeers];   // per warp, per destination: hits of the lower warps (exclusive prefix after block_run_ranks)
	uint32_t cpre[kMaxPeers + 1];  // per destination: first position of its run in the block's concatenated run list; [world] = total
};
// Collective over the 256 threads of a block (every thread calls it, `mask` = destinations of this thread's Gaussian, 0 if none).
// Afterwards the position of this thread's record in destination d's run is  run_rank(rs, mask, d).
__device__ __forceinline__ void block_run_ranks(RunScratch &rs, uint32_t mask, int world) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (int d = 0; d < world; d++) {
		const unsigned b = __ballot_sync(0xffffffffu, (mask >> d) & 1u);
		if (lane == 0) rs.wcnt[warp][d] = (uint32_t)__popc(b);
	}
	__syncthreads();
	if (warp == 0) {  // lane d: exclusive prefix of destination d's hits over the 8 warps, then (shuffles) over the destinations
		uint32_t run = 0u;
		if (lane < world) {
			for (int w = 0; w < 8; w++) {
				const uint32_t t = rs.wcnt[w][lane];
				rs.wcnt[w][lane] = run;
				run += t;
			}
		}
		uint32_t incl = run;
#pragma unroll
		for (int o = 1; o < kMaxPeers; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= o) incl += t;
		}
		if (lane < world) rs.cpre[lane + 1] = incl;
		if (lane == 0) rs.cpre[0] = 0u;
	}
	__syncthreads();
}
__device__ __forceinline__ uint32_t run_rank(const RunScratch &rs, uint32_t mask, int d) {
	const unsigned b = __ballot_sync(0xffffffffu, (mask >> d) & 1u);  // (all lanes of the warp call this together)
	return rs.wcnt[threadIdx.x >> 5][d] + (uint32_t)__popc(b & ((1u << (threadIdx.x & 31)) - 1u));
}
// destination of position `pos` of the block's concatenated run list
__device__ __forceinline__ int run_dest(const RunScratch &rs, uint32_t pos, int world) {
	int d = 0;
	while (d + 1 < world && pos >= rs.cpre[d + 1]) d++;
	return d;
}
// Block-run gather: the rows this block's Gaussians accumulated on rank d are the first c(d) rows of the block's 256
// slots in rank d's partial grad2d — one contiguous run per rank, fetched with lane-contiguous 16-B loads (whole 128-B lines over
// NVLink) into shared memory, 256 rows per round; every thread then adds its own rows in ascending rank order.  Collective over the
// block; `mask` must be the destination mask the forward stored for this thread's Gaussian (0 for none).
__device__ __forceinline__ void gather_runs(const PeerTable &pt, const uint32_t mask, RunScratch &rs, float4 *s_g, float4 &g0v, float4 &g1v,
                                            float4 &g2v) {
	block_run_ranks(rs, mask, pt.world);
	const uint32_t total = rs.cpre[pt.world];
	const size_t slot0 = (size_t)pt.rank * (size_t)pt.chunk + (size_t)blockIdx.x * kRunBlock;
	auto fetch = [&](uint32_t base, float4 (&v)[3]) {  // this thread's (up to) three 16-B pieces of the round that starts at `base`
		const uint32_t n = base < total ? min((uint32_t)kRunBlock, total - base) : 0u;
#pragma unroll
		for (int k = 0; k < 3; k++) {
			const uint32_t e = threadIdx.x + (uint32_t)k * kRunBlock;
			if (e < 3u * n) {
				const uint32_t pos = base + e / 3u, part = e % 3u;
				const int d = run_dest(rs, pos, pt.world);
				v[k] = reinterpret_cast<const float4 *>(pt.grad2d[d] + (slot0 + (pos - rs.cpre[d])) * 12)[part];
			}
		}
	};
	auto consume = [&](uint32_t base, const float4 (&v)[3]) {  // collective: publish the round, add the rows that fall into it
		const uint32_t n = min((uint32_t)kRunBlock, total - base);
#pragma unroll
		for (int k = 0; k < 3; k++) {
			const uint32_t e = threadIdx.x + (uint32_t)k * kRunBlock;
			if (e < 3u * n) s_g[e] = v[k];
		}
		__syncthreads();
		for (int d = 0; d < pt.world; d++) {
			const uint32_t r = run_rank(rs, mask, d);
			const uint32_t pos = rs.cpre[d] + r;
			if (((mask >> d) & 1u) && pos >= base && pos < base + kRunBlock) {
				const float4 a = s_g[(pos - base) * 3u], b = s_g[(pos - base) * 3u + 1u], c = s_g[(pos - base) * 3u + 2u];
				g0v.x += a.x; g0v.y += a.y; g0v.z += a.z; g0v.w += a.w;
				g1v.x += b.x; g1v.y += b.y; g1v.z += b.z; g1v.w += b.w;
				g2v.x += c.x; g2v.y += c.y; g2v.z += c.z; g2v.w += c.w;
			}
		}
		__syncthreads();
	};
	// rounds of 256 rows, two in flight: the loads of the second are requested before the first is waited for (the typical block has
	// 1.2-1.4 rows per Gaussian, i.e. exactly two rounds, so one NVLink round trip replaces two)
	for (uint32_t base = 0; base < total; base += 2u * kRunBlock) {
		float4 va[3], vb[3];
		fetch(base, va);
		fetch(base + kRunBlock, vb);
		consume(base, va);
		if (base + kRunBlock < total) consume(base + kRunBlock, vb);
	}
}

cudaError_t launch_peer_barrier(const PeerTable &pt, uint32_t epoch, uint32_t *status, cudaStream_t st);
// sgr_project fused with sgr_scatter_records: one pass over the rank's chunk (f.P local Gaussians, pt.chunk slots)
// The feature sections of the fused step's peer workspace: sem[P_total, S] and gsem[P_total, S] of every rank, rows by slot.
struct SemPeers {
	float *sem[kMaxPeers];
	float *gsem[kMaxPeers];
};
cudaError_t launch_scatter_semantics(const PeerTable &pt, const SemPeers &sp, int P, int S, const uint32_t *masks, const float *sem, cudaStream_t st);
cudaError_t launch_gather_semantics(const PeerTable &pt, const SemPeers &sp, int P, int S, const uint32_t *masks, float *out, cudaStream_t st);
// Render layers of the fused step (sgr_sharded_*_layers): the layer sections of the peer workspace, layer_mask[P_total] (bit k = layer k,
// rows by slot) and layer_grad2d[L, P_total, 12] of every rank; a layer's rows [begin, end) of the owner's Gaussians.
constexpr int kMaxShardedLayers = SGR_MAX_SHARDED_LAYERS;
struct LayerPeers {
	uint8_t *mask[kMaxPeers];
	int n;
	int begin[kMaxShardedLayers], end[kMaxShardedLayers];
};
cudaError_t launch_scatter_layer_mask(const PeerTable &pt, const LayerPeers &lp, int P, const uint32_t *masks, cudaStream_t st);
struct LayerRows {  // this rank's layer sections to clear
	int n;
	float *rows[kMaxShardedLayers];
};
cudaError_t launch_layer_zero_rows(GeomView g, int n, const LayerRows &t, cudaStream_t st);
struct LayerGatherTable {  // the live layers (those with a gradient) in table order; sec[k].grad2d[p] = rank p's section of layer k
	int n;
	int begin[kMaxShardedLayers], end[kMaxShardedLayers];
	float *sink[kMaxShardedLayers];
	PeerTable sec[kMaxShardedLayers];
};
cudaError_t launch_layer_gather(int P, const PeerTable &pt, const LayerGatherTable &t, const int32_t *radii, const uint32_t *masks, float *out,
                                float *dL_dmeans2D, cudaStream_t st);
cudaError_t launch_project_scatter(const FrameDev &f, const PeerTable &pt, const float *means3D, const float *shs,
                                   const float *colors_precomp, const float *opacities, const float *scales, const float *rotations,
                                   const float *cov3D_precomp, int32_t *radii_local, GaussRec *rec_local, float4 *jac_local,
                                   uint32_t *masks_local, size_t cnt_offset, cudaStream_t st);
cudaError_t launch_scatter_records(const FrameDev &f, const PeerTable &pt, const GaussRec *rec, const int32_t *radii, cudaStream_t st);
cudaError_t launch_gather_grad2d(const FrameDev &f, const PeerTable &pt, const GaussRec *rec, const int32_t *radii, float *out,
                                 cudaStream_t st);
// Gaussian-sharded mode: tile counts / depth keys of gathered records against this rank's band (binning.cu)
cudaError_t launch_count_tiles(const FrameDev &f, GeomView g, const int32_t *radii, cudaStream_t st, float *zero_rows = nullptr);
size_t geom_temp_bytes(int P);
size_t sort_temp_bytes(int64_t R);
size_t bucket_scratch_bytes(int64_t R);
// cap < 0: exact mode, R is the host-known instance count.  cap >= 0: bounded mode, R is ignored, the arrays hold `cap`
// slots and the true count lives in g.big_count[1..3].
cudaError_t launch_binning(const FrameDev &f, GeomView g, const int32_t *radii, BinView b, ImgView img, int64_t R,
                           cudaStream_t st, int64_t cap = -1, int n_order = -1);
// saturation split: whether a forward of this frame takes it, then its passes.  It applies to a whole-image frame that buckets, has
// no semantic channels and R > 0 instances, projected by this process (the records of the Gaussian-sharded mode keep the one-pass
// binning), with a near budget below R (budget < 0: automatic; a budget that covers every instance the binning can hold is the
// one-pass binning).
// near: split + near emission + bucketing; far (after launch_blend_fwd kBlendNear): far count / emission + the final bucketing.
bool split_applies(const FrameDev &f, int64_t R, int64_t budget, bool from_records);
cudaError_t launch_near_binning(const FrameDev &f, GeomView g, const int32_t *radii, BinView b, ImgView img, int64_t slots, cudaStream_t st,
                                int64_t cap, int n_order, int64_t budget);
cudaError_t launch_far_binning(const FrameDev &f, GeomView g, const int32_t *radii, BinView b, ImgView img, int64_t slots, cudaStream_t st,
                               int64_t cap, int n_order);
// pass != kBlendFull needs f.S == 0
cudaError_t launch_blend_fwd(const FrameDev &f, GeomView g, BinView b, ImgView img, const float *semantics, float *out_color,
                             float *out_depth, float *out_alpha, float *out_sem, cudaStream_t st, BlendPass pass = kBlendFull);
cudaError_t launch_blend_bwd(const FrameDev &f, GeomView g, BinView b, ImgView img, const float *semantics,
                             const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                             const float *dL_dsem, float *grad2d, float *dL_dsemantics, cudaStream_t st, bool grad2d_zeroed = false);
cudaError_t launch_blend_bwd2(const FrameDev &f, GeomView g, BinView b, ImgView img, const float *out_alpha, const float *dL_dcolor,
                              const float *dL_ddepth, const float *dL_dalpha, float *grad2d, cudaStream_t st, bool grad2d_zeroed = false);
// pt == nullptr: grad2d holds the f.P x 12 screen-space sums of this process.  With a peer table (sgr_sharded_backward, with
// sgr_gather_grad2d fused in) the sums of each local Gaussian are summed from the ranks that rendered it while the chain rule runs,
// and grad2d carries instead the destination masks (u32[f.P]) the forward stored.
cudaError_t launch_preprocess_bwd(const FrameDev &f, const PeerTable *pt, const float *means3D, const float *shs, const float *colors_precomp,
                                  const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                                  const float4 *jac, const float *grad2d, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh,
                                  float *dL_dcolors, float *dL_dopacity, float *dL_dscales, float *dL_drot, float *dL_dcov3D, cudaStream_t st);
// render layers (layers.cu)
cudaError_t launch_layer_lists(const FrameDev &f, ImgView main_img, BinView main_bin, int begin, int end, ImgView layer_img, uint32_t *layer_list,
                               cudaStream_t st);
cudaError_t launch_layer_lists_masked(const FrameDev &f, ImgView main_img, BinView main_bin, const uint8_t *mask, int bit, ImgView layer_img,
                                      uint32_t *layer_list, cudaStream_t st);
cudaError_t launch_layer_fill(const FrameDev &f, const float *bg, float *color, float *depth, float *alpha, cudaStream_t st);
cudaError_t launch_layer_stash(const float *grad2d, int lo, int hi, float *stash, bool restore, float *dL_dmeans2D, cudaStream_t st);
cudaError_t launch_layer_merge(float *grad2d, const SgrLayerGrad *layers, int n, cudaStream_t st);
cudaError_t launch_compose_fwd(const SgrSegment *segs, int nseg, int M, const float *poses, const float *idft, const uint8_t *flip,
                               const float *flip_quat, float *xyz, float *rot, float *scale, float *opac, float *sh, const float *corr,
                               cudaStream_t st);
cudaError_t launch_compose_bwd(const SgrSegment *segs, const SgrSegmentGrads *grads, int nseg, int M, const float *poses, const float *idft,
                               const uint8_t *flip, const float *flip_quat, const float *g_xyz, const float *g_rot, const float *g_scale,
                               const float *g_opac, const float *g_sh, float *acc, float *dposes, const float *corr, float *dcorr,
                               cudaStream_t st);
cudaError_t launch_compose_bwd_rows(const SgrSegment *segs, const SgrSegmentGrads *grads, int nseg, int M, const float *poses,
                                    const float *idft, const uint8_t *flip, const float *flip_quat, const float *g_xyz, const float *g_rot,
                                    const float *g_scale, const float *g_opac, const float *g_sh, float *acc, const float *corr,
                                    cudaStream_t st);
cudaError_t launch_compose_pose_finalize(const SgrSegment *segs, int nseg, const float *poses, const float *acc, float *dposes,
                                         const float *corr, float *dcorr, cudaStream_t st);
// every rank's composer accumulator section (SgrPeers.pose_acc): SGR_POSE_ACC_ROWS rows of 16 floats
struct PoseAccPeers {
	int world;
	float *sec[kMaxPeers];
};
cudaError_t launch_compose_pose_reduce(const PeerTable &pt, const PoseAccPeers &pp, float *acc, int rows, cudaStream_t st);
cudaError_t launch_color_correct_fwd(int64_t N, const float *image, const float *affine, float *out, cudaStream_t st);
size_t color_correct_scratch_bytes(int64_t N);
cudaError_t launch_color_correct_bwd(int64_t N, const float *image, const float *affine, const float *g_out, float *g_image, float *g_affine,
                                     void *scratch, cudaStream_t st);
// the same on a tile-row band: the band's rows of out / g_image, and the band's 12 sums g_i [x_j, 1] accumulated in double into sums[12]
cudaError_t launch_color_correct_fwd(int H, int W, Band band, const float *image, const float *affine, float *out, cudaStream_t st);
size_t color_correct_band_scratch_bytes(int H, int W);
cudaError_t launch_color_correct_bwd(int H, int W, Band band, const float *image, const float *affine, const float *g_out, float *g_image,
                                     double *sums, void *scratch, cudaStream_t st);
cudaError_t launch_color_correct_affine_grad(const double *sums, float *g_affine, cudaStream_t st);
cudaError_t launch_color_correction_reg(const float *affine, const float *affine_sky, float weight, float *value, float *g_affine,
                                        float *g_affine_sky, cudaStream_t st);
cudaError_t launch_sky_composite_fwd(int H, int W, int R, int mode, float fill, const float *rgb, const float *acc, const uint8_t *mask,
                                     const float *cube, const float *K, const float *w2c, const float *jx, const float *jy, float *out,
                                     cudaStream_t st);
cudaError_t launch_sky_composite_bwd(int H, int W, int R, int mode, float fill, const float *acc, const uint8_t *mask, const float *cube,
                                     const float *K, const float *w2c, const float *jx, const float *jy, const float *gout, float *gacc,
                                     float *gcube, cudaStream_t st);
cudaError_t launch_sky_composite_fwd(int H, int W, Band band, int R, int mode, float fill, const float *rgb, const float *acc, const uint8_t *mask,
                                     const float *cube, const float *K, const float *w2c, const float *jx, const float *jy, float *out,
                                     cudaStream_t st);
cudaError_t launch_sky_composite_bwd(int H, int W, Band band, int R, int mode, float fill, const float *acc, const uint8_t *mask, const float *cube,
                                     const float *K, const float *w2c, const float *jx, const float *jy, const float *gout, float *gacc,
                                     float *gcube, cudaStream_t st, uint8_t *block_map = nullptr, bool clear_map = true);
cudaError_t launch_sky_cube_to_latlong(int R, const float *cube, int H, int W, float *out, uint8_t *u8, cudaStream_t st);
// tracked actor poses (actor_pose.cu): the device-resident track table and one call's camera
constexpr int kActorPoseChunk = 256;  // actors per launch: their track slots travel as a kernel parameter
struct ActorPoseTable {
	int num_tracks, K, num_cams;
	const int32_t *track_off, *entry_fc, *track_frames, *cam_off;
	const double *entry_ts, *track_span, *cam_ts;
	const float *input_trans, *input_rots;
};
struct ActorPoseCall {
	double timestamp, fourier_scale;
	int cam, is_val, opt_track, frame, fourier_dim;
	const float *ego_pose, *opt_trans, *opt_rots;
};
size_t actor_pose_scratch_bytes(int n);
cudaError_t launch_actor_pose_fwd(const ActorPoseTable &T, const ActorPoseCall &c, const int32_t *slots, int n, float *poses, float *idft,
                                  cudaStream_t st);
cudaError_t launch_actor_pose_bwd(const ActorPoseTable &T, const ActorPoseCall &c, const int32_t *slots, int n, const float *g_poses, float *g_trans,
                                  float *g_rots, void *scratch, cudaStream_t st);
// feature channels (features.cu)
cudaError_t launch_gaussian_normals_fwd(int P, const float *means, const float *rots, const float *scales, const float *center, float *normals,
                                        uint8_t *decision, cudaStream_t st);
cudaError_t launch_gaussian_normals_bwd(int P, const float *rots, const uint8_t *decision, const float *g_normals, float *g_rots, cudaStream_t st);
cudaError_t launch_compose_semantics_fwd(int n_bg, int K, int mode, const float *bg, int n_act, const int32_t *start, const int32_t *label,
                                         const float *const *actor, float *out, cudaStream_t st);
cudaError_t launch_compose_semantics_bwd(int n_bg, int K, int mode, const float *out, const float *g, float *g_bg, int n_act, const int32_t *start,
                                         const int32_t *label, float *const *g_actor, cudaStream_t st);
cudaError_t launch_finish_features_fwd(int S, int H, int W, int nc, int mode, const float *in, float *nout, float *sout, cudaStream_t st);
cudaError_t launch_finish_features_bwd(int S, int H, int W, int nc, int mode, const float *in, const float *gn, const float *gs, float *gin,
                                       cudaStream_t st);
// the same on the pixels of a tile-row band only (multi-GPU)
cudaError_t launch_finish_features_fwd(int S, int H, int W, Band band, int nc, int mode, const float *in, float *nout, float *sout, cudaStream_t st);
cudaError_t launch_finish_features_bwd(int S, int H, int W, Band band, int nc, int mode, const float *in, const float *gn, const float *gs,
                                       float *gin, cudaStream_t st);
// the 11-tap SSIM window of loss_utils.py (losses.cu), shared by the image loss and the evaluation metrics
constexpr int kSsimWin = 11;
struct GaussWin {
	float w[kSsimWin];
};
const GaussWin &ssim_window();
size_t image_loss_scratch_bytes(int C, int H, int W);
cudaError_t launch_image_loss(int C, int H, int W, const float *img, const float *gt, const uint8_t *mask, float w_l1, float w_ssim, float *grad,
                              float *scalars, void *scratch, cudaStream_t st);
cudaError_t launch_sky_loss(size_t N, const float *accm, const uint8_t *sky, float weight, float *grad, float *scalars, void *scratch, cudaStream_t st);
cudaError_t launch_obj_acc_loss(size_t N, const float *accm, const uint8_t *obj_bound, float weight, float *grad, float *scalars, void *scratch,
                                cudaStream_t st);
size_t lidar_depth_loss_scratch_bytes(size_t N);
cudaError_t launch_lidar_depth_loss(size_t N, const float *depth, const float *acc, const float *lidar, const uint8_t *mask, double keep, float weight,
                                    float *dL_ddepth, float *dL_dacc, float *scalars, void *scratch, cudaStream_t st);
// the losses on a tile-row band (losses.cu)
constexpr int kBandHalo = 10;  // image rows past a band's edge the photometric loss reads: 5 for the SSIM window, 5 for its derivative maps
struct HaloStrips {
	int first, count, step, offset;
};
HaloStrips halo_strips(int H, Band band, int side);
int64_t halo_rows(int H, const HaloStrips &h);
cudaError_t launch_halo_copy(bool pack, int C, int H, int W, Band band, int side, float *image, float *buf, cudaStream_t st);
// the band losses' exchanges over peer memory (peer_exchange.cu): every rank's loss section (SgrPeers.loss)
struct LossPeers {
	int world;
	char *sec[kMaxPeers];
};
size_t band_halo_slot_bytes(int C, int H, int W);
size_t band_peer_bytes(int C, int H, int W);
cudaError_t launch_band_halo_exchange(const PeerTable &pt, const LossPeers &lp, int C, int H, int W, Band band, const float *image, float *out,
                                      cudaStream_t st);
cudaError_t launch_band_peer_sum(const PeerTable &pt, const LossPeers &lp, bool f64, long long count, const void *local, void *out, cudaStream_t st);
// the sky cube gradient's exchange over peer memory (peer_exchange.cu): every rank's sky section [6 R^2 3 fp32 | block map]
// (SgrSkyPeers).  A block is kSkyBlock x kSkyBlock texels of one face, clipped at the face's last row and column.
constexpr int kSkyBlock = 32;
struct SkyPeers {
	char *sec[kMaxPeers];
};
__host__ __device__ __forceinline__ int sky_blocks_per_side(int R) { return (R + kSkyBlock - 1) / kSkyBlock; }
__host__ __device__ __forceinline__ int64_t sky_block_count(int R) { return 6 * (int64_t)sky_blocks_per_side(R) * sky_blocks_per_side(R); }
__host__ __device__ __forceinline__ size_t sky_cube_section_bytes(int R) { return ((size_t)18 * R * R * sizeof(float) + 255) / 256 * 256; }
__host__ __device__ __forceinline__ size_t sky_peer_bytes(int R) { return (sky_cube_section_bytes(R) + (size_t)sky_block_count(R) + 255) / 256 * 256; }
cudaError_t launch_sky_grad_peer_sum(const PeerTable &pt, const SkyPeers &sp, int R, const uint8_t *map, float *gcube, cudaStream_t st,
                                     uint8_t *union_map = nullptr);
cudaError_t launch_image_loss_stats(int C, int H, int W, Band band, const float *img, const float *gt, const uint8_t *mask, double *acc,
                                    void *scratch, cudaStream_t st);
cudaError_t launch_image_loss_grad(int C, int H, int W, Band band, const float *img, const float *gt, const uint8_t *mask, const double *acc,
                                   float w_l1, float w_ssim, float *grad, float *scalars, void *scratch, cudaStream_t st);
cudaError_t launch_acc_loss_band(int form, int H, int W, Band band, const float *accm, const uint8_t *flag, float weight, float *grad, double *sum,
                                 cudaStream_t st);
cudaError_t launch_acc_loss_value(size_t N, float weight, const double *sum, float *scalars, cudaStream_t st);
size_t lidar_band_scratch_bytes(int H, int W);
cudaError_t launch_lidar_band_keys(int H, int W, Band band, const float *depth, const float *acc, const float *lidar, const uint8_t *mask,
                                   SgrLidarState *s, void *scratch, cudaStream_t st);
cudaError_t launch_lidar_band_select(int level, double keep, int H, int W, Band band, SgrLidarState *s, double *sums, void *scratch, cudaStream_t st);
cudaError_t launch_lidar_band_grad(int H, int W, Band band, const float *depth, const float *acc, const float *lidar, float weight,
                                   const SgrLidarState *s, const double *sums, float *dL_ddepth, float *dL_dacc, float *scalars, void *scratch,
                                   cudaStream_t st);
// evaluation metrics (metrics.cu)
size_t eval_metrics_scratch_bytes(int V, int C, int H, int W);
cudaError_t launch_eval_metrics(int V, int C, int H, int W, Band band, int flags, const float *img, const float *gt, const uint8_t *mask,
                                SgrEvalSums *sums, void *scratch, cudaStream_t st);
cudaError_t launch_eval_metrics_finish(int V, const SgrEvalSums *sums, float *out, cudaStream_t st);
cudaError_t launch_densify_stats(const SgrStatSegment *segs, int nseg, const int32_t *radii, const float *grad2d, cudaStream_t st);
cudaError_t launch_adam(const SgrAdamTensor *ts, int n_tensors, double beta1, double beta2, double eps, cudaStream_t st);
cudaError_t launch_sparse_adam(const SgrSparseAdamSegment *segs, int nseg, const int32_t *radii, double beta1, double beta2, double eps,
                               cudaStream_t st);
cudaError_t launch_cube_sparse_adam(int R, const SgrAdamTensor &a, uint8_t *map, double beta1, double beta2, double eps, cudaStream_t st);
size_t densify_scratch_bytes(int nseg, long long P);
cudaError_t launch_densify_plan(const SgrDensifySegment *segs, int nseg, unsigned long long seed, const float *draws, void *scratch,
                                long long *result_host, cudaStream_t st);
cudaError_t launch_densify_apply(const SgrDensifySegment *segs, const SgrDensifyOutput *outs, int nseg, unsigned long long seed, const float *draws,
                                 void *scratch, cudaStream_t st);
cudaError_t launch_reset_opacity(const SgrDensifySegment *segs, int nseg, cudaStream_t st);
// rebalancing (rebalance.cu): one flat copy of n floats
struct RebalanceSpan {
	const float *src;
	float *dst;
	long long n;
};
size_t rebalance_scratch_bytes(long long nspans);
long long rebalance_blocks(const RebalanceSpan *spans, int nspans);
cudaError_t launch_rebalance_copy(const RebalanceSpan *spans, int nspans, void *scratch, cudaStream_t st);
size_t knn_scratch_bytes(int P);
cudaError_t launch_knn(int P, const float *points, float *out, void *scratch, size_t scratch_bytes, cudaStream_t st);

}  // namespace sgr
