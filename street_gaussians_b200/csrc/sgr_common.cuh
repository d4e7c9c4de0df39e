// sgr_common.cuh — shared device helpers, state layout and the exact tile-cull test.
//
// Data layout in HBM (all caller-owned, see include/sgr.h):
//   geom state   : GaussRec[P] (48 B packed record, 3 x float4 — one 16-B aligned gather of 3 vectors per splat
//                  instance in the blend passes), then tiles_touched / depth_key / iota / depth_sorted / perm / offsets
//                  (u32[P] each) and cub temp storage.
//   img state    : ranges uint2[Ntile], n_contrib u32[H*W], block-max n_contrib u32[Ntile]
//   binning state: keys_in u32[R], keys_out u32[R] (tile ids), vals_in u32[R], vals_out u32[R] (= tile-ordered,
//                  depth-sorted point list), sort temp
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
	uint32_t *ckey, *cval;    // compacted depth-sort input (keys / Gaussian indices), Gaussian-sharded forward only
	void *temp;               // cub temp storage: max(scan, depth sort)
	size_t temp_bytes;
	size_t total_bytes;
};
struct ImgView {
	uint2 *ranges;
	uint32_t *n_contrib;
	uint32_t *tile_max_contrib;
	size_t total_bytes;
};
struct BinView {
	uint32_t *keys_in, *keys_out;  // tile ids
	uint32_t *vals_in, *vals_out;  // Gaussian indices; vals_out is the tile-ordered, depth-sorted point list
	void *sort_temp;
	size_t sort_temp_bytes;
	size_t total_bytes;
};

static inline size_t align_up(size_t v, size_t a = SGR_ALIGN) { return (v + a - 1) / a * a; }

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
ImgView carve_img(void *base, int W, int H);
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
                           int32_t *radii, GaussRec *rec, cudaStream_t st);
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
cudaError_t launch_peer_barrier(const PeerTable &pt, uint32_t epoch, uint32_t *status, cudaStream_t st);
// sgr_project fused with sgr_scatter_records: one pass over the rank's chunk (f.P local Gaussians, pt.chunk slots)
cudaError_t launch_project_scatter(const FrameDev &f, const PeerTable &pt, const float *means3D, const float *shs,
                                   const float *colors_precomp, const float *opacities, const float *scales, const float *rotations,
                                   const float *cov3D_precomp, int32_t *radii_local, GaussRec *rec_local, uint32_t *masks_local,
                                   size_t cnt_offset, cudaStream_t st);
cudaError_t launch_scatter_records(const FrameDev &f, const PeerTable &pt, const GaussRec *rec, const int32_t *radii, cudaStream_t st);
cudaError_t launch_gather_grad2d(const FrameDev &f, const PeerTable &pt, const GaussRec *rec, const int32_t *radii, float *out,
                                 cudaStream_t st);
// Gaussian-sharded mode: tile counts / depth keys of gathered records against this rank's band (binning.cu)
cudaError_t launch_count_tiles(const FrameDev &f, GeomView g, const int32_t *radii, cudaStream_t st, float *zero_rows = nullptr);
size_t geom_temp_bytes(int P);
size_t sort_temp_bytes(int64_t R);
// cap < 0: exact mode, R is the host-known instance count.  cap >= 0: bounded mode, R is ignored, the arrays hold `cap`
// slots and the true count lives in g.big_count[1..3].
cudaError_t launch_binning(const FrameDev &f, GeomView g, const int32_t *radii, BinView b, ImgView img, int64_t R,
                           cudaStream_t st, int64_t cap = -1, int n_order = -1);
cudaError_t launch_blend_fwd(const FrameDev &f, GeomView g, BinView b, ImgView img, const float *semantics, float *out_color,
                             float *out_depth, float *out_alpha, float *out_sem, cudaStream_t st);
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
                                  const GaussRec *rec, const float *grad2d, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh,
                                  float *dL_dcolors, float *dL_dopacity, float *dL_dscales, float *dL_drot, float *dL_dcov3D, cudaStream_t st);
// render layers (layers.cu)
cudaError_t launch_layer_lists(const FrameDev &f, ImgView main_img, BinView main_bin, int begin, int end, ImgView layer_img, uint32_t *layer_list,
                               cudaStream_t st);
cudaError_t launch_layer_fill(const FrameDev &f, const float *bg, float *color, float *depth, float *alpha, cudaStream_t st);
cudaError_t launch_layer_stash(const float *grad2d, int lo, int hi, float *stash, bool restore, float *dL_dmeans2D, cudaStream_t st);
cudaError_t launch_layer_merge(float *grad2d, const SgrLayerGrad *layers, int n, cudaStream_t st);
cudaError_t launch_compose_fwd(const SgrSegment *segs, int nseg, int M, const float *poses, const float *idft, const uint8_t *flip,
                               const float *flip_quat, float *xyz, float *rot, float *scale, float *opac, float *sh, cudaStream_t st);
cudaError_t launch_compose_bwd(const SgrSegment *segs, const SgrSegmentGrads *grads, int nseg, int M, const float *poses, const float *idft,
                               const uint8_t *flip, const float *flip_quat, const float *g_xyz, const float *g_rot, const float *g_scale,
                               const float *g_opac, const float *g_sh, float *acc, float *dposes, cudaStream_t st);
size_t image_loss_scratch_bytes(int C, int H, int W);
cudaError_t launch_image_loss(int C, int H, int W, const float *img, const float *gt, const uint8_t *mask, float w_l1, float w_ssim, float *grad,
                              float *scalars, void *scratch, cudaStream_t st);
cudaError_t launch_sky_loss(size_t N, const float *accm, const uint8_t *sky, float weight, float *grad, float *scalars, void *scratch, cudaStream_t st);
cudaError_t launch_obj_acc_loss(size_t N, const float *accm, const uint8_t *obj_bound, float weight, float *grad, float *scalars, void *scratch,
                                cudaStream_t st);
size_t lidar_depth_loss_scratch_bytes(size_t N);
cudaError_t launch_lidar_depth_loss(size_t N, const float *depth, const float *acc, const float *lidar, const uint8_t *mask, double keep, float weight,
                                    float *dL_ddepth, float *dL_dacc, float *scalars, void *scratch, cudaStream_t st);
cudaError_t launch_densify_stats(const SgrStatSegment *segs, int nseg, const int32_t *radii, const float *grad2d, cudaStream_t st);
cudaError_t launch_adam(const SgrAdamTensor *ts, int n_tensors, double beta1, double beta2, double eps, cudaStream_t st);
cudaError_t launch_sparse_adam(const SgrSparseAdamSegment *segs, int nseg, const int32_t *radii, double beta1, double beta2, double eps,
                               cudaStream_t st);
size_t densify_scratch_bytes(int nseg, long long P);
cudaError_t launch_densify_plan(const SgrDensifySegment *segs, int nseg, unsigned long long seed, const float *draws, void *scratch,
                                long long *result_host, cudaStream_t st);
cudaError_t launch_densify_apply(const SgrDensifySegment *segs, const SgrDensifyOutput *outs, int nseg, unsigned long long seed, const float *draws,
                                 void *scratch, cudaStream_t st);
cudaError_t launch_reset_opacity(const SgrDensifySegment *segs, int nseg, cudaStream_t st);
size_t knn_scratch_bytes(int P);
cudaError_t launch_knn(int P, const float *points, float *out, void *scratch, size_t scratch_bytes, cudaStream_t st);

}  // namespace sgr
