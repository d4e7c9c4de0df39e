// peer_exchange.cu — the two exchange steps of the Gaussian-sharded mode done with plain loads/stores on NVLink peer
// memory instead of NCCL collectives (include/sgr.h: sgr_scatter_records, sgr_gather_grad2d).
//
// With cyclic tile-row bands (row r belongs to rank r % world) a Gaussian whose tile rectangle spans h rows is needed by
// min(h, world) ranks only — 1 or 2 for the bulk of a street scene — while an all-gather ships every record to every
// rank.  So the owner WRITES each 48-B record straight into the gathered array of exactly the ranks that need it (and a
// 4-B radius, 0 = "not yours", to everyone), and in backward READS the partial grad2d rows back from exactly those
// ranks.  Arrays stay indexed by the global Gaussian id, so binning order and results are bit-identical to the NCCL
// path; the caller brackets the two steps with device-side barriers (torch symmetric memory).
#include "sgr_common.cuh"

namespace sgr {

__device__ __forceinline__ uint32_t ranks_of(const FrameDev &f, const float4 q0, int radius, int world) {
	int x0, y0, x1, y1;
	tile_rect(q0.x, q0.y, radius, f.gx, f.gy, x0, y0, x1, y1);
	return x1 > x0 ? touched_ranks(y0, y1, world) : 0u;
}

// one thread per slot of this rank's chunk (slots past f.P are padding: radius 0 everywhere)
__global__ void __launch_bounds__(256) scatter_records_kernel(const FrameDev f, const PeerTable pt, const GaussRec *__restrict__ rec,
                                                             const int32_t *__restrict__ radii) {
	const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= pt.chunk) return;
	int r = 0;
	uint32_t mask = 0u;
	GaussRec v;
	v.q0 = v.q1 = v.q2 = make_float4(0.f, 0.f, 0.f, 0.f);
	if (idx < f.P) {
		r = radii[idx];
		if (r > 0) {
			v = rec[idx];
			mask = ranks_of(f, v.q0, r, pt.world);
		}
	}
	const size_t g = (size_t)pt.rank * (size_t)pt.chunk + (size_t)idx;
	for (int p = 0; p < pt.world; p++) {
		const bool hit = (mask >> p) & 1u;
		if (hit) pt.rec[p][g] = v;
		pt.radii[p][g] = hit ? r : 0;
	}
}

// grad2d_local[i] = sum over the ranks that rendered Gaussian i of their partial row (fixed ascending-rank order)
__global__ void __launch_bounds__(256) gather_grad2d_kernel(const FrameDev f, const PeerTable pt, const GaussRec *__restrict__ rec,
                                                           const int32_t *__restrict__ radii, float *__restrict__ out) {
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= f.P) return;
	float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a, c = a;
	const int r = radii[idx];
	if (r > 0) {
		const uint32_t mask = ranks_of(f, rec[idx].q0, r, pt.world);
		const size_t g = (size_t)pt.rank * (size_t)pt.chunk + (size_t)idx;
		for (int p = 0; p < pt.world; p++) {
			if (!((mask >> p) & 1u)) continue;
			const float4 *src = reinterpret_cast<const float4 *>(pt.grad2d[p] + g * 12);
			const float4 x = src[0], y = src[1], z = src[2];
			a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w;
			b.x += y.x; b.y += y.y; b.z += y.z; b.w += y.w;
			c.x += z.x; c.y += z.y; c.z += z.z; c.w += z.w;
		}
	}
	float4 *dst = reinterpret_cast<float4 *>(out + (size_t)idx * 12);
	dst[0] = a; dst[1] = b; dst[2] = c;
}

// ---- feature channels of the fused step (sgr_sharded_forward_features / sgr_sharded_backward_features) ----
// The S floats of each Gaussian travel like its record: the Gaussians of one block of kRunBlock own slots that rank d needs form ONE
// contiguous run of rows in the block's slots of rank d's `sem` section, in ascending Gaussian order, into the same slots as the records
// preprocess_fwd_kernel<false, SCATTER> sent.  The runs are re-derived from the destination masks that kernel stored (the same
// block_run_ranks over the same masks), so records and rows agree slot for slot.  A run's rows are consecutive in the destination, so a
// block writes each run as one stream of consecutive floats (whole 128-B lines).
__global__ void __launch_bounds__(kRunBlock) scatter_semantics_kernel(const int P, const int S, const PeerTable pt, const SemPeers sp,
                                                                     const uint32_t *__restrict__ masks, const float *__restrict__ sem) {
	__shared__ RunScratch rs;
	__shared__ uint8_t s_src[kRunBlock * kMaxPeers];
	const long long idx = (long long)blockIdx.x * kRunBlock + threadIdx.x;
	const uint32_t mask = idx < P ? masks[idx] : 0u;
	block_run_ranks(rs, mask, pt.world);
	for (int d = 0; d < pt.world; d++) {
		const uint32_t r = run_rank(rs, mask, d);
		if ((mask >> d) & 1u) s_src[rs.cpre[d] + r] = (uint8_t)threadIdx.x;
	}
	__syncthreads();
	const uint32_t total = rs.cpre[pt.world];
	const size_t slot0 = (size_t)pt.rank * (size_t)pt.chunk + (size_t)blockIdx.x * kRunBlock;
	const float *src = sem + (size_t)blockIdx.x * kRunBlock * (size_t)S;
	for (uint32_t e = threadIdx.x; e < total * (uint32_t)S; e += kRunBlock) {
		const uint32_t pos = e / (uint32_t)S, c = e - pos * (uint32_t)S;
		const int d = run_dest(rs, pos, pt.world);
		sp.sem[d][(slot0 + (pos - rs.cpre[d])) * (size_t)S + c] = src[(size_t)s_src[pos] * S + c];
	}
}

// dL/dsemantics of the own Gaussians: the partial rows the ranks' blend backward left in their `gsem` sections, fetched as the same runs
// and added in ascending rank order (from 0, one fp32 add per rank that rendered the Gaussian); a Gaussian no rank received gets 0.
__global__ void __launch_bounds__(kRunBlock) gather_semantics_kernel(const int P, const int S, const PeerTable pt, const SemPeers sp,
                                                                    const uint32_t *__restrict__ masks, float *__restrict__ out) {
	__shared__ RunScratch rs;
	__shared__ uint8_t s_pos[kMaxPeers][kRunBlock];  // thread t's position in destination d's run (where bit d of its mask is set)
	__shared__ uint32_t s_mask[kRunBlock];
	const long long first = (long long)blockIdx.x * kRunBlock;
	const uint32_t mask = first + threadIdx.x < P ? masks[first + threadIdx.x] : 0u;
	block_run_ranks(rs, mask, pt.world);
	for (int d = 0; d < pt.world; d++) {
		const uint32_t r = run_rank(rs, mask, d);
		s_pos[d][threadIdx.x] = (uint8_t)r;
	}
	s_mask[threadIdx.x] = mask;
	__syncthreads();
	const int n = (int)min((long long)kRunBlock, (long long)P - first);
	const size_t slot0 = (size_t)pt.rank * (size_t)pt.chunk + (size_t)first;
	for (int e = threadIdx.x; e < n * S; e += kRunBlock) {
		const int t = e / S, c = e - t * S;
		const uint32_t m = s_mask[t];
		float v = 0.f;
		for (int d = 0; d < pt.world; d++)
			if ((m >> d) & 1u) v += sp.gsem[d][(slot0 + s_pos[d][t]) * (size_t)S + c];
		out[(size_t)first * S + e] = v;
	}
}

// ---- render layers of the fused step (sgr_sharded_forward_layers) ----
// One byte per Gaussian (bit k = the Gaussian lies in layer k's rows), delivered like its record: the same block runs, the same slots of
// rank d's mask section.  The runs are re-derived from the destination masks preprocess_fwd_kernel<false, SCATTER> stored, as above.
__global__ void __launch_bounds__(kRunBlock) scatter_layer_mask_kernel(const int P, const PeerTable pt, const LayerPeers lp,
                                                                      const uint32_t *__restrict__ masks) {
	__shared__ RunScratch rs;
	const int idx = blockIdx.x * kRunBlock + threadIdx.x;
	const uint32_t mask = idx < P ? masks[idx] : 0u;
	uint32_t bits = 0u;
	for (int k = 0; k < lp.n; k++) bits |= (idx >= lp.begin[k] && idx < lp.end[k]) ? 1u << k : 0u;
	block_run_ranks(rs, mask, pt.world);
	const size_t slot0 = (size_t)pt.rank * (size_t)pt.chunk + (size_t)blockIdx.x * kRunBlock;
	for (int d = 0; d < pt.world; d++) {
		const uint32_t r = run_rank(rs, mask, d);
		if ((mask >> d) & 1u) lp.mask[d][slot0 + r] = (uint8_t)bits;
	}
}

cudaError_t launch_scatter_layer_mask(const PeerTable &pt, const LayerPeers &lp, int P, const uint32_t *masks, cudaStream_t st) {
	if (P == 0) return cudaSuccess;
	count_launch();
	scatter_layer_mask_kernel<<<(unsigned)((P + kRunBlock - 1) / kRunBlock), kRunBlock, 0, st>>>(P, pt, lp, masks);
	return cudaGetLastError();
}

cudaError_t launch_scatter_semantics(const PeerTable &pt, const SemPeers &sp, int P, int S, const uint32_t *masks, const float *sem, cudaStream_t st) {
	if (P == 0) return cudaSuccess;
	count_launch();
	scatter_semantics_kernel<<<(unsigned)((P + kRunBlock - 1) / kRunBlock), kRunBlock, 0, st>>>(P, S, pt, sp, masks, sem);
	return cudaGetLastError();
}

cudaError_t launch_gather_semantics(const PeerTable &pt, const SemPeers &sp, int P, int S, const uint32_t *masks, float *out, cudaStream_t st) {
	if (P == 0) return cudaSuccess;
	count_launch();
	gather_semantics_kernel<<<(unsigned)((P + kRunBlock - 1) / kRunBlock), kRunBlock, 0, st>>>(P, S, pt, sp, masks, out);
	return cudaGetLastError();
}

// Cross-rank barrier on the caller's stream: thread p announces this rank's arrival in rank p's pad (a release store at system
// scope, after a system-scope fence that orders this rank's earlier peer stores — issued by previous kernels of the stream —
// before it) and then waits until rank p has announced itself in this rank's pad.  Epochs increase by one per barrier and every
// rank issues the same sequence of barriers, so one pad suffices: a peer that is already one barrier ahead has written a larger
// epoch, which also satisfies the wait.  epoch == 0 ("auto"): the epoch is kept ON THE DEVICE — slot kMaxPeers of the rank's own pad
// counts its barriers — so the launch carries no per-step host value and a captured CUDA graph of a step can be replayed.
// The spin is bounded (2 s) so a missing peer cannot wedge the GPU; a timeout sets status[5] and the frame is garbage.
__global__ void peer_barrier_kernel(const PeerTable pt, uint32_t epoch, uint32_t *__restrict__ status) {
	const int p = threadIdx.x;
	if (epoch == 0u) {
		uint32_t e = 0u;
		if (p == 0) {
			uint32_t *counter = pt.flags[pt.rank] + kMaxPeers;
			e = *counter + 1u;
			*counter = e;
		}
		epoch = __shfl_sync(0xffffffffu, e, 0);
	}
	if (p >= pt.world) return;
	__threadfence_system();
	uint32_t *theirs = pt.flags[p] + pt.rank;
	asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(theirs), "r"(epoch) : "memory");
	const uint32_t *mine = pt.flags[pt.rank] + p;
	unsigned long long t0;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
	for (;;) {
		uint32_t v;
		asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
		if ((int32_t)(v - epoch) >= 0) break;
		__nanosleep(40);
		unsigned long long t1;
		asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
		if (t1 - t0 > 2000000000ull) {
			if (status) atomicExch(&status[5], epoch);
			break;
		}
	}
}
cudaError_t launch_peer_barrier(const PeerTable &pt, uint32_t epoch, uint32_t *status, cudaStream_t st) {
	if (pt.world <= 1) return cudaSuccess;
	count_launch();
	peer_barrier_kernel<<<1, 32, 0, st>>>(pt, epoch, status);
	return cudaGetLastError();
}

// ---- the band losses' exchanges (sgr_band_halo_exchange_peers / sgr_band_peer_sum) ----
// A rank's loss section is [SEND_UP slot | SEND_DOWN slot] for the halo and [count elements] for a sum; the two never overlap in time
// because each call ends with a barrier after which no peer reads the section any more.  A slot holds the largest message of any band:
// with step >= 2 a band owns at most ceil(rows / 2) tile rows, each sending at most one strip per side; with step 1 one strip per side.
size_t band_halo_slot_bytes(int C, int H, int W) {
	const size_t rows = (size_t)(H + 15) / 16;
	const size_t bytes = (size_t)C * kBandHalo * ((rows + 1) / 2) * (size_t)W * sizeof(float);
	return (bytes + 255) / 256 * 256;
}
size_t band_peer_bytes(int C, int H, int W) {
	const size_t rows = (size_t)(H + 15) / 16;
	size_t sums = (size_t)SGR_LIDAR_LEVEL0_WORDS * 4;  // the largest of the summed arrays: LiDAR level-0 words, a level's
	if ((size_t)SGR_LIDAR_BINS * 4 > sums) sums = (size_t)SGR_LIDAR_BINS * 4;  // histogram, the level-3 sums, the frame losses' partials
	if ((1 + rows) * 8 > sums) sums = (1 + rows) * 8;
	if (5 * 8 > sums) sums = 5 * 8;
	const size_t halo = 2 * band_halo_slot_bytes(C, H, W);
	return ((halo > sums ? halo : sums) + 255) / 256 * 256;
}

cudaError_t launch_band_halo_exchange(const PeerTable &pt, const LossPeers &lp, int C, int H, int W, Band band, const float *image, float *out,
                                      cudaStream_t st) {
	const size_t slot = band_halo_slot_bytes(C, H, W);
	const int up = (pt.rank + pt.world - 1) % pt.world, down = (pt.rank + 1) % pt.world;
	float *img = const_cast<float *>(image);
	cudaError_t e = cudaSuccess;
	if (pt.world > 1) {  // publish: the rows the neighbours need, in sgr_band_halo_pack's layout (an empty band has no message)
		if ((e = launch_halo_copy(true, C, H, W, band, SGR_HALO_SEND_UP, img, reinterpret_cast<float *>(lp.sec[pt.rank]), st)) != cudaSuccess) return e;
		if ((e = launch_halo_copy(true, C, H, W, band, SGR_HALO_SEND_DOWN, img, reinterpret_cast<float *>(lp.sec[pt.rank] + slot), st)) != cudaSuccess)
			return e;
	}
	if ((e = launch_peer_barrier(pt, 0u, nullptr, st)) != cudaSuccess) return e;
	if (pt.world > 1) {  // pull: the upper neighbour's SEND_DOWN is this rank's RECV_UP, the lower one's SEND_UP its RECV_DOWN
		if ((e = launch_halo_copy(false, C, H, W, band, SGR_HALO_RECV_UP, out, reinterpret_cast<float *>(lp.sec[up] + slot), st)) != cudaSuccess) return e;
		if ((e = launch_halo_copy(false, C, H, W, band, SGR_HALO_RECV_DOWN, out, reinterpret_cast<float *>(lp.sec[down]), st)) != cudaSuccess) return e;
	}
	return launch_peer_barrier(pt, 0u, nullptr, st);
}

// T: uint32_t for the int32 sums (wrap-around adds are the two's-complement ones), double for fp64
template <typename T>
__global__ void __launch_bounds__(256) loss_stage_kernel(const T *__restrict__ src, T *__restrict__ dst, const long long n) {
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) dst[i] = src[i];
}
template <typename T>
__global__ void __launch_bounds__(256) loss_sum_kernel(const LossPeers lp, const long long n, T *__restrict__ out) {
	const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	T v = T(0);
	for (int p = 0; p < lp.world; p++) v += reinterpret_cast<const T *>(lp.sec[p])[i];
	out[i] = v;
}

template <typename T>
static cudaError_t peer_sum(const PeerTable &pt, const LossPeers &lp, long long n, const T *local, T *out, cudaStream_t st) {
	const unsigned nblk = (unsigned)((n + 255) / 256);
	if (n > 0) {
		count_launch();
		loss_stage_kernel<T><<<nblk, 256, 0, st>>>(local, reinterpret_cast<T *>(lp.sec[pt.rank]), n);
	}
	cudaError_t e = launch_peer_barrier(pt, 0u, nullptr, st);
	if (e != cudaSuccess) return e;
	if (n > 0) {
		count_launch();
		loss_sum_kernel<T><<<nblk, 256, 0, st>>>(lp, n, out);
	}
	return launch_peer_barrier(pt, 0u, nullptr, st);
}

cudaError_t launch_band_peer_sum(const PeerTable &pt, const LossPeers &lp, bool f64, long long count, const void *local, void *out, cudaStream_t st) {
	if (f64) return peer_sum<double>(pt, lp, count, static_cast<const double *>(local), static_cast<double *>(out), st);
	return peer_sum<uint32_t>(pt, lp, count, static_cast<const uint32_t *>(local), static_cast<uint32_t *>(out), st);
}

// ---- the sky cube gradient's exchange (sgr_sky_grad_peer_sum) ----
// A rank's sky section is [6 R^2 3 fp32, padded to 256 B | one byte per block].  Block b (face f, block row br, block column bc) is
// owned by rank b % world.  Stage: the rank copies its marked blocks and its whole map into its section.  Owner sum: the owner adds,
// from rank 0 up, the block of every rank that marked it and writes the sum into its own section (only the owner reads block b of any
// section, so the in-place write races with nothing).  Gather: every rank copies each block of the union from the owner's section into
// its dense gradient.  Barriers separate the three and end the call.  Grids are one CTA per block: they depend on R only.
constexpr int kSkyXThreads = 256;

// op.vec(i) on the 16-byte aligned float4 at float offset i, op.one(i) on a single float, over every float of block b's texels: one warp
// per texel row of the block, the row's unaligned head and tail (when 3 R is not a multiple of 4) one float at a time.
template <class Op>
__device__ __forceinline__ void sky_block_floats(const int b, const int R, Op &op) {
	const int nb = sky_blocks_per_side(R), f = b / (nb * nb), br = (b / nb) % nb, bc = b % nb;
	const int r0 = br * kSkyBlock, r1 = min(R, r0 + kSkyBlock), c0 = bc * kSkyBlock, len = (min(R, c0 + kSkyBlock) - c0) * 3;
	const int lane = threadIdx.x & 31;
	for (int r = r0 + (int)(threadIdx.x >> 5); r < r1; r += kSkyXThreads / 32) {
		const size_t s = ((size_t)(f * R + r) * R + c0) * 3;
		const int head = min(len, (int)((4 - (s & 3)) & 3)), nv = (len - head) >> 2, tail = len - head - 4 * nv;
		if (lane < head) op.one(s + lane);
		for (int v = lane; v < nv; v += 32) op.vec(s + head + 4 * (size_t)v);
		if (lane < tail) op.one(s + head + 4 * (size_t)nv + lane);
	}
}

struct SkyCopy {
	float *__restrict__ dst;
	const float *__restrict__ src;
	__device__ __forceinline__ void vec(size_t i) { *reinterpret_cast<float4 *>(dst + i) = *reinterpret_cast<const float4 *>(src + i); }
	__device__ __forceinline__ void one(size_t i) { dst[i] = src[i]; }
};

// v = 0; for p = 0 .. world - 1 (bit p of `ranks` set): v += section p — the same adds per component for a float4 and a float
struct SkySum {
	float *__restrict__ dst;
	const SkyPeers *sp;
	uint32_t ranks;
	int world;
	__device__ __forceinline__ void vec(size_t i) {
		float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
		for (int p = 0; p < world; p++) {
			if (!((ranks >> p) & 1u)) continue;
			const float4 x = *reinterpret_cast<const float4 *>(reinterpret_cast<const float *>(sp->sec[p]) + i);
			v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
		}
		*reinterpret_cast<float4 *>(dst + i) = v;
	}
	__device__ __forceinline__ void one(size_t i) {
		float v = 0.f;
		for (int p = 0; p < world; p++)
			if ((ranks >> p) & 1u) v += reinterpret_cast<const float *>(sp->sec[p])[i];
		dst[i] = v;
	}
};

__device__ __forceinline__ uint8_t *sky_section_map(char *sec, int R) { return reinterpret_cast<uint8_t *>(sec + sky_cube_section_bytes(R)); }

// bit p set: rank p's staged map marks block b
__device__ __forceinline__ uint32_t sky_block_ranks(const SkyPeers &sp, const int world, const int R, const int b) {
	__shared__ uint32_t s_ranks;
	if (threadIdx.x == 0) {
		uint32_t bits = 0u;
		for (int p = 0; p < world; p++) bits |= sky_section_map(sp.sec[p], R)[b] ? 1u << p : 0u;
		s_ranks = bits;
	}
	__syncthreads();
	return s_ranks;
}

__global__ void __launch_bounds__(kSkyXThreads) sky_stage_kernel(const __grid_constant__ SkyPeers sp, const int R, const int rank, const uint8_t *__restrict__ map,
                                                                 const float *__restrict__ gcube) {
	const int b = blockIdx.x;
	const uint8_t m = map[b];
	char *sec = sp.sec[rank];
	if (threadIdx.x == 0) sky_section_map(sec, R)[b] = m ? 1 : 0;
	if (!m) return;
	SkyCopy op{reinterpret_cast<float *>(sec), gcube};
	sky_block_floats(b, R, op);
}

__global__ void __launch_bounds__(kSkyXThreads) sky_owner_sum_kernel(const __grid_constant__ SkyPeers sp, const int R, const int world,
                                                                     const int rank) {
	const int b = blockIdx.x;
	if (b % world != rank) return;
	const uint32_t ranks = sky_block_ranks(sp, world, R, b);
	if (!ranks) return;
	SkySum op{reinterpret_cast<float *>(sp.sec[rank]), &sp, ranks, world};
	sky_block_floats(b, R, op);
}

__global__ void __launch_bounds__(kSkyXThreads) sky_gather_kernel(const __grid_constant__ SkyPeers sp, const int R, const int world, float *__restrict__ gcube) {
	const int b = blockIdx.x;
	if (!sky_block_ranks(sp, world, R, b)) return;  // outside the union: the rank's partial is already zero there
	SkyCopy op{gcube, reinterpret_cast<const float *>(sp.sec[b % world])};
	sky_block_floats(b, R, op);
}

// The gather that also sets union_map[b] for every block some rank marked (sgr_sky_grad_peer_sum_union): every rank reads the same
// staged maps, so every rank writes the same bytes.
__global__ void __launch_bounds__(kSkyXThreads) sky_gather_union_kernel(const __grid_constant__ SkyPeers sp, const int R, const int world,
                                                                        float *__restrict__ gcube, uint8_t *__restrict__ union_map) {
	const int b = blockIdx.x;
	if (!sky_block_ranks(sp, world, R, b)) return;
	if (threadIdx.x == 0) union_map[b] = 1;
	SkyCopy op{gcube, reinterpret_cast<const float *>(sp.sec[b % world])};
	sky_block_floats(b, R, op);
}

cudaError_t launch_sky_grad_peer_sum(const PeerTable &pt, const SkyPeers &sp, int R, const uint8_t *map, float *gcube, cudaStream_t st,
                                     uint8_t *union_map) {
	const unsigned nblk = (unsigned)sky_block_count(R);
	count_launch();
	sky_stage_kernel<<<nblk, kSkyXThreads, 0, st>>>(sp, R, pt.rank, map, gcube);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess || (e = launch_peer_barrier(pt, 0u, nullptr, st)) != cudaSuccess) return e;
	count_launch();
	sky_owner_sum_kernel<<<nblk, kSkyXThreads, 0, st>>>(sp, R, pt.world, pt.rank);
	if ((e = cudaGetLastError()) != cudaSuccess || (e = launch_peer_barrier(pt, 0u, nullptr, st)) != cudaSuccess) return e;
	count_launch();
	if (union_map)
		sky_gather_union_kernel<<<nblk, kSkyXThreads, 0, st>>>(sp, R, pt.world, gcube, union_map);
	else
		sky_gather_kernel<<<nblk, kSkyXThreads, 0, st>>>(sp, R, pt.world, gcube);
	if ((e = cudaGetLastError()) != cudaSuccess) return e;
	return launch_peer_barrier(pt, 0u, nullptr, st);
}

// ---- buffers moved through the staging regions (sgr_peer_exchange_round) ----
// One CTA copies kPieceVec x 256 consecutive float4 of one piece: every thread issues its kPieceVec 16-B loads before its first store,
// and the lanes of a warp touch consecutive 16-B pieces, so every load request is whole 128-B lines (over NVLink in the pull).  The
// piece's last (floats mod 4) floats are copied one by one by the CTA that holds its end.
constexpr int kPieceThreads = 256, kPieceVec = 4;
constexpr long long kPieceFloats = 4LL * kPieceThreads * kPieceVec;
long long peer_piece_blocks(long long floats) { return (floats + kPieceFloats - 1) / kPieceFloats; }

__global__ void __launch_bounds__(kPieceThreads) copy_pieces_kernel(const __grid_constant__ PieceTable t) {
	int i = 0;
	while (i + 1 < t.n && (int)blockIdx.x >= t.block_start[i + 1]) i++;
	const long long e0 = (long long)(blockIdx.x - t.block_start[i]) * kPieceFloats;
	const long long n = min(kPieceFloats, t.floats[i] - e0);
	const int nv = (int)(n >> 2);
	const float4 *src = reinterpret_cast<const float4 *>(t.src[i] + e0);
	float4 *dst = reinterpret_cast<float4 *>(t.dst[i] + e0);
	float4 v[kPieceVec];
#pragma unroll
	for (int j = 0; j < kPieceVec; j++) {
		const int k = threadIdx.x + j * kPieceThreads;
		if (k < nv) v[j] = src[k];
	}
#pragma unroll
	for (int j = 0; j < kPieceVec; j++) {
		const int k = threadIdx.x + j * kPieceThreads;
		if (k < nv) dst[k] = v[j];
	}
	if (threadIdx.x < (int)(n & 3)) t.dst[i][e0 + 4 * nv + threadIdx.x] = t.src[i][e0 + 4 * nv + threadIdx.x];
}

static cudaError_t launch_pieces(PieceTable &t, cudaStream_t st) {
	long long blocks = 0;
	for (int i = 0; i < t.n; i++) {
		t.block_start[i] = (int)blocks;
		blocks += peer_piece_blocks(t.floats[i]);
	}
	t.block_start[t.n] = (int)blocks;
	if (blocks == 0) return cudaSuccess;
	count_launch();
	copy_pieces_kernel<<<(unsigned)blocks, kPieceThreads, 0, st>>>(t);
	return cudaGetLastError();
}

// stage launch, barrier, pull launch (the pieces without floats are dropped by the caller; a side without pieces launches nothing)
cudaError_t launch_peer_exchange_round(const PeerTable &pt, PieceTable stage, PieceTable pull, cudaStream_t st) {
	cudaError_t e = launch_pieces(stage, st);
	if (e != cudaSuccess || (e = launch_peer_barrier(pt, 0u, nullptr, st)) != cudaSuccess) return e;
	return launch_pieces(pull, st);
}

cudaError_t launch_scatter_records(const FrameDev &f, const PeerTable &pt, const GaussRec *rec, const int32_t *radii, cudaStream_t st) {
	if (pt.chunk == 0) return cudaSuccess;
	count_launch();
	scatter_records_kernel<<<(unsigned)((pt.chunk + 255) / 256), 256, 0, st>>>(f, pt, rec, radii);
	return cudaGetLastError();
}
cudaError_t launch_gather_grad2d(const FrameDev &f, const PeerTable &pt, const GaussRec *rec, const int32_t *radii, float *out,
                                 cudaStream_t st) {
	if (f.P == 0) return cudaSuccess;
	count_launch();
	gather_grad2d_kernel<<<(f.P + 255) / 256, 256, 0, st>>>(f, pt, rec, radii, out);
	return cudaGetLastError();
}

}  // namespace sgr
