// preprocess_bwd.cu — per-Gaussian chain rule: screen-space sums -> (mean3D, SH | colour, opacity, scale, rotation | cov3D).
//
// Replaces the reference's computeCov2DCUDA + preprocessCUDA(backward) pair (DGR/cuda_rasterizer/backward.cu:144-274,
// 346-412, with computeColorFromSH :20-139 and computeCov3D :278-341) by ONE kernel:
//   * reads the 12-float grad2d record produced by blend_bwd (one 48-B aligned load) instead of five separate arrays;
//   * recomputes cov3D from scale/rotation instead of reading a stored copy;
//   * WRITES every output element (zeros for culled Gaussians), so the caller allocates with torch.empty and the
//     reference's 304 B/Gaussian of torch::zeros (rasterize_points.cu:166-176) disappears;
//   * dL/dmean3D is accumulated in registers across the three contributions and stored once (the reference does
//     one store + two read-modify-writes + one more inside the SH routine).
//   * SH coefficients in / SH gradients out are staged through shared memory per warp: the 32 Gaussians of a warp own
//     one contiguous 32 x M x 3 float block of `shs` / `dL_dsh`, which the warp moves with fully coalesced 16-B accesses
//     (rows padded to 49 floats in smem so the per-thread row walks are bank-conflict free).  The direct per-thread
//     version (48 strided scalar loads + 48 strided scalar stores per Gaussian) wastes most of each memory transaction.
// Formulas and evaluation order follow the reference so gradients agree to fp32 rounding.  The geometry (covariances, EWA
// Jacobian, projective divide, depth, scale / rotation) is gaussian_geom.cuh's, the same functions the forward calls; the two
// kernels below differ in how they load their inputs, the gather, their SH backward loop and their stores.
#include <cstdlib>

#include "gaussian_geom.cuh"

namespace sgr {

constexpr int kShRow = 49;  // padded smem row (floats) for up to 16 x 3 SH coefficients
constexpr int kBwdStride = 52;  // row stride (floats) of the TMA variant's stage: 208 B

// Block-run gather (sgr_common.cuh): the rows this block's Gaussians accumulated on rank d are the first c(d) rows of the block's 256
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

// GATHER = true (sgr_sharded_backward): grad2d is not a local array — the 12 sums of local Gaussian idx (global id
// rank*chunk + idx) are read from the partial grad2d of every rank whose cyclic band its rectangle meets (NVLink peer loads)
// and added in ascending rank order, exactly what sgr_gather_grad2d produced as a separate pass.
template <bool STAGED, bool GATHER = false>
__global__ void __launch_bounds__(256) preprocess_bwd_kernel(
    const FrameDev f, const PeerTable pt, const float *__restrict__ means3D, const float *__restrict__ shs, const float *__restrict__ colors_precomp,
    const float *__restrict__ scales, const float *__restrict__ rotations, const float *__restrict__ cov3D_precomp,
    const int32_t *__restrict__ radii, const GaussRec *__restrict__ rec, const float *__restrict__ grad2d,
    float *__restrict__ dL_dmeans3D, float *__restrict__ dL_dmeans2D, float *__restrict__ dL_dsh, float *__restrict__ dL_dcolors,
    float *__restrict__ dL_dopacity, float *__restrict__ dL_dscales, float *__restrict__ dL_drot, float *__restrict__ dL_dcov3D) {
	extern __shared__ float s_sh[];  // [warps][32][kShRow] when STAGED
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const bool in_range = idx < f.P;
	const size_t i = (size_t)idx;
	const int nsh = f.M * 3;
	const bool visible = in_range && radii[idx] > 0;
	float *srow = STAGED ? (s_sh + ((size_t)warp * 32 + lane) * kShRow) : nullptr;

	if (STAGED && shs != nullptr) {
		// coalesced stage-in of this warp's 32 x nsh block (visible rows only)
		const unsigned vis_mask = __ballot_sync(0xffffffffu, visible);
		const size_t g0 = (size_t)(blockIdx.x * blockDim.x + warp * 32);
		const int rows = (int)min((size_t)32, g0 < (size_t)f.P ? (size_t)f.P - g0 : (size_t)0);
		float *wbase = s_sh + (size_t)warp * 32 * kShRow;
		if ((nsh & 3) == 0) {
			const float4 *src = reinterpret_cast<const float4 *>(shs + g0 * nsh);
			const int n4 = rows * nsh / 4;
			for (int e = lane; e < n4; e += 32) {
				const int row = (4 * e) / nsh, col = (4 * e) - row * nsh;
				if ((vis_mask >> row) & 1u) {
					const float4 v = __ldg(src + e);
					float *d = wbase + row * kShRow + col;
					d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
				}
			}
		} else {
			const float *src = shs + g0 * nsh;
			for (int e = lane; e < rows * nsh; e += 32) {
				const int row = e / nsh, col = e - row * nsh;
				if ((vis_mask >> row) & 1u) wbase[row * kShRow + col] = __ldg(src + e);
			}
		}
		__syncwarp();
	}

	float4 g0v = make_float4(0.f, 0.f, 0.f, 0.f), g1v = g0v, g2v = g0v;
	if (GATHER) {  // (`grad2d` carries the destination masks the forward stored)
		__shared__ RunScratch rs;
		__shared__ float4 s_g[3 * kRunBlock];
		const uint32_t mask = visible ? reinterpret_cast<const uint32_t *>(grad2d)[idx] : 0u;
		gather_runs(pt, mask, rs, s_g, g0v, g1v, g2v);
	}
	if (in_range) {
		if (!GATHER) {
			g0v = reinterpret_cast<const float4 *>(grad2d)[3 * i];      // mean2D.x, .y, .z(abs), conic.xx
			g1v = reinterpret_cast<const float4 *>(grad2d)[3 * i + 1];  // conic.xy, conic.yy, opacity, color.r
			g2v = reinterpret_cast<const float4 *>(grad2d)[3 * i + 2];  // color.g, color.b, depth, pad
		}
		dL_dmeans2D[3 * i] = g0v.x; dL_dmeans2D[3 * i + 1] = g0v.y; dL_dmeans2D[3 * i + 2] = g0v.z;
		dL_dopacity[i] = g1v.z;
		if (dL_dcolors) { dL_dcolors[3 * i] = g1v.w; dL_dcolors[3 * i + 1] = g2v.x; dL_dcolors[3 * i + 2] = g2v.y; }
	}
	const float4 g0 = g0v, g1 = g1v, g2 = g2v;

	if (in_range && !visible) {
		dL_dmeans3D[3 * i] = 0.f; dL_dmeans3D[3 * i + 1] = 0.f; dL_dmeans3D[3 * i + 2] = 0.f;
		if (dL_dscales) { dL_dscales[3 * i] = 0.f; dL_dscales[3 * i + 1] = 0.f; dL_dscales[3 * i + 2] = 0.f; }
		if (dL_drot) reinterpret_cast<float4 *>(dL_drot)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
		if (dL_dcov3D)
			for (int k = 0; k < 6; k++) dL_dcov3D[6 * i + k] = 0.f;
		if (dL_dsh) {
			if (STAGED) {
				for (int k = 0; k < nsh; k++) srow[k] = 0.f;
			} else {
				for (int k = 0; k < nsh; k++) dL_dsh[i * nsh + k] = 0.f;
			}
		}
	}
	if (visible) {
	const float *view = f.view, *proj = f.proj;
	const float3 mean = make_float3(means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]);
	const ShapeIn g = load_shape(idx, scales, rotations, cov3D_precomp);
	float c6[6];
	const float3 s_mod = make_float3(f.mod * g.s.x, f.mod * g.s.y, f.mod * g.s.z);
	const float4 q = g.q;
	M3 R;
	if (cov3D_precomp != nullptr) {
#pragma unroll
		for (int k = 0; k < 6; k++) c6[k] = g.c6[k];
	} else {
		R = quat_rot_colmajor(q);
		cov3d_from_scale_rot(s_mod, R, c6);
	}
	Ewa ewa;
	ewa_cov2d(ewa, mean, f.fx, f.fy, f.tanx, f.tany, c6, view);
	float dcov[6];
	float3 dmean = ewa_cov2d_bwd(ewa, make_float3(g0.w, g1.x, g1.y), f.fx, f.fy, view, dcov);
	if (dL_dcov3D) {
#pragma unroll
		for (int k = 0; k < 6; k++) dL_dcov3D[6 * i + k] = dcov[k];
	}
	add_to(dmean, mean2d_bwd(mean, proj, g0.x, g0.y));
	add_to(dmean, depth_bwd(mean, view, g2.z));

	// ---- SH backward (reference backward.cu:20-139) ----
	if (shs != nullptr) {
		const float *sh = STAGED ? srow : shs + i * nsh;
		float *dsh = STAGED ? srow : dL_dsh + i * nsh;
		const uint32_t clamp_bits = __float_as_uint(rec[idx].q2.w) & 7u;  // (the fused forward keeps the radius in the upper bits)
		const float3 campos = make_float3(f.campos[0], f.campos[1], f.campos[2]);
		const float3 dir_orig = make_float3(mean.x - campos.x, mean.y - campos.y, mean.z - campos.z);
		const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
		const float x = dir_orig.x / len, y = dir_orig.y / len, z = dir_orig.z / len;
		float dRGB[3] = {g1.w, g2.x, g2.y};
		dRGB[0] *= (clamp_bits & 1u) ? 0 : 1;
		dRGB[1] *= (clamp_bits & 2u) ? 0 : 1;
		dRGB[2] *= (clamp_bits & 4u) ? 0 : 1;
		const int deg = f.D;
		const int ncoef = min(f.M, (deg + 1) * (deg + 1));
		float ddir[3] = {0.f, 0.f, 0.f};
		// coefficients beyond the active degree receive zero gradient
		for (int k = ncoef * 3; k < nsh; k++) dsh[k] = 0.f;
#pragma unroll
		for (int ch = 0; ch < 3; ch++) {
			// all coefficients of this channel are read before any gradient is written: sh and dsh may alias (staged rows)
			float cf[16];
#pragma unroll
			for (int k = 0; k < 16; k++) cf[k] = k < ncoef ? sh[k * 3 + ch] : 0.f;
#define SHC(k) cf[k]
#define DSH(k) dsh[(k) * 3 + ch]
			const float g = dRGB[ch];
			float dx = 0.f, dy = 0.f, dz = 0.f;
			DSH(0) = kC0 * g;
			if (deg > 0 && ncoef >= 4) {
				DSH(1) = (-kC1 * y) * g; DSH(2) = (kC1 * z) * g; DSH(3) = (-kC1 * x) * g;
				dx = -kC1 * SHC(3); dy = -kC1 * SHC(1); dz = kC1 * SHC(2);
				if (deg > 1 && ncoef >= 9) {
					const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
					DSH(4) = (kC2[0] * xy) * g; DSH(5) = (kC2[1] * yz) * g; DSH(6) = (kC2[2] * (2.f * zz - xx - yy)) * g;
					DSH(7) = (kC2[3] * xz) * g; DSH(8) = (kC2[4] * (xx - yy)) * g;
					dx += kC2[0] * y * SHC(4) + kC2[2] * 2.f * -x * SHC(6) + kC2[3] * z * SHC(7) + kC2[4] * 2.f * x * SHC(8);
					dy += kC2[0] * x * SHC(4) + kC2[1] * z * SHC(5) + kC2[2] * 2.f * -y * SHC(6) + kC2[4] * 2.f * -y * SHC(8);
					dz += kC2[1] * y * SHC(5) + kC2[2] * 2.f * 2.f * z * SHC(6) + kC2[3] * x * SHC(7);
					if (deg > 2 && ncoef >= 16) {
						DSH(9) = (kC3[0] * y * (3.f * xx - yy)) * g; DSH(10) = (kC3[1] * xy * z) * g;
						DSH(11) = (kC3[2] * y * (4.f * zz - xx - yy)) * g; DSH(12) = (kC3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy)) * g;
						DSH(13) = (kC3[4] * x * (4.f * zz - xx - yy)) * g; DSH(14) = (kC3[5] * z * (xx - yy)) * g;
						DSH(15) = (kC3[6] * x * (xx - 3.f * yy)) * g;
						dx += (kC3[0] * SHC(9) * 3.f * 2.f * xy + kC3[1] * SHC(10) * yz + kC3[2] * SHC(11) * -2.f * xy +
						       kC3[3] * SHC(12) * -3.f * 2.f * xz + kC3[4] * SHC(13) * (-3.f * xx + 4.f * zz - yy) +
						       kC3[5] * SHC(14) * 2.f * xz + kC3[6] * SHC(15) * 3.f * (xx - yy));
						dy += (kC3[0] * SHC(9) * 3.f * (xx - yy) + kC3[1] * SHC(10) * xz + kC3[2] * SHC(11) * (-3.f * yy + 4.f * zz - xx) +
						       kC3[3] * SHC(12) * -3.f * 2.f * yz + kC3[4] * SHC(13) * -2.f * xy + kC3[5] * SHC(14) * -2.f * yz +
						       kC3[6] * SHC(15) * -3.f * 2.f * xy);
						dz += (kC3[1] * SHC(10) * xy + kC3[2] * SHC(11) * 4.f * 2.f * yz + kC3[3] * SHC(12) * 3.f * (2.f * zz - xx - yy) +
						       kC3[4] * SHC(13) * 4.f * 2.f * xz + kC3[5] * SHC(14) * (xx - yy));
					}
				}
			}
#undef SHC
#undef DSH
			ddir[0] += dx * g; ddir[1] += dy * g; ddir[2] += dz * g;
		}
		add_to(dmean, dnormvdv(dir_orig, make_float3(ddir[0], ddir[1], ddir[2])));
	}
	dL_dmeans3D[3 * i] = dmean.x; dL_dmeans3D[3 * i + 1] = dmean.y; dL_dmeans3D[3 * i + 2] = dmean.z;

	if (cov3D_precomp == nullptr) {
		float3 dscale;
		float4 dq;
		cov3d_bwd(s_mod, q, R, dcov, dscale, dq);
		dL_dscales[3 * i] = dscale.x; dL_dscales[3 * i + 1] = dscale.y; dL_dscales[3 * i + 2] = dscale.z;
		reinterpret_cast<float4 *>(dL_drot)[i] = dq;
	}
	}  // visible

	if (STAGED && dL_dsh != nullptr) {
		// coalesced stage-out of the warp's 32 x nsh gradient block (rows of culled Gaussians were zero-filled above)
		__syncwarp();
		const size_t g0s = (size_t)(blockIdx.x * blockDim.x + warp * 32);
		const int rows = (int)min((size_t)32, g0s < (size_t)f.P ? (size_t)f.P - g0s : (size_t)0);
		const float *wbase = s_sh + (size_t)warp * 32 * kShRow;
		if ((nsh & 3) == 0) {
			float4 *dst = reinterpret_cast<float4 *>(dL_dsh + g0s * nsh);
			const int n4 = rows * nsh / 4;
			for (int e = lane; e < n4; e += 32) {
				const int row = (4 * e) / nsh, col = (4 * e) - row * nsh;
				const float *sp = wbase + row * kShRow + col;
				dst[e] = make_float4(sp[0], sp[1], sp[2], sp[3]);
			}
		} else {
			float *dst = dL_dsh + g0s * nsh;
			for (int e = lane; e < rows * nsh; e += 32) {
				const int row = e / nsh, col = e - row * nsh;
				dst[e] = wbase[row * kShRow + col];
			}
		}
	}
}

// ---------------------------------------------------------------------------------------------------------------------------------
// TMA variant (rows of 12*M bytes with M in {4, 8, 12, 16}, 16-B aligned: SH degree 1 and 3).  Same geometry functions as the kernel
// above; what changes is how the two big streams of this kernel — the SH coefficients in (12M B per Gaussian) and their gradients out
// (12M B) — move:
//   * at the very top every lane issues ONE cp.async.bulk of its coefficient row into a padded shared-memory row (stride
//     kBwdStride floats = 208 B: 16-B aligned for TMA / LDS.128, and 13 x 16 B so the 8 lanes of a quarter-warp hit 8 distinct
//     16-B bank groups); one mbarrier per warp counts the bytes.  The round-1 kernel staged the block with a per-lane loop of
//     "load 16 B, store to shared" — one DRAM round trip per iteration, 12 iterations; the profiler's source view put a large share of
//     the warp stalls on those two STS, and the padded-row scalar stores caused bank conflicts;
//   * every other per-Gaussian input (radius, the 12 screen-space sums, position, scale, rotation, clamp bits) is requested before
//     any arithmetic, so the whole kernel waits for DRAM once;
//   * the SH backward runs IN PLACE on the row with LDS.128 / STS.128 (coefficient e = 3k + ch of float4 j = e / 4 is read, its
//     contribution to d colour / d direction accumulated, and its gradient basis_k * dL/dRGB[ch] written back to the same slot);
//   * each lane then issues ONE cp.async.bulk shared -> global of its gradient row (zeros for culled Gaussians).
template <bool GATHER>
__global__ void __launch_bounds__(256, 3) preprocess_bwd_tma_kernel(
    const FrameDev f, const PeerTable pt, const float *__restrict__ means3D, const float *__restrict__ shs, const float *__restrict__ scales,
    const float *__restrict__ rotations, const float *__restrict__ cov3D_precomp, const int32_t *__restrict__ radii,
    const GaussRec *__restrict__ rec, const float *__restrict__ grad2d, float *__restrict__ dL_dmeans3D, float *__restrict__ dL_dmeans2D,
    float *__restrict__ dL_dsh, float *__restrict__ dL_dopacity, float *__restrict__ dL_dscales, float *__restrict__ dL_drot,
    float *__restrict__ dL_dcov3D) {
	extern __shared__ __align__(16) unsigned char s_stage[];
	__shared__ float s_cam[36];
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const bool in_range = idx < f.P;
	const size_t i = (size_t)idx;
	const int nsh = f.M * 3;
	const uint32_t row_bytes = (uint32_t)nsh * 4u;
	const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(s_stage);
	const uint32_t row = sbase + (uint32_t)((warp * 32 + lane) * kBwdStride) * 4u;
	const uint32_t bar = sbase + (uint32_t)(8 * 32 * kBwdStride) * 4u + (uint32_t)warp * 8u;
	const int first = blockIdx.x * blockDim.x + warp * 32;
	const int rows = min(32, f.P - first);
	if (rows > 0) {
		if (lane == 0) {
			mbar_init(bar, 1);
			fence_proxy_async();
		}
		__syncwarp();
		if (in_range) bulk_g2s(row, shs + i * nsh, row_bytes, bar);
		if (lane == 0) mbar_expect_tx(bar, row_bytes * (uint32_t)rows);
	}
	// ---- every small input up front ----
	int radius = 0;
	float4 g0v = make_float4(0.f, 0.f, 0.f, 0.f), g1v = g0v, g2v = g0v;
	float3 mean = make_float3(0.f, 0.f, 0.f);
	float3 sc = make_float3(0.f, 0.f, 0.f);
	float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
	float c6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
	uint32_t clamp_bits = 0u;
	if (in_range) {
		radius = radii[idx];
		mean = make_float3(means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]);
		if (cov3D_precomp != nullptr) {
#pragma unroll
			for (int k = 0; k < 6; k++) c6[k] = cov3D_precomp[6 * i + k];
		} else {
			q = *reinterpret_cast<const float4 *>(rotations + 4 * i);
			sc = make_float3(scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]);
		}
		clamp_bits = __float_as_uint(rec[idx].q2.w) & 7u;  // (the fused forward keeps the radius in the upper bits)
		if (!GATHER) {
			g0v = reinterpret_cast<const float4 *>(grad2d)[3 * i];      // mean2D.x, .y, .z(abs), conic.xx
			g1v = reinterpret_cast<const float4 *>(grad2d)[3 * i + 1];  // conic.xy, conic.yy, opacity, color.r
			g2v = reinterpret_cast<const float4 *>(grad2d)[3 * i + 2];  // color.g, color.b, depth, pad
		}
	}
	if (threadIdx.x < 16) s_cam[threadIdx.x] = f.view[threadIdx.x];
	else if (threadIdx.x < 32) s_cam[threadIdx.x] = f.proj[threadIdx.x - 16];
	else if (threadIdx.x < 35) s_cam[threadIdx.x] = f.campos[threadIdx.x - 32];
	__syncthreads();
	const float *view = s_cam, *proj = s_cam + 16;
	const bool visible = in_range && radius > 0;
	if (GATHER) {  // (`grad2d` carries the destination masks the forward stored)
		__shared__ RunScratch rs;
		__shared__ float4 s_g[3 * kRunBlock];
		const uint32_t mask = visible ? reinterpret_cast<const uint32_t *>(grad2d)[idx] : 0u;
		gather_runs(pt, mask, rs, s_g, g0v, g1v, g2v);
	}
	const float4 g0 = g0v, g1 = g1v, g2 = g2v;
	if (in_range) {
		dL_dmeans2D[3 * i] = g0.x; dL_dmeans2D[3 * i + 1] = g0.y; dL_dmeans2D[3 * i + 2] = g0.z;
		dL_dopacity[i] = g1.z;
	}
	float3 dmean = make_float3(0.f, 0.f, 0.f);
	float dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
	float3 dscale = make_float3(0.f, 0.f, 0.f);
	float4 dq = make_float4(0.f, 0.f, 0.f, 0.f);
	float dRGB[3] = {0.f, 0.f, 0.f};
	float3 dir_orig = make_float3(0.f, 0.f, 1.f);
	if (visible) {
		float3 s_mod = make_float3(f.mod * sc.x, f.mod * sc.y, f.mod * sc.z);
		M3 R;
		if (cov3D_precomp == nullptr) {
			R = quat_rot_colmajor(q);
			cov3d_from_scale_rot(s_mod, R, c6);
		}
		Ewa ewa;
		ewa_cov2d(ewa, mean, f.fx, f.fy, f.tanx, f.tany, c6, view);
		dmean = ewa_cov2d_bwd(ewa, make_float3(g0.w, g1.x, g1.y), f.fx, f.fy, view, dcov);
		add_to(dmean, mean2d_bwd(mean, proj, g0.x, g0.y));
		add_to(dmean, depth_bwd(mean, view, g2.z));
		if (cov3D_precomp == nullptr) cov3d_bwd(s_mod, q, R, dcov, dscale, dq);
		dRGB[0] = (clamp_bits & 1u) ? 0.f : g1.w;
		dRGB[1] = (clamp_bits & 2u) ? 0.f : g2.x;
		dRGB[2] = (clamp_bits & 4u) ? 0.f : g2.y;
		dir_orig = make_float3(mean.x - s_cam[32], mean.y - s_cam[33], mean.z - s_cam[34]);
	}
	if (in_range) {
		if (dL_dscales) { dL_dscales[3 * i] = dscale.x; dL_dscales[3 * i + 1] = dscale.y; dL_dscales[3 * i + 2] = dscale.z; }
		if (dL_drot) reinterpret_cast<float4 *>(dL_drot)[i] = dq;
		if (dL_dcov3D) {
#pragma unroll
			for (int k = 0; k < 6; k++) dL_dcov3D[6 * i + k] = dcov[k];
		}
	}
	// ---- SH backward in place on the staged row (reference backward.cu:20-139) ----
	if (rows > 0) mbar_wait(bar, 0);  // the warp's rows have landed; nobody may touch (or abandon) the stage before this
	if (in_range) {
		const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
		const float x = dir_orig.x / len, y = dir_orig.y / len, z = dir_orig.z / len;
		const int deg = f.D;
		const int ncoef = visible ? min(f.M, (deg + 1) * (deg + 1)) : 0;  // culled: every gradient 0
		// basis_k and its partial derivatives w.r.t. the unit direction; coefficients beyond the active degree get zeros
		float B[16], Bx[16], By[16], Bz[16];
#pragma unroll
		for (int k = 0; k < 16; k++) { B[k] = 0.f; Bx[k] = 0.f; By[k] = 0.f; Bz[k] = 0.f; }
		const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
		if (ncoef >= 1) B[0] = kC0;
		if (deg > 0 && ncoef >= 4) {
			B[1] = -kC1 * y; B[2] = kC1 * z; B[3] = -kC1 * x;
			By[1] = -kC1; Bz[2] = kC1; Bx[3] = -kC1;
		}
		if (deg > 1 && ncoef >= 9) {
			B[4] = kC2[0] * xy; B[5] = kC2[1] * yz; B[6] = kC2[2] * (2.f * zz - xx - yy); B[7] = kC2[3] * xz; B[8] = kC2[4] * (xx - yy);
			Bx[4] = kC2[0] * y; By[4] = kC2[0] * x;
			By[5] = kC2[1] * z; Bz[5] = kC2[1] * y;
			Bx[6] = kC2[2] * 2.f * -x; By[6] = kC2[2] * 2.f * -y; Bz[6] = kC2[2] * 2.f * 2.f * z;
			Bx[7] = kC2[3] * z; Bz[7] = kC2[3] * x;
			Bx[8] = kC2[4] * 2.f * x; By[8] = kC2[4] * 2.f * -y;
		}
		if (deg > 2 && ncoef >= 16) {
			B[9] = kC3[0] * y * (3.f * xx - yy); B[10] = kC3[1] * xy * z; B[11] = kC3[2] * y * (4.f * zz - xx - yy);
			B[12] = kC3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy); B[13] = kC3[4] * x * (4.f * zz - xx - yy); B[14] = kC3[5] * z * (xx - yy);
			B[15] = kC3[6] * x * (xx - 3.f * yy);
			Bx[9] = kC3[0] * 3.f * 2.f * xy; By[9] = kC3[0] * 3.f * (xx - yy);
			Bx[10] = kC3[1] * yz; By[10] = kC3[1] * xz; Bz[10] = kC3[1] * xy;
			Bx[11] = kC3[2] * -2.f * xy; By[11] = kC3[2] * (-3.f * yy + 4.f * zz - xx); Bz[11] = kC3[2] * 4.f * 2.f * yz;
			Bx[12] = kC3[3] * -3.f * 2.f * xz; By[12] = kC3[3] * -3.f * 2.f * yz; Bz[12] = kC3[3] * 3.f * (2.f * zz - xx - yy);
			Bx[13] = kC3[4] * (-3.f * xx + 4.f * zz - yy); By[13] = kC3[4] * -2.f * xy; Bz[13] = kC3[4] * 4.f * 2.f * xz;
			Bx[14] = kC3[5] * 2.f * xz; By[14] = kC3[5] * -2.f * yz; Bz[14] = kC3[5] * (xx - yy);
			Bx[15] = kC3[6] * 3.f * (xx - yy); By[15] = kC3[6] * -3.f * 2.f * xy;
		}
		float ddx = 0.f, ddy = 0.f, ddz = 0.f;
#pragma unroll
		for (int j = 0; j < 12; j++) {
			if (4 * j < nsh) {
				float4 v;
				asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(row + 16u * j));
				const float cv[4] = {v.x, v.y, v.z, v.w};
				float o[4];
#pragma unroll
				for (int tt = 0; tt < 4; tt++) {
					const int e = 4 * j + tt, k = e / 3, ch = e % 3;  // compile-time after unrolling
					const float cg = cv[tt] * dRGB[ch];
					ddx += Bx[k] * cg; ddy += By[k] * cg; ddz += Bz[k] * cg;
					o[tt] = B[k] * dRGB[ch];
				}
				asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(row + 16u * j), "f"(o[0]), "f"(o[1]), "f"(o[2]), "f"(o[3]) : "memory");
			}
		}
		if (visible) add_to(dmean, dnormvdv(dir_orig, make_float3(ddx, ddy, ddz)));
		dL_dmeans3D[3 * i] = dmean.x; dL_dmeans3D[3 * i + 1] = dmean.y; dL_dmeans3D[3 * i + 2] = dmean.z;
		// this lane's gradient row leaves through the async proxy
		fence_proxy_async();
		bulk_s2g(dL_dsh + i * nsh, row, row_bytes);
		bulk_commit();
		bulk_wait_all_read();  // the stage must stay intact until the copy engine has read it (the CTA may exit right after)
	}
}

static bool bwd_rows_fit_tma(const FrameDev &f, const float *shs, const float *dL_dsh) {
	static const bool disabled = getenv("SGR_NO_TMA") != nullptr;
	if (disabled) return false;
	return shs != nullptr && dL_dsh != nullptr && f.M > 0 && f.M <= 16 && (f.M * 12) % 16 == 0 && (reinterpret_cast<uintptr_t>(shs) & 15u) == 0 &&
	       (reinterpret_cast<uintptr_t>(dL_dsh) & 15u) == 0;
}
constexpr size_t kBwdStageBytes = (size_t)8 * 32 * kBwdStride * sizeof(float) + 8 * sizeof(uint64_t);

cudaError_t launch_preprocess_bwd(const FrameDev &f, const PeerTable *pt, const float *means3D, const float *shs, const float *colors_precomp,
                                  const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                                  const GaussRec *rec, const float *grad2d, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh,
                                  float *dL_dcolors, float *dL_dopacity, float *dL_dscales, float *dL_drot, float *dL_dcov3D, cudaStream_t st) {
	if (f.P == 0) return cudaSuccess;
	const bool gather = pt != nullptr;  // pt == nullptr: the local path, grad2d holds this process's screen-space sums
	const PeerTable peers = gather ? *pt : PeerTable{};
	const unsigned grid = (unsigned)((f.P + 255) / 256);
	cudaError_t e;
	if (bwd_rows_fit_tma(f, shs, dL_dsh)) {
		static std::atomic<uint64_t> configured[2];
		const auto kernel = gather ? preprocess_bwd_tma_kernel<true> : preprocess_bwd_tma_kernel<false>;
		if ((e = ensure_dynamic_smem(kernel, (int)kBwdStageBytes, configured[gather])) != cudaSuccess) return e;
		count_launch();
		kernel<<<grid, 256, kBwdStageBytes, st>>>(f, peers, means3D, shs, scales, rotations, cov3D_precomp, radii, rec, grad2d, dL_dmeans3D,
		                                          dL_dmeans2D, dL_dsh, dL_dopacity, dL_dscales, dL_drot, dL_dcov3D);
		return cudaGetLastError();
	}
	const bool staged = shs != nullptr && f.M <= 16;  // rows of up to 48 floats fit the padded smem row
	const auto kernel = staged ? (gather ? preprocess_bwd_kernel<true, true> : preprocess_bwd_kernel<true, false>)
	                           : (gather ? preprocess_bwd_kernel<false, true> : preprocess_bwd_kernel<false, false>);
	const size_t smem = staged ? (size_t)8 * 32 * kShRow * sizeof(float) : 0;  // 50,176 B: above the 48 KB static limit -> opt in
	if (staged) {
		static std::atomic<uint64_t> configured[2];
		if ((e = ensure_dynamic_smem(kernel, (int)smem, configured[gather])) != cudaSuccess) return e;
	}
	count_launch();
	kernel<<<grid, 256, smem, st>>>(f, peers, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii, rec, grad2d, dL_dmeans3D,
	                                dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drot, dL_dcov3D);
	return cudaGetLastError();
}

}  // namespace sgr
