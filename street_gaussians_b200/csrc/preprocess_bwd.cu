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
//   * the SH coefficients are NOT read: dL/dsh = B_k(dir) dL/dRGB needs only the view direction, and dL/ddir = J^T dL/dRGB takes
//     the colour Jacobian J (3 x 3, with the clamp bits) that the forward stored while it held the coefficient row — 48 B per
//     visible Gaussian instead of the 12 M-byte row plus a sector of the blend record;
//   * SH gradients out are staged through shared memory per warp: the 32 Gaussians of a warp own one contiguous 32 x M x 3
//     float block of `dL_dsh`, which leaves with fully coalesced 16-B stores (rows padded to 49 floats in smem so the per-thread
//     row writes are bank-conflict free).  Direct per-thread stores (48 strided scalar stores per Gaussian) waste most of each
//     memory transaction.
// Formulas and evaluation order follow the reference so gradients agree to fp32 rounding.  The geometry (covariances, EWA
// Jacobian, projective divide, depth, scale / rotation) and the SH basis and colour Jacobian are gaussian_geom.cuh's, the same
// functions the forward calls; the two kernels below differ in how they load their inputs, the gather and their stores.
#include <cstdlib>

#include "gaussian_geom.cuh"

namespace sgr {

constexpr int kShRow = 49;  // padded smem row (floats) for up to 16 x 3 SH coefficients
constexpr int kBwdStride = 52;  // row stride (floats) of the TMA variant's stage: 208 B

// reached (nullable, !GATHER only): the forward's reached words (GeomView::reached).  A Gaussian without one loads nothing but its word
// and writes zeros: its grad2d row may hold anything (launch_blend_bwd cleared only the reached rows), and with a zero row and finite
// inputs its chain rule gives zeros (+-0) anyway — the forward marked every visible Gaussian whose inputs are not all finite.
// GATHER = true (sgr_sharded_backward): grad2d is not a local array — the 12 sums of local Gaussian idx (global id
// rank*chunk + idx) are read from the partial grad2d of every rank whose cyclic band its rectangle meets (NVLink peer loads)
// and added in ascending rank order, exactly what sgr_gather_grad2d produced as a separate pass.
template <bool STAGED, bool GATHER = false>
__global__ void __launch_bounds__(256) preprocess_bwd_kernel(
    const FrameDev f, const PeerTable pt, const float *__restrict__ means3D, const float *__restrict__ shs, const float *__restrict__ colors_precomp,
    const float *__restrict__ scales, const float *__restrict__ rotations, const float *__restrict__ cov3D_precomp,
    const int32_t *__restrict__ radii, const float4 *__restrict__ jac, const float *__restrict__ grad2d,
    float *__restrict__ dL_dmeans3D, float *__restrict__ dL_dmeans2D, float *__restrict__ dL_dsh, float *__restrict__ dL_dcolors,
    float *__restrict__ dL_dopacity, float *__restrict__ dL_dscales, float *__restrict__ dL_drot, float *__restrict__ dL_dcov3D,
    const uint32_t *__restrict__ reached) {
	extern __shared__ float s_sh[];  // [warps][32][kShRow] when STAGED
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const bool in_range = idx < f.P;
	const bool need = in_range && (GATHER || reached == nullptr || reached[idx] != 0u);
	const size_t i = (size_t)idx;
	const int nsh = f.M * 3;
	const bool visible = need && radii[idx] > 0;
	float *srow = STAGED ? (s_sh + ((size_t)warp * 32 + lane) * kShRow) : nullptr;

	float4 g0v = make_float4(0.f, 0.f, 0.f, 0.f), g1v = g0v, g2v = g0v;
	if (GATHER) {  // (`grad2d` carries the destination masks the forward stored)
		__shared__ RunScratch rs;
		__shared__ float4 s_g[3 * kRunBlock];
		const uint32_t mask = visible ? reinterpret_cast<const uint32_t *>(grad2d)[idx] : 0u;
		gather_runs(pt, mask, rs, s_g, g0v, g1v, g2v);
	}
	if (in_range) {
		if (!GATHER && need) {
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

	// ---- SH backward (reference backward.cu:20-139) from the direction basis and the forward's colour Jacobian ----
	if (shs != nullptr) {
		float *dsh = STAGED ? srow : dL_dsh + i * nsh;
		const ColorJac cj = load_color_jac(jac + 3 * i);
		const float3 campos = make_float3(f.campos[0], f.campos[1], f.campos[2]);
		const float3 dir_orig = make_float3(mean.x - campos.x, mean.y - campos.y, mean.z - campos.z);
		const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
		const float x = dir_orig.x / len, y = dir_orig.y / len, z = dir_orig.z / len;
		float dRGB[3];
		masked_drgb(cj, g1.w, g2.x, g2.y, dRGB);
		const int ncoef = min(f.M, (f.D + 1) * (f.D + 1));
		float B[16];
		sh_basis(f.D, x, y, z, B);
		// coefficients beyond the active degree receive +0 gradient
#pragma unroll
		for (int e = 0; e < 48; e++)
			if (e < nsh) dsh[e] = e / 3 < ncoef ? B[e / 3] * dRGB[e % 3] : 0.f;
		for (int e = 48; e < nsh; e++) dsh[e] = 0.f;
		add_to(dmean, dnormvdv(dir_orig, color_jac_dir_grad(cj, dRGB)));
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
// above; what changes is how the biggest stream of this kernel — the SH gradients out (12M B per Gaussian) — leaves, and the load order:
//   * every per-Gaussian input (radius, the 12 screen-space sums, position, scale, rotation, and for visible Gaussians the colour
//     Jacobian) is requested before any arithmetic, so the kernel waits for DRAM about once;
//   * each lane writes its gradient row basis_k * dL/dRGB[ch] with STS.128 into a padded shared-memory row (stride kBwdStride floats
//     = 208 B: 16-B aligned for the bulk copy, and 13 x 16 B so the 8 lanes of a quarter-warp hit 8 distinct 16-B bank groups) and
//     issues ONE cp.async.bulk shared -> global of it (zeros for culled Gaussians).
template <bool GATHER>
__global__ void __launch_bounds__(256, 3) preprocess_bwd_tma_kernel(
    const FrameDev f, const PeerTable pt, const float *__restrict__ means3D, const float *__restrict__ scales,
    const float *__restrict__ rotations, const float *__restrict__ cov3D_precomp, const int32_t *__restrict__ radii,
    const float4 *__restrict__ jac, const float *__restrict__ grad2d, float *__restrict__ dL_dmeans3D, float *__restrict__ dL_dmeans2D,
    float *__restrict__ dL_dsh, float *__restrict__ dL_dopacity, float *__restrict__ dL_dscales, float *__restrict__ dL_drot,
    float *__restrict__ dL_dcov3D, const uint32_t *__restrict__ reached) {
	extern __shared__ __align__(16) unsigned char s_stage[];
	__shared__ float s_cam[36];
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const bool in_range = idx < f.P;
	// (an unreached Gaussian keeps radius 0 below: every gradient it writes is then the zero of a culled one)
	const bool need = in_range && (GATHER || reached == nullptr || reached[idx] != 0u);
	const size_t i = (size_t)idx;
	const int nsh = f.M * 3;
	const uint32_t row_bytes = (uint32_t)nsh * 4u;
	const uint32_t row = (uint32_t)__cvta_generic_to_shared(s_stage) + (uint32_t)((warp * 32 + lane) * kBwdStride) * 4u;
	// ---- every input up front ----
	int radius = 0;
	float4 g0v = make_float4(0.f, 0.f, 0.f, 0.f), g1v = g0v, g2v = g0v;
	float3 mean = make_float3(0.f, 0.f, 0.f);
	float3 sc = make_float3(0.f, 0.f, 0.f);
	float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
	float c6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
	ColorJac cj = {g0v, g0v, g0v};
	if (need) {
		radius = radii[idx];
		mean = make_float3(means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]);
		if (cov3D_precomp != nullptr) {
#pragma unroll
			for (int k = 0; k < 6; k++) c6[k] = cov3D_precomp[6 * i + k];
		} else {
			q = *reinterpret_cast<const float4 *>(rotations + 4 * i);
			sc = make_float3(scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]);
		}
		if (!GATHER) {
			g0v = reinterpret_cast<const float4 *>(grad2d)[3 * i];      // mean2D.x, .y, .z(abs), conic.xx
			g1v = reinterpret_cast<const float4 *>(grad2d)[3 * i + 1];  // conic.xy, conic.yy, opacity, color.r
			g2v = reinterpret_cast<const float4 *>(grad2d)[3 * i + 2];  // color.g, color.b, depth, pad
		}
		// (the forward writes it for visible Gaussians only; the gather keeps it out of its registers)
		if (!GATHER && radius > 0) cj = load_color_jac(jac + 3 * i);
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
		if (visible) cj = load_color_jac(jac + 3 * i);
	}
	const float4 g0 = g0v, g1 = g1v, g2 = g2v;
	if (in_range) {
		dL_dmeans2D[3 * i] = g0.x; dL_dmeans2D[3 * i + 1] = g0.y; dL_dmeans2D[3 * i + 2] = g0.z;
		dL_dopacity[i] = g1.z;
	}
	// the colour terms first: 6 live floats instead of the 12 of the Jacobian through the geometry below
	float dRGB[3] = {0.f, 0.f, 0.f};
	float3 ddir = make_float3(0.f, 0.f, 0.f);
	if (visible) {
		masked_drgb(cj, g1.w, g2.x, g2.y, dRGB);
		ddir = color_jac_dir_grad(cj, dRGB);
	}
	float3 dmean = make_float3(0.f, 0.f, 0.f);
	float dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
	float3 dscale = make_float3(0.f, 0.f, 0.f);
	float4 dq = make_float4(0.f, 0.f, 0.f, 0.f);
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
	// ---- SH backward (reference backward.cu:20-139) into the staged row ----
	if (in_range) {
		const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
		const float x = dir_orig.x / len, y = dir_orig.y / len, z = dir_orig.z / len;
		const int ncoef = visible ? min(f.M, (f.D + 1) * (f.D + 1)) : 0;  // culled: every gradient 0
		float B[16];
		sh_basis(f.D, x, y, z, B);
#pragma unroll
		for (int j = 0; j < 12; j++) {
			if (4 * j < nsh) {
				float o[4];
#pragma unroll
				for (int tt = 0; tt < 4; tt++) {
					const int e = 4 * j + tt, k = e / 3, ch = e % 3;  // compile-time after unrolling
					// coefficients beyond the active degree get +0 (B[k] = 0 times a negative dL/dRGB would store -0)
					o[tt] = k < ncoef ? B[k] * dRGB[ch] : 0.f;
				}
				asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(row + 16u * j), "f"(o[0]), "f"(o[1]), "f"(o[2]), "f"(o[3]) : "memory");
			}
		}
		if (visible) add_to(dmean, dnormvdv(dir_orig, ddir));
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
constexpr size_t kBwdStageBytes = (size_t)8 * 32 * kBwdStride * sizeof(float);

cudaError_t launch_preprocess_bwd(const FrameDev &f, const PeerTable *pt, const float *means3D, const float *shs, const float *colors_precomp,
                                  const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                                  const float4 *jac, const float *grad2d, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh,
                                  float *dL_dcolors, float *dL_dopacity, float *dL_dscales, float *dL_drot, float *dL_dcov3D, cudaStream_t st,
                                  const uint32_t *reached) {
	if (f.P == 0) return cudaSuccess;
	const bool gather = pt != nullptr;  // pt == nullptr: the local path, grad2d holds this process's screen-space sums
	if (gather) reached = nullptr;      // (the gathered sums come from other ranks' emissions)
	const PeerTable peers = gather ? *pt : PeerTable{};
	const unsigned grid = (unsigned)((f.P + 255) / 256);
	cudaError_t e;
	if (bwd_rows_fit_tma(f, shs, dL_dsh)) {
		static std::atomic<uint64_t> configured[2];
		const auto kernel = gather ? preprocess_bwd_tma_kernel<true> : preprocess_bwd_tma_kernel<false>;
		if ((e = ensure_dynamic_smem(kernel, (int)kBwdStageBytes, configured[gather])) != cudaSuccess) return e;
		count_launch();
		kernel<<<grid, 256, kBwdStageBytes, st>>>(f, peers, means3D, scales, rotations, cov3D_precomp, radii, jac, grad2d, dL_dmeans3D,
		                                          dL_dmeans2D, dL_dsh, dL_dopacity, dL_dscales, dL_drot, dL_dcov3D, reached);
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
	kernel<<<grid, 256, smem, st>>>(f, peers, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii, jac, grad2d, dL_dmeans3D,
	                                dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drot, dL_dcov3D, reached);
	return cudaGetLastError();
}

}  // namespace sgr
