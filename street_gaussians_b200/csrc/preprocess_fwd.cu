// preprocess_fwd.cu — per-Gaussian forward stage: project, EWA covariance, conic, radius, SH -> RGB, exact tile count.
//
// One thread per Gaussian (HBM-bound; algorithmic bytes per Gaussian in DESIGN.md §4).  Replaces the reference's
// preprocessCUDA / filter_preprocessCUDA / checkFrustum (DGR/cuda_rasterizer/forward.cu:155-334,
// rasterizer_impl.cu:54-66).  The arithmetic keeps the reference's expression shapes so that depth, conic, radius and
// RGB are bit-equal (the tile sort key is the raw depth bits; a 1-ulp difference could swap two splats).
//
// What is new relative to the reference: (1) the packed 48-B GaussRec output, (2) cov3D is not stored (backward
// recomputes it), (3) tiles_touched counts only the tiles of the 3-sigma rectangle that can actually receive a
// contribution (exact opacity-aware row-span cull, tile_visit.cuh) and that lie in this process's tile-row band,
// (4) large rectangles are counted warp-cooperatively instead of by one thread, (5) a 32-bit depth key per Gaussian
// feeds the depth pre-sort of binning.cu, (6) the SH colour's 3 x 3 direction Jacobian (+ clamp bits) is stored for the backward,
// which then never reads the coefficient rows, (7) the reached word (GeomView::reached) starts here: 1 for a visible Gaussian whose
// chain-rule inputs (position, shape, camera, colour Jacobian) are not all finite, so that the backward runs its chain rule on a zero
// row exactly as it runs every other one and turns a non-finite input into the same NaN / Inf; 0 otherwise, until the emission marks it.
// The per-Gaussian geometry it shares with the backward is in gaussian_geom.cuh.
#include "gaussian_geom.cuh"
#include "tile_visit.cuh"

namespace sgr {

struct Projected {
	bool ok;
	float depth, px, py;
	float3 conic;
	int radius;
	int x0, y0, x1, y1;
};

// Shared front half of preprocess / visible_filter: cull, project, conic, radius, tile rectangle.  `view` / `proj` may point at
// a shared-memory copy of the camera matrices.
__device__ __forceinline__ Projected project_gaussian(const FrameDev &f, const float *view, const float *proj, const float3 p, ShapeIn g,
                                                      const bool precomp) {
	Projected o;
	o.ok = false;
	o.radius = 0;
	const float4 p_hom = xform4x4(p, proj);
	const float p_w = 1.0f / (p_hom.w + 0.0000001f);
	const float3 p_proj = make_float3(p_hom.x * p_w, p_hom.y * p_w, p_hom.z * p_w);
	const float3 p_view = xform4x3(p, view);
	if (p_view.z <= 0.2f) return o;  // near cull only (reference auxiliary.h:154)
	float c6[6];
	if (precomp) {
#pragma unroll
		for (int k = 0; k < 6; k++) c6[k] = g.c6[k];
	} else {
		cov3d_from_scale_rot(make_float3(f.mod * g.s.x, f.mod * g.s.y, f.mod * g.s.z), quat_rot_colmajor(g.q), c6);
	}
	Ewa ewa;
	ewa_cov2d(ewa, p, f.fx, f.fy, f.tanx, f.tany, c6, view);
	const float3 cov = ewa.cov;
	const float det = (cov.x * cov.z - cov.y * cov.y);
	if (det == 0.0f) return o;
	const float det_inv = 1.f / det;
	o.conic = make_float3(cov.z * det_inv, -cov.y * det_inv, cov.x * det_inv);
	const float mid = 0.5f * (cov.x + cov.z);
	const float lambda1 = mid + sqrtf(fmaxf(0.1f, mid * mid - det));
	const float lambda2 = mid - sqrtf(fmaxf(0.1f, mid * mid - det));
	const float my_radius = ceilf(3.f * sqrtf(fmaxf(lambda1, lambda2)));
	o.px = ndc2pix(p_proj.x, f.W);
	o.py = ndc2pix(p_proj.y, f.H);
	o.radius = (int)my_radius;
	tile_rect(o.px, o.py, o.radius, f.gx, f.gy, o.x0, o.y0, o.x1, o.y1);
	if ((o.x1 - o.x0) * (o.y1 - o.y0) == 0) {
		o.radius = 0;
		return o;
	}
	o.depth = p_view.z;
	o.ok = true;
	return o;
}

// SH (degree <= 3) -> RGB with +0.5 and clamp-at-zero flags (reference forward.cu:20-71).  c[] holds this Gaussian's
// coefficient row (coefficient-major, RGB innermost), loaded by load_sh_global: each thread walks its own 12*M-byte row in
// global memory, with 16-B loads when the row size is a multiple of 16 B (M = 4, 8, 12, 16).
__device__ __forceinline__ void load_sh_global(float *c, const float *__restrict__ sh, int M, int n) {
	if (((M * 3) & 3) == 0) {
		const float4 *s4 = reinterpret_cast<const float4 *>(sh);
#pragma unroll
		for (int k = 0; k < 12; k++)
			if (4 * k < n) {
				const float4 v = __ldg(s4 + k);
				c[4 * k] = v.x; c[4 * k + 1] = v.y; c[4 * k + 2] = v.z; c[4 * k + 3] = v.w;
			}
	} else {
#pragma unroll
		for (int k = 0; k < 48; k++)
			if (k < n) c[k] = __ldg(sh + k);
	}
}

// (x, y, z) = the unit view direction (mean - campos) / |mean - campos|
__device__ __forceinline__ float3 sh_eval(int deg, const float x, const float y, const float z, const float *c, uint32_t &clamp_bits) {
	float res[3];
#pragma unroll
	for (int ch = 0; ch < 3; ch++) {
#define SHC(k) c[(k) * 3 + ch]
		float r = kC0 * SHC(0);
		if (deg > 0) {
			r = r - kC1 * y * SHC(1) + kC1 * z * SHC(2) - kC1 * x * SHC(3);
			if (deg > 1) {
				const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
				r = r + kC2[0] * xy * SHC(4) + kC2[1] * yz * SHC(5) + kC2[2] * (2.0f * zz - xx - yy) * SHC(6) +
				    kC2[3] * xz * SHC(7) + kC2[4] * (xx - yy) * SHC(8);
				if (deg > 2) {
					r = r + kC3[0] * y * (3.0f * xx - yy) * SHC(9) + kC3[1] * xy * z * SHC(10) +
					    kC3[2] * y * (4.0f * zz - xx - yy) * SHC(11) + kC3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * SHC(12) +
					    kC3[4] * x * (4.0f * zz - xx - yy) * SHC(13) + kC3[5] * z * (xx - yy) * SHC(14) +
					    kC3[6] * x * (xx - 3.0f * yy) * SHC(15);
				}
			}
		}
#undef SHC
		r += 0.5f;
		res[ch] = r;
	}
	clamp_bits = (res[0] < 0 ? 1u : 0u) | (res[1] < 0 ? 2u : 0u) | (res[2] < 0 ? 4u : 0u);
	return make_float3(fmaxf(res[0], 0.0f), fmaxf(res[1], 0.0f), fmaxf(res[2], 0.0f));
}

// COUNT = false: records + radii only (sgr_project; the tile counts are taken after the all-gather, per band)
// SCATTER = true (with COUNT = false): sgr_sharded_forward — the record additionally goes straight from registers into the
// gathered arrays of exactly the ranks whose cyclic tile-row band its 3-sigma rectangle meets (NVLink peer stores), and the
// radius (0 = "not yours") to every rank; threads f.P .. pt.chunk-1 are the padding slots of this rank's chunk.
template <bool COUNT, bool SCATTER = false>
__global__ void __launch_bounds__(256) preprocess_fwd_kernel(const FrameDev f, const PeerTable pt, const float *__restrict__ means3D,
                                                             const float *__restrict__ shs, const float *__restrict__ colors_precomp,
                                                             const float *__restrict__ opacities, const float *__restrict__ scales,
                                                             const float *__restrict__ rotations, const float *__restrict__ cov3D_precomp,
                                                             int32_t *__restrict__ radii, GaussRec *__restrict__ rec,
                                                             float4 *__restrict__ jac, uint32_t *__restrict__ tiles_touched, uint32_t *__restrict__ depth_key,
                                                             uint32_t *__restrict__ iota, uint32_t *__restrict__ reached,
                                                             const size_t cnt_offset = 0) {
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const bool in_range = idx < f.P;
	// every small per-Gaussian input is requested up front, before any arithmetic: one DRAM round trip instead of three
	Projected pr;
	pr.ok = false;
	pr.radius = 0;
	CullParams cp = {};
	float3 p = make_float3(0.f, 0.f, 0.f);
	float opacity = 0.f;
	ShapeIn shape;
	if (in_range) {
		p = make_float3(means3D[3 * (size_t)idx], means3D[3 * (size_t)idx + 1], means3D[3 * (size_t)idx + 2]);
		opacity = opacities[idx];
		shape = load_shape(idx, scales, rotations, cov3D_precomp);
	}
	// camera constants through shared memory: every thread needs all 35 floats, and read through the settings' device pointers
	// they were per-thread global loads at the head of the dependency chain
	__shared__ float s_cam[36];
	if (threadIdx.x < 16) s_cam[threadIdx.x] = f.view[threadIdx.x];
	else if (threadIdx.x < 32) s_cam[threadIdx.x] = f.proj[threadIdx.x - 16];
	else if (threadIdx.x < 35) s_cam[threadIdx.x] = f.campos[threadIdx.x - 32];
	const bool cam_finite = __syncthreads_and(threadIdx.x >= 35 || isfinite(s_cam[threadIdx.x])) &&
	                        isfinite(f.fx + f.fy + f.tanx + f.tany + f.mod);
	if (in_range) pr = project_gaussian(f, s_cam, s_cam + 16, p, shape, cov3D_precomp != nullptr);
	// the inputs of the backward's chain rule (the colour Jacobian's entries are added below): a sum of finite values that overflows
	// marks a Gaussian too, which only costs it the shortcut
	float in_sum = p.x + p.y + p.z;
	if (cov3D_precomp != nullptr) {
#pragma unroll
		for (int k = 0; k < 6; k++) in_sum += shape.c6[k];
	} else {
		in_sum += shape.s.x + shape.s.y + shape.s.z + shape.q.x + shape.q.y + shape.q.z + shape.q.w;
	}
	GaussRec rec_out;
	rec_out.q0 = rec_out.q1 = rec_out.q2 = make_float4(0.f, 0.f, 0.f, 0.f);
	if (in_range) {
		if (pr.ok) {
			float3 rgb;
			uint32_t clamp_bits = 0;
			if (colors_precomp == nullptr) {
				const float3 campos = make_float3(s_cam[32], s_cam[33], s_cam[34]);
				float c[48];
				const int n = min(f.M, (f.D + 1) * (f.D + 1)) * 3;
				load_sh_global(c, shs + (size_t)idx * f.M * 3, f.M, n);
				const float3 d = make_float3(p.x - campos.x, p.y - campos.y, p.z - campos.z);
				const float len = sqrtf(d.x * d.x + d.y * d.y + d.z * d.z);
				const float x = d.x / len, y = d.y / len, z = d.z / len;
				rgb = sh_eval(f.D, x, y, z, c, clamp_bits);
				// the colour's direction Jacobian for the backward, taken while the row is in registers: the backward then reads 48 B
				// per Gaussian instead of the 12 M-byte row
				float J[9];
				sh_color_jacobian(f.D, x, y, z, c, J);
				store_color_jac(jac + 3 * (size_t)idx, J, clamp_bits);
#pragma unroll
				for (int k = 0; k < 9; k++) in_sum += J[k];
			} else {
				rgb = make_float3(colors_precomp[3 * (size_t)idx], colors_precomp[3 * (size_t)idx + 1], colors_precomp[3 * (size_t)idx + 2]);
			}
			GaussRec r;
			cp = make_cull(pr.px, pr.py, pr.conic.x, pr.conic.y, pr.conic.z, opacity);
			r.q0 = make_float4(pr.px, pr.py, pr.conic.x, pr.conic.y);
			r.q1 = make_float4(pr.conic.z, opacity, -0.5f * cp.qmax, pr.depth);
			r.q2 = make_float4(rgb.x, rgb.y, rgb.z, __uint_as_float(clamp_bits));
			if (!SCATTER) rec[idx] = r;
			else rec_out = r;
		}
		radii[idx] = pr.radius;
	}
	if (SCATTER) {
		// Block-run delivery (sgr_common.cuh): the records of this block that rank d needs leave as ONE contiguous run into the block's
		// 256 slots of rank d's gathered array, copied out of shared memory as lane-contiguous 16-B pieces (whole 128-B lines), and the
		// run lengths go to rank d's count table.  Per-lane 48-B stores at the global index and
		// warp-staged lines with per-Gaussian radius stores were both tried first: they send half-empty NVLink packets, and the
		// barrier after them waits for those posted writes to drain.
		// Here `depth_key` = this rank's destination masks (kept for the backward), `iota`/cnt_offset = the count tables.
		__shared__ float4 s_out[8][96];
		__shared__ RunScratch rs;
		__shared__ uint8_t s_src[kRunBlock * kMaxPeers];
		const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
		const bool slot = (long long)idx < pt.chunk;
		const uint32_t mask = pr.ok ? touched_ranks(pr.y0, pr.y1, pt.world) : 0u;
		rec_out.q2.w = pack_radius_clamp(pr.ok ? pr.radius : 0, __float_as_uint(rec_out.q2.w));
		s_out[warp][lane * 3] = rec_out.q0; s_out[warp][lane * 3 + 1] = rec_out.q1; s_out[warp][lane * 3 + 2] = rec_out.q2;
		if (slot) depth_key[idx] = mask;
		if (slot && !in_range) radii[idx] = 0;  // padding slot of the local arrays
		block_run_ranks(rs, mask, pt.world);    // (contains the barriers that publish s_out)
		// own copy, kept for the backward (all 256 records, coalesced)
		{
			const long long first = (long long)blockIdx.x * kRunBlock;
			const int nrec = (int)min((long long)kRunBlock, (long long)f.P - first);
			float4 *dst = reinterpret_cast<float4 *>(rec + first);
			const float4 *src = &s_out[0][0];
			for (int e = threadIdx.x; e < 3 * nrec; e += kRunBlock) dst[e] = src[e];
		}
		for (int d = 0; d < pt.world; d++) {
			const uint32_t r = run_rank(rs, mask, d);
			if ((mask >> d) & 1u) s_src[rs.cpre[d] + r] = (uint8_t)threadIdx.x;
		}
		__syncthreads();
		const uint32_t total = rs.cpre[pt.world];
		const size_t slot0 = (size_t)pt.rank * (size_t)pt.chunk + (size_t)blockIdx.x * kRunBlock;
		for (uint32_t e = threadIdx.x; e < 3u * total; e += kRunBlock) {
			const uint32_t pos = e / 3u, part = e - 3u * pos;
			const int d = run_dest(rs, pos, pt.world);
			const uint32_t t = s_src[pos];
			reinterpret_cast<float4 *>(pt.rec[d] + slot0 + (pos - rs.cpre[d]))[part] = s_out[t >> 5][(t & 31u) * 3u + part];
		}
		if ((int)threadIdx.x < pt.world) {
			uint32_t *cnt = reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(pt.rec[threadIdx.x]) + cnt_offset);
			const uint32_t nblk = (uint32_t)((pt.chunk + kRunBlock - 1) / kRunBlock);
			cnt[(size_t)pt.rank * nblk + blockIdx.x] = rs.cpre[threadIdx.x + 1] - rs.cpre[threadIdx.x];
		}
	}
	if (!COUNT) return;
	uint32_t count = 0;
	visit_tiles<false, uint32_t>(pr.ok, pr.x0, pr.y0, pr.x1, pr.y1, cp, f.band, f.gx, 0u, 0u, nullptr, nullptr, count);
	if (in_range) {
		tiles_touched[idx] = count;
		// sort key of the depth pre-sort: Gaussians that emit nothing go to the very end
		depth_key[idx] = count > 0 ? __float_as_uint(pr.depth) : 0xffffffffu;
		iota[idx] = (uint32_t)idx;
		reached[idx] = pr.ok && !(cam_finite && isfinite(in_sum)) ? 1u : 0u;
	}
}

// radii + means2D only (reference filter_preprocessCUDA, forward.cu:259-334)
__global__ void __launch_bounds__(256) filter_kernel(const FrameDev f, const float *__restrict__ means3D, const float *__restrict__ scales,
                                                     const float *__restrict__ rotations, const float *__restrict__ cov3D_precomp,
                                                     int32_t *__restrict__ radii, float *__restrict__ means2D) {
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= f.P) return;
	const float3 p = make_float3(means3D[3 * (size_t)idx], means3D[3 * (size_t)idx + 1], means3D[3 * (size_t)idx + 2]);
	const Projected pr = project_gaussian(f, f.view, f.proj, p, load_shape(idx, scales, rotations, cov3D_precomp), cov3D_precomp != nullptr);
	radii[idx] = pr.radius;
	means2D[2 * (size_t)idx] = pr.ok ? pr.px : 0.f;
	means2D[2 * (size_t)idx + 1] = pr.ok ? pr.py : 0.f;
}

// present = z_view > 0.2 (reference checkFrustum, rasterizer_impl.cu:54-66)
__global__ void __launch_bounds__(256) mark_visible_kernel(int P, const float *__restrict__ means3D, const float *__restrict__ view,
                                                           uint8_t *__restrict__ present) {
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P) return;
	const float3 p = make_float3(means3D[3 * (size_t)idx], means3D[3 * (size_t)idx + 1], means3D[3 * (size_t)idx + 2]);
	const float3 pv = xform4x3(p, view);
	present[idx] = pv.z > 0.2f ? 1 : 0;
}

cudaError_t launch_preprocess_fwd(const FrameDev &f, const float *means3D, const float *shs, const float *colors_precomp,
                                  const float *opacities, const float *scales, const float *rotations,
                                  const float *cov3D_precomp, int32_t *radii, GeomView g, cudaStream_t st) {
	if (f.P == 0) return cudaSuccess;
	count_launch();
	preprocess_fwd_kernel<true><<<(f.P + 255) / 256, 256, 0, st>>>(f, PeerTable{}, means3D, shs, colors_precomp, opacities, scales, rotations,
	                                                                  cov3D_precomp, radii, g.rec, g.jac, g.tiles_touched, g.depth_key, g.iota,
	                                                                  g.reached);
	return cudaGetLastError();
}
cudaError_t launch_project(const FrameDev &f, const float *means3D, const float *shs, const float *colors_precomp,
                           const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp,
                           int32_t *radii, GaussRec *rec, float4 *jac, cudaStream_t st) {
	if (f.P == 0) return cudaSuccess;
	count_launch();
	preprocess_fwd_kernel<false><<<(f.P + 255) / 256, 256, 0, st>>>(f, PeerTable{}, means3D, shs, colors_precomp, opacities, scales, rotations,
	                                                                   cov3D_precomp, radii, rec, jac, nullptr, nullptr, nullptr, nullptr);
	return cudaGetLastError();
}
cudaError_t launch_project_scatter(const FrameDev &f, const PeerTable &pt, const float *means3D, const float *shs,
                                   const float *colors_precomp, const float *opacities, const float *scales, const float *rotations,
                                   const float *cov3D_precomp, int32_t *radii_local, GaussRec *rec_local, float4 *jac_local,
                                   uint32_t *masks_local, size_t cnt_offset, cudaStream_t st) {
	if (pt.chunk == 0) return cudaSuccess;
	count_launch();
	const unsigned nblk = (unsigned)((pt.chunk + kRunBlock - 1) / kRunBlock);
	preprocess_fwd_kernel<false, true><<<nblk, 256, 0, st>>>(f, pt, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
	                                                         radii_local, rec_local, jac_local, nullptr, masks_local, nullptr, nullptr,
	                                                         cnt_offset);
	return cudaGetLastError();
}
cudaError_t launch_filter(const FrameDev &f, const float *means3D, const float *scales, const float *rotations,
                          const float *cov3D_precomp, int32_t *radii, float *means2D, cudaStream_t st) {
	if (f.P == 0) return cudaSuccess;
	count_launch();
	filter_kernel<<<(f.P + 255) / 256, 256, 0, st>>>(f, means3D, scales, rotations, cov3D_precomp, radii, means2D);
	return cudaGetLastError();
}
cudaError_t launch_mark_visible(int P, const float *means3D, const float *view, uint8_t *present, cudaStream_t st) {
	if (P == 0) return cudaSuccess;
	count_launch();
	mark_visible_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, view, present);
	return cudaGetLastError();
}

}  // namespace sgr
