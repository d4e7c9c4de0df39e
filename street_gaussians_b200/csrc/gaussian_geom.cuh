// gaussian_geom.cuh — per-Gaussian geometry shared by the forward (preprocess_fwd.cu) and the chain rule (preprocess_bwd.cu).
//
// One copy of each reference expression: the SH constants, the world covariance from scale and rotation, the EWA screen-space
// covariance, and the backward's pieces (reference backward.cu:144-274, 375-403, 278-341, auxiliary.h:107-117).  The backward
// recomputes cov2D with the very function the forward calls, so the two agree by construction.  Every expression keeps the
// reference's shape and association: how nvcc contracts them into FMAs is what makes depth, radius and pixel position bit-equal
// to the reference (DESIGN.md §5).  Camera matrices are passed as pointers, to global memory or to a shared-memory copy.
#pragma once
#include "sgr_common.cuh"

namespace sgr {

// real SH basis constants up to degree 3 (reference forward.cu:20-31)
static __device__ __constant__ float kC0 = 0.28209479177387814f;
static __device__ __constant__ float kC1 = 0.4886025119029199f;
static __device__ __constant__ float kC2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
                                               0.5462742152960396f};
static __device__ __constant__ float kC3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                                               -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

// Real SH basis B_k of the unit view direction (x, y, z) for k < (deg + 1)^2, 0 beyond (reference forward.cu:20-71).
__device__ __forceinline__ void sh_basis(int deg, float x, float y, float z, float (&B)[16]) {
#pragma unroll
	for (int k = 0; k < 16; k++) B[k] = 0.f;
	B[0] = kC0;
	if (deg > 0) {
		B[1] = -kC1 * y; B[2] = kC1 * z; B[3] = -kC1 * x;
		if (deg > 1) {
			const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
			B[4] = kC2[0] * xy; B[5] = kC2[1] * yz; B[6] = kC2[2] * (2.f * zz - xx - yy); B[7] = kC2[3] * xz; B[8] = kC2[4] * (xx - yy);
			if (deg > 2) {
				B[9] = kC3[0] * y * (3.f * xx - yy); B[10] = kC3[1] * xy * z; B[11] = kC3[2] * y * (4.f * zz - xx - yy);
				B[12] = kC3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy); B[13] = kC3[4] * x * (4.f * zz - xx - yy); B[14] = kC3[5] * z * (xx - yy);
				B[15] = kC3[6] * x * (xx - 3.f * yy);
			}
		}
	}
}

// Colour Jacobian of one coefficient row c (coefficient-major, RGB innermost) at the unit direction: J[3 a + ch] = d colour_ch /
// d dir_a for a = x, y, z — the reference's per-channel dRGBdx / dRGBdy / dRGBdz sums (backward.cu:20-139).  It does not depend on
// the upstream gradient, so the forward evaluates it while it holds the row, and the backward never reads the coefficients.
__device__ __forceinline__ void sh_color_jacobian(int deg, float x, float y, float z, const float *c, float (&J)[9]) {
#pragma unroll
	for (int ch = 0; ch < 3; ch++) {
#define SHC(k) c[(k) * 3 + ch]
		float dx = 0.f, dy = 0.f, dz = 0.f;
		if (deg > 0) {
			dx = -kC1 * SHC(3); dy = -kC1 * SHC(1); dz = kC1 * SHC(2);
			if (deg > 1) {
				const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
				dx += kC2[0] * y * SHC(4) + kC2[2] * 2.f * -x * SHC(6) + kC2[3] * z * SHC(7) + kC2[4] * 2.f * x * SHC(8);
				dy += kC2[0] * x * SHC(4) + kC2[1] * z * SHC(5) + kC2[2] * 2.f * -y * SHC(6) + kC2[4] * 2.f * -y * SHC(8);
				dz += kC2[1] * y * SHC(5) + kC2[2] * 2.f * 2.f * z * SHC(6) + kC2[3] * x * SHC(7);
				if (deg > 2) {
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
		J[ch] = dx; J[3 + ch] = dy; J[6 + ch] = dz;
	}
}

// The colour Jacobian as the forward stores it, three float4 per Gaussian: {J0 J1 J2 J3} {J4 J5 J6 J7} {J8, clamp bits, 0, 0}.
// The clamp bits (bit ch: colour channel ch was clamped at 0, so no gradient flows through it) travel with it, so the backward reads
// nothing of the 48-B blend record.
__device__ __forceinline__ void store_color_jac(float4 *dst, const float (&J)[9], uint32_t clamp_bits) {
	dst[0] = make_float4(J[0], J[1], J[2], J[3]);
	dst[1] = make_float4(J[4], J[5], J[6], J[7]);
	dst[2] = make_float4(J[8], __uint_as_float(clamp_bits), 0.f, 0.f);
}
struct ColorJac {
	float4 a, b, c;
};
__device__ __forceinline__ ColorJac load_color_jac(const float4 *__restrict__ src) {
	return ColorJac{__ldg(src), __ldg(src + 1), __ldg(src + 2)};
}
// dL/dRGB with the clamped channels zeroed
__device__ __forceinline__ void masked_drgb(const ColorJac &cj, float r, float g, float b, float (&dRGB)[3]) {
	const uint32_t clamp_bits = __float_as_uint(cj.c.y);
	dRGB[0] = (clamp_bits & 1u) ? 0.f : r;
	dRGB[1] = (clamp_bits & 2u) ? 0.f : g;
	dRGB[2] = (clamp_bits & 4u) ? 0.f : b;
}
// dL/d(unit direction) = J^T dL/dRGB, summed over the channels in the reference's order
__device__ __forceinline__ float3 color_jac_dir_grad(const ColorJac &cj, const float (&dRGB)[3]) {
	const float J[9] = {cj.a.x, cj.a.y, cj.a.z, cj.a.w, cj.b.x, cj.b.y, cj.b.z, cj.b.w, cj.c.x};
	float3 d = make_float3(0.f, 0.f, 0.f);
#pragma unroll
	for (int ch = 0; ch < 3; ch++) {
		d.x += J[ch] * dRGB[ch]; d.y += J[3 + ch] * dRGB[ch]; d.z += J[6 + ch] * dRGB[ch];
	}
	return d;
}

// The per-Gaussian shape inputs.  The forward loads them at the TOP of its kernel together with the position and the opacity: the
// round-1 kernel loaded them where they were used (after the near cull, inside the projection), which serialised three DRAM round
// trips per thread (the profiler's source view put most long-scoreboard stalls on exactly these loads).
struct ShapeIn {
	float3 s;
	float4 q;
	float c6[6];
};
__device__ __forceinline__ ShapeIn load_shape(int idx, const float *__restrict__ scales, const float *__restrict__ rotations,
                                              const float *__restrict__ cov3D_precomp) {
	ShapeIn g;
	g.s = make_float3(0.f, 0.f, 0.f);
	g.q = make_float4(1.f, 0.f, 0.f, 0.f);
	if (cov3D_precomp != nullptr) {
#pragma unroll
		for (int k = 0; k < 6; k++) g.c6[k] = cov3D_precomp[6 * (size_t)idx + k];
	} else {
		g.s = make_float3(scales[3 * (size_t)idx], scales[3 * (size_t)idx + 1], scales[3 * (size_t)idx + 2]);
		g.q = *reinterpret_cast<const float4 *>(rotations + 4 * (size_t)idx);
	}
	return g;
}

// World-space covariance from (modifier * scale, rotation R of the raw quaternion), upper triangle xx xy xz yy yz zz.  The
// quaternion is deliberately not normalised (reference forward.cu:127).
__device__ __forceinline__ void cov3d_from_scale_rot(const float3 s_mod, const M3 &R, float *c6) {
	const M3 S = {{{s_mod.x, 0.f, 0.f}, {0.f, s_mod.y, 0.f}, {0.f, 0.f, s_mod.z}}};
	const M3 Mm = m3_mul(S, R);
	const M3 Sg = m3_mul(m3_t(Mm), Mm);
	c6[0] = Sg.m[0][0]; c6[1] = Sg.m[0][1]; c6[2] = Sg.m[0][2]; c6[3] = Sg.m[1][1]; c6[4] = Sg.m[1][2]; c6[5] = Sg.m[2][2];
}

// EWA screen-space covariance (+0.3 low-pass), reference forward.cu:74-113.  Besides cov2D it keeps what the backward
// differentiates through; the forward uses `cov` only and the compiler drops the rest.  Two choices here are about code generation,
// observed with nvcc 12.9 for sm_90a: ewa_cov2d fills an Ewa the caller owns (returned by value, the struct changed which product
// nvcc fuses in the backward's dL/dT sums), and the clamp flags are integers converted where the backward uses them (float flags
// were converted early and cost the gather instantiations of preprocess_bwd_kernel a spill).  After touching these functions,
// compare `python -m street_gaussians_b200.build --force --ptxas` and the per-kernel counts of floating-point SASS opcodes
// (`cuobjdump -sass libsgr.so`) with the previous build.
struct Ewa {
	float3 t;                      // view-space mean, x and y clamped to 1.3 tan(fov / 2) z
	unsigned x_in, y_in;           // 0 where that clamp was active (no gradient flows through it), else 1
	M3 W, T, V;                    // view rotation, T = W J, world covariance
	float3 cov;                    // cov2D (xx, xy, yy)
};
__device__ __forceinline__ void ewa_cov2d(Ewa &e, const float3 mean, float fx, float fy, float tanx, float tany, const float *c6,
                                         const float *__restrict__ view) {
	float3 t = xform4x3(mean, view);
	const float limx = 1.3f * tanx, limy = 1.3f * tany;
	const float txtz = t.x / t.z, tytz = t.y / t.z;
	t.x = fminf(limx, fmaxf(-limx, txtz)) * t.z;
	t.y = fminf(limy, fmaxf(-limy, tytz)) * t.z;
	e.t = t;
	e.x_in = txtz < -limx || txtz > limx ? 0 : 1;
	e.y_in = tytz < -limy || tytz > limy ? 0 : 1;
	const M3 J = {{{fx / t.z, 0.0f, -(fx * t.x) / (t.z * t.z)}, {0.0f, fy / t.z, -(fy * t.y) / (t.z * t.z)}, {0.f, 0.f, 0.f}}};
	e.W = M3{{{view[0], view[4], view[8]}, {view[1], view[5], view[9]}, {view[2], view[6], view[10]}}};
	e.T = m3_mul(e.W, J);
	e.V = M3{{{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}}};
	M3 cov = m3_mul(m3_mul(m3_t(e.T), m3_t(e.V)), e.T);
	cov.m[0][0] += 0.3f;
	cov.m[1][1] += 0.3f;
	e.cov = make_float3(cov.m[0][0], cov.m[0][1], cov.m[1][1]);
}

// conic -> cov2D -> cov3D (dcov, upper triangle like c6) and the mean through the EWA Jacobian (reference backward.cu:144-274);
// returns the mean's gradient of this path.
__device__ __forceinline__ float3 ewa_cov2d_bwd(const Ewa &e, const float3 dL_dconic, float h_x, float h_y, const float *view, float *dcov) {
	const float a = e.cov.x, b = e.cov.y, c = e.cov.z;
	const float denom = a * c - b * b;
	float dL_da = 0, dL_db = 0, dL_dc = 0;
	const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
#pragma unroll
	for (int k = 0; k < 6; k++) dcov[k] = 0.f;
#define T_(c_, r_) e.T.m[c_][r_]
	if (denom2inv != 0) {
		dL_da = denom2inv * (-c * c * dL_dconic.x + 2 * b * c * dL_dconic.y + (denom - a * c) * dL_dconic.z);
		dL_dc = denom2inv * (-a * a * dL_dconic.z + 2 * a * b * dL_dconic.y + (denom - a * c) * dL_dconic.x);
		dL_db = denom2inv * 2 * (b * c * dL_dconic.x - (denom + 2 * b * b) * dL_dconic.y + a * b * dL_dconic.z);
		dcov[0] = (T_(0, 0) * T_(0, 0) * dL_da + T_(0, 0) * T_(1, 0) * dL_db + T_(1, 0) * T_(1, 0) * dL_dc);
		dcov[3] = (T_(0, 1) * T_(0, 1) * dL_da + T_(0, 1) * T_(1, 1) * dL_db + T_(1, 1) * T_(1, 1) * dL_dc);
		dcov[5] = (T_(0, 2) * T_(0, 2) * dL_da + T_(0, 2) * T_(1, 2) * dL_db + T_(1, 2) * T_(1, 2) * dL_dc);
		dcov[1] = 2 * T_(0, 0) * T_(0, 1) * dL_da + (T_(0, 0) * T_(1, 1) + T_(0, 1) * T_(1, 0)) * dL_db + 2 * T_(1, 0) * T_(1, 1) * dL_dc;
		dcov[2] = 2 * T_(0, 0) * T_(0, 2) * dL_da + (T_(0, 0) * T_(1, 2) + T_(0, 2) * T_(1, 0)) * dL_db + 2 * T_(1, 0) * T_(1, 2) * dL_dc;
		dcov[4] = 2 * T_(0, 2) * T_(0, 1) * dL_da + (T_(0, 1) * T_(1, 2) + T_(0, 2) * T_(1, 1)) * dL_db + 2 * T_(1, 1) * T_(1, 2) * dL_dc;
	}
#define V_(c_, r_) e.V.m[c_][r_]
	const float dL_dT00 = 2 * (T_(0, 0) * V_(0, 0) + T_(0, 1) * V_(0, 1) + T_(0, 2) * V_(0, 2)) * dL_da +
	                      (T_(1, 0) * V_(0, 0) + T_(1, 1) * V_(0, 1) + T_(1, 2) * V_(0, 2)) * dL_db;
	const float dL_dT01 = 2 * (T_(0, 0) * V_(1, 0) + T_(0, 1) * V_(1, 1) + T_(0, 2) * V_(1, 2)) * dL_da +
	                      (T_(1, 0) * V_(1, 0) + T_(1, 1) * V_(1, 1) + T_(1, 2) * V_(1, 2)) * dL_db;
	const float dL_dT02 = 2 * (T_(0, 0) * V_(2, 0) + T_(0, 1) * V_(2, 1) + T_(0, 2) * V_(2, 2)) * dL_da +
	                      (T_(1, 0) * V_(2, 0) + T_(1, 1) * V_(2, 1) + T_(1, 2) * V_(2, 2)) * dL_db;
	const float dL_dT10 = 2 * (T_(1, 0) * V_(0, 0) + T_(1, 1) * V_(0, 1) + T_(1, 2) * V_(0, 2)) * dL_dc +
	                      (T_(0, 0) * V_(0, 0) + T_(0, 1) * V_(0, 1) + T_(0, 2) * V_(0, 2)) * dL_db;
	const float dL_dT11 = 2 * (T_(1, 0) * V_(1, 0) + T_(1, 1) * V_(1, 1) + T_(1, 2) * V_(1, 2)) * dL_dc +
	                      (T_(0, 0) * V_(1, 0) + T_(0, 1) * V_(1, 1) + T_(0, 2) * V_(1, 2)) * dL_db;
	const float dL_dT12 = 2 * (T_(1, 0) * V_(2, 0) + T_(1, 1) * V_(2, 1) + T_(1, 2) * V_(2, 2)) * dL_dc +
	                      (T_(0, 0) * V_(2, 0) + T_(0, 1) * V_(2, 1) + T_(0, 2) * V_(2, 2)) * dL_db;
#undef V_
#undef T_
	const float dL_dJ00 = e.W.m[0][0] * dL_dT00 + e.W.m[0][1] * dL_dT01 + e.W.m[0][2] * dL_dT02;
	const float dL_dJ02 = e.W.m[2][0] * dL_dT00 + e.W.m[2][1] * dL_dT01 + e.W.m[2][2] * dL_dT02;
	const float dL_dJ11 = e.W.m[1][0] * dL_dT10 + e.W.m[1][1] * dL_dT11 + e.W.m[1][2] * dL_dT12;
	const float dL_dJ12 = e.W.m[2][0] * dL_dT10 + e.W.m[2][1] * dL_dT11 + e.W.m[2][2] * dL_dT12;
	const float3 t = e.t;
	const float tz = 1.f / t.z, tz2 = tz * tz, tz3 = tz2 * tz;
	const float x_grad_mul = (float)e.x_in, y_grad_mul = (float)e.y_in;
	const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
	const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
	const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * t.x) * tz3 * dL_dJ02 + (2 * h_y * t.y) * tz3 * dL_dJ12;
	// view^T (3x3 part) applied to (dtx, dty, dtz)
	return make_float3(view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz, view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz,
	                   view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz);
}

__device__ __forceinline__ void add_to(float3 &acc, const float3 d) {
	acc.x += d.x; acc.y += d.y; acc.z += d.z;
}

// mean2D -> mean3D through the projective divide (reference backward.cu:375-389)
__device__ __forceinline__ float3 mean2d_bwd(const float3 mean, const float *proj, const float dL_dpx, const float dL_dpy) {
	const float4 m_hom = xform4x4(mean, proj);
	const float m_w = 1.0f / (m_hom.w + 0.0000001f);
	const float mul1 = (proj[0] * mean.x + proj[4] * mean.y + proj[8] * mean.z + proj[12]) * m_w * m_w;
	const float mul2 = (proj[1] * mean.x + proj[5] * mean.y + proj[9] * mean.z + proj[13]) * m_w * m_w;
	return make_float3((proj[0] * m_w - proj[3] * mul1) * dL_dpx + (proj[1] * m_w - proj[3] * mul2) * dL_dpy,
	                   (proj[4] * m_w - proj[7] * mul1) * dL_dpx + (proj[5] * m_w - proj[7] * mul2) * dL_dpy,
	                   (proj[8] * m_w - proj[11] * mul1) * dL_dpx + (proj[9] * m_w - proj[11] * mul2) * dL_dpy);
}

// blended depth -> mean3D (reference backward.cu:392-403)
__device__ __forceinline__ float3 depth_bwd(const float3 mean, const float *view, const float dL_ddepth) {
	const float mul3 = view[2] * mean.x + view[6] * mean.y + view[10] * mean.z + view[14];
	return make_float3((view[2] - view[3] * mul3) * dL_ddepth, (view[6] - view[7] * mul3) * dL_ddepth, (view[10] - view[11] * mul3) * dL_ddepth);
}

// cov3D -> scale, raw quaternion (reference backward.cu:278-341; no normalisation Jacobian, scale_modifier quirk kept).
// `s_mod` and `R` are what cov3d_from_scale_rot was given.
__device__ __forceinline__ void cov3d_bwd(const float3 s_mod, const float4 q, const M3 &R, const float *dcov, float3 &dscale, float4 &dq) {
	const float r = q.x, x = q.y, y = q.z, z = q.w;
	const M3 S = {{{s_mod.x, 0.f, 0.f}, {0.f, s_mod.y, 0.f}, {0.f, 0.f, s_mod.z}}};
	const M3 Mm = m3_mul(S, R);
	const M3 dSig = {{{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]}, {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]}, {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}}};
	M3 M2;
#pragma unroll
	for (int cc = 0; cc < 3; cc++)
#pragma unroll
		for (int rr = 0; rr < 3; rr++) M2.m[cc][rr] = Mm.m[cc][rr] * 2.0f;
	const M3 dL_dM = m3_mul(M2, dSig);
	const M3 Rt = m3_t(R);
	M3 dMt = m3_t(dL_dM);
	dscale.x = Rt.m[0][0] * dMt.m[0][0] + Rt.m[0][1] * dMt.m[0][1] + Rt.m[0][2] * dMt.m[0][2];
	dscale.y = Rt.m[1][0] * dMt.m[1][0] + Rt.m[1][1] * dMt.m[1][1] + Rt.m[1][2] * dMt.m[1][2];
	dscale.z = Rt.m[2][0] * dMt.m[2][0] + Rt.m[2][1] * dMt.m[2][1] + Rt.m[2][2] * dMt.m[2][2];
#pragma unroll
	for (int k = 0; k < 3; k++) { dMt.m[0][k] *= s_mod.x; dMt.m[1][k] *= s_mod.y; dMt.m[2][k] *= s_mod.z; }
#define D_(c_, r_) dMt.m[c_][r_]
	dq.x = 2 * z * (D_(0, 1) - D_(1, 0)) + 2 * y * (D_(2, 0) - D_(0, 2)) + 2 * x * (D_(1, 2) - D_(2, 1));
	dq.y = 2 * y * (D_(1, 0) + D_(0, 1)) + 2 * z * (D_(2, 0) + D_(0, 2)) + 2 * r * (D_(1, 2) - D_(2, 1)) - 4 * x * (D_(2, 2) + D_(1, 1));
	dq.z = 2 * x * (D_(1, 0) + D_(0, 1)) + 2 * r * (D_(2, 0) - D_(0, 2)) + 2 * z * (D_(1, 2) + D_(2, 1)) - 4 * y * (D_(2, 2) + D_(0, 0));
	dq.w = 2 * r * (D_(0, 1) - D_(1, 0)) + 2 * x * (D_(2, 0) + D_(0, 2)) + 2 * y * (D_(1, 2) + D_(2, 1)) - 4 * z * (D_(1, 1) + D_(0, 0));
#undef D_
}

// through the normalisation of the view direction `dir` = mean - campos (reference dnormvdv, auxiliary.h:107-117)
__device__ __forceinline__ float3 dnormvdv(const float3 dir, const float3 ddir) {
	const float sum2 = dir.x * dir.x + dir.y * dir.y + dir.z * dir.z;
	const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
	return make_float3(((+sum2 - dir.x * dir.x) * ddir.x - dir.y * dir.x * ddir.y - dir.z * dir.x * ddir.z) * invsum32,
	                   (-dir.x * dir.y * ddir.x + (sum2 - dir.y * dir.y) * ddir.y - dir.z * dir.y * ddir.z) * invsum32,
	                   (-dir.x * dir.z * ddir.x - dir.y * dir.z * ddir.y + (sum2 - dir.z * dir.z) * ddir.z) * invsum32);
}

}  // namespace sgr
