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
