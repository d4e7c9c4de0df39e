// actor_pose.cu — the tracked actor poses of street_gaussians (lib/models/actor_pose.py, ActorPose, as
// StreetGaussianModel.parse_camera uses it at street_gaussian_model.py:257-271), from the tracklets and their learned offsets
// opt_trans / opt_rots, composed with the ego pose, and their gradient back to the offsets.
//
// One warp per visible actor.  The warp finds the two tracklet entries nearest the timestamp (find_closest_indices,
// actor_pose.py:83-90) and, for a validation camera, the two nearest training timestamps of that camera inside the track's span
// (find_closest_camera_timestamps, :93-105); then every lane runs the pose arithmetic and lane 0 writes.  The arithmetic is the
// reference's fp32 torch lines op by op, with no FMA contraction:
//   translation  (trans1 a + trans2 b) / c            :107-122, with a, b, c the float64 differences rounded once to fp32 and / c taken
//                                                     as * (1 / c), as torch does on CUDA for a Python-scalar divisor
//   rotation     slerp(q1 (x) theta1, q1 (x) theta1 (x) theta2, r)   :138-158 — theta2 = opt_rots[frame_ind1, column_ind2] and the
//                second frame's input_rots is never read (DESIGN.md §5); r = (t - t1) / (t2 - t1) in float64, rounded once
//   validation   the two of them at the two camera timestamps, interpolated again (:124-136, :160-173); fewer than two
//                camera timestamps in the span fall back to the training path (:127)
//   ego          matrix_to_quaternion(ego[:3, :3]) (x) rot and ego[:3, :3] trans + ego[:3, 3]   street_gaussian_model.py:260-265
//   (x) theta    quaternion_raw_multiply_theta (general_utils.py:240-259), a yaw about z
//   slerp        quaternion_slerp (general_utils.py:277-303): F.normalize, then the shortest-arc slerp DESIGN.md §5 states
//   idft         IDFT(fourier_scale (frame - start_frame) / (end_frame - start_frame), C)   sh_utils.py:120-130, gaussian_model_actor.py:71-77
// Ties in distance go to the entry that comes first in the track's argwhere order (DESIGN.md §5).  The backward recomputes the
// forward, writes each actor's (row, value) contributions to scratch, and one more kernel adds them up row by row in actor order, so
// repeated calls give bit-identical gradients.  Grids depend on the number of actors only; nothing is read back to the host.
#include <climits>
#include <cstring>

#include "sgr_common.cuh"

namespace sgr {

constexpr int kPoseWarps = 4;  // actors per block
constexpr int kAccumThreads = 256;

struct Near {
	double d;
	int i;
};
__device__ __forceinline__ bool nearer(const Near a, const Near b) { return a.d < b.d || (a.d == b.d && a.i < b.i); }

// The two entries of ts[lo, hi) nearest tq (ties: the lower index), counting only entries inside [span_lo, span_hi] when `filter`.
// Warp-collective; every lane returns the same result.  i1 / i2 are -1 when fewer than one / two entries qualify.
__device__ __forceinline__ int nearest_two(const double *__restrict__ ts, const int lo, const int hi, const double tq, const bool filter,
                                           const double span_lo, const double span_hi, int &i1, int &i2) {
	const unsigned full = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	Near b1{INFINITY, INT_MAX}, b2{INFINITY, INT_MAX};
	int count = 0;
	for (int e = lo + lane; e < hi; e += 32) {
		const double x = __ldg(ts + e);
		if (filter && !(x >= span_lo && x <= span_hi)) continue;
		count++;
		const Near c{fabs(x - tq), e};
		if (nearer(c, b1)) { b2 = b1; b1 = c; }
		else if (nearer(c, b2)) b2 = c;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		const Near p1{__shfl_xor_sync(full, b1.d, o), __shfl_xor_sync(full, b1.i, o)};
		const Near p2{__shfl_xor_sync(full, b2.d, o), __shfl_xor_sync(full, b2.i, o)};
		// best two of {b1, b2, p1, p2}; b1 < b2 and p1 < p2, and all indices differ
		if (nearer(p1, b1)) { b2 = nearer(b1, p2) ? b1 : p2; b1 = p1; }
		else if (nearer(p1, b2)) b2 = p1;
	}
	i1 = b1.i == INT_MAX ? -1 : b1.i;
	i2 = b2.i == INT_MAX ? -1 : b2.i;
	return __reduce_add_sync(full, count);
}

struct PoseArgs {
	int n, base, K, opt_track, is_val, cam, frame, fourier_dim;
	double t, fourier_scale;
	const int *track_off, *entry_fc, *track_frames, *cam_off;
	const double *entry_ts, *track_span, *cam_ts;
	const float *in_trans, *in_rots, *opt_trans, *opt_rots, *ego;
	float *poses, *idft;
	const float *gposes;
	int *trow, *rrow;
	float *tval, *rval;
	int slot[kActorPoseChunk];
};

// The two tracklet entries of a track nearest tq: (frame, column) of each and their timestamps.
struct Pick {
	int f1, c1, f2, c2;
	double t1, t2;
};
__device__ __forceinline__ Pick pick_entries(const PoseArgs &a, const int trk, const double tq) {
	int i1, i2;
	nearest_two(a.entry_ts, __ldg(a.track_off + trk), __ldg(a.track_off + trk + 1), tq, false, 0.0, 0.0, i1, i2);
	Pick p;
	const bool ok = i2 >= 0;
	p.f1 = ok ? __ldg(a.entry_fc + 2 * i1) : 0;
	p.c1 = ok ? __ldg(a.entry_fc + 2 * i1 + 1) : 0;
	p.f2 = ok ? __ldg(a.entry_fc + 2 * i2) : 0;
	p.c2 = ok ? __ldg(a.entry_fc + 2 * i2 + 1) : 0;
	p.t1 = ok ? __ldg(a.entry_ts + i1) : NAN;
	p.t2 = ok ? __ldg(a.entry_ts + i2) : NAN;
	return p;
}

// torch's clamp_min / maximum against a constant: NaN propagates (fmaxf would drop it)
__device__ __forceinline__ float clamp_lo(const float x, const float lo) { return x < lo ? lo : x; }

// ---- quaternion pieces, (w, x, y, z) ----
__device__ __forceinline__ void mul_theta(const float q[4], const float th, float o[4]) {  // general_utils.py:252-258
	const float c = cosf(th), s = sinf(th);
	o[0] = __fsub_rn(__fmul_rn(q[0], c), __fmul_rn(q[3], s));
	o[1] = __fadd_rn(__fmul_rn(q[1], c), __fmul_rn(q[2], s));
	o[2] = __fsub_rn(__fmul_rn(q[2], c), __fmul_rn(q[1], s));
	o[3] = __fadd_rn(__fmul_rn(q[3], c), __fmul_rn(q[0], s));
}
// dL/dq of mul_theta added to gq, and dL/dtheta returned, for the upstream gradient g.
__device__ __forceinline__ float mul_theta_bwd(const float q[4], const float th, const float g[4], float gq[4]) {
	const float c = cosf(th), s = sinf(th);
	gq[0] += c * g[0] + s * g[3];
	gq[1] += c * g[1] - s * g[2];
	gq[2] += s * g[1] + c * g[2];
	gq[3] += c * g[3] - s * g[0];
	return g[0] * (-q[0] * s - q[3] * c) + g[1] * (-q[1] * s + q[2] * c) + g[2] * (-q[2] * s - q[1] * c) + g[3] * (-q[3] * s + q[0] * c);
}
__device__ __forceinline__ void quat_mul(const float a[4], const float b[4], float o[4]) {  // quaternion_raw_multiply, :232-238
	o[0] = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2])), __fmul_rn(a[3], b[3]));
	o[1] = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0])), __fmul_rn(a[2], b[3])), __fmul_rn(a[3], b[2]));
	o[2] = __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(a[0], b[2]), __fmul_rn(a[1], b[3])), __fmul_rn(a[2], b[0])), __fmul_rn(a[3], b[1]));
	o[3] = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(a[0], b[3]), __fmul_rn(a[1], b[2])), __fmul_rn(a[2], b[1])), __fmul_rn(a[3], b[0]));
}

// matrix_to_quaternion (general_utils.py:159-218) of ego[:3, :3], ego row-major [4, 4].
__device__ __forceinline__ void ego_quat(const float *__restrict__ ego, float q[4]) {
	float m[3][3];
#pragma unroll
	for (int i = 0; i < 3; i++)
#pragma unroll
		for (int j = 0; j < 3; j++) m[i][j] = __ldg(ego + 4 * i + j);
	const float x[4] = {__fadd_rn(__fadd_rn(__fadd_rn(1.f, m[0][0]), m[1][1]), m[2][2]), __fsub_rn(__fsub_rn(__fadd_rn(1.f, m[0][0]), m[1][1]), m[2][2]),
	                    __fsub_rn(__fadd_rn(__fsub_rn(1.f, m[0][0]), m[1][1]), m[2][2]), __fadd_rn(__fsub_rn(__fsub_rn(1.f, m[0][0]), m[1][1]), m[2][2])};
	float qa[4];
	int k = 0;
#pragma unroll
	for (int i = 0; i < 4; i++) {
		qa[i] = x[i] > 0.f ? __fsqrt_rn(x[i]) : 0.f;
		if (qa[i] > qa[k]) k = i;  // argmax: the first of equal maxima
	}
	float r[4];
	const float sq = __fmul_rn(qa[k], qa[k]);
	if (k == 0) { r[0] = sq; r[1] = __fsub_rn(m[2][1], m[1][2]); r[2] = __fsub_rn(m[0][2], m[2][0]); r[3] = __fsub_rn(m[1][0], m[0][1]); }
	else if (k == 1) { r[0] = __fsub_rn(m[2][1], m[1][2]); r[1] = sq; r[2] = __fadd_rn(m[1][0], m[0][1]); r[3] = __fadd_rn(m[0][2], m[2][0]); }
	else if (k == 2) { r[0] = __fsub_rn(m[0][2], m[2][0]); r[1] = __fadd_rn(m[1][0], m[0][1]); r[2] = sq; r[3] = __fadd_rn(m[1][2], m[2][1]); }
	else { r[0] = __fsub_rn(m[1][0], m[0][1]); r[1] = __fadd_rn(m[2][0], m[0][2]); r[2] = __fadd_rn(m[2][1], m[1][2]); r[3] = sq; }
	const float den = __fmul_rn(2.f, clamp_lo(qa[k], 0.1f));
#pragma unroll
	for (int i = 0; i < 4; i++) q[i] = __fdiv_rn(r[i], den);
}

// ---- slerp: F.normalize both, shortest arc, then w0 u + w1 v with the small-angle weights (1 - t, t) where |sin theta| < 1e-6 ----
struct Slerp {
	float u[4], v[4], n0, n1, sigma, w0, w1, theta, s, dc;
	bool small, inside;  // inside: |u . q1n| <= 1, where the clamp passes the gradient
};
__device__ __forceinline__ float norm4(const float q[4]) {
	return __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[0], q[0]), __fmul_rn(q[1], q[1])), __fmul_rn(q[2], q[2])), __fmul_rn(q[3], q[3])));
}
__device__ __forceinline__ Slerp slerp_fwd(const float q0[4], const float q1[4], const float t, float out[4]) {
	Slerp S;
	S.n0 = clamp_lo(norm4(q0), 1e-12f);
	S.n1 = clamp_lo(norm4(q1), 1e-12f);
	float v0[4];
#pragma unroll
	for (int i = 0; i < 4; i++) { S.u[i] = __fdiv_rn(q0[i], S.n0); v0[i] = __fdiv_rn(q1[i], S.n1); }
	// (q0 * q1).sum(-1) in x, y, z, w order
	const float d = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(S.u[1], v0[1]), __fmul_rn(S.u[2], v0[2])), __fmul_rn(S.u[3], v0[3])), __fmul_rn(S.u[0], v0[0]));
	S.sigma = d < 0.f ? -1.f : 1.f;
#pragma unroll
	for (int i = 0; i < 4; i++) S.v[i] = d < 0.f ? -v0[i] : v0[i];
	const float ad = fabsf(d);
	S.inside = ad <= 1.f;
	S.dc = ad > 1.f ? 1.f : ad;  // torch's clamp: NaN stays NaN (fminf would return 1)
	S.theta = acosf(S.dc);
	S.s = sinf(S.theta);
	S.small = fabsf(S.s) < 1e-6f;
	const float omt = __fsub_rn(1.f, t);
	S.w0 = S.small ? omt : __fdiv_rn(sinf(__fmul_rn(omt, S.theta)), S.s);
	S.w1 = S.small ? t : __fdiv_rn(sinf(__fmul_rn(t, S.theta)), S.s);
#pragma unroll
	for (int i = 0; i < 4; i++) out[i] = __fadd_rn(__fmul_rn(S.w0, S.u[i]), __fmul_rn(S.w1, S.v[i]));
	return S;
}
// dL/dq0, dL/dq1 (before the normalisation) for the upstream gradient g.  In the small-angle branch the weights are constants, so no
// gradient reaches the angle: the finite value, where the reference's autograd multiplies that zero by acos'(1) = -inf at q0 == q1.
__device__ __forceinline__ void slerp_bwd(const float q0[4], const float q1[4], const float t, const float g[4], float gq0[4], float gq1[4]) {
	float out[4];
	const Slerp S = slerp_fwd(q0, q1, t, out);
	float gu[4], gv[4], gw0 = 0.f, gw1 = 0.f;
#pragma unroll
	for (int i = 0; i < 4; i++) {
		gu[i] = S.w0 * g[i];
		gv[i] = S.w1 * g[i];
		gw0 += g[i] * S.u[i];
		gw1 += g[i] * S.v[i];
	}
	float dd = 0.f;
	if (!S.small) {
		const float omt = 1.f - t;
		const float dth = gw0 / S.s * omt * cosf(omt * S.theta) + gw1 / S.s * t * cosf(t * S.theta) - (gw0 * S.w0 + gw1 * S.w1) / S.s * cosf(S.theta);
		dd = S.inside ? -dth / sqrtf(1.f - S.dc * S.dc) : 0.f;
	}
	float gn0[4], gn1[4];
#pragma unroll
	for (int i = 0; i < 4; i++) {
		gn0[i] = gu[i] + dd * S.v[i];
		gn1[i] = S.sigma * (gv[i] + dd * S.u[i]);
	}
	// F.normalize: x / N  ->  dx = gn / N - (gn . x) x / N^3 (N = max(|x|, 1e-12); the norm's gradient is cut where the clamp acts)
	float dot0 = 0.f, dot1 = 0.f;
#pragma unroll
	for (int i = 0; i < 4; i++) { dot0 += gn0[i] * q0[i]; dot1 += gn1[i] * q1[i]; }
	const float k0 = S.n0 > 1e-12f ? dot0 / (S.n0 * S.n0 * S.n0) : 0.f, k1 = S.n1 > 1e-12f ? dot1 / (S.n1 * S.n1 * S.n1) : 0.f;
#pragma unroll
	for (int i = 0; i < 4; i++) {
		gq0[i] = gn0[i] / S.n0 - k0 * q0[i];
		gq1[i] = gn1[i] / S.n1 - k1 * q1[i];
	}
}

__device__ __forceinline__ void load3(const float *__restrict__ p, float o[3]) {
#pragma unroll
	for (int i = 0; i < 3; i++) o[i] = __ldg(p + i);
}
__device__ __forceinline__ void load4(const float *__restrict__ p, float o[4]) {
#pragma unroll
	for (int i = 0; i < 4; i++) o[i] = __ldg(p + i);
}

// get_tracking_translation_ and get_tracking_rotation_ at tq (actor_pose.py:107-122, 138-158).
struct Sub {
	float a, b, ic, r;          // fp32 interpolation factors of the translation, and the slerp step
	float qa[4], q1[4], q2[4];  // input_rots[f1, c1]; the slerp's two ends
	float th1, th2;
};
__device__ __forceinline__ Sub sub_eval(const PoseArgs &A, const Pick &p, const double tq, float trans[3], float rot[4]) {
	Sub S;
	S.a = (float)(p.t2 - tq);
	S.b = (float)(tq - p.t1);
	S.ic = __fdiv_rn(1.f, (float)(p.t2 - p.t1));
	S.r = (float)((tq - p.t1) / (p.t2 - p.t1));
	const int r1 = p.f1 * A.K + p.c1, r2 = p.f2 * A.K + p.c2;
	float t1[3], t2[3];
	load3(A.in_trans + 3 * r1, t1);
	load3(A.in_trans + 3 * r2, t2);
	if (A.opt_track) {
		float o1[3], o2[3];
		load3(A.opt_trans + 3 * r1, o1);
		load3(A.opt_trans + 3 * r2, o2);
#pragma unroll
		for (int i = 0; i < 3; i++) { t1[i] = __fadd_rn(t1[i], o1[i]); t2[i] = __fadd_rn(t2[i], o2[i]); }
	}
#pragma unroll
	for (int i = 0; i < 3; i++) trans[i] = __fmul_rn(__fadd_rn(__fmul_rn(t1[i], S.a), __fmul_rn(t2[i], S.b)), S.ic);
	load4(A.in_rots + 4 * r1, S.qa);
	if (A.opt_track) {
		S.th1 = __ldg(A.opt_rots + r1);
		S.th2 = __ldg(A.opt_rots + p.f1 * A.K + p.c2);  // actor_pose.py:148: frame_ind1, column_ind2
		mul_theta(S.qa, S.th1, S.q1);
		mul_theta(S.q1, S.th2, S.q2);
	} else {
		S.th1 = S.th2 = 0.f;
#pragma unroll
		for (int i = 0; i < 4; i++) S.q1[i] = S.qa[i];
		load4(A.in_rots + 4 * r2, S.q2);
	}
	slerp_fwd(S.q1, S.q2, S.r, rot);
	return S;
}
// Gradient of one sub_eval for upstream (gt, gr): contributions to opt_trans rows (f1, c1), (f2, c2) and opt_rots rows (f1, c1), (f1, c2)
// written to scratch slots 2k and 2k + 1.
__device__ __forceinline__ void sub_bwd(const PoseArgs &A, const Pick &p, const Sub &S, const float gt[3], const float gr[4], const int actor, const int k,
                                        const bool write) {
	const int r1 = p.f1 * A.K + p.c1, r2 = p.f2 * A.K + p.c2, rt2 = p.f1 * A.K + p.c2;
	float gq1[4], gq2[4], gqa[4] = {0.f, 0.f, 0.f, 0.f};
	slerp_bwd(S.q1, S.q2, S.r, gr, gq1, gq2);
	const float dth2 = mul_theta_bwd(S.q1, S.th2, gq2, gq1);
	const float dth1 = mul_theta_bwd(S.qa, S.th1, gq1, gqa);
	if (!write) return;
	const int s0 = 4 * actor + 2 * k;
	A.trow[s0] = r1;
	A.trow[s0 + 1] = r2;
	A.rrow[s0] = r1;
	A.rrow[s0 + 1] = rt2;
#pragma unroll
	for (int i = 0; i < 3; i++) {
		const float gx = __fmul_rn(gt[i], S.ic);
		A.tval[3 * s0 + i] = __fmul_rn(gx, S.a);
		A.tval[3 * (s0 + 1) + i] = __fmul_rn(gx, S.b);
	}
	A.rval[s0] = dth1;
	A.rval[s0 + 1] = dth2;
}

// The validation path's two camera timestamps, or false for the training path (not opt_track / not is_val / fewer than two in span).
__device__ __forceinline__ bool val_stamps(const PoseArgs &A, const int trk, double &c1, double &c2) {
	if (!(A.opt_track && A.is_val)) return false;
	int i1, i2;
	const int n = nearest_two(A.cam_ts, __ldg(A.cam_off + A.cam), __ldg(A.cam_off + A.cam + 1), A.t, true, __ldg(A.track_span + 2 * trk),
	                          __ldg(A.track_span + 2 * trk + 1), i1, i2);
	if (n < 2) return false;
	c1 = __ldg(A.cam_ts + i1);
	c2 = __ldg(A.cam_ts + i2);
	return true;
}

__global__ void __launch_bounds__(32 * kPoseWarps) actor_pose_fwd_kernel(const PoseArgs A) {
	const int w = blockIdx.x * kPoseWarps + (threadIdx.x >> 5);
	if (w >= A.n) return;  // whole warps leave together
	const bool lead = (threadIdx.x & 31) == 0;
	const int trk = A.slot[w];
	const int out = A.base + w;
	float trans[3], rot[4];
	double c1, c2;
	if (val_stamps(A, trk, c1, c2)) {
		const Pick p1 = pick_entries(A, trk, c1), p2 = pick_entries(A, trk, c2);
		float ta[3], tb[3], ra[4], rb[4];
		sub_eval(A, p1, c1, ta, ra);
		sub_eval(A, p2, c2, tb, rb);
		const float a = (float)(c2 - A.t), b = (float)(A.t - c1), ic = __fdiv_rn(1.f, (float)(c2 - c1)), r = (float)((A.t - c1) / (c2 - c1));
#pragma unroll
		for (int i = 0; i < 3; i++) trans[i] = __fmul_rn(__fadd_rn(__fmul_rn(ta[i], a), __fmul_rn(tb[i], b)), ic);
		slerp_fwd(ra, rb, r, rot);
	} else {
		const Pick p = pick_entries(A, trk, A.t);
		sub_eval(A, p, A.t, trans, rot);
	}
	if (lead) {
		float e[4], q[4];
		ego_quat(A.ego, e);
		quat_mul(e, rot, q);
		float *o = A.poses + 7 * (size_t)out;
#pragma unroll
		for (int i = 0; i < 4; i++) o[i] = q[i];
#pragma unroll
		for (int i = 0; i < 3; i++) {
			const float *m = A.ego + 4 * i;
			o[4 + i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(m), trans[0]), __fmul_rn(__ldg(m + 1), trans[1])), __fmul_rn(__ldg(m + 2), trans[2])),
			                     __ldg(m + 3));
		}
		if (A.idft) {  // IDFT(time, C)[0] with time = fourier_scale * (frame - start) / (end - start) formed in float64, then fp32
			const int sf = __ldg(A.track_frames + 2 * trk), ef = __ldg(A.track_frames + 2 * trk + 1);
			const float tf = (float)(A.fourier_scale * ((double)(A.frame - sf) / (double)(ef - sf)));
			const float x = __fmul_rn((float)M_PI, tf);
			for (int k = 0; k < A.fourier_dim; k++)
				A.idft[(size_t)out * A.fourier_dim + k] = (k & 1) ? sinf(__fmul_rn(x, (float)(k + 1))) : cosf(__fmul_rn(x, (float)k));
		}
	}
}

__global__ void __launch_bounds__(32 * kPoseWarps) actor_pose_bwd_kernel(const PoseArgs A) {
	const int w = blockIdx.x * kPoseWarps + (threadIdx.x >> 5);
	if (w >= A.n) return;
	const bool lead = (threadIdx.x & 31) == 0;
	const int trk = A.slot[w];
	const int out = A.base + w;
	// dL/dtrans = R_ego^T dL/dt;  dL/drot = L(e)^T dL/dq for q = e (x) rot
	float g[7], e[4], gt[3], gr[4];
#pragma unroll
	for (int i = 0; i < 7; i++) g[i] = __ldg(A.gposes + 7 * (size_t)out + i);
#pragma unroll
	for (int j = 0; j < 3; j++) gt[j] = __ldg(A.ego + j) * g[4] + __ldg(A.ego + 4 + j) * g[5] + __ldg(A.ego + 8 + j) * g[6];
	ego_quat(A.ego, e);
	gr[0] = e[0] * g[0] + e[1] * g[1] + e[2] * g[2] + e[3] * g[3];
	gr[1] = -e[1] * g[0] + e[0] * g[1] + e[3] * g[2] - e[2] * g[3];
	gr[2] = -e[2] * g[0] - e[3] * g[1] + e[0] * g[2] + e[1] * g[3];
	gr[3] = -e[3] * g[0] + e[2] * g[1] - e[1] * g[2] + e[0] * g[3];
	const int s0 = 4 * (A.base + w);
	double c1, c2;
	if (val_stamps(A, trk, c1, c2)) {
		const Pick p1 = pick_entries(A, trk, c1), p2 = pick_entries(A, trk, c2);
		float ta[3], tb[3], ra[4], rb[4];
		const Sub S1 = sub_eval(A, p1, c1, ta, ra), S2 = sub_eval(A, p2, c2, tb, rb);
		const float a = (float)(c2 - A.t), b = (float)(A.t - c1), ic = __fdiv_rn(1.f, (float)(c2 - c1)), r = (float)((A.t - c1) / (c2 - c1));
		float gta[3], gtb[3], gra[4], grb[4];
#pragma unroll
		for (int i = 0; i < 3; i++) {
			const float gx = __fmul_rn(gt[i], ic);
			gta[i] = __fmul_rn(gx, a);
			gtb[i] = __fmul_rn(gx, b);
		}
		slerp_bwd(ra, rb, r, gr, gra, grb);
		sub_bwd(A, p1, S1, gta, gra, A.base + w, 0, lead);
		sub_bwd(A, p2, S2, gtb, grb, A.base + w, 1, lead);
	} else {
		const Pick p = pick_entries(A, trk, A.t);
		float tr[3], ro[4];
		const Sub S = sub_eval(A, p, A.t, tr, ro);
		sub_bwd(A, p, S, gt, gr, A.base + w, 0, lead);
		if (lead) {
			A.trow[s0 + 2] = A.trow[s0 + 3] = -1;
			A.rrow[s0 + 2] = A.rrow[s0 + 3] = -1;
		}
	}
}

// Each row's contributions summed in slot order (actor order, then slot) by the thread of its first slot, and added once.
__global__ void __launch_bounds__(kAccumThreads) actor_pose_accum_kernel(const int nslots, const int *__restrict__ trow, const float *__restrict__ tval,
                                                                          const int *__restrict__ rrow, const float *__restrict__ rval,
                                                                          float *__restrict__ g_trans, float *__restrict__ g_rots) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= 2 * nslots) return;
	const bool rot = i >= nslots;
	const int s = rot ? i - nslots : i;
	const int *__restrict__ rows = rot ? rrow : trow;
	const int row = __ldg(rows + s);
	if (row < 0) return;
	for (int j = 0; j < s; j++)
		if (__ldg(rows + j) == row) return;
	if (rot) {
		float acc = __ldg(rval + s);
		for (int j = s + 1; j < nslots; j++)
			if (__ldg(rrow + j) == row) acc = __fadd_rn(acc, __ldg(rval + j));
		g_rots[row] = __fadd_rn(g_rots[row], acc);
	} else {
		float acc[3] = {__ldg(tval + 3 * s), __ldg(tval + 3 * s + 1), __ldg(tval + 3 * s + 2)};
		for (int j = s + 1; j < nslots; j++)
			if (__ldg(trow + j) == row) {
#pragma unroll
				for (int c = 0; c < 3; c++) acc[c] = __fadd_rn(acc[c], __ldg(tval + 3 * j + c));
			}
#pragma unroll
		for (int c = 0; c < 3; c++) g_trans[3 * (size_t)row + c] = __fadd_rn(g_trans[3 * (size_t)row + c], acc[c]);
	}
}

size_t actor_pose_scratch_bytes(int n) { return (size_t)n * 4 * (2 * sizeof(int) + 4 * sizeof(float)); }

static PoseArgs pose_args(const ActorPoseTable &T, const ActorPoseCall &c) {
	PoseArgs A;
	memset(&A, 0, sizeof(A));
	A.K = T.K;
	A.opt_track = c.opt_track;
	A.is_val = c.is_val;
	A.cam = c.cam;
	A.frame = c.frame;
	A.fourier_dim = c.fourier_dim;
	A.t = c.timestamp;
	A.fourier_scale = c.fourier_scale;
	A.track_off = T.track_off;
	A.entry_fc = T.entry_fc;
	A.track_frames = T.track_frames;
	A.cam_off = T.cam_off;
	A.entry_ts = T.entry_ts;
	A.track_span = T.track_span;
	A.cam_ts = T.cam_ts;
	A.in_trans = T.input_trans;
	A.in_rots = T.input_rots;
	A.opt_trans = c.opt_trans;
	A.opt_rots = c.opt_rots;
	A.ego = c.ego_pose;
	return A;
}

static int pose_blocks(int n) { return (n + kPoseWarps - 1) / kPoseWarps; }

cudaError_t launch_actor_pose_fwd(const ActorPoseTable &T, const ActorPoseCall &c, const int32_t *slots, int n, float *poses, float *idft,
                                  cudaStream_t st) {
	PoseArgs A = pose_args(T, c);
	A.poses = poses;
	A.idft = idft;
	for (int base = 0; base < n; base += kActorPoseChunk) {
		A.base = base;
		A.n = n - base < kActorPoseChunk ? n - base : kActorPoseChunk;
		for (int i = 0; i < A.n; i++) A.slot[i] = slots[base + i];
		count_launch();
		actor_pose_fwd_kernel<<<pose_blocks(A.n), 32 * kPoseWarps, 0, st>>>(A);
		if (cudaError_t e = cudaGetLastError()) return e;
	}
	return cudaSuccess;
}

cudaError_t launch_actor_pose_bwd(const ActorPoseTable &T, const ActorPoseCall &c, const int32_t *slots, int n, const float *g_poses, float *g_trans,
                                  float *g_rots, void *scratch, cudaStream_t st) {
	PoseArgs A = pose_args(T, c);
	A.gposes = g_poses;
	char *p = reinterpret_cast<char *>(scratch);
	const int ns = 4 * n;
	A.trow = reinterpret_cast<int *>(p);
	A.rrow = A.trow + ns;
	A.tval = reinterpret_cast<float *>(A.rrow + ns);
	A.rval = A.tval + 3 * ns;
	for (int base = 0; base < n; base += kActorPoseChunk) {
		A.base = base;
		A.n = n - base < kActorPoseChunk ? n - base : kActorPoseChunk;
		for (int i = 0; i < A.n; i++) A.slot[i] = slots[base + i];
		count_launch();
		actor_pose_bwd_kernel<<<pose_blocks(A.n), 32 * kPoseWarps, 0, st>>>(A);
		if (cudaError_t e = cudaGetLastError()) return e;
	}
	count_launch();
	actor_pose_accum_kernel<<<(2 * ns + kAccumThreads - 1) / kAccumThreads, kAccumThreads, 0, st>>>(ns, A.trow, A.tval, A.rrow, A.rval, g_trans, g_rots);
	return cudaGetLastError();
}

}  // namespace sgr
