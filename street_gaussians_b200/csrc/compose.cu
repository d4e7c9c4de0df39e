// compose.cu — the scene-graph composer of street_gaussians as two kernels (SURVEY.md §8 row f1).
//
// The reference re-materialises the 59 floats per Gaussian that the rasterizer consumes with ~40 small PyTorch kernels per
// frame: per-model activations (lib/models/gaussian_model.py:224-251), the actors' Fourier DC colour
// (lib/models/gaussian_model_actor.py:71-80), the rigid pose of every actor applied to positions and rotations with an optional
// mirror augmentation (lib/models/street_gaussian_model.py:305-363), and five torch.cat (:287-449).  Here one kernel reads the
// raw parameters of every sub-model in place (a table of segments: background + actors) and writes the composed
// means3D / rotations / scales / opacities / shs once; one kernel sends the gradients back to the raw parameter layouts and
// reduces the tracked-pose gradients per actor.  Per-frame inputs are tiny (7 floats of pose + the IDFT row per actor), so a
// training step uploads poses, not parameters.
//
// Both kernels are HBM-bound streams: thread = Gaussian for the 11 + 4 small values, warp-cooperative (coalesced) copies for
// the SH rows, which are 80 % of the bytes.
#include "sgr_common.cuh"

namespace sgr {

constexpr int kMaxSeg = SGR_MAX_SEGMENTS_PER_LAUNCH;
static_assert(kMaxSeg <= 32, "compose_pose_finalize_kernel takes the posed flags of a group as one 32-bit mask");

struct SegDev {
	const float *xyz, *rotation, *scaling, *opacity, *fdc, *frest;
};
struct SegGradDev {
	float *xyz, *rotation, *scaling, *opacity, *fdc, *frest;
};
struct SegTable {
	int n;                   // segments in this launch
	int first;               // index of segment 0 of this launch in the caller's table (poses / idft / dposes rows)
	int start[kMaxSeg + 1];  // composed index of each segment's first Gaussian; start[n] = end
	int fourier[kMaxSeg];
	int posed[kMaxSeg];
	SegDev seg[kMaxSeg];
};
struct SegGradTable {
	SegGradDev seg[kMaxSeg];
};

__device__ __forceinline__ int find_segment(const SegTable &t, int i) {
	int lo = 0, hi = t.n - 1;  // largest s with start[s] <= i
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (t.start[mid] <= i) lo = mid; else hi = mid - 1;
	}
	return lo;
}

__device__ __forceinline__ float4 qmul(const float4 a, const float4 b) {  // (w,x,y,z) in (.x,.y,.z,.w); general_utils.py:232-238
	return make_float4(a.x * b.x - a.y * b.y - a.z * b.z - a.w * b.w, a.x * b.y + a.y * b.x + a.z * b.w - a.w * b.z,
	                   a.x * b.z - a.y * b.w + a.z * b.x + a.w * b.y, a.x * b.w + a.y * b.z - a.z * b.y + a.w * b.x);
}
__device__ __forceinline__ float4 qconj(const float4 a) { return make_float4(a.x, -a.y, -a.z, -a.w); }
__device__ __forceinline__ float qnorm_clamped(const float4 q) {  // F.normalize: x / max(||x||, 1e-12)
	return fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);
}
// rotation matrix (row-major) of the NORMALISED quaternion (general_utils.py:125-146)
__device__ __forceinline__ void quat_to_rot(const float4 r, float R[9]) {
	const float n = sqrtf(r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w);
	const float w = r.x / n, x = r.y / n, y = r.z / n, z = r.w / n;
	R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - w * z); R[2] = 2.f * (x * z + w * y);
	R[3] = 2.f * (x * y + w * z); R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - w * x);
	R[6] = 2.f * (x * z - w * y); R[7] = 2.f * (y * z + w * x); R[8] = 1.f - 2.f * (x * x + y * y);
}

// What a warp needs to move its SH rows cooperatively: all 32 lanes in one segment, consecutive local indices.
__device__ __forceinline__ bool warp_is_contiguous(int seg, int li, bool active) {
	const unsigned full = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int s0 = __shfl_sync(full, seg, 0), l0 = __shfl_sync(full, li, 0);
	return __all_sync(full, active && seg == s0 && li == l0 + lane);
}

// Warp-cooperative copy of 32 rows of R3 floats between a dense block (row stride R3) and rows embedded at `off` in rows of stride
// `wide`.  Loads are issued in batches of kCopyBatch before the dependent stores: the naive "load one, store one" loop kept ONE
// request in flight per lane and left the composer waiting on memory (long-scoreboard stalls on the store) far below the HBM roofline.
constexpr int kCopyBatch = 9;
template <bool TO_WIDE>
__device__ __forceinline__ void warp_copy_rows(const float *__restrict__ src, float *__restrict__ dst, const int R3, const int wide, const int off,
                                               const int lane) {
	const int total = 32 * R3;
	int row = lane / R3, col = lane - row * R3;  // position of element e = lane in the dense block
	for (int e0 = lane; e0 < total; e0 += 32 * kCopyBatch) {
		float v[kCopyBatch];
		int r[kCopyBatch], c[kCopyBatch];
#pragma unroll
		for (int u = 0; u < kCopyBatch; u++) {
			const int e = e0 + 32 * u;
			r[u] = row; c[u] = col;
			if (e < total) v[u] = TO_WIDE ? __ldg(src + e) : __ldg(src + (size_t)row * wide + off + col);
			col += 32;
			while (col >= R3) { col -= R3; row++; }
		}
#pragma unroll
		for (int u = 0; u < kCopyBatch; u++) {
			const int e = e0 + 32 * u;
			if (e < total) {
				if (TO_WIDE) dst[(size_t)r[u] * wide + off + c[u]] = v[u];
				else dst[e] = v[u];
			}
		}
	}
}

__global__ void __launch_bounds__(256) compose_fwd_kernel(const SegTable t, const int M, const float *__restrict__ poses,
                                                         const float *__restrict__ idft, const uint8_t *__restrict__ flip,
                                                         const float *__restrict__ flip_quat, float *__restrict__ o_xyz,
                                                         float *__restrict__ o_rot, float *__restrict__ o_scale, float *__restrict__ o_opac,
                                                         float *__restrict__ o_sh) {
	const int i = t.start[0] + blockIdx.x * blockDim.x + threadIdx.x;
	const bool active = i < t.start[t.n];
	const int lane = threadIdx.x & 31;
	int s = 0, li = 0;
	if (active) {
		s = find_segment(t, i);
		li = i - t.start[s];
		const SegDev sg = t.seg[s];
		const size_t l = (size_t)li, g = (size_t)i;
		// all per-Gaussian inputs are requested before any arithmetic (one DRAM round trip)
		float3 p = make_float3(sg.xyz[3 * l], sg.xyz[3 * l + 1], sg.xyz[3 * l + 2]);
		float4 q = *reinterpret_cast<const float4 *>(sg.rotation + 4 * l);
		const float3 ls = make_float3(sg.scaling[3 * l], sg.scaling[3 * l + 1], sg.scaling[3 * l + 2]);
		const float lo = sg.opacity[l];
		const int C = t.fourier[s];
		const float *fd = sg.fdc + l * C * 3;
		const float3 dc0 = make_float3(fd[0], fd[1], fd[2]);
		const float qn = qnorm_clamped(q);
		q = make_float4(q.x / qn, q.y / qn, q.z / qn, q.w / qn);  // gaussian_model.py:229-230
		if (t.posed[s]) {
			const float *ps = poses + (size_t)(t.first + s) * 8;
			const float4 qo = make_float4(ps[0], ps[1], ps[2], ps[3]);
			const bool fl = flip != nullptr && flip[i] != 0;
			if (fl) {  // mirror across the actor's local x-z plane (street_gaussian_model.py:319-323, 347-349)
				p.y = -p.y;
				q = qmul(make_float4(flip_quat[0], flip_quat[1], flip_quat[2], flip_quat[3]), q);
			}
			float R[9];
			quat_to_rot(qo, R);
			p = make_float3(R[0] * p.x + R[1] * p.y + R[2] * p.z + ps[4], R[3] * p.x + R[4] * p.y + R[5] * p.z + ps[5],
			                R[6] * p.x + R[7] * p.y + R[8] * p.z + ps[6]);
			q = qmul(qo, q);  // raw product with the (un-normalised) actor quaternion, then normalise (:324-325)
			const float n2 = qnorm_clamped(q);
			q = make_float4(q.x / n2, q.y / n2, q.z / n2, q.w / n2);
		}
		o_xyz[3 * g] = p.x; o_xyz[3 * g + 1] = p.y; o_xyz[3 * g + 2] = p.z;
		*reinterpret_cast<float4 *>(o_rot + 4 * g) = q;
		o_scale[3 * g] = expf(ls.x); o_scale[3 * g + 1] = expf(ls.y); o_scale[3 * g + 2] = expf(ls.z);
		o_opac[g] = 1.0f / (1.0f + expf(-lo));
		// DC colour: background = its single row; actors = sum_c dc[c] * IDFT(t)[c] (gaussian_model_actor.py:76-77)
		float d0 = dc0.x, d1 = dc0.y, d2 = dc0.z;
		if (t.posed[s]) {
			const float *w = idft + (size_t)(t.first + s) * SGR_MAX_FOURIER;
			d0 *= w[0]; d1 *= w[0]; d2 *= w[0];
			for (int c = 1; c < C; c++) {
				const float *f = fd + c * 3;
				d0 += f[0] * w[c]; d1 += f[1] * w[c]; d2 += f[2] * w[c];
			}
		}
		float *dst = o_sh + g * M * 3;
		dst[0] = d0; dst[1] = d1; dst[2] = d2;
	}
	// higher SH bands: rows of (M-1)*3 floats -> rows of M*3 floats, offset 3
	const int R3 = (M - 1) * 3;
	if (R3 <= 0) return;
	if (warp_is_contiguous(s, li, active)) {
		const int s0 = __shfl_sync(0xffffffffu, s, 0), l0 = __shfl_sync(0xffffffffu, li, 0), i0 = __shfl_sync(0xffffffffu, i, 0);
		warp_copy_rows<true>(t.seg[s0].frest + (size_t)l0 * R3, o_sh + (size_t)i0 * M * 3, R3, M * 3, 3, lane);
	} else if (active) {
		const float *src = t.seg[s].frest + (size_t)li * R3;
		float *dst = o_sh + (size_t)i * M * 3 + 3;
		for (int k = 0; k < R3; k++) dst[k] = __ldg(src + k);
	}
}

// acc[16] per segment: G = sum g_xyz (x) x_local (9, row-major), g_a = sum over the rotation path (4), sum g_xyz (3)
__global__ void __launch_bounds__(256) compose_bwd_kernel(const SegTable t, const SegGradTable gt, const int M, const float *__restrict__ poses,
                                                         const float *__restrict__ idft, const uint8_t *__restrict__ flip,
                                                         const float *__restrict__ flip_quat, const float *__restrict__ g_xyz,
                                                         const float *__restrict__ g_rot, const float *__restrict__ g_scale,
                                                         const float *__restrict__ g_opac, const float *__restrict__ g_sh,
                                                         float *__restrict__ acc) {
	const int i = t.start[0] + blockIdx.x * blockDim.x + threadIdx.x;
	const bool active = i < t.start[t.n];
	const int lane = threadIdx.x & 31;
	const unsigned full = 0xffffffffu;
	int s = 0, li = 0;
	float a16[16];
#pragma unroll
	for (int k = 0; k < 16; k++) a16[k] = 0.f;
	bool posed = false;
	if (active) {
		s = find_segment(t, i);
		li = i - t.start[s];
		posed = t.posed[s] != 0;
		const SegDev sg = t.seg[s];
		const SegGradDev og = gt.seg[s];
		const size_t l = (size_t)li, g = (size_t)i;
		// all per-Gaussian inputs are requested before any arithmetic or store (one DRAM round trip)
		const float3 ls = make_float3(sg.scaling[3 * l], sg.scaling[3 * l + 1], sg.scaling[3 * l + 2]);
		const float3 gs = make_float3(g_scale[3 * g], g_scale[3 * g + 1], g_scale[3 * g + 2]);
		const float lo = sg.opacity[l], go = g_opac[g];
		const float gd0 = g_sh[g * M * 3], gd1 = g_sh[g * M * 3 + 1], gd2 = g_sh[g * M * 3 + 2];
		const float4 raw = *reinterpret_cast<const float4 *>(sg.rotation + 4 * l);
		float4 gn = *reinterpret_cast<const float4 *>(g_rot + 4 * g);  // gradient w.r.t. the composed (unit) rotation
		float3 gx = make_float3(g_xyz[3 * g], g_xyz[3 * g + 1], g_xyz[3 * g + 2]);
		float3 xl = posed ? make_float3(sg.xyz[3 * l], sg.xyz[3 * l + 1], sg.xyz[3 * l + 2]) : make_float3(0.f, 0.f, 0.f);
		// activations (gaussian_model.py:224-251): d exp = exp, d sigmoid = o (1 - o)
		og.scaling[3 * l] = gs.x * expf(ls.x); og.scaling[3 * l + 1] = gs.y * expf(ls.y); og.scaling[3 * l + 2] = gs.z * expf(ls.z);
		const float o = 1.0f / (1.0f + expf(-lo));
		og.opacity[l] = go * o * (1.f - o);
		// DC colour
		const int C = t.fourier[s];
		if (posed) {
			const float *w = idft + (size_t)(t.first + s) * SGR_MAX_FOURIER;
			for (int c = 0; c < C; c++) {
				float *f = og.fdc + (l * C + c) * 3;
				f[0] = gd0 * w[c]; f[1] = gd1 * w[c]; f[2] = gd2 * w[c];
			}
		} else {
			float *f = og.fdc + l * C * 3;
			f[0] = gd0; f[1] = gd1; f[2] = gd2;
			for (int k = 3; k < C * 3; k++) f[k] = 0.f;  // (a background with C > 1 only ever uses row 0)
		}
		// rotation: z = normalize(y), y = q_obj (x) b, b = [flip_quat (x)] n, n = normalize(raw)
		const float rn = qnorm_clamped(raw);
		const float4 n = make_float4(raw.x / rn, raw.y / rn, raw.z / rn, raw.w / rn);
		if (posed) {
			const float *ps = poses + (size_t)(t.first + s) * 8;
			const float4 qo = make_float4(ps[0], ps[1], ps[2], ps[3]);
			const bool fl = flip != nullptr && flip[i] != 0;
			const float4 fq = fl ? make_float4(flip_quat[0], flip_quat[1], flip_quat[2], flip_quat[3]) : make_float4(1.f, 0.f, 0.f, 0.f);
			const float4 b = fl ? qmul(fq, n) : n;
			const float4 y = qmul(qo, b);
			const float yn = qnorm_clamped(y);
			const float4 z = make_float4(y.x / yn, y.y / yn, y.z / yn, y.w / yn);
			const float dz = z.x * gn.x + z.y * gn.y + z.z * gn.z + z.w * gn.w;
			const float4 gy = make_float4((gn.x - z.x * dz) / yn, (gn.y - z.y * dz) / yn, (gn.z - z.z * dz) / yn, (gn.w - z.w * dz) / yn);
			const float4 ga = qmul(gy, qconj(b));  // d/d q_obj of q_obj (x) b
			float4 gb = qmul(qconj(qo), gy);       // d/d b
			if (fl) gb = qmul(qconj(fq), gb);
			gn = gb;
			a16[9] = ga.x; a16[10] = ga.y; a16[11] = ga.z; a16[12] = ga.w;
			// position: x_w = R(q_obj) x_l + t
			if (fl) xl.y = -xl.y;
			float R[9];
			quat_to_rot(qo, R);
			a16[0] = gx.x * xl.x; a16[1] = gx.x * xl.y; a16[2] = gx.x * xl.z;
			a16[3] = gx.y * xl.x; a16[4] = gx.y * xl.y; a16[5] = gx.y * xl.z;
			a16[6] = gx.z * xl.x; a16[7] = gx.z * xl.y; a16[8] = gx.z * xl.z;
			a16[13] = gx.x; a16[14] = gx.y; a16[15] = gx.z;
			float3 gl = make_float3(R[0] * gx.x + R[3] * gx.y + R[6] * gx.z, R[1] * gx.x + R[4] * gx.y + R[7] * gx.z,
			                        R[2] * gx.x + R[5] * gx.y + R[8] * gx.z);  // R^T g
			if (fl) gl.y = -gl.y;
			gx = gl;
		}
		og.xyz[3 * l] = gx.x; og.xyz[3 * l + 1] = gx.y; og.xyz[3 * l + 2] = gx.z;
		const float dn = n.x * gn.x + n.y * gn.y + n.z * gn.z + n.w * gn.w;  // through n = raw / max(|raw|, eps)
		*reinterpret_cast<float4 *>(og.rotation + 4 * l) =
		    make_float4((gn.x - n.x * dn) / rn, (gn.y - n.y * dn) / rn, (gn.z - n.z * dn) / rn, (gn.w - n.w * dn) / rn);
	}
	// tracked-pose sums: one atomic per (warp, component) when the whole warp sits in one actor
	const bool contiguous = warp_is_contiguous(s, li, active);
	const bool any_posed = __any_sync(full, posed);
	if (any_posed) {
		const int s0 = __shfl_sync(full, s, 0);
		const bool uniform = __all_sync(full, !active || s == s0);
		if (uniform) {
#pragma unroll
			for (int k = 0; k < 16; k++) {
				float v = a16[k];
#pragma unroll
				for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(full, v, o);
				if (lane == k) atomicAdd(acc + (size_t)(t.first + s0) * 16 + k, v);
			}
		} else if (posed) {
#pragma unroll
			for (int k = 0; k < 16; k++) atomicAdd(acc + (size_t)(t.first + s) * 16 + k, a16[k]);
		}
	}
	// higher SH bands back to the per-model rows
	const int R3 = (M - 1) * 3;
	if (R3 <= 0) return;
	if (contiguous) {
		const int s0 = __shfl_sync(full, s, 0), l0 = __shfl_sync(full, li, 0), i0 = __shfl_sync(full, i, 0);
		warp_copy_rows<false>(g_sh + (size_t)i0 * M * 3, gt.seg[s0].frest + (size_t)l0 * R3, R3, M * 3, 3, lane);
	} else if (active) {
		float *dst = gt.seg[s].frest + (size_t)li * R3;
		const float *src = g_sh + (size_t)i * M * 3 + 3;
		for (int k = 0; k < R3; k++) dst[k] = __ldg(src + k);
	}
}

// acc[16] -> d pose (4 + 3, padded to 8): the matrix path goes through quaternion_to_matrix's normalisation.  One warp per group of
// kMaxSeg segments; bit k of `posed` is segment first + k.  Rows of unposed segments are written as zeros: their pose row is not
// read by the other kernels and may hold anything, a zero quaternion included (composer.py leaves the background's row zero).
__global__ void compose_pose_finalize_kernel(const int first, const int n, const unsigned posed, const float *__restrict__ poses,
                                             const float *__restrict__ acc, float *__restrict__ dposes) {
	if ((int)threadIdx.x >= n) return;
	const size_t s = (size_t)first + threadIdx.x;
	float *o = dposes + s * 8;
	if (!((posed >> threadIdx.x) & 1u)) {
		for (int k = 0; k < 8; k++) o[k] = 0.f;
		return;
	}
	const float *a = acc + s * 16, *ps = poses + s * 8;
	const float nr = sqrtf(ps[0] * ps[0] + ps[1] * ps[1] + ps[2] * ps[2] + ps[3] * ps[3]);
	const float w = ps[0] / nr, x = ps[1] / nr, y = ps[2] / nr, z = ps[3] / nr;
	const float G00 = a[0], G01 = a[1], G02 = a[2], G10 = a[3], G11 = a[4], G12 = a[5], G20 = a[6], G21 = a[7], G22 = a[8];
	const float dw = 2.f * (-z * G01 + y * G02 + z * G10 - x * G12 - y * G20 + x * G21);
	const float dx = 2.f * (y * G01 + z * G02 + y * G10 - 2.f * x * G11 - w * G12 + z * G20 + w * G21 - 2.f * x * G22);
	const float dy = 2.f * (-2.f * y * G00 + x * G01 + w * G02 + x * G10 + z * G12 - w * G20 + z * G21 - 2.f * y * G22);
	const float dz = 2.f * (-2.f * z * G00 - w * G01 + x * G02 + w * G10 - 2.f * z * G11 + y * G12 + x * G20 + y * G21);
	const float dot = w * dw + x * dx + y * dy + z * dz;
	o[0] = a[9] + (dw - w * dot) / nr; o[1] = a[10] + (dx - x * dot) / nr; o[2] = a[11] + (dy - y * dot) / nr; o[3] = a[12] + (dz - z * dot) / nr;
	o[4] = a[13]; o[5] = a[14]; o[6] = a[15]; o[7] = 0.f;
}

static void fill_table(SegTable &t, const SgrSegment *segs, int first, int n) {
	t.n = n;
	t.first = first;
	for (int k = 0; k < n; k++) {
		const SgrSegment &s = segs[first + k];
		t.start[k] = s.start;
		t.fourier[k] = s.fourier_dim;
		t.posed[k] = s.posed;
		t.seg[k] = SegDev{s.xyz, s.rotation, s.scaling, s.opacity, s.features_dc, s.features_rest};
	}
	t.start[n] = segs[first + n - 1].start + segs[first + n - 1].count;
}

cudaError_t launch_compose_fwd(const SgrSegment *segs, int nseg, int M, const float *poses, const float *idft, const uint8_t *flip,
                               const float *flip_quat, float *xyz, float *rot, float *scale, float *opac, float *sh, cudaStream_t st) {
	for (int first = 0; first < nseg; first += kMaxSeg) {
		SegTable t;
		fill_table(t, segs, first, nseg - first < kMaxSeg ? nseg - first : kMaxSeg);
		const int count = t.start[t.n] - t.start[0];
		if (count <= 0) continue;
		count_launch();
		compose_fwd_kernel<<<(count + 255) / 256, 256, 0, st>>>(t, M, poses, idft, flip, flip_quat, xyz, rot, scale, opac, sh);
	}
	return cudaGetLastError();
}

cudaError_t launch_compose_bwd(const SgrSegment *segs, const SgrSegmentGrads *grads, int nseg, int M, const float *poses, const float *idft,
                               const uint8_t *flip, const float *flip_quat, const float *g_xyz, const float *g_rot, const float *g_scale,
                               const float *g_opac, const float *g_sh, float *acc, float *dposes, cudaStream_t st) {
	cudaError_t e = cudaMemsetAsync(acc, 0, (size_t)nseg * 16 * sizeof(float), st);
	if (e != cudaSuccess) return e;
	for (int first = 0; first < nseg; first += kMaxSeg) {
		SegTable t;
		SegGradTable gt;
		const int n = nseg - first < kMaxSeg ? nseg - first : kMaxSeg;
		fill_table(t, segs, first, n);
		for (int k = 0; k < n; k++) {
			const SgrSegmentGrads &g = grads[first + k];
			gt.seg[k] = SegGradDev{g.xyz, g.rotation, g.scaling, g.opacity, g.features_dc, g.features_rest};
		}
		const int count = t.start[t.n] - t.start[0];
		if (count <= 0) continue;
		count_launch();
		compose_bwd_kernel<<<(count + 255) / 256, 256, 0, st>>>(t, gt, M, poses, idft, flip, flip_quat, g_xyz, g_rot, g_scale, g_opac, g_sh, acc);
	}
	for (int first = 0; first < nseg; first += kMaxSeg) {
		const int n = nseg - first < kMaxSeg ? nseg - first : kMaxSeg;
		unsigned posed = 0;
		for (int k = 0; k < n; k++) posed |= (segs[first + k].posed ? 1u : 0u) << k;
		count_launch();
		compose_pose_finalize_kernel<<<1, kMaxSeg, 0, st>>>(first, n, posed, poses, acc, dposes);
	}
	return cudaGetLastError();
}

}  // namespace sgr
