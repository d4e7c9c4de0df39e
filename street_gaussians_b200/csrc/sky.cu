// sky.cu — the sky cube map of street_gaussians (lib/models/sky_cubemap.py:77-123, composited at street_gaussian_renderer.py:107-111)
// as one fused kernel each way.
//
// Per pixel (column i, row j): the ray Rm^T K^-1 (i + a, j + b, 1) (graphics_utils.py:186-207; a = b = 0.5 without jitter), the mask
// (training with a sky mask: the mask or rows 0-49; otherwise 1 - acc > 1e-3), the cube lookup dr.texture(linear, cube) restates
// (face of the largest component, face coordinates inverting cube_to_dir, sky_cubemap.py:154-161, bilinear over four taps with edge
// and corner wrap), the clamp to [0, 1] and rgb + sky (1 - acc).  The backward recomputes the ray and the taps from the saved jitter.
// Nothing depends on how many pixels are sky: grids depend on H x W only and nothing is read back to the host.  The band forms run the
// same kernels over the pixels of a tile-row band only (multi-GPU, DESIGN.md §8): grids depend on H x W and the band.  The marking band
// backward also records which kSkyBlock x kSkyBlock blocks of the cube its atomics wrote, for the peer-memory exchange (peer_exchange.cu).
#include "sgr_common.cuh"

namespace sgr {

constexpr int kSkyThreads = 256;
constexpr int kSkyTopRows = 50;  // sky_cubemap.py:83: mask[:50, :] = True
constexpr float kThird = 1.f / 3.f;

// Face frames of cube_to_dir: direction = N + gx U + gy V.  An axis is coded as 1 + axis index, negated for the negative direction.
__constant__ int8_t kFaceN[6] = {1, -1, 2, -2, 3, -3};
__constant__ int8_t kFaceU[6] = {-3, 3, 1, 1, 1, -1};
__constant__ int8_t kFaceV[6] = {-2, -2, 3, -3, -2, -2};

__device__ __forceinline__ int axis_of(int code) { return (code < 0 ? -code : code) - 1; }
__device__ __forceinline__ int sign_of(int code) { return code < 0 ? -1 : 1; }
// The signed component of (x, y, z) along an axis code, by selects (an indexed array would live in local memory).
template <typename T>
__device__ __forceinline__ T along(int code, T x, T y, T z) {
	const int a = axis_of(code);
	const T v = a == 0 ? x : (a == 1 ? y : z);
	return code < 0 ? -v : v;
}
// The component on axis q of the unit vector an axis code names.
__device__ __forceinline__ int unit(int code, int q) { return axis_of(code) == q ? sign_of(code) : 0; }

struct SkyCam {
	float m[9];  // Rm^T K^-1, row-major
};

// K^-1 by the adjugate, then Rm^T K^-1; Rm = w2c[:3, :3] (w2c row-major [4, 4]).
__device__ __forceinline__ SkyCam sky_camera(const float *__restrict__ K, const float *__restrict__ w2c) {
	float k[9], r[9], inv[9];
#pragma unroll
	for (int e = 0; e < 9; e++) k[e] = __ldg(K + e);
#pragma unroll
	for (int a = 0; a < 3; a++)
#pragma unroll
		for (int b = 0; b < 3; b++) r[a * 3 + b] = __ldg(w2c + a * 4 + b);
	inv[0] = k[4] * k[8] - k[5] * k[7];
	inv[1] = k[2] * k[7] - k[1] * k[8];
	inv[2] = k[1] * k[5] - k[2] * k[4];
	inv[3] = k[5] * k[6] - k[3] * k[8];
	inv[4] = k[0] * k[8] - k[2] * k[6];
	inv[5] = k[2] * k[3] - k[0] * k[5];
	inv[6] = k[3] * k[7] - k[4] * k[6];
	inv[7] = k[1] * k[6] - k[0] * k[7];
	inv[8] = k[0] * k[4] - k[1] * k[3];
	const float rdet = __frcp_rn(k[0] * inv[0] + k[1] * inv[3] + k[2] * inv[6]);
#pragma unroll
	for (int e = 0; e < 9; e++) inv[e] = inv[e] * rdet;
	SkyCam c;
#pragma unroll
	for (int a = 0; a < 3; a++)
#pragma unroll
		for (int b = 0; b < 3; b++) c.m[a * 3 + b] = r[0 * 3 + a] * inv[0 * 3 + b] + r[1 * 3 + a] * inv[1 * 3 + b] + r[2 * 3 + a] * inv[2 * 3 + b];
	return c;
}

// Texel of tap (c, r) on face f, c and r in [-1, R]: the flat texel index into [6, R, R], or -1 for the tap past a cube corner.
// A tap past one edge is read from the adjacent face: the extrapolated texel centre, as the integer lattice direction
// D = R N + (2c + 1 - R) U + (2r + 1 - R) V, has its largest component on the neighbour's axis; there the component that was the old
// face's axis (+-R) names the neighbour's edge row or column, and the other (|.| < R) the same position along the shared edge.
__device__ __forceinline__ int sky_texel(const int f, const int c, const int r, const int R) {
	const bool oc = c < 0 || c >= R, orow = r < 0 || r >= R;
	if (!oc && !orow) return (f * R + r) * R + c;
	if (oc && orow) return -1;
	const int n = kFaceN[f], uc = kFaceU[f], vc = kFaceV[f], du = 2 * c + 1 - R, dv = 2 * r + 1 - R;
	const int Dx = unit(n, 0) * R + unit(uc, 0) * du + unit(vc, 0) * dv, Dy = unit(n, 1) * R + unit(uc, 1) * du + unit(vc, 1) * dv,
	          Dz = unit(n, 2) * R + unit(uc, 2) * du + unit(vc, 2) * dv;
	const int out_code = oc ? uc * (c < 0 ? -1 : 1) : vc * (r < 0 ? -1 : 1);  // the neighbour's N
	int nf = 0;
#pragma unroll
	for (int q = 0; q < 6; q++)
		if (kFaceN[q] == out_code) nf = q;
	const int a = along(kFaceU[nf], Dx, Dy, Dz), b = along(kFaceV[nf], Dx, Dy, Dz);
	const int nc = a >= R ? R - 1 : (a <= -R ? 0 : (a + R - 1) / 2);
	const int nr = b >= R ? R - 1 : (b <= -R ? 0 : (b + R - 1) / 2);
	return (nf * R + nr) * R + nc;
}

struct SkyTaps {
	int idx[4];    // texels of taps (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1); -1 for a corner tap
	float w[4];    // bilinear weights
	int corner;    // which tap is past a cube corner, or -1
};

// Face, coordinates and taps of direction d on a cube of R x R faces.
__device__ __forceinline__ SkyTaps sky_taps(const float d[3], const int R) {
	const float ax = fabsf(d[0]), ay = fabsf(d[1]), az = fabsf(d[2]);
	int f;
	float ma;
	if (az > ax && az > ay) { f = d[2] >= 0.f ? 4 : 5; ma = az; }
	else if (ay > ax) { f = d[1] >= 0.f ? 2 : 3; ma = ay; }
	else { f = d[0] >= 0.f ? 0 : 1; ma = ax; }
	const float rma = __frcp_rn(ma);
	const float gx = __fmul_rn(along(kFaceU[f], d[0], d[1], d[2]), rma), gy = __fmul_rn(along(kFaceV[f], d[0], d[1], d[2]), rma);
	const float u = fminf(fmaxf(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f), 0.f), 1.f), v = fminf(fmaxf(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f), 0.f), 1.f);
	const float x = __fsub_rn(__fmul_rn(u, (float)R), 0.5f), y = __fsub_rn(__fmul_rn(v, (float)R), 0.5f);
	const float x0 = floorf(x), y0 = floorf(y);
	const float fx = x - x0, fy = y - y0;
	const int c0 = (int)x0, r0 = (int)y0;
	SkyTaps t;
	t.w[0] = __fmul_rn(1.f - fx, 1.f - fy);
	t.w[1] = __fmul_rn(fx, 1.f - fy);
	t.w[2] = __fmul_rn(1.f - fx, fy);
	t.w[3] = __fmul_rn(fx, fy);
	t.corner = -1;
#pragma unroll
	for (int k = 0; k < 4; k++) {
		t.idx[k] = sky_texel(f, c0 + (k & 1), r0 + (k >> 1), R);
		if (t.idx[k] < 0) t.corner = k;
	}
	return t;
}

// The lookup: the weighted taps, a corner tap taking the mean of the three taps that exist.
__device__ __forceinline__ void sky_sample(const SkyTaps t, const float *__restrict__ cube, float s[3]) {
	float v[4][3];
#pragma unroll
	for (int k = 0; k < 4; k++)
#pragma unroll
		for (int ch = 0; ch < 3; ch++) v[k][ch] = t.idx[k] >= 0 ? __ldg(cube + (size_t)t.idx[k] * 3 + ch) : 0.f;
	if (t.corner >= 0) {
#pragma unroll
		for (int ch = 0; ch < 3; ch++) {
			const float mean = __fmul_rn(__fadd_rn(__fadd_rn(v[0][ch], v[1][ch]), __fadd_rn(v[2][ch], v[3][ch])), kThird);
#pragma unroll
			for (int k = 0; k < 4; k++)
				if (k == t.corner) v[k][ch] = mean;
		}
	}
#pragma unroll
	for (int ch = 0; ch < 3; ch++)
		s[ch] = __fadd_rn(__fadd_rn(__fmul_rn(t.w[0], v[0][ch]), __fmul_rn(t.w[1], v[1][ch])),
		                  __fadd_rn(__fmul_rn(t.w[2], v[2][ch]), __fmul_rn(t.w[3], v[3][ch])));
}

// The pixel's ray (unnormalised: the lookup only uses ratios of its components) and whether it samples the cube.
__device__ __forceinline__ bool sky_pixel(const SkyCam &cam, const int64_t pix, const int W, const int mode, const float accv,
                                          const uint8_t *__restrict__ mask, const float *__restrict__ jx, const float *__restrict__ jy,
                                          float d[3]) {
	const int j = (int)(pix / W), i = (int)(pix - (int64_t)j * W);
	const float px = __fadd_rn((float)i, jx ? __ldg(jx + pix) : 0.5f), py = __fadd_rn((float)j, jy ? __ldg(jy + pix) : 0.5f);
#pragma unroll
	for (int a = 0; a < 3; a++) d[a] = cam.m[a * 3] * px + cam.m[a * 3 + 1] * py + cam.m[a * 3 + 2];
	if (mode == SGR_SKY_MASK_GIVEN) return j < kSkyTopRows || __ldg(mask + pix) != 0;
	return __fsub_rn(1.f, accv) > 1e-3f;
}

// Work item t of M: pixel t of the frame (M = N), or with kBand pixel t of the band's tile rows (M = band_rows * 16 W, band_pixel).
// Every pixel is indexed by its global (i, j): the ray and the rows-0-49 rule depend on the row in the frame.
template <bool kBand>
__global__ void __launch_bounds__(kSkyThreads) sky_composite_fwd_kernel(const int64_t N, const int64_t M, const Band band, const int W, const int R,
                                                                        const int mode, const float fill,
                                                                        const float *__restrict__ rgb, const float *__restrict__ acc,
                                                                        const uint8_t *__restrict__ mask, const float *__restrict__ cube,
                                                                        const float *__restrict__ K, const float *__restrict__ w2c,
                                                                        const float *__restrict__ jx, const float *__restrict__ jy,
                                                                        float *__restrict__ out) {
	const int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (item >= M) return;
	const int64_t pix = kBand ? band_pixel(item, band, (int64_t)kBandTileRows * W) : item;
	if (kBand && pix >= N) return;
	const SkyCam cam = sky_camera(K, w2c);
	const float accv = __ldg(acc + pix);
	float d[3], sky[3] = {fill, fill, fill};
	if (sky_pixel(cam, pix, W, mode, accv, mask, jx, jy, d)) {
		sky_sample(sky_taps(d, R), cube, sky);
#pragma unroll
		for (int ch = 0; ch < 3; ch++) sky[ch] = fminf(fmaxf(sky[ch], 0.f), 1.f);
	}
	const float t = __fsub_rn(1.f, accv);
#pragma unroll
	for (int ch = 0; ch < 3; ch++) out[ch * N + pix] = __fadd_rn(__ldg(rgb + ch * N + pix), __fmul_rn(sky[ch], t));
}

// One tap's three gradient values added into texel `idx` (-1: nothing).  The warp's pixels are consecutive, so equal texels come in
// runs of lanes: a segmented suffix sum leaves each run's total in its first lane, which issues the only atomics of the run.  kMark:
// that lane also sets the byte of the texel's kSkyBlock x kSkyBlock block in `map`, so the map holds exactly the blocks written.
template <bool kMark>
__device__ __forceinline__ void sky_scatter(const int idx, float g0, float g1, float g2, float *__restrict__ gcube, uint8_t *__restrict__ map,
                                            const int R) {
	const unsigned full = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int prev = __shfl_up_sync(full, idx, 1);
	const unsigned heads = __ballot_sync(full, lane == 0 || prev != idx);
	const unsigned later = heads & ~((2u << lane) - 1u);  // heads above this lane (2u << 31 wraps to 0: none)
	const int end = later ? __ffs(later) - 1 : 32;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		const float a = __shfl_down_sync(full, g0, o), b = __shfl_down_sync(full, g1, o), c = __shfl_down_sync(full, g2, o);
		if (lane + o < end) { g0 += a; g1 += b; g2 += c; }
	}
	if (idx >= 0 && ((heads >> lane) & 1u)) {
		atomicAdd(gcube + (size_t)idx * 3, g0);
		atomicAdd(gcube + (size_t)idx * 3 + 1, g1);
		atomicAdd(gcube + (size_t)idx * 3 + 2, g2);
	}
	if (kMark) {  // one store per distinct block of the warp, and none where the block is already marked: few blocks, many writers
		int blk = -1;
		if (idx >= 0 && ((heads >> lane) & 1u)) {
			const int RR = R * R, f = idx / RR, rem = idx - f * RR, r = rem / R, c = rem - r * R, nb = sky_blocks_per_side(R);
			blk = (f * nb + r / kSkyBlock) * nb + c / kSkyBlock;
		}
		const unsigned same = __match_any_sync(full, blk);
		if (blk >= 0 && lane == __ffs(same) - 1 && !map[blk]) map[blk] = 1;
	}
}

// dL/dacc = -sum_c sky_c g_c; dL/dcube: each tap's weight times g (1 - acc) where 0 <= s <= 1, a corner tap's weight shared by thirds
// among the three taps that exist.  dL/drgb is dL/dout itself.  Every lane of a warp reaches sky_scatter (idx = -1 past the image or the band).
// kMark (band form only): also mark the blocks of the texels written in `map` (sky_scatter).
template <bool kBand, bool kMark = false>
__global__ void __launch_bounds__(kSkyThreads) sky_composite_bwd_kernel(const int64_t N, const int64_t M, const Band band, const int W, const int R,
                                                                        const int mode, const float fill,
                                                                        const float *__restrict__ acc, const uint8_t *__restrict__ mask,
                                                                        const float *__restrict__ cube, const float *__restrict__ K,
                                                                        const float *__restrict__ w2c, const float *__restrict__ jx,
                                                                        const float *__restrict__ jy, const float *__restrict__ gout,
                                                                        float *__restrict__ gacc, float *__restrict__ gcube,
                                                                        uint8_t *__restrict__ map) {
	const int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	const int64_t pix = kBand ? band_pixel(item, band, (int64_t)kBandTileRows * W) : item;
	const bool live = item < M && pix < N;
	const SkyCam cam = sky_camera(K, w2c);
	const float accv = live ? __ldg(acc + pix) : 1.f;
	float d[3] = {1.f, 0.f, 0.f};
	const bool masked = live && sky_pixel(cam, pix, W, mode, accv, mask, jx, jy, d);
	SkyTaps t = sky_taps(d, R);
	float ds[3] = {0.f, 0.f, 0.f};
	if (!masked) {
#pragma unroll
		for (int k = 0; k < 4; k++) t.idx[k] = -1;
	}
	if (live) {
		const float g[3] = {__ldg(gout + pix), __ldg(gout + N + pix), __ldg(gout + 2 * N + pix)};
		const float tm = __fsub_rn(1.f, accv);
		float sky[3] = {fill, fill, fill};
		if (masked) {
			sky_sample(t, cube, sky);
#pragma unroll
			for (int ch = 0; ch < 3; ch++) {
				ds[ch] = (sky[ch] >= 0.f && sky[ch] <= 1.f) ? __fmul_rn(g[ch], tm) : 0.f;
				sky[ch] = fminf(fmaxf(sky[ch], 0.f), 1.f);
			}
			if (t.corner >= 0) {
				float wc = 0.f;
#pragma unroll
				for (int k = 0; k < 4; k++)
					if (k == t.corner) wc = t.w[k];
				const float share = __fmul_rn(wc, kThird);
#pragma unroll
				for (int k = 0; k < 4; k++) t.w[k] = k == t.corner ? 0.f : __fadd_rn(t.w[k], share);
			}
		}
		if (gacc) gacc[pix] = -__fadd_rn(__fadd_rn(__fmul_rn(sky[0], g[0]), __fmul_rn(sky[1], g[1])), __fmul_rn(sky[2], g[2]));
	}
	if (!gcube) return;  // uniform over the grid
#pragma unroll
	for (int k = 0; k < 4; k++)
		sky_scatter<kMark>(t.idx[k], __fmul_rn(t.w[k], ds[0]), __fmul_rn(t.w[k], ds[1]), __fmul_rn(t.w[k], ds[2]), gcube, map, R);
}

static int sky_blocks(int64_t N) { return (int)((N + kSkyThreads - 1) / kSkyThreads); }

cudaError_t launch_sky_composite_fwd(int H, int W, int R, int mode, float fill, const float *rgb, const float *acc, const uint8_t *mask,
                                     const float *cube, const float *K, const float *w2c, const float *jx, const float *jy, float *out,
                                     cudaStream_t st) {
	const int64_t N = (int64_t)H * W;
	count_launch();
	sky_composite_fwd_kernel<false><<<sky_blocks(N), kSkyThreads, 0, st>>>(N, N, Band{0, 1, 1}, W, R, mode, fill, rgb, acc, mask, cube, K, w2c, jx,
	                                                                       jy, out);
	return cudaGetLastError();
}

cudaError_t launch_sky_composite_bwd(int H, int W, int R, int mode, float fill, const float *acc, const uint8_t *mask, const float *cube,
                                     const float *K, const float *w2c, const float *jx, const float *jy, const float *gout, float *gacc,
                                     float *gcube, cudaStream_t st) {
	const int64_t N = (int64_t)H * W;
	count_launch();
	sky_composite_bwd_kernel<false><<<sky_blocks(N), kSkyThreads, 0, st>>>(N, N, Band{0, 1, 1}, W, R, mode, fill, acc, mask, cube, K, w2c, jx, jy,
	                                                                       gout, gacc, gcube, nullptr);
	return cudaGetLastError();
}

// The band's forms: one thread per pixel of the band's tile rows (an empty band launches nothing).
cudaError_t launch_sky_composite_fwd(int H, int W, Band band, int R, int mode, float fill, const float *rgb, const float *acc, const uint8_t *mask,
                                     const float *cube, const float *K, const float *w2c, const float *jx, const float *jy, float *out,
                                     cudaStream_t st) {
	const int64_t N = (int64_t)H * W, M = (int64_t)band_rows(band) * kBandTileRows * W;
	if (M == 0) return cudaSuccess;
	count_launch();
	sky_composite_fwd_kernel<true><<<sky_blocks(M), kSkyThreads, 0, st>>>(N, M, band, W, R, mode, fill, rgb, acc, mask, cube, K, w2c, jx, jy, out);
	return cudaGetLastError();
}

// With a block map (sgr_band_sky_composite_backward_marked): the map is cleared first, also for an empty band, then marked.  Without
// clear_map (sgr_band_sky_composite_backward_or_marks) the marks are added to what the map holds.
cudaError_t launch_sky_composite_bwd(int H, int W, Band band, int R, int mode, float fill, const float *acc, const uint8_t *mask, const float *cube,
                                     const float *K, const float *w2c, const float *jx, const float *jy, const float *gout, float *gacc,
                                     float *gcube, cudaStream_t st, uint8_t *block_map, bool clear_map) {
	const int64_t N = (int64_t)H * W, M = (int64_t)band_rows(band) * kBandTileRows * W;
	if (block_map && clear_map) {
		cudaError_t e = cudaMemsetAsync(block_map, 0, (size_t)sky_block_count(R), st);
		if (e != cudaSuccess) return e;
	}
	if (M == 0) return cudaSuccess;
	count_launch();
	if (block_map)
		sky_composite_bwd_kernel<true, true><<<sky_blocks(M), kSkyThreads, 0, st>>>(N, M, band, W, R, mode, fill, acc, mask, cube, K, w2c, jx, jy, gout,
		                                                                            gacc, gcube, block_map);
	else
		sky_composite_bwd_kernel<true><<<sky_blocks(M), kSkyThreads, 0, st>>>(N, M, band, W, R, mode, fill, acc, mask, cube, K, w2c, jx, jy, gout, gacc,
		                                                                      gcube, nullptr);
	return cudaGetLastError();
}

}  // namespace sgr
