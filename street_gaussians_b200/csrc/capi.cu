// capi.cu — the extern "C" surface of libsgr.so (include/sgr.h): argument validation, state carving, launch order.
// Host-side only; every device kernel lives in its own translation unit.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "sgr_common.cuh"

namespace sgr {

static thread_local char g_err[512] = "";
static thread_local int64_t g_near_budget = SGR_NEAR_BUDGET_AUTO;  // sgr_set_near_budget
std::atomic<uint64_t> g_kernel_launches{0};

// cub's temp-storage size queries (two per carve_geom, two per carve_bin) walk cub's dispatch layer every time; every C-ABI
// call carves its state, so the answers are memoised per thread for the last few problem sizes.
template <typename F>
static size_t memo_bytes(int64_t n, F compute) {
	struct Slot { int64_t n; size_t bytes; };
	static thread_local Slot slots[4] = {{-1, 0}, {-1, 0}, {-1, 0}, {-1, 0}};
	static thread_local unsigned next = 0;
	for (const Slot &s : slots)
		if (s.n == n) return s.bytes;
	const size_t b = compute(n);
	slots[next++ & 3u] = Slot{n, b};
	return b;
}

static int fail(int code, const char *fmt, ...) {
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof(g_err), fmt, ap);
	va_end(ap);
	return code;
}

// ---- state carving: bump-pointer layout inside the caller's buffers (all sub-arrays 256-B aligned) ----
template <typename T>
static T *take(char *&p, size_t count) {
	T *r = reinterpret_cast<T *>(p);
	p += align_up(count * sizeof(T));
	return r;
}
GeomView carve_geom(void *base, int P) {
	GeomView g;
	char *p = reinterpret_cast<char *>(base);
	const size_t n = P > 0 ? P : 1;
	g.rec = take<GaussRec>(p, n);
	g.tiles_touched = take<uint32_t>(p, n);
	g.depth_key = take<uint32_t>(p, n);
	g.iota = take<uint32_t>(p, n);
	g.depth_sorted = take<uint32_t>(p, n);
	g.perm = take<uint32_t>(p, n);
	g.offsets = take<uint32_t>(p, n);
	g.big_list = take<uint32_t>(p, n);
	g.big_count = take<uint32_t>(p, 64);
	g.jac = take<float4>(p, 3 * n);
	g.ckey = take<uint32_t>(p, n);
	g.cval = take<uint32_t>(p, n);
	g.reached = g.cval;
	g.temp_bytes = memo_bytes((int64_t)P, [](int64_t n) { return geom_temp_bytes((int)n); });
	g.temp = take<char>(p, g.temp_bytes);
	g.total_bytes = (size_t)(p - reinterpret_cast<char *>(base));
	return g;
}
// blend_state: the per-pixel T of the saturation split (forward img states; a layer's img has none)
ImgView carve_img(void *base, int W, int H, bool blend_state) {
	ImgView v;
	char *p = reinterpret_cast<char *>(base);
	const size_t gx = (W + SGR_TILE - 1) / SGR_TILE, gy = (H + SGR_TILE - 1) / SGR_TILE;
	v.ranges = take<uint2>(p, gx * gy + 1);
	v.tile_max_contrib = take<uint32_t>(p, gx * gy + 1);
	v.n_contrib = take<uint32_t>(p, (size_t)W * H + 1);
	v.blend_T = blend_state ? take<float>(p, (size_t)W * H) : nullptr;
	v.far_ranges = blend_state ? take<uint2>(p, gx * gy + 1) : nullptr;
	v.split = blend_state ? take<uint2>(p, gx * gy + 1) : nullptr;
	v.total_bytes = (size_t)(p - reinterpret_cast<char *>(base));
	return v;
}
BinView carve_bin(void *base, int64_t R) {
	BinView b;
	char *p = reinterpret_cast<char *>(base);
	const size_t n = R > 0 ? (size_t)R : 1;
	b.keys_in = take<uint32_t>(p, n);
	b.keys_out = take<uint32_t>(p, n);
	b.vals_in = take<uint32_t>(p, n);
	b.vals_out = take<uint32_t>(p, n);
	b.sort_temp_bytes = std::max(memo_bytes(R, [](int64_t n) { return sort_temp_bytes(n); }), n * sizeof(uint32_t));
	b.sort_temp = take<char>(p, b.sort_temp_bytes);
	b.bucket_bytes = bucket_scratch_bytes(R);
	b.bucket = take<char>(p, b.bucket_bytes);
	b.total_bytes = (size_t)(p - reinterpret_cast<char *>(base));
	return b;
}

static int make_frame(const SgrFrame *fr, FrameDev &f) {
	if (!fr) return fail(SGR_EINVAL, "frame is NULL");
	if (fr->P < 0 || fr->width <= 0 || fr->height <= 0) return fail(SGR_EINVAL, "bad sizes P=%d W=%d H=%d", fr->P, fr->width, fr->height);
	if (fr->S < 0 || fr->M < 0 || fr->D < 0 || fr->D > 3) return fail(SGR_EINVAL, "bad S=%d M=%d D=%d (SH degree must be 0..3)", fr->S, fr->M, fr->D);
	f.P = fr->P; f.D = fr->D; f.M = fr->M; f.S = fr->S; f.W = fr->width; f.H = fr->height;
	f.gx = (f.W + SGR_TILE - 1) / SGR_TILE; f.gy = (f.H + SGR_TILE - 1) / SGR_TILE;
	f.tanx = fr->tan_fovx; f.tany = fr->tan_fovy; f.mod = fr->scale_modifier;
	// focal lengths exactly as the reference derives them (rasterizer_impl.cu:225-226)
	f.fy = f.H / (2.0f * f.tany);
	f.fx = f.W / (2.0f * f.tanx);
	if (fr->row_step == 0 && fr->row_begin == 0 && fr->row_end == 0) f.band = Band{0, f.gy, 1};
	else {
		if (fr->row_step <= 0 || fr->row_begin < 0 || fr->row_end > f.gy || fr->row_begin > fr->row_end)
			return fail(SGR_EINVAL, "bad tile-row band [%d,%d) step %d for %d tile rows", fr->row_begin, fr->row_end, fr->row_step, f.gy);
		f.band = Band{fr->row_begin, fr->row_end, fr->row_step};
	}
	f.bg = fr->bg; f.view = fr->viewmatrix; f.proj = fr->projmatrix; f.campos = fr->campos;
	return SGR_OK;
}

static int check(cudaError_t e, const char *what, bool debug, cudaStream_t st) {
	if (e == cudaSuccess && debug) e = cudaStreamSynchronize(st);
	if (e == cudaSuccess && debug) e = cudaGetLastError();
	if (e != cudaSuccess) return fail(SGR_ECUDA, "%s: %s", what, cudaGetErrorString(e));
	return SGR_OK;
}
// The one host<->device round trip of the exact mode: 4 bytes into a pinned, thread-local staging word, then a
// BLOCKING wait on an event (the thread sleeps instead of spinning in cudaStreamSynchronize).  With one process per GPU
// on a host with fewer cores than 2 x GPUs (e.g. a cgroup quota of 16 cores for 8 GPUs) eight spinning main threads plus
// eight autograd threads exhaust the quota and every rank gets throttled, which shows up as a step time well above the sum
// of its stages.
static cudaError_t read_back_u32(uint32_t *dst, const uint32_t *src_dev, cudaStream_t st) {
	static thread_local uint32_t *pinned = nullptr;
	static thread_local cudaEvent_t ev = nullptr;
	static thread_local int ev_dev = -1;
	// policy: SGR_SYNC_MODE=spin|block wins; otherwise spin when this is the only rank on the node (slightly faster
	// at N=1) and sleep when torchrun-style launchers announce several local ranks
	static const bool spin = [] {
		const char *m = getenv("SGR_SYNC_MODE");
		if (m) return strcmp(m, "spin") == 0;
		const char *w = getenv("LOCAL_WORLD_SIZE");
		if (!w) w = getenv("WORLD_SIZE");
		return !(w && atoi(w) > 1);
	}();
	cudaError_t e;
	if (!pinned && (e = cudaHostAlloc(reinterpret_cast<void **>(&pinned), 64, cudaHostAllocDefault)) != cudaSuccess) return e;
	int dev = 0;
	if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
	if (!spin && (ev == nullptr || ev_dev != dev)) {
		if (ev) cudaEventDestroy(ev);
		if ((e = cudaEventCreateWithFlags(&ev, cudaEventBlockingSync | cudaEventDisableTiming)) != cudaSuccess) return e;
		ev_dev = dev;
	}
	if ((e = cudaMemcpyAsync(pinned, src_dev, sizeof(uint32_t), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
	if (spin) {
		if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
	} else {
		if ((e = cudaEventRecord(ev, st)) != cudaSuccess) return e;
		if ((e = cudaEventSynchronize(ev)) != cudaSuccess) return e;
	}
	*dst = *pinned;
	return cudaSuccess;
}

#define SGR_TRY(expr, what)                                             \
	do {                                                                \
		int rc_ = check((expr), what, debug, st);                       \
		if (rc_ != SGR_OK) return rc_;                                  \
	} while (0)

// The kernels read rotation rows and SH rows with 16-B vector loads (and store their gradients so); a pointer into the middle of
// a larger buffer can break that alignment, which faults on the device.  NULL passes.
static int check_aligned16(const char *what, const void *p) {
	if ((reinterpret_cast<uintptr_t>(p) & 15u) != 0) return fail(SGR_EINVAL, "%s is not 16-byte aligned (%p)", what, p);
	return SGR_OK;
}

// colour and covariance inputs of a projection: exactly one source of each, SH coefficients only with M > 0 and at least the
// (D + 1)^2 the active degree evaluates, and the rows read as float4 aligned
static int check_gaussian_inputs(const FrameDev &f, const float *shs, const float *colors_precomp, const float *scales,
                                 const float *rotations, const float *cov3D_precomp) {
	if ((shs == nullptr) == (colors_precomp == nullptr)) return fail(SGR_EINVAL, "provide exactly one of shs / colors_precomp");
	const bool sr = scales != nullptr && rotations != nullptr;
	if (sr == (cov3D_precomp != nullptr) || ((scales != nullptr) != (rotations != nullptr)))
		return fail(SGR_EINVAL, "provide exactly one of (scales, rotations) / cov3D_precomp");
	if (shs && f.M <= 0) return fail(SGR_EINVAL, "shs given but M == 0");
	if (shs && f.M < (f.D + 1) * (f.D + 1))
		return fail(SGR_EINVAL, "SH degree %d needs %d coefficients per Gaussian, shs has M = %d", f.D, (f.D + 1) * (f.D + 1), f.M);
	int rc;
	if ((rc = check_aligned16("shs", shs)) != SGR_OK) return rc;
	return check_aligned16("rotations", rotations);
}

// pointers of the per-Gaussian chain rule; `inputs_ok` is the caller's check of its own input pointers
static int check_geom_grads(const char *fn, const FrameDev &f, bool inputs_ok, const float *shs, const float *scales, const float *rotations,
                            const float *cov3D_precomp, const float *dL_dmeans3D, const float *dL_dmeans2D, const float *dL_dsh,
                            const float *dL_dopacity, const float *dL_dscales, const float *dL_drotations) {
	if (!inputs_ok || !dL_dmeans3D || !dL_dmeans2D || !dL_dopacity) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (shs && !dL_dsh) return fail(SGR_EINVAL, "shs given but dL_dsh is NULL");
	if (!cov3D_precomp && (!scales || !rotations || !dL_dscales || !dL_drotations))
		return fail(SGR_EINVAL, "scale/rotation path needs scales, rotations, dL_dscales, dL_drotations");
	if (shs && f.M < (f.D + 1) * (f.D + 1))
		return fail(SGR_EINVAL, "SH degree %d needs %d coefficients per Gaussian, shs has M = %d", f.D, (f.D + 1) * (f.D + 1), f.M);
	int rc;
	if ((rc = check_aligned16("shs", shs)) != SGR_OK || (rc = check_aligned16("rotations", rotations)) != SGR_OK) return rc;
	if (shs && (rc = check_aligned16("dL_dsh", dL_dsh)) != SGR_OK) return rc;
	if (!cov3D_precomp && (rc = check_aligned16("dL_drotations", dL_drotations)) != SGR_OK) return rc;
	return SGR_OK;
}

}  // namespace sgr

using namespace sgr;

extern "C" {

int sgr_abi_version(void) { return SGR_ABI_VERSION; }
int64_t sgr_set_near_budget(int64_t budget) {
	const int64_t prev = g_near_budget;
	g_near_budget = budget < 0 ? SGR_NEAR_BUDGET_AUTO : budget;
	return prev;
}
uint64_t sgr_launch_count(void) { return g_kernel_launches.load(std::memory_order_relaxed); }
const char *sgr_last_error(void) { return g_err; }

int sgr_state_sizes(const SgrFrame *frame, size_t *geom_bytes, size_t *img_bytes) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	if (geom_bytes) *geom_bytes = carve_geom(nullptr, f.P).total_bytes;
	if (img_bytes) *img_bytes = carve_img(nullptr, f.W, f.H).total_bytes;
	return SGR_OK;
}

size_t sgr_binning_bytes(int64_t R) { return carve_bin(nullptr, R).total_bytes; }

int sgr_state_layout(const SgrFrame *frame, int64_t num_instances, int32_t bounded, SgrStateLayout *out) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	if (!out || num_instances < 0) return fail(SGR_EINVAL, "out is NULL or num_instances %lld < 0", (long long)num_instances);
	// carved from a null base, every section pointer is its byte offset
	const GeomView g = carve_geom(nullptr, f.P);
	const ImgView v = carve_img(nullptr, f.W, f.H);
	const BinView b = carve_bin(nullptr, num_instances);
	const auto at = [](const void *p) { return (size_t)reinterpret_cast<uintptr_t>(p); };
	SgrStateLayout &l = *out;
	l.rec = at(g.rec); l.tiles_touched = at(g.tiles_touched); l.depth_key = at(g.depth_key); l.iota = at(g.iota);
	l.depth_sorted = at(g.depth_sorted); l.perm = at(g.perm); l.offsets = at(g.offsets); l.big_list = at(g.big_list);
	l.status = at(g.big_count); l.jac = at(g.jac); l.ckey = at(g.ckey); l.cval = at(g.cval); l.geom_bytes = g.total_bytes;
	l.ranges = at(v.ranges); l.tile_max_contrib = at(v.tile_max_contrib); l.n_contrib = at(v.n_contrib); l.blend_T = at(v.blend_T);
	l.far_ranges = at(v.far_ranges); l.split = at(v.split); l.img_bytes = v.total_bytes;
	l.keys_in = at(b.keys_in); l.keys_out = at(b.keys_out); l.vals_in = at(b.vals_in); l.vals_out = at(b.vals_out);
	l.sort_temp = at(b.sort_temp); l.bucket = at(b.bucket); l.binning_bytes = b.total_bytes;
	l.key_bytes = tile_key_bytes(f.gx * f.gy, bounded != 0);
	return SGR_OK;
}

// shared body of sgr_forward (exact: reads the instance count back, asks the caller's allocator) and sgr_forward_bounded
// (no host synchronisation: caller-sized binning state, count stays on the device)
static int forward_impl(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                        const float *semantics, const float *opacities, const float *scales, const float *rotations,
                        const float *cov3D_precomp, float *out_color, float *out_depth, float *out_alpha, float *out_semantic,
                        int32_t *radii, void *geom_state, size_t geom_bytes, void *img_state, size_t img_bytes, sgr_alloc_fn alloc,
                        void *alloc_user, void **binning_state, int64_t *num_instances, void *bounded_state, size_t bounded_bytes,
                        int64_t capacity, void *stream, bool from_records = false) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	const bool bounded = capacity >= 0;
	if (binning_state) *binning_state = nullptr;
	if (num_instances) *num_instances = 0;
	if (!out_color || !out_depth || !out_alpha || (f.S > 0 && !out_semantic)) return fail(SGR_EINVAL, "output image pointer is NULL");
	if (!f.bg || !f.view || !f.proj || !f.campos) return fail(SGR_EINVAL, "camera pointer (bg/viewmatrix/projmatrix/campos) is NULL");
	if (f.P > 0 && from_records) {
		if (!radii) return fail(SGR_EINVAL, "radii is NULL");
		if (f.S > 0 && !semantics) return fail(SGR_EINVAL, "S > 0 but semantics is NULL");
	} else if (f.P > 0) {
		if (!means3D || !opacities || !radii) return fail(SGR_EINVAL, "means3D / opacities / radii is NULL");
		if ((rc = check_gaussian_inputs(f, shs, colors_precomp, scales, rotations, cov3D_precomp)) != SGR_OK) return rc;
		if (f.S > 0 && !semantics) return fail(SGR_EINVAL, "S > 0 but semantics is NULL");
	}
	const GeomView g = carve_geom(geom_state, f.P);
	const ImgView img = carve_img(img_state, f.W, f.H);
	if (!geom_state || geom_bytes < g.total_bytes) return fail(SGR_ENOMEM, "geom_state too small: %zu < %zu", geom_bytes, g.total_bytes);
	if (!img_state || img_bytes < img.total_bytes) return fail(SGR_ENOMEM, "img_state too small: %zu < %zu", img_bytes, img.total_bytes);
	if (bounded) {
		if (capacity > 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "capacity %lld exceeds 2^31-1", (long long)capacity);
		const size_t need = carve_bin(nullptr, capacity).total_bytes;
		if (capacity > 0 && (!bounded_state || bounded_bytes < need))
			return fail(SGR_ENOMEM, "binning_state too small for capacity %lld: %zu < %zu", (long long)capacity, bounded_bytes, need);
	}

	int64_t R = 0;
	int n_order = f.P;
	BinView b = carve_bin(nullptr, 0);
	if (f.P > 0) {
		SGR_TRY(cudaMemsetAsync(g.big_count, 0, 64 * sizeof(uint32_t), st), "status reset");
		if (from_records) SGR_TRY(launch_count_tiles(f, g, radii, st), "count_tiles");
		else
			SGR_TRY(launch_preprocess_fwd(f, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, radii, g, st),
			        "preprocess_fwd");
		SGR_TRY(launch_depth_order(f, g, st), "depth_order");
		if (!bounded) {
			uint32_t r32 = 0;
			cudaError_t e = read_back_u32(&r32, g.offsets + (n_order - 1), st);
			if (e != cudaSuccess) return fail(SGR_ECUDA, "instance count read-back: %s", cudaGetErrorString(e));
			R = (int64_t)r32;
			if (R > 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "instance count %lld exceeds 2^31-1", (long long)R);
		}
	}
	if (bounded) {
		R = capacity;
		if (capacity > 0) b = carve_bin(bounded_state, capacity);
	} else if (R > 0) {
		if (!alloc) return fail(SGR_EINVAL, "alloc callback is NULL");
		const size_t need = carve_bin(nullptr, R).total_bytes;
		void *bin = alloc(alloc_user, need);
		if (!bin) return fail(SGR_ENOMEM, "binning allocator returned NULL for %zu bytes", need);
		b = carve_bin(bin, R);
		if (binning_state) *binning_state = bin;
	}
	if (num_instances) *num_instances = R;
	const int64_t budget = g_near_budget;
	if (split_applies(f, R, budget, from_records)) {
		const int64_t cap = bounded ? capacity : -1;
		SGR_TRY(launch_near_binning(f, g, radii, b, img, R, st, cap, n_order, budget), "near binning");
		SGR_TRY(launch_blend_fwd(f, g, split_near_lists(b), img, nullptr, out_color, out_depth, out_alpha, nullptr, st, kBlendNear),
		        "near blend_fwd");
		SGR_TRY(launch_far_binning(f, g, radii, b, img, R, st, cap, n_order), "far binning");
		SGR_TRY(launch_blend_fwd(f, g, b, img, nullptr, out_color, out_depth, out_alpha, nullptr, st, kBlendResume), "resume blend_fwd");
		return SGR_OK;
	}
	SGR_TRY(launch_binning(f, g, radii, b, img, R, st, bounded ? capacity : -1, n_order), "binning");
	SGR_TRY(launch_blend_fwd(f, g, b, img, semantics, out_color, out_depth, out_alpha, out_semantic, st), "blend_fwd");
	return SGR_OK;
}

int sgr_forward(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                const float *semantics, const float *opacities, const float *scales, const float *rotations,
                const float *cov3D_precomp, float *out_color, float *out_depth, float *out_alpha, float *out_semantic,
                int32_t *radii, void *geom_state, size_t geom_bytes, void *img_state, size_t img_bytes, sgr_alloc_fn alloc,
                void *alloc_user, void **binning_state, int64_t *num_instances, void *stream) {
	return forward_impl(frame, means3D, shs, colors_precomp, semantics, opacities, scales, rotations, cov3D_precomp, out_color, out_depth,
	                    out_alpha, out_semantic, radii, geom_state, geom_bytes, img_state, img_bytes, alloc, alloc_user, binning_state,
	                    num_instances, nullptr, 0, -1, stream);
}

int sgr_forward_bounded(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                        const float *semantics, const float *opacities, const float *scales, const float *rotations,
                        const float *cov3D_precomp, float *out_color, float *out_depth, float *out_alpha, float *out_semantic,
                        int32_t *radii, void *geom_state, size_t geom_bytes, void *img_state, size_t img_bytes,
                        void *binning_state, size_t binning_bytes, int64_t capacity, void *stream) {
	if (capacity < 0) return fail(SGR_EINVAL, "capacity must be >= 0");
	return forward_impl(frame, means3D, shs, colors_precomp, semantics, opacities, scales, rotations, cov3D_precomp, out_color, out_depth,
	                    out_alpha, out_semantic, radii, geom_state, geom_bytes, img_state, img_bytes, nullptr, nullptr, nullptr, nullptr,
	                    binning_state, binning_bytes, capacity, stream);
}

size_t sgr_record_bytes(void) { return sizeof(GaussRec); }

int sgr_project(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp, const float *opacities,
                const float *scales, const float *rotations, const float *cov3D_precomp, int32_t *radii, void *records, void *stream) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	if (f.P == 0) return SGR_OK;
	if (!f.view || !f.proj || !f.campos) return fail(SGR_EINVAL, "camera pointer (viewmatrix/projmatrix/campos) is NULL");
	if (!means3D || !opacities || !radii || !records) return fail(SGR_EINVAL, "means3D / opacities / radii / records is NULL");
	if ((rc = check_gaussian_inputs(f, shs, colors_precomp, scales, rotations, cov3D_precomp)) != SGR_OK) return rc;
	// `records` is the head of a geom state for frame.P: the records go there, the colour Jacobian that sgr_backward_geom reads after them
	const GeomView g = carve_geom(records, f.P);
	SGR_TRY(launch_project(f, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, radii, g.rec, g.jac, st),
	        "project");
	return SGR_OK;
}

int sgr_forward_records(const SgrFrame *frame, const int32_t *radii, const float *semantics, float *out_color, float *out_depth,
                        float *out_alpha, float *out_semantic, void *geom_state, size_t geom_bytes, void *img_state, size_t img_bytes,
                        sgr_alloc_fn alloc, void *alloc_user, void **binning_state_out, int64_t *num_instances, void *binning_state,
                        size_t binning_bytes, int64_t capacity, void *stream) {
	return forward_impl(frame, nullptr, nullptr, nullptr, semantics, nullptr, nullptr, nullptr, nullptr, out_color, out_depth, out_alpha,
	                    out_semantic, const_cast<int32_t *>(radii), geom_state, geom_bytes, img_state, img_bytes, alloc, alloc_user,
	                    binning_state_out, num_instances, capacity >= 0 ? binning_state : nullptr, capacity >= 0 ? binning_bytes : 0,
	                    capacity >= 0 ? capacity : -1, stream, true);
}

static int make_peers(const SgrPeers *peers, const FrameDev &f, bool need_grad, PeerTable &pt) {
	if (!peers) return fail(SGR_EINVAL, "peers is NULL");
	if (peers->world < 1 || peers->world > SGR_MAX_PEERS || peers->rank < 0 || peers->rank >= peers->world)
		return fail(SGR_EINVAL, "bad peer table: world=%d rank=%d (at most %d ranks)", peers->world, peers->rank, SGR_MAX_PEERS);
	if (peers->chunk < f.P) return fail(SGR_EINVAL, "chunk %lld smaller than the local Gaussian count %d", (long long)peers->chunk, f.P);
	if ((long long)peers->chunk * peers->world > 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "world*chunk exceeds 2^31-1");
	pt.world = peers->world; pt.rank = peers->rank; pt.chunk = peers->chunk;
	for (int p = 0; p < peers->world; p++) {
		if (!peers->records[p] || !peers->radii[p] || (need_grad && !peers->grad2d[p])) return fail(SGR_EINVAL, "peer table entry %d is NULL", p);
		pt.rec[p] = reinterpret_cast<GaussRec *>(peers->records[p]);
		pt.radii[p] = peers->radii[p];
		pt.grad2d[p] = peers->grad2d[p];
		pt.flags[p] = peers->flags[p];
	}
	return SGR_OK;
}

int sgr_scatter_records(const SgrFrame *frame, const SgrPeers *peers, const void *records_local, const int32_t *radii_local, void *stream) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	PeerTable pt = {};
	if ((rc = make_peers(peers, f, false, pt)) != SGR_OK) return rc;
	if (f.P > 0 && (!records_local || !radii_local)) return fail(SGR_EINVAL, "records_local / radii_local is NULL");
	SGR_TRY(launch_scatter_records(f, pt, reinterpret_cast<const GaussRec *>(records_local), radii_local, st), "scatter_records");
	return SGR_OK;
}

int sgr_gather_grad2d(const SgrFrame *frame, const SgrPeers *peers, const void *records_local, const int32_t *radii_local,
                      float *grad2d_local, void *stream) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	PeerTable pt = {};
	if ((rc = make_peers(peers, f, true, pt)) != SGR_OK) return rc;
	if (f.P == 0) return SGR_OK;
	if (!records_local || !radii_local || !grad2d_local) return fail(SGR_EINVAL, "NULL pointer passed to sgr_gather_grad2d");
	SGR_TRY(launch_gather_grad2d(f, pt, reinterpret_cast<const GaussRec *>(records_local), radii_local, grad2d_local, st), "gather_grad2d");
	return SGR_OK;
}

int sgr_peer_barrier(const SgrPeers *peers, uint32_t epoch, void *stream) {
	if (!peers) return fail(SGR_EINVAL, "peers is NULL");
	FrameDev f = {};
	PeerTable pt = {};
	int rc = make_peers(peers, f, false, pt);
	if (rc) return rc;
	for (int p = 0; p < pt.world; p++)
		if (!pt.flags[p]) return fail(SGR_EINVAL, "peer table entry %d has no barrier pad", p);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_peer_barrier(pt, epoch, nullptr, st), "peer_barrier");
	return SGR_OK;
}

// layer state: the img-state layout (ranges, tile_max_contrib, n_contrib) of the layer, then its tile lists u32[num_instances]
struct LayerView {
	ImgView img;
	uint32_t *list;
	size_t total_bytes;
};
static LayerView carve_layer(void *base, int W, int H, int64_t R) {
	LayerView v;
	v.img = carve_img(base, W, H, false);
	char *p = reinterpret_cast<char *>(base) + v.img.total_bytes;
	v.list = take<uint32_t>(p, R > 0 ? (size_t)R : 1);
	v.total_bytes = (size_t)(p - reinterpret_cast<char *>(base));
	return v;
}
// a layer of the fused Gaussian-sharded step: carve_layer's lists for `capacity` instances, then the backward's scratch rows of the P local
// Gaussians (the summed main + layer rows [P, 12] the chain rule reads, and [P, 3] for the dL/dmeans2D it writes from them)
struct ShardedLayerView {
	LayerView lv;
	float *rows, *means2D;
	size_t total_bytes;
};
static ShardedLayerView carve_sharded_layer(void *base, int W, int H, int64_t capacity, int P) {
	ShardedLayerView v;
	v.lv = carve_layer(base, W, H, capacity);
	char *p = reinterpret_cast<char *>(base) + v.lv.total_bytes;
	const size_t n = P > 0 ? (size_t)P : 1;
	v.rows = take<float>(p, 12 * n);
	v.means2D = take<float>(p, 3 * n);
	v.total_bytes = (size_t)(p - reinterpret_cast<char *>(base));
	return v;
}

// the layer table of sgr_sharded_forward_layers / sgr_sharded_backward_layers, checked before the main call's arguments
static int check_sharded_layers(const char *fn, const SgrFrame *frame, const SgrShardedLayer *layers, int32_t n, int64_t capacity, bool backward) {
	if (!frame) return fail(SGR_EINVAL, "frame is NULL");
	if (!layers) return fail(SGR_EINVAL, "%s: layer table is NULL", fn);
	if (n < 1 || n > SGR_MAX_SHARDED_LAYERS) return fail(SGR_EINVAL, "%s: %d layers (1 to %d)", fn, n, SGR_MAX_SHARDED_LAYERS);
	if (frame->S != 0) return fail(SGR_EINVAL, "%s: layers take no feature channels (S = %d)", fn, frame->S);
	if (frame->width <= 0 || frame->height <= 0 || frame->P < 0) return fail(SGR_EINVAL, "bad sizes P=%d W=%d H=%d", frame->P, frame->width, frame->height);
	if (capacity < 0 || capacity > 0x7fffffffLL) return fail(SGR_EINVAL, "capacity must be in [0, 2^31)");
	const size_t need = carve_sharded_layer(nullptr, frame->width, frame->height, capacity, frame->P).total_bytes;
	for (int k = 0; k < n; k++) {
		const SgrShardedLayer &l = layers[k];
		if (l.begin < 0 || l.begin > l.end || l.end > frame->P)
			return fail(SGR_EINVAL, "%s: bad layer %d range [%d, %d) for %d local Gaussians", fn, k, l.begin, l.end, frame->P);
		if (!l.bg) return fail(SGR_EINVAL, "%s: layer %d bg is NULL", fn, k);
		if (!l.state) return fail(SGR_EINVAL, "%s: layer %d state is NULL", fn, k);
		if (l.state_bytes < need) return fail(SGR_ENOMEM, "%s: layer %d state too small: %zu < %zu", fn, k, l.state_bytes, need);
		if (!l.alpha || (!backward && (!l.color || !l.depth))) return fail(SGR_EINVAL, "%s: layer %d image pointer is NULL", fn, k);
		const int given = (l.dL_dcolor != nullptr) + (l.dL_ddepth != nullptr) + (l.dL_dalpha != nullptr);
		if (backward && given != 0 && given != 3)
			return fail(SGR_EINVAL, "%s: layer %d has %d of its 3 upstream gradients (all or none)", fn, k, given);
	}
	return SGR_OK;
}
// both directions use every section: the forward writes the masks and clears its own layer rows, the backward writes and reads the rows
static int layer_peers(const SgrLayerPeers *peers, const PeerTable &pt, int nl) {
	if (!peers) return fail(SGR_EINVAL, "layer_peers is NULL");
	if (peers->layers < nl) return fail(SGR_EINVAL, "the layer sections hold %d layers, the call has %d", peers->layers, nl);
	for (int p = 0; p < pt.world; p++)
		if (!peers->layer_mask[p] || !peers->layer_grad2d[p]) return fail(SGR_EINVAL, "peer table entry %d has no layer section", p);
	return SGR_OK;
}
// layer k's rows of rank p: its part of p's layer_grad2d section
static float *layer_section(const SgrLayerPeers *peers, int p, int k, const FrameDev &ft) {
	return peers->layer_grad2d[p] + (size_t)k * (size_t)ft.P * 12;
}

// FrameDev of the gathered problem (all world*chunk slots) seen through this rank's band
static int make_total_frame(const SgrFrame *frame, const SgrPeers *peers, FrameDev &fl, FrameDev &ft, PeerTable &pt, bool need_grad,
                            SemPeers *sp = nullptr) {
	int rc = make_frame(frame, fl);
	if (rc) return rc;
	if ((rc = make_peers(peers, fl, need_grad, pt)) != SGR_OK) return rc;
	if (!sp && fl.S != 0)
		return fail(SGR_EUNSUPPORTED, "sgr_sharded_forward / _backward take S == 0 only (feature channels: sgr_sharded_*_features)");
	if (sp) {
		if (fl.S < 1 || fl.S > SGR_MAX_SEMANTIC_BWD)
			return fail(SGR_EUNSUPPORTED, "the fused step carries 1 to %d feature channels, got S = %d", SGR_MAX_SEMANTIC_BWD, fl.S);
		for (int p = 0; p < pt.world; p++) {
			if (!peers->sem[p] || (need_grad && !peers->gsem[p])) return fail(SGR_EINVAL, "peer table entry %d has no feature section", p);
			sp->sem[p] = peers->sem[p];
			sp->gsem[p] = peers->gsem[p];
		}
	}
	for (int p = 0; p < pt.world; p++)
		if (pt.world > 1 && !pt.flags[p]) return fail(SGR_EINVAL, "peer table entry %d has no barrier pad", p);
	// a rank past the last tile row (more ranks than tile rows) owns no row: its cyclic band is empty (cyclic_band passes [0, 0)), it
	// receives no record and renders nothing, but it still projects, scatters and gathers its own Gaussians and takes every barrier
	const bool no_rows = pt.rank >= fl.gy && band_rows(fl.band) == 0;
	if (pt.world > 1 && !no_rows && !(fl.band.step == pt.world && fl.band.begin == pt.rank))
		return fail(SGR_EINVAL, "the peer exchange needs the cyclic band of this rank: begin == rank, step == world (got [%d,%d) step %d)",
		            fl.band.begin, fl.band.end, fl.band.step);
	ft = fl;
	ft.P = (int)(pt.chunk * pt.world);
	return SGR_OK;
}

// sp != nullptr: the feature form (sgr_sharded_forward_features)
static int sharded_forward(const SgrFrame *frame, const SgrPeers *peers, const float *means3D, const float *shs, const float *colors_precomp,
                           const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp, float *out_color,
                           float *out_depth, float *out_alpha, int32_t *radii_local, void *records_local, size_t geom_bytes, void *img_state,
                           size_t img_bytes, void *binning_state, size_t binning_bytes, int64_t capacity, int64_t gaussian_capacity,
                           uint32_t barrier_epoch, int32_t pre_barrier, SemPeers *sp, const float *semantics, float *out_semantic,
                           void *stream, const SgrLayerPeers *lpeers = nullptr, const SgrShardedLayer *layers = nullptr, int nl = 0) {
	FrameDev fl, ft;
	PeerTable pt = {};
	int rc = make_total_frame(frame, peers, fl, ft, pt, false, sp);
	if (rc) return rc;
	if (nl && (rc = layer_peers(lpeers, pt, nl)) != SGR_OK) return rc;
	if (sp && (!out_semantic || (fl.P > 0 && !semantics))) return fail(SGR_EINVAL, "semantics / out_semantic is NULL");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	if (capacity < 0 || capacity > 0x7fffffffLL) return fail(SGR_EINVAL, "capacity must be in [0, 2^31)");
	if (!out_color || !out_depth || !out_alpha) return fail(SGR_EINVAL, "output image pointer is NULL");
	if (!fl.bg || !fl.view || !fl.proj || !fl.campos) return fail(SGR_EINVAL, "camera pointer (bg/viewmatrix/projmatrix/campos) is NULL");
	if (pt.chunk > 0 && (!radii_local || !records_local)) return fail(SGR_EINVAL, "radii_local / records_local is NULL");
	if (fl.P > 0) {
		if (!means3D || !opacities) return fail(SGR_EINVAL, "means3D / opacities is NULL");
		if ((rc = check_gaussian_inputs(fl, shs, colors_precomp, scales, rotations, cov3D_precomp)) != SGR_OK) return rc;
	}
	void *geom_state = pt.rec[pt.rank];  // this rank's gathered records ARE the head of its geom state
	GeomView g = carve_geom(geom_state, ft.P);
	g.reached = nullptr;  // (cval holds the compacted depth-sort input, which the layer rows' reset reads after the binning)
	const ImgView img = carve_img(img_state, ft.W, ft.H);
	if (geom_bytes < g.total_bytes) return fail(SGR_ENOMEM, "geom_state too small: %zu < %zu", geom_bytes, g.total_bytes);
	if (!img_state || img_bytes < img.total_bytes) return fail(SGR_ENOMEM, "img_state too small: %zu < %zu", img_bytes, img.total_bytes);
	const size_t need = carve_bin(nullptr, capacity).total_bytes;
	if (capacity > 0 && (!binning_state || binning_bytes < need))
		return fail(SGR_ENOMEM, "binning_state too small for capacity %lld: %zu < %zu", (long long)capacity, binning_bytes, need);
	// a forward that follows a forward (no backward in between) must not overwrite records a peer may still be blending
	if (pre_barrier) SGR_TRY(launch_peer_barrier(pt, barrier_epoch ? barrier_epoch - 1u : 0u, nullptr, st), "pre-barrier");
	// (g.depth_key of this rank = the destination masks of its own Gaussians, kept for the backward; g.iota of rank d = the run-length
	// table the owners fill — same offset inside every rank's geom state)
	SGR_TRY(launch_project_scatter(fl, pt, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, radii_local,
	                               reinterpret_cast<GaussRec *>(records_local), g.jac, g.depth_key,
	                               (size_t)(reinterpret_cast<char *>(g.iota) - reinterpret_cast<char *>(geom_state)), st),
	        "project+scatter");
	if (sp) SGR_TRY(launch_scatter_semantics(pt, *sp, fl.P, fl.S, g.depth_key, semantics, st), "scatter semantics");
	LayerPeers lp = {};
	if (nl) {  // layer membership travels with the records, before the barrier
		for (int p = 0; p < pt.world; p++) lp.mask[p] = lpeers->layer_mask[p];
		lp.n = nl;
		for (int k = 0; k < nl; k++) { lp.begin[k] = layers[k].begin; lp.end[k] = layers[k].end; }
		SGR_TRY(launch_scatter_layer_mask(pt, lp, fl.P, g.depth_key, st), "scatter layer mask");
	}
	if (ft.P == 0) return SGR_OK;
	SGR_TRY(cudaMemsetAsync(g.big_count, 0, 64 * sizeof(uint32_t), st), "status reset");
	SGR_TRY(launch_peer_barrier(pt, barrier_epoch, g.big_count, st), "barrier");
	int n_order = ft.P;
	SGR_TRY(launch_count_and_order_runs(ft, g, pt.radii[pt.rank], pt.world, pt.chunk, st, gaussian_capacity, const_cast<float *>(pt.grad2d[pt.rank]), &n_order),
	        "count + depth_order");
	const BinView b = capacity > 0 ? carve_bin(binning_state, capacity) : carve_bin(nullptr, 0);
	SGR_TRY(launch_binning(ft, g, pt.radii[pt.rank], b, img, capacity, st, capacity, n_order), "binning");
	SGR_TRY(launch_blend_fwd(ft, g, b, img, sp ? sp->sem[pt.rank] : nullptr, out_color, out_depth, out_alpha, sp ? out_semantic : nullptr, st),
	        "blend_fwd");
	if (nl) {
		LayerRows zr = {};
		zr.n = nl;
		for (int k = 0; k < nl; k++) zr.rows[k] = layer_section(lpeers, pt.rank, k, ft);
		SGR_TRY(launch_layer_zero_rows(g, n_order, zr, st), "layer rows reset");
		for (int k = 0; k < nl; k++) {
			const LayerView lv = carve_sharded_layer(layers[k].state, ft.W, ft.H, capacity, fl.P).lv;
			SGR_TRY(launch_layer_lists_masked(ft, img, b, lp.mask[pt.rank], k, lv.img, lv.list, st), "layer_lists");
			BinView lb = b;
			lb.vals_out = lv.list;
			FrameDev fk = ft;
			fk.bg = layers[k].bg;
			SGR_TRY(launch_blend_fwd(fk, g, lb, lv.img, nullptr, layers[k].color, layers[k].depth, layers[k].alpha, nullptr, st), "layer blend_fwd");
		}
	}
	return SGR_OK;
}

int sgr_sharded_forward(const SgrFrame *frame, const SgrPeers *peers, const float *means3D, const float *shs, const float *colors_precomp,
                        const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp, float *out_color,
                        float *out_depth, float *out_alpha, int32_t *radii_local, void *records_local, size_t geom_bytes, void *img_state,
                        size_t img_bytes, void *binning_state, size_t binning_bytes, int64_t capacity, int64_t gaussian_capacity,
                        uint32_t barrier_epoch, int32_t pre_barrier, void *stream) {
	return sharded_forward(frame, peers, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, out_color, out_depth, out_alpha,
	                       radii_local, records_local, geom_bytes, img_state, img_bytes, binning_state, binning_bytes, capacity, gaussian_capacity,
	                       barrier_epoch, pre_barrier, nullptr, nullptr, nullptr, stream);
}

int sgr_sharded_forward_features(const SgrFrame *frame, const SgrPeers *peers, const float *means3D, const float *shs, const float *colors_precomp,
                                 const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp,
                                 float *out_color, float *out_depth, float *out_alpha, int32_t *radii_local, void *records_local,
                                 size_t geom_bytes, void *img_state, size_t img_bytes, void *binning_state, size_t binning_bytes,
                                 int64_t capacity, int64_t gaussian_capacity, uint32_t barrier_epoch, int32_t pre_barrier,
                                 const float *semantics, float *out_semantic, void *stream) {
	SemPeers sp = {};
	return sharded_forward(frame, peers, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, out_color, out_depth, out_alpha,
	                       radii_local, records_local, geom_bytes, img_state, img_bytes, binning_state, binning_bytes, capacity, gaussian_capacity,
	                       barrier_epoch, pre_barrier, &sp, semantics, out_semantic, stream);
}

static int sharded_backward(const SgrFrame *frame, const SgrPeers *peers, int64_t capacity, const float *means3D, const float *shs,
                            const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                            const int32_t *radii_local, const void *records_local, const void *img_state, const void *binning_state,
                            const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                            float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                            float *dL_dscales, float *dL_drotations, float *dL_dcov3D, uint32_t barrier_epoch, SemPeers *sp,
                            const float *dL_dsemantic, float *dL_dsemantics, void *stream, const SgrLayerPeers *lpeers = nullptr, const SgrShardedLayer *layers = nullptr, int nl = 0) {
	FrameDev fl, ft;
	PeerTable pt = {};
	int rc = make_total_frame(frame, peers, fl, ft, pt, true, sp);
	if (rc) return rc;
	if (nl && (rc = layer_peers(lpeers, pt, nl)) != SGR_OK) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	if (!img_state || !out_alpha || !dL_dcolor || !dL_ddepth || !dL_dalpha) return fail(SGR_EINVAL, "NULL pointer passed to sgr_sharded_backward");
	if (sp && (!dL_dsemantic || (fl.P > 0 && !dL_dsemantics))) return fail(SGR_EINVAL, "dL_dsemantic / dL_dsemantics is NULL");
	if (capacity > 0 && !binning_state) return fail(SGR_EINVAL, "capacity > 0 but binning_state is NULL");
	if (fl.P > 0 && (rc = check_geom_grads("sgr_sharded_backward", fl, means3D && radii_local && records_local, shs, scales, rotations, cov3D_precomp,
	                                       dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dopacity, dL_dscales, dL_drotations)) != SGR_OK)
		return rc;
	const GeomView g = carve_geom(pt.rec[pt.rank], ft.P);
	const ImgView img = carve_img(const_cast<void *>(img_state), ft.W, ft.H);
	const BinView b = carve_bin(const_cast<void *>(binning_state), capacity);
	float *grad2d = const_cast<float *>(pt.grad2d[pt.rank]);
	// (S > 0: the blend backward zeroes grad2d and gsem of every slot first; that is after the forward barrier, which a peer passes only
	// after the gather of its previous backward, the last reader of both)
	if (ft.P > 0)
		SGR_TRY(launch_blend_bwd(ft, g, b, img, sp ? sp->sem[pt.rank] : nullptr, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, sp ? dL_dsemantic : nullptr,
		                         grad2d, sp ? sp->gsem[pt.rank] : nullptr, st, true),
		        "blend_bwd");
	if (nl) {  // the live layers (this call takes them only when one has a gradient): blend backward by slot into the layer sections
		for (int k = 0; k < nl && ft.P > 0; k++) {
			if (!layers[k].dL_dcolor) continue;
			const LayerView lv = carve_sharded_layer(layers[k].state, ft.W, ft.H, capacity, fl.P).lv;
			BinView lb = b;
			lb.vals_out = lv.list;
			FrameDev fk = ft;  // (the background term of the blend's alpha gradient is the layer's)
			fk.bg = layers[k].bg;
			SGR_TRY(launch_blend_bwd2(fk, g, lb, lv.img, layers[k].alpha, layers[k].dL_dcolor, layers[k].dL_ddepth, layers[k].dL_dalpha,
			                          layer_section(lpeers, pt.rank, k, ft), st, true),
			        "layer blend_bwd");
		}
	}
	SGR_TRY(launch_peer_barrier(pt, barrier_epoch, ft.P > 0 ? g.big_count : nullptr, st), "barrier");
	if (nl) {  // owner side: main + live layer rows summed from the ranks, then the chain rule once on them
		const ShardedLayerView sv = carve_sharded_layer(layers[0].state, ft.W, ft.H, capacity, fl.P);
		LayerGatherTable t = {};
		for (int k = 0; k < nl; k++) {
			if (!layers[k].dL_dcolor || layers[k].end == layers[k].begin) continue;
			t.begin[t.n] = layers[k].begin; t.end[t.n] = layers[k].end; t.sink[t.n] = layers[k].dL_dmeans2D;
			t.sec[t.n] = pt;
			for (int p = 0; p < pt.world; p++) t.sec[t.n].grad2d[p] = layer_section(lpeers, p, k, ft);
			t.n++;
		}
		SGR_TRY(launch_layer_gather(fl.P, pt, t, radii_local, g.depth_key, sv.rows, dL_dmeans2D, st), "layer gather");
		SGR_TRY(launch_preprocess_bwd(fl, nullptr, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii_local, g.jac, sv.rows,
		                              dL_dmeans3D, sv.means2D, shs ? dL_dsh : nullptr, dL_dcolors_precomp, dL_dopacity,
		                              cov3D_precomp ? nullptr : dL_dscales, cov3D_precomp ? nullptr : dL_drotations, dL_dcov3D, st),
		        "preprocess_bwd");
		return SGR_OK;
	}
	SGR_TRY(launch_preprocess_bwd(fl, &pt, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii_local,
	                              g.jac, reinterpret_cast<const float *>(g.depth_key), dL_dmeans3D,
	                              dL_dmeans2D, shs ? dL_dsh : nullptr, dL_dcolors_precomp, dL_dopacity, cov3D_precomp ? nullptr : dL_dscales,
	                              cov3D_precomp ? nullptr : dL_drotations, dL_dcov3D, st),
	        "preprocess_bwd+gather");
	if (sp) SGR_TRY(launch_gather_semantics(pt, *sp, fl.P, fl.S, g.depth_key, dL_dsemantics, st), "gather semantics");
	return SGR_OK;
}

int sgr_sharded_backward(const SgrFrame *frame, const SgrPeers *peers, int64_t capacity, const float *means3D, const float *shs,
                         const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                         const int32_t *radii_local, const void *records_local, const void *img_state, const void *binning_state,
                         const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                         float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                         float *dL_dscales, float *dL_drotations, float *dL_dcov3D, uint32_t barrier_epoch, void *stream) {
	return sharded_backward(frame, peers, capacity, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii_local, records_local,
	                        img_state, binning_state, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors_precomp,
	                        dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D, barrier_epoch, nullptr, nullptr, nullptr, stream);
}

int sgr_sharded_backward_features(const SgrFrame *frame, const SgrPeers *peers, int64_t capacity, const float *means3D, const float *shs,
                                  const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                                  const int32_t *radii_local, const void *records_local, const void *img_state, const void *binning_state,
                                  const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                                  float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                                  float *dL_dscales, float *dL_drotations, float *dL_dcov3D, uint32_t barrier_epoch,
                                  const float *dL_dsemantic, float *dL_dsemantics, void *stream) {
	SemPeers sp = {};
	return sharded_backward(frame, peers, capacity, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii_local, records_local,
	                        img_state, binning_state, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors_precomp,
	                        dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D, barrier_epoch, &sp, dL_dsemantic, dL_dsemantics, stream);
}

int sgr_sharded_layer_state_sizes(const SgrFrame *frame, int64_t capacity, size_t *layer_bytes) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	if (capacity < 0 || capacity > 0x7fffffffLL) return fail(SGR_EINVAL, "capacity must be in [0, 2^31)");
	if (layer_bytes) *layer_bytes = carve_sharded_layer(nullptr, f.W, f.H, capacity, f.P).total_bytes;
	return SGR_OK;
}

int sgr_sharded_forward_layers(const SgrFrame *frame, const SgrPeers *peers, const float *means3D, const float *shs, const float *colors_precomp,
                               const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp, float *out_color,
                               float *out_depth, float *out_alpha, int32_t *radii_local, void *records_local, size_t geom_bytes, void *img_state,
                               size_t img_bytes, void *binning_state, size_t binning_bytes, int64_t capacity, int64_t gaussian_capacity,
                               uint32_t barrier_epoch, int32_t pre_barrier, const SgrLayerPeers *layer_peers, const SgrShardedLayer *layers,
                               int32_t num_layers, void *stream) {
	int rc = check_sharded_layers("sgr_sharded_forward_layers", frame, layers, num_layers, capacity, false);
	if (rc) return rc;
	return sharded_forward(frame, peers, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, out_color, out_depth, out_alpha,
	                       radii_local, records_local, geom_bytes, img_state, img_bytes, binning_state, binning_bytes, capacity, gaussian_capacity,
	                       barrier_epoch, pre_barrier, nullptr, nullptr, nullptr, stream, layer_peers, layers, num_layers);
}

int sgr_sharded_backward_layers(const SgrFrame *frame, const SgrPeers *peers, int64_t capacity, const float *means3D, const float *shs,
                                const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                                const int32_t *radii_local, const void *records_local, const void *img_state, const void *binning_state,
                                const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                                float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                                float *dL_dscales, float *dL_drotations, float *dL_dcov3D, uint32_t barrier_epoch, const SgrLayerPeers *layer_peers,
                                const SgrShardedLayer *layers, int32_t num_layers, void *stream) {
	int rc = check_sharded_layers("sgr_sharded_backward_layers", frame, layers, num_layers, capacity, true);
	if (rc) return rc;
	bool live = false;  // a layer whose images got no gradient costs nothing: without one this is sgr_sharded_backward
	for (int k = 0; k < num_layers; k++) live = live || layers[k].dL_dcolor != nullptr;
	return sharded_backward(frame, peers, capacity, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii_local, records_local,
	                        img_state, binning_state, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors_precomp,
	                        dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D, barrier_epoch, nullptr, nullptr, nullptr, stream, layer_peers,
	                        live ? layers : nullptr, live ? num_layers : 0);
}

int sgr_forward_status_async(const SgrFrame *frame, const void *geom_state, uint32_t *host_status, void *stream) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	if (!geom_state || !host_status) return fail(SGR_EINVAL, "NULL pointer passed to sgr_forward_status_async");
	for (int k = 0; k < 8; k++) host_status[k] = 0;
	if (f.P == 0) return SGR_OK;
	const GeomView g = carve_geom(const_cast<void *>(geom_state), f.P);
	cudaError_t e = cudaMemcpyAsync(host_status, g.big_count + 1, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, reinterpret_cast<cudaStream_t>(stream));
	if (e != cudaSuccess) return fail(SGR_ECUDA, "status copy: %s", cudaGetErrorString(e));
	return SGR_OK;
}

int sgr_forward_status(const SgrFrame *frame, const void *geom_state, int64_t *num_instances, int32_t *overflowed, void *stream) {
	uint32_t h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
	int rc = sgr_forward_status_async(frame, geom_state, h, stream);
	if (rc) return rc;
	cudaError_t e = cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(stream));
	if (e != cudaSuccess) return fail(SGR_ECUDA, "status sync: %s", cudaGetErrorString(e));
	if (num_instances) *num_instances = (int64_t)h[0];
	if (overflowed) *overflowed = (int32_t)h[1];
	return SGR_OK;
}

// shared body of sgr_backward_blend (every grad2d row written) and sgr_backward (grad2d is scratch for the chain rule: `reached_only`
// clears the rows of the Gaussians the forward reached, and only those are read back)
static int backward_blend(const SgrFrame *frame, int64_t num_instances, const float *semantics, const void *geom_state,
                          const void *binning_state, const void *img_state, const float *out_alpha, const float *dL_dcolor,
                          const float *dL_ddepth, const float *dL_dalpha, const float *dL_dsemantic, float *grad2d,
                          float *dL_dsemantics, bool reached_only, void *stream) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	if (f.P == 0) return SGR_OK;
	if (f.S > SGR_MAX_SEMANTIC_BWD) return fail(SGR_EUNSUPPORTED, "backward supports at most %d semantic channels, got %d", SGR_MAX_SEMANTIC_BWD, f.S);
	if (!geom_state || !img_state || !out_alpha || !dL_dcolor || !dL_ddepth || !dL_dalpha || !grad2d)
		return fail(SGR_EINVAL, "NULL pointer passed to sgr_backward_blend");
	if (f.S > 0 && (!semantics || !dL_dsemantic || !dL_dsemantics)) return fail(SGR_EINVAL, "S > 0 but a semantic pointer is NULL");
	if (num_instances > 0 && !binning_state) return fail(SGR_EINVAL, "num_instances > 0 but binning_state is NULL");
	const GeomView g = carve_geom(const_cast<void *>(geom_state), f.P);
	const ImgView img = carve_img(const_cast<void *>(img_state), f.W, f.H);
	const BinView b = carve_bin(const_cast<void *>(binning_state), num_instances);
	SGR_TRY(launch_blend_bwd(f, g, b, img, semantics, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, dL_dsemantic, grad2d, dL_dsemantics, st,
	                         false, reached_only ? g.reached : nullptr),
	        "blend_bwd");
	return SGR_OK;
}
int sgr_backward_blend(const SgrFrame *frame, int64_t num_instances, const float *semantics, const void *geom_state,
                       const void *binning_state, const void *img_state, const float *out_alpha, const float *dL_dcolor,
                       const float *dL_ddepth, const float *dL_dalpha, const float *dL_dsemantic, float *grad2d,
                       float *dL_dsemantics, void *stream) {
	return backward_blend(frame, num_instances, semantics, geom_state, binning_state, img_state, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha,
	                      dL_dsemantic, grad2d, dL_dsemantics, false, stream);
}

// shared body of sgr_backward_geom (no layer table) and sgr_backward_geom_layered; `fn` names the entry point in error messages.
// With a live layer (grad2d set, non-empty range) the layers' rows are merged into grad2d before the chain rule, and the main
// dL_dmeans2D of their range is restored from the pre-merge rows afterwards.  reached_only (sgr_backward, no layers): only the rows of
// the Gaussians the forward reached are read.
static int backward_geom(const char *fn, const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                         const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                         const void *geom_state, float *grad2d, const SgrLayerGrad *layers, int32_t num_layers, float *scratch,
                         float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                         float *dL_dscales, float *dL_drotations, float *dL_dcov3D, void *stream, bool reached_only = false) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	if (num_layers < 0 || (num_layers > 0 && !layers)) return fail(SGR_EINVAL, "bad layer table");
	int lo = 0x7fffffff, hi = 0;
	for (int k = 0; k < num_layers; k++) {
		const SgrLayerGrad &l = layers[k];
		if (l.begin < 0 || l.begin > l.end || l.end > f.P) return fail(SGR_EINVAL, "bad layer %d range [%d, %d) for P = %d", k, l.begin, l.end, f.P);
		if (!l.grad2d || l.end == l.begin) continue;
		lo = l.begin < lo ? l.begin : lo;
		hi = l.end > hi ? l.end : hi;
	}
	if (f.P == 0) return SGR_OK;
	if ((rc = check_geom_grads(fn, f, means3D && radii && geom_state && grad2d, shs, scales, rotations, cov3D_precomp, dL_dmeans3D,
	                           dL_dmeans2D, dL_dsh, dL_dopacity, dL_dscales, dL_drotations)) != SGR_OK)
		return rc;
	if (hi > lo && !scratch) return fail(SGR_EINVAL, "scratch is NULL");
	const GeomView g = carve_geom(const_cast<void *>(geom_state), f.P);
	if (hi > lo) {
		SGR_TRY(launch_layer_stash(grad2d, lo, hi, scratch, false, nullptr, st), "layer stash");
		SGR_TRY(launch_layer_merge(grad2d, layers, num_layers, st), "layer merge");
	}
	SGR_TRY(launch_preprocess_bwd(f, nullptr, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii, g.jac, grad2d, dL_dmeans3D,
	                              dL_dmeans2D, shs ? dL_dsh : nullptr, dL_dcolors_precomp, dL_dopacity,
	                              cov3D_precomp ? nullptr : dL_dscales, cov3D_precomp ? nullptr : dL_drotations, dL_dcov3D, st,
	                              reached_only ? g.reached : nullptr),
	        "preprocess_bwd");
	if (hi > lo) SGR_TRY(launch_layer_stash(grad2d, lo, hi, scratch, true, dL_dmeans2D, st), "layer restore");
	return SGR_OK;
}

int sgr_backward_geom(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                      const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                      const void *geom_state, const float *grad2d, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh,
                      float *dL_dcolors_precomp, float *dL_dopacity, float *dL_dscales, float *dL_drotations,
                      float *dL_dcov3D, void *stream) {
	// without layers grad2d is only read
	return backward_geom("sgr_backward_geom", frame, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii, geom_state,
	                     const_cast<float *>(grad2d), nullptr, 0, nullptr, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors_precomp, dL_dopacity,
	                     dL_dscales, dL_drotations, dL_dcov3D, stream);
}

int sgr_backward(const SgrFrame *frame, int64_t num_instances, const float *means3D, const float *shs,
                 const float *colors_precomp, const float *semantics, const float *scales, const float *rotations,
                 const float *cov3D_precomp, const int32_t *radii, const void *geom_state, const void *binning_state,
                 const void *img_state, const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth,
                 const float *dL_dalpha, const float *dL_dsemantic, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh,
                 float *dL_dcolors_precomp, float *dL_dsemantics, float *dL_dopacity, float *dL_dscales,
                 float *dL_drotations, float *dL_dcov3D, float *grad2d_scratch, void *stream) {
	int rc = backward_blend(frame, num_instances, semantics, geom_state, binning_state, img_state, out_alpha, dL_dcolor, dL_ddepth,
	                        dL_dalpha, dL_dsemantic, grad2d_scratch, dL_dsemantics, true, stream);
	if (rc) return rc;
	return backward_geom("sgr_backward", frame, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii, geom_state,
	                     grad2d_scratch, nullptr, 0, nullptr, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors_precomp, dL_dopacity, dL_dscales,
	                     dL_drotations, dL_dcov3D, stream, true);
}

// ---- render layers ----
// the frame of a layer: the main call's, whole image, no feature channels, the layer's background
static int make_layer_frame(const SgrFrame *frame, const SgrLayer *layer, FrameDev &f) {
	int rc = make_frame(frame, f);
	if (rc) return rc;
	if (!layer) return fail(SGR_EINVAL, "layer is NULL");
	if (layer->begin < 0 || layer->begin > layer->end || layer->end > f.P)
		return fail(SGR_EINVAL, "bad layer range [%d, %d) for P = %d", layer->begin, layer->end, f.P);
	if (!layer->bg) return fail(SGR_EINVAL, "layer bg is NULL");
	if (!(f.band.begin == 0 && f.band.end == f.gy && f.band.step == 1))
		return fail(SGR_EUNSUPPORTED, "layers need the whole image (a tile-row band was given)");
	f.S = 0;
	f.bg = layer->bg;
	return SGR_OK;
}

int sgr_layer_state_sizes(const SgrFrame *frame, int64_t num_instances, size_t *layer_bytes) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	if (num_instances < 0 || num_instances > 0x7fffffffLL) return fail(SGR_EINVAL, "num_instances %lld outside [0, 2^31)", (long long)num_instances);
	if (layer_bytes) *layer_bytes = carve_layer(nullptr, f.W, f.H, num_instances).total_bytes;
	return SGR_OK;
}

int sgr_forward_layer(const SgrFrame *frame, const SgrLayer *layer, int64_t num_instances, const void *geom_state, const void *binning_state,
                      const void *img_state, void *layer_state, size_t layer_bytes, float *out_color, float *out_depth, float *out_alpha,
                      void *stream) {
	FrameDev f;
	int rc = make_layer_frame(frame, layer, f);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	if (!out_color || !out_depth || !out_alpha) return fail(SGR_EINVAL, "output image pointer is NULL");
	if (num_instances < 0 || num_instances > 0x7fffffffLL) return fail(SGR_EINVAL, "num_instances %lld outside [0, 2^31)", (long long)num_instances);
	if (layer->begin == layer->end) {
		SGR_TRY(launch_layer_fill(f, f.bg, out_color, out_depth, out_alpha, st), "layer_fill");
		return SGR_OK;
	}
	if (!f.view || !f.proj || !f.campos) return fail(SGR_EINVAL, "camera pointer (viewmatrix/projmatrix/campos) is NULL");
	if (!geom_state || !img_state || !layer_state) return fail(SGR_EINVAL, "NULL state passed to sgr_forward_layer");
	if (num_instances > 0 && !binning_state) return fail(SGR_EINVAL, "num_instances > 0 but binning_state is NULL");
	const LayerView lv = carve_layer(layer_state, f.W, f.H, num_instances);
	if (layer_bytes < lv.total_bytes) return fail(SGR_ENOMEM, "layer_state too small: %zu < %zu", layer_bytes, lv.total_bytes);
	const GeomView g = carve_geom(const_cast<void *>(geom_state), f.P);
	const ImgView img = carve_img(const_cast<void *>(img_state), f.W, f.H);
	const BinView b = carve_bin(const_cast<void *>(binning_state), num_instances);
	SGR_TRY(launch_layer_lists(f, img, b, layer->begin, layer->end, lv.img, lv.list, st), "layer_lists");
	BinView lb = b;
	lb.vals_out = lv.list;
	SGR_TRY(launch_blend_fwd(f, g, lb, lv.img, nullptr, out_color, out_depth, out_alpha, nullptr, st), "layer blend_fwd");
	return SGR_OK;
}

int sgr_backward_blend_layer(const SgrFrame *frame, const SgrLayer *layer, const void *geom_state, const void *layer_state, const float *out_alpha,
                             const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha, float *grad2d, void *stream) {
	FrameDev f;
	int rc = make_layer_frame(frame, layer, f);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	if (layer->begin == layer->end) return SGR_OK;
	if (!geom_state || !layer_state || !out_alpha || !dL_dcolor || !dL_ddepth || !dL_dalpha || !grad2d)
		return fail(SGR_EINVAL, "NULL pointer passed to sgr_backward_blend_layer");
	const LayerView lv = carve_layer(const_cast<void *>(layer_state), f.W, f.H, 0);
	const GeomView g = carve_geom(const_cast<void *>(geom_state), f.P);
	BinView lb = carve_bin(nullptr, 0);
	lb.vals_out = lv.list;
	const size_t rows = (size_t)(layer->end - layer->begin);
	SGR_TRY(cudaMemsetAsync(grad2d, 0, rows * 12 * sizeof(float), st), "layer grad2d reset");
	// the layer's lists hold ids in [begin, end) only: a base `begin` rows before the layer's array keeps blend_bwd2's global indexing in bounds
	float *base = grad2d - (size_t)layer->begin * 12;
	SGR_TRY(launch_blend_bwd2(f, g, lb, lv.img, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, base, st, true), "layer blend_bwd");
	return SGR_OK;
}

int sgr_backward_geom_layered(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                              const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                              const void *geom_state, float *grad2d, const SgrLayerGrad *layers, int32_t num_layers, float *scratch,
                              float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                              float *dL_dscales, float *dL_drotations, float *dL_dcov3D, void *stream) {
	return backward_geom("sgr_backward_geom_layered", frame, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii,
	                     geom_state, grad2d, layers, num_layers, scratch, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors_precomp, dL_dopacity,
	                     dL_dscales, dL_drotations, dL_dcov3D, stream);
}

int sgr_mark_visible(int32_t P, const float *means3D, const float *viewmatrix, const float *projmatrix, uint8_t *present,
                     void *stream) {
	(void)projmatrix;  // the reference passes it too but the test only uses the view-space depth
	if (P < 0) return fail(SGR_EINVAL, "P < 0");
	if (P == 0) return SGR_OK;
	if (!means3D || !viewmatrix || !present) return fail(SGR_EINVAL, "NULL pointer passed to sgr_mark_visible");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_mark_visible(P, means3D, viewmatrix, present, st), "mark_visible");
	return SGR_OK;
}

int sgr_visible_filter(const SgrFrame *frame, const float *means3D, const float *scales, const float *rotations,
                       const float *cov3D_precomp, int32_t *radii, float *means2D, void *stream) {
	FrameDev f;
	int rc = make_frame(frame, f);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	if (f.P == 0) return SGR_OK;
	if (!means3D || !radii || !means2D || !f.view || !f.proj) return fail(SGR_EINVAL, "NULL pointer passed to sgr_visible_filter");
	if (!cov3D_precomp && (!scales || !rotations)) return fail(SGR_EINVAL, "provide (scales, rotations) or cov3D_precomp");
	if ((rc = check_aligned16("rotations", cov3D_precomp ? nullptr : rotations)) != SGR_OK) return rc;
	SGR_TRY(launch_filter(f, means3D, scales, rotations, cov3D_precomp, radii, means2D, st), "visible_filter");
	return SGR_OK;
}

static int check_segments(const SgrSegment *segs, int32_t n, int32_t M, int64_t &P) {
	if (!segs || n <= 0) return fail(SGR_EINVAL, "segment table is empty");
	if (M < 1 || M > 16) return fail(SGR_EINVAL, "M = %d SH coefficients per Gaussian (must be 1..16)", M);
	int64_t at = segs[0].start;
	if (at != 0) return fail(SGR_EINVAL, "segment 0 must start at composed index 0");
	for (int k = 0; k < n; k++) {
		const SgrSegment &s = segs[k];
		if (s.start != at || s.count < 0) return fail(SGR_EINVAL, "segment %d: start %d (expected %lld), count %d — segments must be ascending and gap-free", k, s.start, (long long)at, s.count);
		if (s.fourier_dim < 1 || s.fourier_dim > SGR_MAX_FOURIER) return fail(SGR_EINVAL, "segment %d: fourier_dim %d outside 1..%d", k, s.fourier_dim, SGR_MAX_FOURIER);
		if (s.count > 0 && (!s.xyz || !s.rotation || !s.scaling || !s.opacity || !s.features_dc || (M > 1 && !s.features_rest)))
			return fail(SGR_EINVAL, "segment %d has a NULL parameter array", k);
		at += s.count;
	}
	if (at > 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "composed Gaussian count exceeds 2^31-1");
	P = at;
	return SGR_OK;
}

static int compose_forward_impl(const char *fn, const SgrSegment *segments, int32_t num_segments, int32_t M, const float *poses,
                                const float *idft, const uint8_t *flip, const float *flip_quat, float *means3D, float *rotations, float *scales,
                                float *opacities, float *shs, const float *correction, void *stream) {
	int64_t P = 0;
	int rc = check_segments(segments, num_segments, M, P);
	if (rc) return rc;
	if (P == 0) return SGR_OK;
	if (!poses || !idft || !means3D || !rotations || !scales || !opacities || !shs) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (flip && !flip_quat) return fail(SGR_EINVAL, "flip mask given without flip_quat");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_compose_fwd(segments, num_segments, M, poses, idft, flip, flip_quat, means3D, rotations, scales, opacities, shs, correction, st),
	        "compose_fwd");
	return SGR_OK;
}

int sgr_compose_forward(const SgrSegment *segments, int32_t num_segments, int32_t M, const float *poses, const float *idft,
                        const uint8_t *flip, const float *flip_quat, float *means3D, float *rotations, float *scales, float *opacities,
                        float *shs, void *stream) {
	return compose_forward_impl("sgr_compose_forward", segments, num_segments, M, poses, idft, flip, flip_quat, means3D, rotations, scales,
	                            opacities, shs, nullptr, stream);
}

int sgr_compose_forward_corrected(const SgrSegment *segments, int32_t num_segments, int32_t M, const float *poses, const float *idft,
                                  const uint8_t *flip, const float *flip_quat, const float *bkgd_correction, float *means3D, float *rotations,
                                  float *scales, float *opacities, float *shs, void *stream) {
	if (!bkgd_correction) return fail(SGR_EINVAL, "NULL bkgd_correction passed to sgr_compose_forward_corrected");
	return compose_forward_impl("sgr_compose_forward_corrected", segments, num_segments, M, poses, idft, flip, flip_quat, means3D, rotations,
	                            scales, opacities, shs, bkgd_correction, stream);
}

static int compose_backward_impl(const char *fn, const SgrSegment *segments, const SgrSegmentGrads *grads, int32_t num_segments, int32_t M,
                                 const float *poses, const float *idft, const uint8_t *flip, const float *flip_quat, const float *correction,
                                 const float *dL_dmeans3D, const float *dL_drotations, const float *dL_dscales, const float *dL_dopacities,
                                 const float *dL_dshs, float *dposes, float *dcorrection, float *pose_scratch, void *stream) {
	int64_t P = 0;
	int rc = check_segments(segments, num_segments, M, P);
	if (rc) return rc;
	if (!grads || !dposes || !pose_scratch || !poses || !idft) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (P > 0 && (!dL_dmeans3D || !dL_drotations || !dL_dscales || !dL_dopacities || !dL_dshs)) return fail(SGR_EINVAL, "NULL upstream gradient");
	if (flip && !flip_quat) return fail(SGR_EINVAL, "flip mask given without flip_quat");
	for (int k = 0; k < num_segments; k++) {
		const SgrSegmentGrads &g = grads[k];
		if (segments[k].count > 0 && (!g.xyz || !g.rotation || !g.scaling || !g.opacity || !g.features_dc || (M > 1 && !g.features_rest)))
			return fail(SGR_EINVAL, "segment %d has a NULL gradient array", k);
	}
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_compose_bwd(segments, grads, num_segments, M, poses, idft, flip, flip_quat, dL_dmeans3D, dL_drotations, dL_dscales,
	                           dL_dopacities, dL_dshs, pose_scratch, dposes, correction, dcorrection, st),
	        "compose_bwd");
	return SGR_OK;
}

int sgr_compose_backward(const SgrSegment *segments, const SgrSegmentGrads *grads, int32_t num_segments, int32_t M, const float *poses,
                         const float *idft, const uint8_t *flip, const float *flip_quat, const float *dL_dmeans3D,
                         const float *dL_drotations, const float *dL_dscales, const float *dL_dopacities, const float *dL_dshs,
                         float *dposes, float *pose_scratch, void *stream) {
	return compose_backward_impl("sgr_compose_backward", segments, grads, num_segments, M, poses, idft, flip, flip_quat, nullptr, dL_dmeans3D,
	                             dL_drotations, dL_dscales, dL_dopacities, dL_dshs, dposes, nullptr, pose_scratch, stream);
}

int sgr_compose_backward_corrected(const SgrSegment *segments, const SgrSegmentGrads *grads, int32_t num_segments, int32_t M,
                                   const float *poses, const float *idft, const uint8_t *flip, const float *flip_quat,
                                   const float *bkgd_correction, const float *dL_dmeans3D, const float *dL_drotations, const float *dL_dscales,
                                   const float *dL_dopacities, const float *dL_dshs, float *dposes, float *dcorrection, float *pose_scratch,
                                   void *stream) {
	if (!bkgd_correction || !dcorrection) return fail(SGR_EINVAL, "NULL bkgd_correction / dcorrection passed to sgr_compose_backward_corrected");
	return compose_backward_impl("sgr_compose_backward_corrected", segments, grads, num_segments, M, poses, idft, flip, flip_quat, bkgd_correction,
	                             dL_dmeans3D, dL_drotations, dL_dscales, dL_dopacities, dL_dshs, dposes, dcorrection, pose_scratch, stream);
}

int32_t sgr_compose_pose_rows(int32_t num_segments, int32_t corrected) { return num_segments > 0 ? num_segments + (corrected ? 1 : 0) : 0; }

static int check_pose_acc_bytes(const char *fn, int32_t num_segments, const float *bkgd_correction, size_t bytes) {
	const size_t need = (size_t)sgr_compose_pose_rows(num_segments, bkgd_correction != nullptr) * 16 * sizeof(float);
	if (bytes < need) return fail(SGR_ENOMEM, "%s: pose_acc holds %zu bytes, %zu needed", fn, bytes, need);
	return SGR_OK;
}

int sgr_compose_backward_rows(const SgrSegment *segments, const SgrSegmentGrads *grads, int32_t num_segments, int32_t M, const float *poses,
                              const float *idft, const uint8_t *flip, const float *flip_quat, const float *bkgd_correction,
                              const float *dL_dmeans3D, const float *dL_drotations, const float *dL_dscales, const float *dL_dopacities,
                              const float *dL_dshs, float *pose_acc, size_t pose_acc_bytes, void *stream) {
	int64_t P = 0;
	int rc = check_segments(segments, num_segments, M, P);
	if (rc) return rc;
	if (!grads || !pose_acc || !poses || !idft) return fail(SGR_EINVAL, "NULL pointer passed to sgr_compose_backward_rows");
	if (P > 0 && (!dL_dmeans3D || !dL_drotations || !dL_dscales || !dL_dopacities || !dL_dshs)) return fail(SGR_EINVAL, "NULL upstream gradient");
	if (flip && !flip_quat) return fail(SGR_EINVAL, "flip mask given without flip_quat");
	for (int k = 0; k < num_segments; k++) {
		const SgrSegmentGrads &g = grads[k];
		if (segments[k].count > 0 && (!g.xyz || !g.rotation || !g.scaling || !g.opacity || !g.features_dc || (M > 1 && !g.features_rest)))
			return fail(SGR_EINVAL, "segment %d has a NULL gradient array", k);
	}
	if ((rc = check_pose_acc_bytes("sgr_compose_backward_rows", num_segments, bkgd_correction, pose_acc_bytes)) != SGR_OK) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_compose_bwd_rows(segments, grads, num_segments, M, poses, idft, flip, flip_quat, dL_dmeans3D, dL_drotations, dL_dscales,
	                                dL_dopacities, dL_dshs, pose_acc, bkgd_correction, st),
	        "compose_bwd_rows");
	return SGR_OK;
}

// what the finalize reads: the posed flags of the segments and, with a correction, somewhere to put its gradient
static int check_pose_finalize(const char *fn, const SgrSegment *segments, int32_t num_segments, const float *poses, const float *bkgd_correction,
                               const float *pose_acc, size_t pose_acc_bytes, const float *dposes, const float *dcorrection) {
	if (!segments || num_segments <= 0) return fail(SGR_EINVAL, "segment table is empty");
	if (!poses || !pose_acc || !dposes) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (bkgd_correction && !dcorrection) return fail(SGR_EINVAL, "%s: bkgd_correction given without dcorrection", fn);
	if (!bkgd_correction && dcorrection) return fail(SGR_EINVAL, "%s: dcorrection given without bkgd_correction", fn);
	return check_pose_acc_bytes(fn, num_segments, bkgd_correction, pose_acc_bytes);
}

int sgr_compose_pose_finalize(const SgrSegment *segments, int32_t num_segments, const float *poses, const float *bkgd_correction,
                              const float *pose_acc, size_t pose_acc_bytes, float *dposes, float *dcorrection, void *stream) {
	int rc = check_pose_finalize("sgr_compose_pose_finalize", segments, num_segments, poses, bkgd_correction, pose_acc, pose_acc_bytes, dposes,
	                             dcorrection);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_compose_pose_finalize(segments, num_segments, poses, pose_acc, dposes, bkgd_correction, dcorrection, st), "compose_pose_finalize");
	return SGR_OK;
}

int sgr_compose_pose_reduce_peers(const SgrPeers *peers, const SgrSegment *segments, int32_t num_segments, const float *poses,
                                  const float *bkgd_correction, float *pose_acc, size_t pose_acc_bytes, float *dposes, float *dcorrection,
                                  void *stream) {
	if (!peers) return fail(SGR_EINVAL, "peers is NULL");
	int rc = check_pose_finalize("sgr_compose_pose_reduce_peers", segments, num_segments, poses, bkgd_correction, pose_acc, pose_acc_bytes, dposes,
	                             dcorrection);
	if (rc) return rc;
	FrameDev f = {};
	PeerTable pt = {};
	if ((rc = make_peers(peers, f, false, pt)) != SGR_OK) return rc;
	PoseAccPeers pp = {};
	pp.world = pt.world;
	for (int p = 0; p < pt.world; p++) {
		if (!peers->pose_acc[p]) return fail(SGR_EINVAL, "peer table entry %d has no composer accumulator section", p);
		if (pt.world > 1 && !pt.flags[p]) return fail(SGR_EINVAL, "peer table entry %d has no barrier pad", p);
		pp.sec[p] = peers->pose_acc[p];
	}
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_compose_pose_reduce(pt, pp, pose_acc, sgr_compose_pose_rows(num_segments, bkgd_correction != nullptr), st), "compose_pose_reduce");
	SGR_TRY(launch_compose_pose_finalize(segments, num_segments, poses, pose_acc, dposes, bkgd_correction, dcorrection, st), "compose_pose_finalize");
	return SGR_OK;
}

int sgr_color_correct_forward(int32_t H, int32_t W, const float *image, const float *affine, float *out, void *stream) {
	if (H <= 0 || W <= 0) return fail(SGR_EINVAL, "bad image size H=%d W=%d", H, W);
	if (!image || !affine || !out) return fail(SGR_EINVAL, "NULL pointer passed to sgr_color_correct_forward");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_color_correct_fwd((int64_t)H * W, image, affine, out, st), "color_correct_fwd");
	return SGR_OK;
}

size_t sgr_color_correct_scratch_bytes(int32_t H, int32_t W) { return (H > 0 && W > 0) ? color_correct_scratch_bytes((int64_t)H * W) : 0; }

int sgr_color_correct_backward(int32_t H, int32_t W, const float *image, const float *affine, const float *dL_dout, float *dL_dimage,
                               float *dL_daffine, void *scratch, size_t scratch_bytes, void *stream) {
	if (H <= 0 || W <= 0) return fail(SGR_EINVAL, "bad image size H=%d W=%d", H, W);
	if (!image || !affine || !dL_dout || !dL_daffine) return fail(SGR_EINVAL, "NULL pointer passed to sgr_color_correct_backward");
	const int64_t N = (int64_t)H * W;
	if (!scratch || scratch_bytes < color_correct_scratch_bytes(N))
		return fail(SGR_ENOMEM, "colour correction scratch too small: %zu < %zu", scratch_bytes, color_correct_scratch_bytes(N));
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_color_correct_bwd(N, image, affine, dL_dout, dL_dimage, dL_daffine, scratch, st), "color_correct_bwd");
	return SGR_OK;
}

int sgr_color_correction_reg(const float *affine, const float *affine_sky, float weight, float *value, float *g_affine, float *g_affine_sky,
                             void *stream) {
	if (!affine || !value) return fail(SGR_EINVAL, "NULL pointer passed to sgr_color_correction_reg");
	if (affine_sky == nullptr && g_affine_sky != nullptr) return fail(SGR_EINVAL, "g_affine_sky given without affine_sky");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_color_correction_reg(affine, affine_sky, weight, value, g_affine, g_affine_sky, st), "color_correction_reg");
	return SGR_OK;
}

static int sky_check(const char *fn, int32_t H, int32_t W, int32_t R, int32_t mode, const uint8_t *sky_mask) {
	// texel indices are int: 6 R^2 < 2^31
	if (H <= 0 || W <= 0 || R <= 0 || R > 16384) return fail(SGR_EINVAL, "%s: bad sizes H=%d W=%d R=%d", fn, H, W, R);
	if (mode != SGR_SKY_MASK_ACC && mode != SGR_SKY_MASK_GIVEN) return fail(SGR_EINVAL, "%s: unknown mask mode %d", fn, mode);
	if (mode == SGR_SKY_MASK_GIVEN && !sky_mask) return fail(SGR_EINVAL, "%s: SGR_SKY_MASK_GIVEN needs sky_mask", fn);
	return SGR_OK;
}

int sgr_sky_composite_forward(int32_t H, int32_t W, int32_t R, int32_t mode, float fill, const float *rgb, const float *acc,
                              const uint8_t *sky_mask, const float *cube_map, const float *K, const float *w2c, const float *jitter_x,
                              const float *jitter_y, float *rgb_out, void *stream) {
	if (int rc = sky_check("sgr_sky_composite_forward", H, W, R, mode, sky_mask)) return rc;
	if (!rgb || !acc || !cube_map || !K || !w2c || !rgb_out) return fail(SGR_EINVAL, "NULL pointer passed to sgr_sky_composite_forward");
	if (!jitter_x != !jitter_y) return fail(SGR_EINVAL, "sgr_sky_composite_forward: give both jitters or neither");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_sky_composite_fwd(H, W, R, mode, fill, rgb, acc, sky_mask, cube_map, K, w2c, jitter_x, jitter_y, rgb_out, st), "sky_composite_fwd");
	return SGR_OK;
}

int sgr_sky_composite_backward(int32_t H, int32_t W, int32_t R, int32_t mode, float fill, const float *acc, const uint8_t *sky_mask,
                               const float *cube_map, const float *K, const float *w2c, const float *jitter_x, const float *jitter_y,
                               const float *dL_dout, float *dL_dacc, float *dL_dcube, void *stream) {
	if (int rc = sky_check("sgr_sky_composite_backward", H, W, R, mode, sky_mask)) return rc;
	if (!acc || !cube_map || !K || !w2c || !dL_dout) return fail(SGR_EINVAL, "NULL pointer passed to sgr_sky_composite_backward");
	if (!jitter_x != !jitter_y) return fail(SGR_EINVAL, "sgr_sky_composite_backward: give both jitters or neither");
	if (!dL_dacc && !dL_dcube) return SGR_OK;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_sky_composite_bwd(H, W, R, mode, fill, acc, sky_mask, cube_map, K, w2c, jitter_x, jitter_y, dL_dout, dL_dacc, dL_dcube, st),
	        "sky_composite_bwd");
	return SGR_OK;
}

static int actor_pose_check(const char *fn, int32_t num_tracks, int32_t K, const int32_t *track_off, const int32_t *entry_fc, const double *entry_ts,
                            const double *track_span, const int32_t *track_frames, int32_t num_cams, const int32_t *cam_off, const double *cam_ts,
                            const float *input_trans, const float *input_rots, int32_t n_act, const int32_t *tracks, int32_t cam, int32_t is_val,
                            const float *ego_pose, const float *opt_trans, const float *opt_rots) {
	if (num_tracks < 0 || K <= 0 || num_cams < 0 || n_act < 0) return fail(SGR_EINVAL, "%s: bad sizes tracks=%d K=%d cams=%d actors=%d", fn, num_tracks, K, num_cams, n_act);
	if (!track_off || !entry_fc || !entry_ts || !track_span || !track_frames || !input_trans || !input_rots || !ego_pose)
		return fail(SGR_EINVAL, "%s: NULL track table or ego pose", fn);
	if (n_act > 0 && !tracks) return fail(SGR_EINVAL, "%s: tracks is NULL", fn);
	for (int32_t a = 0; a < n_act; a++)
		if (tracks[a] < 0 || tracks[a] >= num_tracks) return fail(SGR_EINVAL, "%s: track slot %d of actor %d is outside [0, %d)", fn, tracks[a], a, num_tracks);
	if ((opt_trans == nullptr) != (opt_rots == nullptr)) return fail(SGR_EINVAL, "%s: give both opt_trans and opt_rots or neither", fn);
	if (opt_trans && is_val) {
		if (cam < 0 || cam >= num_cams) return fail(SGR_EINVAL, "%s: camera %d is outside [0, %d)", fn, cam, num_cams);
		if (!cam_off || !cam_ts) return fail(SGR_EINVAL, "%s: NULL camera timestamps", fn);
	}
	return SGR_OK;
}

static ActorPoseTable actor_pose_table(int32_t num_tracks, int32_t K, const int32_t *track_off, const int32_t *entry_fc, const double *entry_ts,
                                       const double *track_span, const int32_t *track_frames, int32_t num_cams, const int32_t *cam_off,
                                       const double *cam_ts, const float *input_trans, const float *input_rots) {
	return ActorPoseTable{num_tracks, K, num_cams, track_off, entry_fc, track_frames, cam_off, entry_ts, track_span, cam_ts, input_trans, input_rots};
}

int sgr_actor_pose_forward(int32_t num_tracks, int32_t K, const int32_t *track_off, const int32_t *entry_fc, const double *entry_ts,
                           const double *track_span, const int32_t *track_frames, int32_t num_cams, const int32_t *cam_off, const double *cam_ts,
                           const float *input_trans, const float *input_rots, int32_t n_act, const int32_t *tracks, double timestamp, int32_t cam,
                           int32_t is_val, const float *ego_pose, const float *opt_trans, const float *opt_rots, int32_t frame, double fourier_scale,
                           int32_t fourier_dim, float *poses, float *idft, void *stream) {
	const char *fn = "sgr_actor_pose_forward";
	if (int rc = actor_pose_check(fn, num_tracks, K, track_off, entry_fc, entry_ts, track_span, track_frames, num_cams, cam_off, cam_ts, input_trans,
	                              input_rots, n_act, tracks, cam, is_val, ego_pose, opt_trans, opt_rots))
		return rc;
	if (n_act > 0 && !poses) return fail(SGR_EINVAL, "%s: poses is NULL", fn);
	if (idft && (fourier_dim <= 0 || fourier_dim > SGR_MAX_FOURIER)) return fail(SGR_EINVAL, "%s: fourier_dim %d is outside [1, %d]", fn, fourier_dim, SGR_MAX_FOURIER);
	if (n_act == 0) return SGR_OK;
	const ActorPoseTable T = actor_pose_table(num_tracks, K, track_off, entry_fc, entry_ts, track_span, track_frames, num_cams, cam_off, cam_ts,
	                                          input_trans, input_rots);
	const ActorPoseCall c{timestamp, fourier_scale, cam, is_val != 0, opt_trans != nullptr, frame, fourier_dim, ego_pose, opt_trans, opt_rots};
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_actor_pose_fwd(T, c, tracks, n_act, poses, idft, st), "actor_pose_fwd");
	return SGR_OK;
}

size_t sgr_actor_pose_scratch_bytes(int32_t n_act) { return n_act > 0 ? actor_pose_scratch_bytes(n_act) : 0; }

int sgr_actor_pose_backward(int32_t num_tracks, int32_t K, const int32_t *track_off, const int32_t *entry_fc, const double *entry_ts,
                            const double *track_span, const int32_t *track_frames, int32_t num_cams, const int32_t *cam_off, const double *cam_ts,
                            const float *input_trans, const float *input_rots, int32_t n_act, const int32_t *tracks, double timestamp, int32_t cam,
                            int32_t is_val, const float *ego_pose, const float *opt_trans, const float *opt_rots, const float *dL_dposes,
                            float *dL_dopt_trans, float *dL_dopt_rots, void *scratch, size_t scratch_bytes, void *stream) {
	const char *fn = "sgr_actor_pose_backward";
	if (int rc = actor_pose_check(fn, num_tracks, K, track_off, entry_fc, entry_ts, track_span, track_frames, num_cams, cam_off, cam_ts, input_trans,
	                              input_rots, n_act, tracks, cam, is_val, ego_pose, opt_trans, opt_rots))
		return rc;
	if (!opt_trans) return fail(SGR_EINVAL, "%s: without opt_trans / opt_rots the poses have no parameters", fn);
	if (n_act == 0) return SGR_OK;
	if (!dL_dposes || !dL_dopt_trans || !dL_dopt_rots) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (!scratch || scratch_bytes < actor_pose_scratch_bytes(n_act))
		return fail(SGR_EINVAL, "%s: scratch of %zu bytes, needs %zu", fn, scratch_bytes, actor_pose_scratch_bytes(n_act));
	const ActorPoseTable T = actor_pose_table(num_tracks, K, track_off, entry_fc, entry_ts, track_span, track_frames, num_cams, cam_off, cam_ts,
	                                          input_trans, input_rots);
	const ActorPoseCall c{timestamp, 0.0, cam, is_val != 0, 1, 0, 0, ego_pose, opt_trans, opt_rots};
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_actor_pose_bwd(T, c, tracks, n_act, dL_dposes, dL_dopt_trans, dL_dopt_rots, scratch, st), "actor_pose_bwd");
	return SGR_OK;
}

int sgr_gaussian_normals_forward(int32_t P, const float *means3D, const float *rotations, const float *scales, const float *camera_center,
                                 float *normals, uint8_t *decision, void *stream) {
	const char *fn = "sgr_gaussian_normals_forward";
	if (P < 0) return fail(SGR_EINVAL, "%s: bad size P=%d", fn, P);
	if (P == 0) return SGR_OK;
	if (!means3D || !rotations || !scales || !camera_center || !normals || !decision) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (reinterpret_cast<uintptr_t>(rotations) % 16) return fail(SGR_EINVAL, "%s: rotations must be 16-byte aligned", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_gaussian_normals_fwd(P, means3D, rotations, scales, camera_center, normals, decision, st), "gaussian_normals_fwd");
	return SGR_OK;
}

int sgr_gaussian_normals_backward(int32_t P, const float *rotations, const uint8_t *decision, const float *dL_dnormals, float *dL_drotations,
                                  void *stream) {
	const char *fn = "sgr_gaussian_normals_backward";
	if (P < 0) return fail(SGR_EINVAL, "%s: bad size P=%d", fn, P);
	if (P == 0) return SGR_OK;
	if (!rotations || !decision || !dL_dnormals || !dL_drotations) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (reinterpret_cast<uintptr_t>(rotations) % 16 || reinterpret_cast<uintptr_t>(dL_drotations) % 16)
		return fail(SGR_EINVAL, "%s: rotations and dL_drotations must be 16-byte aligned", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_gaussian_normals_bwd(P, rotations, decision, dL_dnormals, dL_drotations, st), "gaussian_normals_bwd");
	return SGR_OK;
}

// Checks what both semantic entries share and builds the actors' composed row starts (starts[a] = n_bg + counts before a).
static int semantics_check(const char *fn, int32_t K, int32_t mode, int32_t n_bg, int32_t n_act, const int32_t *actor_count,
                           const int32_t *class_label, std::vector<int32_t> &starts) {
	if (K < 1) return fail(SGR_EINVAL, "%s: K = %d, need at least one class", fn, K);
	if (mode != SGR_SEMANTIC_LOGITS && mode != SGR_SEMANTIC_PROBABILITIES) return fail(SGR_EINVAL, "%s: unknown semantic mode %d", fn, mode);
	if (n_bg < 0 || n_act < 0) return fail(SGR_EINVAL, "%s: bad sizes n_bg=%d n_act=%d", fn, n_bg, n_act);
	if (n_act > 0 && (!actor_count || !class_label)) return fail(SGR_EINVAL, "%s: NULL actor table", fn);
	starts.assign((size_t)n_act + 1, 0);
	long long at = n_bg;
	for (int32_t a = 0; a < n_act; a++) {
		if (actor_count[a] < 0) return fail(SGR_EINVAL, "%s: actor %d has %d rows", fn, a, actor_count[a]);
		if (class_label[a] < 0 || class_label[a] >= K) return fail(SGR_EINVAL, "%s: class label %d of actor %d is outside [0, %d)", fn, class_label[a], a, K);
		starts[a] = (int32_t)at;
		at += actor_count[a];
		if (at > 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "%s: composed row count exceeds 2^31-1", fn);
	}
	starts[n_act] = (int32_t)at;
	return SGR_OK;
}

int sgr_compose_semantics_forward(int32_t K, int32_t mode, int32_t n_bg, const float *bg_semantic, int32_t n_act, const int32_t *actor_count,
                                  const int32_t *class_label, const float *const *actor_semantic, float *semantics, void *stream) {
	const char *fn = "sgr_compose_semantics_forward";
	std::vector<int32_t> starts;
	if (int rc = semantics_check(fn, K, mode, n_bg, n_act, actor_count, class_label, starts)) return rc;
	if (starts[n_act] == 0) return SGR_OK;
	if (!semantics || (n_bg > 0 && !bg_semantic)) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	for (int32_t a = 0; a < n_act; a++)
		if (actor_count[a] > 0 && (!actor_semantic || !actor_semantic[a])) return fail(SGR_EINVAL, "%s: NULL semantic of actor %d", fn, a);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_compose_semantics_fwd(n_bg, K, mode, bg_semantic, n_act, starts.data(), class_label, actor_semantic, semantics, st),
	        "compose_semantics_fwd");
	return SGR_OK;
}

int sgr_compose_semantics_backward(int32_t K, int32_t mode, int32_t n_bg, int32_t n_act, const int32_t *actor_count, const int32_t *class_label,
                                   const float *semantics, const float *dL_dsemantics, float *dL_dbg, float *const *dL_dactor_semantic,
                                   void *stream) {
	const char *fn = "sgr_compose_semantics_backward";
	std::vector<int32_t> starts;
	if (int rc = semantics_check(fn, K, mode, n_bg, n_act, actor_count, class_label, starts)) return rc;
	if (starts[n_act] == 0) return SGR_OK;
	if (!semantics || !dL_dsemantics) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (dL_dactor_semantic)
		for (int32_t a = 0; a < n_act; a++)
			if (actor_count[a] > 0 && !dL_dactor_semantic[a]) return fail(SGR_EINVAL, "%s: NULL gradient of actor %d", fn, a);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_compose_semantics_bwd(n_bg, K, mode, semantics, dL_dsemantics, dL_dbg, n_act, starts.data(), class_label, dL_dactor_semantic, st),
	        "compose_semantics_bwd");
	return SGR_OK;
}

static int finish_check(const char *fn, int32_t S, int32_t H, int32_t W, int32_t normal_channels, int32_t mode) {
	if (S < 1 || H <= 0 || W <= 0) return fail(SGR_EINVAL, "%s: bad sizes S=%d H=%d W=%d", fn, S, H, W);
	if (normal_channels != 0 && normal_channels != 3) return fail(SGR_EINVAL, "%s: normal_channels must be 0 or 3, got %d", fn, normal_channels);
	if (normal_channels > S) return fail(SGR_EINVAL, "%s: %d normal channels but S = %d", fn, normal_channels, S);
	if (mode != SGR_SEMANTIC_LOGITS && mode != SGR_SEMANTIC_PROBABILITIES) return fail(SGR_EINVAL, "%s: unknown semantic mode %d", fn, mode);
	return SGR_OK;
}

int sgr_finish_features_forward(int32_t S, int32_t H, int32_t W, int32_t normal_channels, int32_t mode, const float *rendered, float *normals,
                                float *semantic, void *stream) {
	const char *fn = "sgr_finish_features_forward";
	if (int rc = finish_check(fn, S, H, W, normal_channels, mode)) return rc;
	if (!rendered || (normal_channels > 0 && !normals) || (S > normal_channels && !semantic)) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_finish_features_fwd(S, H, W, normal_channels, mode, rendered, normals, semantic, st), "finish_features_fwd");
	return SGR_OK;
}

int sgr_finish_features_backward(int32_t S, int32_t H, int32_t W, int32_t normal_channels, int32_t mode, const float *rendered,
                                 const float *dL_dnormals, const float *dL_dsemantic, float *dL_drendered, void *stream) {
	const char *fn = "sgr_finish_features_backward";
	if (int rc = finish_check(fn, S, H, W, normal_channels, mode)) return rc;
	if (!rendered || !dL_drendered) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_finish_features_bwd(S, H, W, normal_channels, mode, rendered, dL_dnormals, dL_dsemantic, dL_drendered, st), "finish_features_bwd");
	return SGR_OK;
}

size_t sgr_image_loss_scratch_bytes(int32_t C, int32_t H, int32_t W) { return (C > 0 && H > 0 && W > 0) ? image_loss_scratch_bytes(C, H, W) : 0; }

int sgr_image_loss(int32_t C, int32_t H, int32_t W, const float *image, const float *gt, const uint8_t *mask, float w_l1, float w_ssim,
                   float *dL_dimage, float *scalars, void *scratch, size_t scratch_bytes, void *stream) {
	if (C <= 0 || H <= 0 || W <= 0) return fail(SGR_EINVAL, "bad image size C=%d H=%d W=%d", C, H, W);
	if (!image || !gt || !scalars) return fail(SGR_EINVAL, "NULL pointer passed to sgr_image_loss");
	if (!scratch || scratch_bytes < image_loss_scratch_bytes(C, H, W))
		return fail(SGR_ENOMEM, "image loss scratch too small: %zu < %zu", scratch_bytes, image_loss_scratch_bytes(C, H, W));
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_image_loss(C, H, W, image, gt, mask, w_l1, w_ssim, dL_dimage, scalars, scratch, st), "image_loss");
	return SGR_OK;
}

int sgr_sky_loss(int64_t N, const float *acc, const uint8_t *sky_mask, float weight, float *dL_dacc, float *scalars, void *scratch, void *stream) {
	if (N <= 0) return fail(SGR_EINVAL, "N must be positive");
	if (!acc || !sky_mask || !scalars || !scratch) return fail(SGR_EINVAL, "NULL pointer passed to sgr_sky_loss");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_sky_loss((size_t)N, acc, sky_mask, weight, dL_dacc, scalars, scratch, st), "sky_loss");
	return SGR_OK;
}

// replaces train.py:114-122 (clamp / where / entropy / mean on the objects-only render's acc)
int sgr_obj_acc_loss(int64_t N, const float *acc, const uint8_t *obj_bound, float weight, float *dL_dacc, float *scalars, void *scratch, void *stream) {
	if (N <= 0) return fail(SGR_EINVAL, "N must be positive");
	if (!acc || !obj_bound || !scalars || !scratch) return fail(SGR_EINVAL, "NULL pointer passed to sgr_obj_acc_loss");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_obj_acc_loss((size_t)N, acc, obj_bound, weight, dL_dacc, scalars, scratch, st), "obj_acc_loss");
	return SGR_OK;
}

// replaces train.py:124-132 (boolean index, torch.topk with a host-side k, mean) and its autograd replay
size_t sgr_lidar_depth_loss_scratch_bytes(int64_t N) { return (N > 0 && N < ((int64_t)1 << 31)) ? lidar_depth_loss_scratch_bytes((size_t)N) : 0; }

int sgr_lidar_depth_loss(int64_t N, const float *depth, const float *acc, const float *lidar_depth, const uint8_t *mask, double keep, float weight,
                         float *dL_ddepth, float *dL_dacc, float *scalars, void *scratch, size_t scratch_bytes, void *stream) {
	if (N <= 0 || N >= ((int64_t)1 << 31)) return fail(SGR_EINVAL, "N must be in [1, 2^31), got %lld", (long long)N);
	if (!(keep > 0.0 && keep <= 1.0)) return fail(SGR_EINVAL, "keep must be in (0, 1], got %g", keep);
	if (!depth || !acc || !lidar_depth || !scalars) return fail(SGR_EINVAL, "NULL pointer passed to sgr_lidar_depth_loss");
	if (!scratch || scratch_bytes < lidar_depth_loss_scratch_bytes((size_t)N))
		return fail(SGR_ENOMEM, "lidar depth loss scratch too small: %zu < %zu", scratch_bytes, lidar_depth_loss_scratch_bytes((size_t)N));
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_lidar_depth_loss((size_t)N, depth, acc, lidar_depth, mask, keep, weight, dL_ddepth, dL_dacc, scalars, scratch, st),
	        "lidar_depth_loss");
	return SGR_OK;
}

// ---- the losses on a tile-row band ----
static int loss_band(const char *fn, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, Band *band) {
	if (H <= 0 || W <= 0 || (int64_t)H * W >= ((int64_t)1 << 31)) return fail(SGR_EINVAL, "%s: bad image size H=%d W=%d", fn, H, W);
	const int rows = (H + 15) / 16;
	if (row_step <= 0 || row_begin < 0 || row_end > rows || row_begin > row_end)
		return fail(SGR_EINVAL, "%s: bad tile-row band [%d,%d) step %d for %d tile rows", fn, row_begin, row_end, row_step, rows);
	*band = Band{row_begin, row_end, row_step};
	return SGR_OK;
}

int64_t sgr_band_halo_rows(int32_t H, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t side) {
	Band band;
	if (loss_band("sgr_band_halo_rows", H, 1, row_begin, row_end, row_step, &band) != SGR_OK) return -1;
	if (side < SGR_HALO_SEND_UP || side > SGR_HALO_RECV_DOWN) return -1;
	return halo_rows(H, halo_strips(H, band, side));
}

static int halo_copy(const char *fn, bool pack, int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t side,
                     float *image, float *buffer, void *stream) {
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (C <= 0) return fail(SGR_EINVAL, "%s: bad channel count %d", fn, C);
	const bool ok = pack ? (side == SGR_HALO_SEND_UP || side == SGR_HALO_SEND_DOWN) : (side == SGR_HALO_RECV_UP || side == SGR_HALO_RECV_DOWN);
	if (!ok) return fail(SGR_EINVAL, "%s: side %d is not a %s side", fn, side, pack ? "send" : "receive");
	if (halo_rows(H, halo_strips(H, band, side)) > 0 && (!image || !buffer)) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_halo_copy(pack, C, H, W, band, side, image, buffer, st), fn);
	return SGR_OK;
}

int sgr_band_halo_pack(int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t side, const float *image,
                       float *buffer, void *stream) {
	return halo_copy("sgr_band_halo_pack", true, C, H, W, row_begin, row_end, row_step, side, const_cast<float *>(image), buffer, stream);
}

int sgr_band_halo_unpack(int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t side,
                         const float *buffer, float *image, void *stream) {
	return halo_copy("sgr_band_halo_unpack", false, C, H, W, row_begin, row_end, row_step, side, image, const_cast<float *>(buffer), stream);
}

static int band_image_loss_check(const char *fn, int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step,
                                 const float *image, const float *gt, const double *partials, void *scratch, size_t scratch_bytes, Band *band) {
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, band)) return rc;
	if (C <= 0) return fail(SGR_EINVAL, "%s: bad channel count %d", fn, C);
	if (!image || !gt || !partials) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (!scratch || scratch_bytes < image_loss_scratch_bytes(C, H, W))
		return fail(SGR_ENOMEM, "%s: scratch too small: %zu < %zu", fn, scratch_bytes, image_loss_scratch_bytes(C, H, W));
	return SGR_OK;
}

int sgr_band_image_loss_stats(int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *image,
                              const float *gt, const uint8_t *mask, double *partials, void *scratch, size_t scratch_bytes, void *stream) {
	Band band;
	if (int rc = band_image_loss_check("sgr_band_image_loss_stats", C, H, W, row_begin, row_end, row_step, image, gt, partials, scratch, scratch_bytes,
	                                   &band))
		return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_image_loss_stats(C, H, W, band, image, gt, mask, partials, scratch, st), "band_image_loss_stats");
	return SGR_OK;
}

int sgr_band_image_loss_grad(int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *image,
                             const float *gt, const uint8_t *mask, float w_l1, float w_ssim, const double *partials, float *dL_dimage,
                             float *scalars, void *scratch, size_t scratch_bytes, void *stream) {
	Band band;
	if (int rc = band_image_loss_check("sgr_band_image_loss_grad", C, H, W, row_begin, row_end, row_step, image, gt, partials, scratch, scratch_bytes,
	                                   &band))
		return rc;
	if (!scalars) return fail(SGR_EINVAL, "NULL pointer passed to sgr_band_image_loss_grad");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_image_loss_grad(C, H, W, band, image, gt, mask, partials, w_l1, w_ssim, dL_dimage, scalars, scratch, st), "band_image_loss_grad");
	return SGR_OK;
}

static int band_acc_loss(const char *fn, int form, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *acc,
                         const uint8_t *flag, float weight, float *dL_dacc, double *partial, void *stream) {
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (!acc || !flag || !partial) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_acc_loss_band(form, H, W, band, acc, flag, weight, dL_dacc, partial, st), fn);
	return SGR_OK;
}

int sgr_band_sky_loss(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *acc, const uint8_t *sky_mask,
                      float weight, float *dL_dacc, double *partial, void *stream) {
	return band_acc_loss("sgr_band_sky_loss", 0, H, W, row_begin, row_end, row_step, acc, sky_mask, weight, dL_dacc, partial, stream);
}

int sgr_band_obj_acc_loss(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *acc, const uint8_t *obj_bound,
                          float weight, float *dL_dacc, double *partial, void *stream) {
	return band_acc_loss("sgr_band_obj_acc_loss", 1, H, W, row_begin, row_end, row_step, acc, obj_bound, weight, dL_dacc, partial, stream);
}

int sgr_band_acc_loss_value(int64_t N, float weight, const double *sum, float *scalars, void *stream) {
	if (N <= 0) return fail(SGR_EINVAL, "N must be positive");
	if (!sum || !scalars) return fail(SGR_EINVAL, "NULL pointer passed to sgr_band_acc_loss_value");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_acc_loss_value((size_t)N, weight, sum, scalars, st), "band_acc_loss_value");
	return SGR_OK;
}

size_t sgr_band_lidar_scratch_bytes(int32_t H, int32_t W) {
	return (H > 0 && W > 0 && (int64_t)H * W < ((int64_t)1 << 31)) ? lidar_band_scratch_bytes(H, W) : 0;
}

static int band_lidar_check(const char *fn, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const void *state,
                            void *scratch, size_t scratch_bytes, Band *band) {
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, band)) return rc;
	if (!state) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (!scratch || scratch_bytes < lidar_band_scratch_bytes(H, W))
		return fail(SGR_ENOMEM, "%s: scratch too small: %zu < %zu", fn, scratch_bytes, lidar_band_scratch_bytes(H, W));
	return SGR_OK;
}

int sgr_band_lidar_keys(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *depth, const float *acc,
                        const float *lidar_depth, const uint8_t *mask, SgrLidarState *state, void *scratch, size_t scratch_bytes, void *stream) {
	const char *fn = "sgr_band_lidar_keys";
	Band band;
	if (int rc = band_lidar_check(fn, H, W, row_begin, row_end, row_step, state, scratch, scratch_bytes, &band)) return rc;
	if (!depth || !acc || !lidar_depth) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_lidar_band_keys(H, W, band, depth, acc, lidar_depth, mask, state, scratch, st), fn);
	return SGR_OK;
}

int sgr_band_lidar_select(int32_t level, double keep, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step,
                          SgrLidarState *state, double *sums, void *scratch, size_t scratch_bytes, void *stream) {
	const char *fn = "sgr_band_lidar_select";
	Band band;
	if (int rc = band_lidar_check(fn, H, W, row_begin, row_end, row_step, state, scratch, scratch_bytes, &band)) return rc;
	if (level < 1 || level > 3) return fail(SGR_EINVAL, "%s: level must be 1, 2 or 3, got %d", fn, level);
	if (!(keep > 0.0 && keep <= 1.0)) return fail(SGR_EINVAL, "keep must be in (0, 1], got %g", keep);
	if (level == 3 && !sums) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_lidar_band_select(level, keep, H, W, band, state, sums, scratch, st), fn);
	return SGR_OK;
}

int sgr_band_lidar_grad(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *depth, const float *acc,
                        const float *lidar_depth, float weight, const SgrLidarState *state, const double *sums, float *dL_ddepth,
                        float *dL_dacc, float *scalars, void *scratch, size_t scratch_bytes, void *stream) {
	const char *fn = "sgr_band_lidar_grad";
	Band band;
	if (int rc = band_lidar_check(fn, H, W, row_begin, row_end, row_step, state, scratch, scratch_bytes, &band)) return rc;
	if (!depth || !acc || !lidar_depth || !sums || !scalars) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_lidar_band_grad(H, W, band, depth, acc, lidar_depth, weight, state, sums, dL_ddepth, dL_dacc, scalars, scratch, st), fn);
	return SGR_OK;
}

// ---- the band losses' exchanges over peer memory ----
size_t sgr_band_peer_bytes(int32_t C, int32_t H, int32_t W) {
	if (C <= 0 || H <= 0 || W <= 0 || (int64_t)H * W >= ((int64_t)1 << 31)) return 0;
	return band_peer_bytes(C, H, W);
}

// the peer table of the loss sections: world, rank and barrier pads, and every rank's section of at least `need` bytes
static int loss_peers(const char *fn, const SgrPeers *peers, size_t need, PeerTable &pt, LossPeers &lp) {
	if (!peers) return fail(SGR_EINVAL, "%s: peers is NULL", fn);
	if (peers->world < 1 || peers->world > SGR_MAX_PEERS || peers->rank < 0 || peers->rank >= peers->world)
		return fail(SGR_EINVAL, "%s: bad peer table: world=%d rank=%d (at most %d ranks)", fn, peers->world, peers->rank, SGR_MAX_PEERS);
	pt.world = lp.world = peers->world;
	pt.rank = peers->rank;
	for (int p = 0; p < peers->world; p++) {
		if (!peers->loss[p]) return fail(SGR_EINVAL, "%s: peer table entry %d has no loss section", fn, p);
		if (peers->world > 1 && !peers->flags[p]) return fail(SGR_EINVAL, "%s: peer table entry %d has no barrier pad", fn, p);
		lp.sec[p] = reinterpret_cast<char *>(peers->loss[p]);
		pt.flags[p] = peers->flags[p];
	}
	if (peers->loss_bytes < need) return fail(SGR_ENOMEM, "%s: the loss sections hold %zu bytes, %zu needed", fn, peers->loss_bytes, need);
	return SGR_OK;
}

int sgr_band_halo_exchange_peers(const SgrPeers *peers, int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step,
                                 const float *image, float *out, void *stream) {
	const char *fn = "sgr_band_halo_exchange_peers";
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (C <= 0) return fail(SGR_EINVAL, "%s: bad channel count %d", fn, C);
	if (!image || !out) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	PeerTable pt = {};
	LossPeers lp = {};
	if (int rc = loss_peers(fn, peers, band_peer_bytes(C, H, W), pt, lp)) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_band_halo_exchange(pt, lp, C, H, W, band, image, out, st), fn);
	return SGR_OK;
}

int sgr_band_peer_sum(const SgrPeers *peers, int32_t type, int64_t count, const void *local, void *out, void *stream) {
	const char *fn = "sgr_band_peer_sum";
	if (type != SGR_PEER_SUM_INT32 && type != SGR_PEER_SUM_FLOAT64) return fail(SGR_EINVAL, "%s: unknown element type %d", fn, type);
	if (count < 0) return fail(SGR_EINVAL, "%s: negative count %lld", fn, (long long)count);
	if (count > 0 && (!local || !out)) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	const size_t elem = type == SGR_PEER_SUM_INT32 ? sizeof(int32_t) : sizeof(double);
	PeerTable pt = {};
	LossPeers lp = {};
	if (int rc = loss_peers(fn, peers, (size_t)count * elem, pt, lp)) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_band_peer_sum(pt, lp, type == SGR_PEER_SUM_FLOAT64, count, local, out, st), fn);
	return SGR_OK;
}

// ---- the sky composite and the colour correction on a tile-row band ----
int sgr_band_sky_composite_forward(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t R, int32_t mode, float fill,
                                   const float *rgb, const float *acc, const uint8_t *sky_mask, const float *cube_map, const float *K,
                                   const float *w2c, const float *jitter_x, const float *jitter_y, float *rgb_out, void *stream) {
	const char *fn = "sgr_band_sky_composite_forward";
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (int rc = sky_check(fn, H, W, R, mode, sky_mask)) return rc;
	if (!rgb || !acc || !cube_map || !K || !w2c || !rgb_out) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (!jitter_x != !jitter_y) return fail(SGR_EINVAL, "%s: give both jitters or neither", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_sky_composite_fwd(H, W, band, R, mode, fill, rgb, acc, sky_mask, cube_map, K, w2c, jitter_x, jitter_y, rgb_out, st), fn);
	return SGR_OK;
}

int sgr_band_sky_composite_backward(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t R, int32_t mode, float fill,
                                    const float *acc, const uint8_t *sky_mask, const float *cube_map, const float *K, const float *w2c,
                                    const float *jitter_x, const float *jitter_y, const float *dL_dout, float *dL_dacc, float *dL_dcube,
                                    void *stream) {
	const char *fn = "sgr_band_sky_composite_backward";
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (int rc = sky_check(fn, H, W, R, mode, sky_mask)) return rc;
	if (!acc || !cube_map || !K || !w2c || !dL_dout) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (!jitter_x != !jitter_y) return fail(SGR_EINVAL, "%s: give both jitters or neither", fn);
	if (!dL_dacc && !dL_dcube) return SGR_OK;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_sky_composite_bwd(H, W, band, R, mode, fill, acc, sky_mask, cube_map, K, w2c, jitter_x, jitter_y, dL_dout, dL_dacc, dL_dcube, st),
	        fn);
	return SGR_OK;
}

int64_t sgr_sky_grad_blocks(int32_t R) { return (R > 0 && R <= 16384) ? sky_block_count(R) : 0; }
size_t sgr_sky_peer_bytes(int32_t R) { return (R > 0 && R <= 16384) ? sky_peer_bytes(R) : 0; }

int sgr_sky_cube_to_latlong(int32_t R, const float *cube_map, int32_t H, int32_t W, float *latlong, uint8_t *latlong_u8, void *stream) {
	const char *fn = "sgr_sky_cube_to_latlong";
	// one thread per pixel in an int grid of 256-thread blocks (sky.cu's kSkyThreads): H W <= (2^31 - 1) 256
	if (R <= 0 || R > 16384 || H <= 0 || W <= 0 || (int64_t)H * W > (int64_t)0x7fffffff * 256)
		return fail(SGR_EINVAL, "%s: bad sizes R=%d H=%d W=%d", fn, R, H, W);
	if (!cube_map || (!latlong && !latlong_u8)) return fail(SGR_EINVAL, "%s: cube_map and at least one output are required", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_sky_cube_to_latlong(R, cube_map, H, W, latlong, latlong_u8, st), fn);
	return SGR_OK;
}

static int sky_backward_marking(const char *fn, bool clear_map, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step,
                                int32_t R, int32_t mode, float fill, const float *acc, const uint8_t *sky_mask, const float *cube_map,
                                const float *K, const float *w2c, const float *jitter_x, const float *jitter_y, const float *dL_dout,
                                float *dL_dacc, float *dL_dcube, uint8_t *block_map, void *stream) {
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (int rc = sky_check(fn, H, W, R, mode, sky_mask)) return rc;
	if (!acc || !cube_map || !K || !w2c || !dL_dout || !dL_dcube || !block_map) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (!jitter_x != !jitter_y) return fail(SGR_EINVAL, "%s: give both jitters or neither", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_sky_composite_bwd(H, W, band, R, mode, fill, acc, sky_mask, cube_map, K, w2c, jitter_x, jitter_y, dL_dout, dL_dacc, dL_dcube, st,
	                                 block_map, clear_map),
	        fn);
	return SGR_OK;
}

int sgr_band_sky_composite_backward_marked(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t R, int32_t mode,
                                           float fill, const float *acc, const uint8_t *sky_mask, const float *cube_map, const float *K,
                                           const float *w2c, const float *jitter_x, const float *jitter_y, const float *dL_dout, float *dL_dacc,
                                           float *dL_dcube, uint8_t *block_map, void *stream) {
	return sky_backward_marking("sgr_band_sky_composite_backward_marked", true, H, W, row_begin, row_end, row_step, R, mode, fill, acc, sky_mask,
	                            cube_map, K, w2c, jitter_x, jitter_y, dL_dout, dL_dacc, dL_dcube, block_map, stream);
}

int sgr_band_sky_composite_backward_or_marks(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t R, int32_t mode,
                                             float fill, const float *acc, const uint8_t *sky_mask, const float *cube_map, const float *K,
                                             const float *w2c, const float *jitter_x, const float *jitter_y, const float *dL_dout, float *dL_dacc,
                                             float *dL_dcube, uint8_t *block_map, void *stream) {
	return sky_backward_marking("sgr_band_sky_composite_backward_or_marks", false, H, W, row_begin, row_end, row_step, R, mode, fill, acc,
	                            sky_mask, cube_map, K, w2c, jitter_x, jitter_y, dL_dout, dL_dacc, dL_dcube, block_map, stream);
}

static int sky_peer_sum(const char *fn, const SgrPeers *peers, const SgrSkyPeers *sky_peers, int32_t R, const uint8_t *block_map, float *dL_dcube,
                        uint8_t *union_map, void *stream) {
	if (!peers) return fail(SGR_EINVAL, "%s: peers is NULL", fn);
	if (!sky_peers) return fail(SGR_EINVAL, "%s: sky_peers is NULL", fn);
	if (peers->world < 1 || peers->world > SGR_MAX_PEERS || peers->rank < 0 || peers->rank >= peers->world)
		return fail(SGR_EINVAL, "%s: bad peer table: world=%d rank=%d (at most %d ranks)", fn, peers->world, peers->rank, SGR_MAX_PEERS);
	if (R <= 0 || R > 16384) return fail(SGR_EINVAL, "%s: bad sizes R=%d", fn, R);
	if (!block_map || !dL_dcube) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (int rc = check_aligned16("dL_dcube", dL_dcube)) return rc;
	PeerTable pt = {};
	SkyPeers sp = {};
	pt.world = peers->world;
	pt.rank = peers->rank;
	for (int p = 0; p < peers->world; p++) {
		if (!sky_peers->sec[p]) return fail(SGR_EINVAL, "%s: sky section table entry %d is NULL", fn, p);
		if (int rc = check_aligned16("a sky section", sky_peers->sec[p])) return rc;
		if (peers->world > 1 && !peers->flags[p]) return fail(SGR_EINVAL, "%s: peer table entry %d has no barrier pad", fn, p);
		sp.sec[p] = reinterpret_cast<char *>(sky_peers->sec[p]);
		pt.flags[p] = peers->flags[p];
	}
	if (sky_peers->bytes < sky_peer_bytes(R))
		return fail(SGR_ENOMEM, "%s: the sky sections hold %zu bytes, %zu needed", fn, sky_peers->bytes, sky_peer_bytes(R));
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_sky_grad_peer_sum(pt, sp, R, block_map, dL_dcube, st, union_map), fn);
	return SGR_OK;
}

int sgr_sky_grad_peer_sum(const SgrPeers *peers, const SgrSkyPeers *sky_peers, int32_t R, const uint8_t *block_map, float *dL_dcube, void *stream) {
	return sky_peer_sum("sgr_sky_grad_peer_sum", peers, sky_peers, R, block_map, dL_dcube, nullptr, stream);
}

int sgr_sky_grad_peer_sum_union(const SgrPeers *peers, const SgrSkyPeers *sky_peers, int32_t R, const uint8_t *block_map, float *dL_dcube,
                                uint8_t *union_map, void *stream) {
	const char *fn = "sgr_sky_grad_peer_sum_union";
	if (!union_map) return fail(SGR_EINVAL, "%s: union_map is NULL", fn);
	if (union_map == block_map) return fail(SGR_EINVAL, "%s: union_map must not be block_map", fn);
	return sky_peer_sum(fn, peers, sky_peers, R, block_map, dL_dcube, union_map, stream);
}

int sgr_band_color_correct_forward(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *image, const float *affine,
                                   float *out, void *stream) {
	const char *fn = "sgr_band_color_correct_forward";
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (!image || !affine || !out) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_color_correct_fwd(H, W, band, image, affine, out, st), fn);
	return SGR_OK;
}

size_t sgr_band_color_correct_scratch_bytes(int32_t H, int32_t W) {
	return (H > 0 && W > 0 && (int64_t)H * W < ((int64_t)1 << 31)) ? color_correct_band_scratch_bytes(H, W) : 0;
}

int sgr_band_color_correct_backward(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *image, const float *affine,
                                    const float *dL_dout, float *dL_dimage, double *partials, void *scratch, size_t scratch_bytes, void *stream) {
	const char *fn = "sgr_band_color_correct_backward";
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (!image || !affine || !dL_dout || !partials) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (!scratch || scratch_bytes < color_correct_band_scratch_bytes(H, W))
		return fail(SGR_ENOMEM, "%s: scratch too small: %zu < %zu", fn, scratch_bytes, color_correct_band_scratch_bytes(H, W));
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_color_correct_bwd(H, W, band, image, affine, dL_dout, dL_dimage, partials, scratch, st), fn);
	return SGR_OK;
}

int sgr_band_color_correct_affine_grad(const double *sums, float *dL_daffine, void *stream) {
	if (!sums || !dL_daffine) return fail(SGR_EINVAL, "NULL pointer passed to sgr_band_color_correct_affine_grad");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_color_correct_affine_grad(sums, dL_daffine, st), "band_color_correct_affine_grad");
	return SGR_OK;
}

// ---- the feature maps' finishing on a tile-row band ----
int sgr_band_finish_features_forward(int32_t S, int32_t H, int32_t W, int32_t normal_channels, int32_t mode, int32_t row_begin, int32_t row_end,
                                     int32_t row_step, const float *rendered, float *normals, float *semantic, void *stream) {
	const char *fn = "sgr_band_finish_features_forward";
	if (int rc = finish_check(fn, S, H, W, normal_channels, mode)) return rc;
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (!rendered || (normal_channels > 0 && !normals) || (S > normal_channels && !semantic)) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_finish_features_fwd(S, H, W, band, normal_channels, mode, rendered, normals, semantic, st), fn);
	return SGR_OK;
}

int sgr_band_finish_features_backward(int32_t S, int32_t H, int32_t W, int32_t normal_channels, int32_t mode, int32_t row_begin, int32_t row_end,
                                      int32_t row_step, const float *rendered, const float *dL_dnormals, const float *dL_dsemantic,
                                      float *dL_drendered, void *stream) {
	const char *fn = "sgr_band_finish_features_backward";
	if (int rc = finish_check(fn, S, H, W, normal_channels, mode)) return rc;
	Band band;
	if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) return rc;
	if (!rendered || !dL_drendered) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_finish_features_bwd(S, H, W, band, normal_channels, mode, rendered, dL_dnormals, dL_dsemantic, dL_drendered, st), fn);
	return SGR_OK;
}

// ---- evaluation metrics ----
static bool eval_sizes_ok(int32_t V, int32_t C, int32_t H, int32_t W) {
	if (V <= 0 || C <= 0 || H <= 0 || W <= 0 || (int64_t)H * W >= ((int64_t)1 << 31)) return false;
	// one grid z per (view, channel), one grid y per tile row; the tile partials of a view are counted in 32 bits
	const int64_t rows = ((int64_t)H + 15) / 16, cols = ((int64_t)W + 15) / 16;
	return (int64_t)V * C <= 65535 && rows <= 65535 && (int64_t)C * rows * cols < ((int64_t)1 << 31);
}

size_t sgr_eval_metrics_scratch_bytes(int32_t V, int32_t C, int32_t H, int32_t W) {
	return eval_sizes_ok(V, C, H, W) ? eval_metrics_scratch_bytes(V, C, H, W) : 0;
}

static int eval_accumulate(const char *fn, int32_t V, int32_t C, int32_t H, int32_t W, bool whole, int32_t row_begin, int32_t row_end,
                           int32_t row_step, int32_t flags, const float *image, const float *gt, const uint8_t *mask, SgrEvalSums *sums,
                           void *scratch, size_t scratch_bytes, void *stream) {
	if (!eval_sizes_ok(V, C, H, W)) return fail(SGR_EINVAL, "%s: bad sizes V=%d C=%d H=%d W=%d", fn, V, C, H, W);
	Band band;
	if (whole) {
		band = Band{0, (int)(((int64_t)H + 15) / 16), 1};
	} else if (int rc = loss_band(fn, H, W, row_begin, row_end, row_step, &band)) {
		return rc;
	}
	const int32_t known = SGR_EVAL_CLAMP | SGR_EVAL_QUANT8 | SGR_EVAL_SSIM_MASKED | SGR_EVAL_NO_SSIM;
	if ((flags & ~known) != 0 || ((flags & SGR_EVAL_QUANT8) && !(flags & SGR_EVAL_CLAMP)))
		return fail(SGR_EINVAL, "%s: bad flags %d (SGR_EVAL_QUANT8 needs SGR_EVAL_CLAMP)", fn, flags);
	if (!image || !gt || !sums) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (!scratch || scratch_bytes < eval_metrics_scratch_bytes(V, C, H, W))
		return fail(SGR_ENOMEM, "%s: scratch too small: %zu < %zu", fn, scratch_bytes, eval_metrics_scratch_bytes(V, C, H, W));
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_eval_metrics(V, C, H, W, band, flags, image, gt, mask, sums, scratch, st), fn);
	return SGR_OK;
}

int sgr_band_eval_metrics_accumulate(int32_t V, int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step,
                                     int32_t flags, const float *image, const float *gt, const uint8_t *mask, SgrEvalSums *sums,
                                     void *scratch, size_t scratch_bytes, void *stream) {
	return eval_accumulate("sgr_band_eval_metrics_accumulate", V, C, H, W, false, row_begin, row_end, row_step, flags, image, gt, mask, sums,
	                       scratch, scratch_bytes, stream);
}

int sgr_eval_metrics_accumulate(int32_t V, int32_t C, int32_t H, int32_t W, int32_t flags, const float *image, const float *gt,
                                const uint8_t *mask, SgrEvalSums *sums, void *scratch, size_t scratch_bytes, void *stream) {
	return eval_accumulate("sgr_eval_metrics_accumulate", V, C, H, W, true, 0, 0, 1, flags, image, gt, mask, sums, scratch, scratch_bytes, stream);
}

int sgr_eval_metrics_finish(int32_t V, const SgrEvalSums *sums, float *out, void *stream) {
	if (V <= 0) return fail(SGR_EINVAL, "sgr_eval_metrics_finish: V must be positive, got %d", V);
	if (!sums || !out) return fail(SGR_EINVAL, "NULL pointer passed to sgr_eval_metrics_finish");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_eval_metrics_finish(V, sums, out, st), "eval_metrics_finish");
	return SGR_OK;
}

int sgr_densify_stats(const SgrStatSegment *segments, int32_t num_segments, const int32_t *radii, const float *means2D_grad, void *stream) {
	if (!segments || num_segments <= 0) return fail(SGR_EINVAL, "segment table is empty");
	int64_t at = 0;
	for (int k = 0; k < num_segments; k++) {
		const SgrStatSegment &s = segments[k];
		if (s.start != at || s.count < 0) return fail(SGR_EINVAL, "segment %d: start %d (expected %lld), count %d", k, s.start, (long long)at, s.count);
		if (s.count > 0 && (!s.max_radii2D || !s.xyz_gradient_accum || !s.denom)) return fail(SGR_EINVAL, "segment %d has a NULL statistics array", k);
		at += s.count;
	}
	if (at == 0) return SGR_OK;
	if (!radii || !means2D_grad) return fail(SGR_EINVAL, "NULL pointer passed to sgr_densify_stats");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_densify_stats(segments, num_segments, radii, means2D_grad, st), "densify_stats");
	return SGR_OK;
}

int sgr_adam_step(const SgrAdamTensor *tensors, int32_t num_tensors, double beta1, double beta2, double eps, void *stream) {
	if (num_tensors < 0 || (num_tensors > 0 && !tensors)) return fail(SGR_EINVAL, "bad tensor table");
	for (int k = 0; k < num_tensors; k++) {
		const SgrAdamTensor &a = tensors[k];
		if (a.numel < 0 || a.step < 1) return fail(SGR_EINVAL, "tensor %d: numel %lld, step %d (step counts from 1)", k, (long long)a.numel, a.step);
		if (a.numel > 0 && (!a.param || !a.grad || !a.exp_avg || !a.exp_avg_sq)) return fail(SGR_EINVAL, "tensor %d has a NULL pointer", k);
	}
	if (!(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0)) return fail(SGR_EINVAL, "betas must lie in [0, 1)");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_adam(tensors, num_tensors, beta1, beta2, eps, st), "adam");
	return SGR_OK;
}

int sgr_cube_sparse_adam_step(int32_t R, const SgrAdamTensor *cube, uint8_t *block_map, double beta1, double beta2, double eps, void *stream) {
	const char *fn = "sgr_cube_sparse_adam_step";
	if (R <= 0 || R > 16384) return fail(SGR_EINVAL, "%s: bad sizes R=%d", fn, R);
	if (!cube || !block_map) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (!cube->param || !cube->grad || !cube->exp_avg || !cube->exp_avg_sq) return fail(SGR_EINVAL, "%s: the cube has a NULL pointer", fn);
	if (cube->numel != (int64_t)18 * R * R)
		return fail(SGR_EINVAL, "%s: numel %lld is not 6 R^2 3 = %lld for R=%d", fn, (long long)cube->numel, (long long)18 * R * R, R);
	if (cube->step < 1) return fail(SGR_EINVAL, "%s: step %d (step counts from 1)", fn, cube->step);
	if (!std::isfinite(cube->lr)) return fail(SGR_EINVAL, "%s: non-finite lr", fn);
	if (!(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0)) return fail(SGR_EINVAL, "%s: betas must lie in [0, 1)", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_cube_sparse_adam(R, *cube, block_map, beta1, beta2, eps, st), fn);
	return SGR_OK;
}

// ---- densification ----
static const char *const kDensifyTensor[SGR_DENSIFY_TENSORS] = {"xyz", "features_dc", "features_rest", "opacity", "scaling", "rotation", "semantic"};

static int densify_width(const SgrDensifySegment &s, int a) {
	const int fixed[SGR_DENSIFY_TENSORS] = {3, s.dc_width, s.rest_width, 1, 3, 4, s.semantic_width};
	return fixed[a];
}

// validates the input table; *P receives the total Gaussian count
static int check_densify_segments(const SgrDensifySegment *segments, int32_t num_segments, int64_t *P) {
	if (!segments || num_segments <= 0) return fail(SGR_EINVAL, "segment table is empty");
	int64_t at = 0;
	for (int k = 0; k < num_segments; k++) {
		const SgrDensifySegment &s = segments[k];
		if (s.kind != SGR_DENSIFY_BACKGROUND && s.kind != SGR_DENSIFY_ACTOR) return fail(SGR_EINVAL, "segment %d: unknown kind %d", k, s.kind);
		if (s.count < 0) return fail(SGR_EINVAL, "segment %d: count %d", k, s.count);
		if (s.dc_width <= 0 || s.rest_width < 0 || s.semantic_width < 0)
			return fail(SGR_EINVAL, "segment %d: bad row widths dc=%d rest=%d semantic=%d", k, s.dc_width, s.rest_width, s.semantic_width);
		if (s.grad_col != 0 && s.grad_col != 1) return fail(SGR_EINVAL, "segment %d: grad_col must be 0 or 1, got %d", k, s.grad_col);
		if (s.count > 0) {
			for (int a = 0; a < SGR_DENSIFY_TENSORS; a++) {
				const bool has = densify_width(s, a) > 0;
				if (has != (s.param[a] != nullptr))
					return fail(SGR_EINVAL, "segment %d: %s is %s", k, kDensifyTensor[a], has ? "NULL" : "given for a zero row width");
				if ((s.exp_avg[a] == nullptr) != (s.exp_avg_sq[a] == nullptr) || (!has && s.exp_avg[a]))
					return fail(SGR_EINVAL, "segment %d: %s needs both Adam moments or neither", k, kDensifyTensor[a]);
			}
			if (!s.max_radii2D || !s.xyz_gradient_accum || !s.denom) return fail(SGR_EINVAL, "segment %d has a NULL statistics array", k);
		}
		at += s.count;
	}
	if (at >= 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "%lld Gaussians in all exceed 2^31-2", (long long)at);
	*P = at;
	return SGR_OK;
}

size_t sgr_densify_scratch_bytes(int32_t num_segments, int64_t P) {
	return num_segments > 0 && P >= 0 ? densify_scratch_bytes(num_segments, (long long)P) : 0;
}

int sgr_densify_plan(const SgrDensifySegment *segments, int32_t num_segments, uint64_t seed, const float *draws, void *scratch,
                     size_t scratch_bytes, int64_t *result, void *stream) {
	int64_t P = 0;
	const int rc = check_densify_segments(segments, num_segments, &P);
	if (rc != SGR_OK) return rc;
	if (!result) return fail(SGR_EINVAL, "result is NULL");
	const size_t need = densify_scratch_bytes(num_segments, (long long)P);
	if (!scratch || scratch_bytes < need) return fail(SGR_ENOMEM, "densify scratch too small: %zu < %zu", scratch_bytes, need);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_densify_plan(segments, num_segments, (unsigned long long)seed, draws, scratch, reinterpret_cast<long long *>(result), st),
	        "densify_plan");
	return SGR_OK;
}

int sgr_densify_apply(const SgrDensifySegment *segments, const SgrDensifyOutput *outputs, int32_t num_segments, uint64_t seed,
                      const float *draws, void *scratch, size_t scratch_bytes, void *stream) {
	int64_t P = 0;
	const int rc = check_densify_segments(segments, num_segments, &P);
	if (rc != SGR_OK) return rc;
	if (!outputs) return fail(SGR_EINVAL, "output table is NULL");
	for (int k = 0; k < num_segments; k++) {
		const SgrDensifySegment &s = segments[k];
		const SgrDensifyOutput &o = outputs[k];
		if (o.count < 0) return fail(SGR_EINVAL, "output %d: count %d", k, o.count);
		if (o.count == 0) continue;
		for (int a = 0; a < SGR_DENSIFY_TENSORS; a++) {
			const bool has = densify_width(s, a) > 0;
			if (has != (o.param[a] != nullptr)) return fail(SGR_EINVAL, "output %d: %s is %s", k, kDensifyTensor[a], has ? "NULL" : "given for a zero row width");
			const bool moments = s.count > 0 && s.exp_avg[a] != nullptr;
			if (moments != (o.exp_avg[a] != nullptr) || moments != (o.exp_avg_sq[a] != nullptr))
				return fail(SGR_EINVAL, "output %d: the Adam moments of %s must be given exactly where the input has them", k, kDensifyTensor[a]);
		}
		if (!o.max_radii2D || !o.xyz_gradient_accum || !o.denom) return fail(SGR_EINVAL, "output %d has a NULL statistics array", k);
	}
	const size_t need = densify_scratch_bytes(num_segments, (long long)P);
	if (!scratch || scratch_bytes < need) return fail(SGR_ENOMEM, "densify scratch too small: %zu < %zu", scratch_bytes, need);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_densify_apply(segments, outputs, num_segments, (unsigned long long)seed, draws, scratch, st), "densify_apply");
	return SGR_OK;
}

int sgr_reset_opacity(const SgrDensifySegment *segments, int32_t num_segments, void *stream) {
	if (!segments || num_segments <= 0) return fail(SGR_EINVAL, "segment table is empty");
	int64_t at = 0;
	for (int k = 0; k < num_segments; k++) {
		const SgrDensifySegment &s = segments[k];
		if (s.count < 0) return fail(SGR_EINVAL, "segment %d: count %d", k, s.count);
		if (s.count > 0 && !s.param[3]) return fail(SGR_EINVAL, "segment %d: opacity is NULL", k);
		if ((s.exp_avg[3] == nullptr) != (s.exp_avg_sq[3] == nullptr)) return fail(SGR_EINVAL, "segment %d: opacity needs both Adam moments or neither", k);
		at += s.count;
	}
	if (at >= 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "%lld Gaussians in all exceed 2^31-2", (long long)at);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_reset_opacity(segments, num_segments, st), "reset_opacity");
	return SGR_OK;
}

// ---- rebalancing: the row format of include/sgr.h as (pointer, floats per row) per tensor, and the span tables of pack / splice ----
constexpr int kRebalanceTensors = 3 * SGR_DENSIFY_TENSORS + 3;

static int rebalance_format_ok(const SgrDensifySegment &s, int k) {
	if (s.count < 0 || s.dc_width <= 0 || s.rest_width < 0 || s.semantic_width < 0)
		return fail(SGR_EINVAL, "segment %d: bad count %d or row widths dc=%d rest=%d semantic=%d", k, s.count, s.dc_width, s.rest_width,
		            s.semantic_width);
	for (int a = 0; a < 32; a++)
		if (((s.moments >> a) & 1) && (a >= SGR_DENSIFY_TENSORS || densify_width(s, a) == 0))
			return fail(SGR_EINVAL, "segment %d: moment bit %d names no tensor with a nonzero width", k, a);
	return SGR_OK;
}

// fills ptr[] / width[] in the row format's order from the given pointer arrays; returns the number of tensors carried
static int rebalance_tensors(const SgrDensifySegment &s, float *const *param, float *const *m, float *const *v, float *mr, float *ga, float *dn,
                             float *ptr[kRebalanceTensors], int width[kRebalanceTensors]) {
	int n = 0;
	for (int a = 0; a < SGR_DENSIFY_TENSORS; a++)
		if (densify_width(s, a) > 0) { ptr[n] = param[a]; width[n++] = densify_width(s, a); }
	for (int j = 0; j < 2; j++)
		for (int a = 0; a < SGR_DENSIFY_TENSORS; a++)
			if ((s.moments >> a) & 1) { ptr[n] = (j ? v : m)[a]; width[n++] = densify_width(s, a); }
	ptr[n] = mr; width[n++] = 1;
	ptr[n] = ga; width[n++] = 2;
	ptr[n] = dn; width[n++] = 1;
	return n;
}

static int64_t rebalance_row_floats(const SgrDensifySegment &s) {
	float *ptr[kRebalanceTensors];
	int width[kRebalanceTensors];
	const int n = rebalance_tensors(s, s.param, s.exp_avg, s.exp_avg_sq, s.max_radii2D, s.xyz_gradient_accum, s.denom, ptr, width);
	int64_t f = 0;
	for (int t = 0; t < n; t++) f += width[t];
	return f;
}

// segments carrying rows must give every tensor of the format (and no moment the format does not carry)
static int check_rebalance_segments(const char *fn, const SgrDensifySegment *segments, int32_t num_segments) {
	if (!segments || num_segments <= 0) return fail(SGR_EINVAL, "%s: segment table is empty", fn);
	for (int k = 0; k < num_segments; k++) {
		const SgrDensifySegment &s = segments[k];
		int rc = rebalance_format_ok(s, k);
		if (rc) return rc;
		if (s.count == 0) continue;
		for (int a = 0; a < SGR_DENSIFY_TENSORS; a++) {
			const bool has = densify_width(s, a) > 0, mom = (s.moments >> a) & 1;
			if (has != (s.param[a] != nullptr)) return fail(SGR_EINVAL, "%s: segment %d: %s is %s", fn, k, kDensifyTensor[a], has ? "NULL" : "given for a zero row width");
			if (mom != (s.exp_avg[a] != nullptr) || mom != (s.exp_avg_sq[a] != nullptr))
				return fail(SGR_EINVAL, "%s: segment %d: the Adam moments of %s must be given exactly where its moment bit is set", fn, k, kDensifyTensor[a]);
		}
		if (!s.max_radii2D || !s.xyz_gradient_accum || !s.denom) return fail(SGR_EINVAL, "%s: segment %d has a NULL statistics array", fn, k);
	}
	return SGR_OK;
}

// checks the ranges against the segments and buffers and appends one span per tensor of each range with rows (pack: rows -> buffer;
// splice: buffer or old rows -> new rows of outs[k])
static int rebalance_spans(const char *fn, const SgrDensifySegment *segments, const SgrDensifyOutput *outs, int32_t num_segments,
                           const SgrRebalanceRange *ranges, int32_t num_ranges, float *const *buffers, const int64_t *buffer_floats,
                           int32_t num_buffers, std::vector<RebalanceSpan> &spans) {
	if (num_ranges < 0 || (num_ranges > 0 && !ranges)) return fail(SGR_EINVAL, "%s: bad range table", fn);
	if (num_buffers < 0 || (num_buffers > 0 && (!buffers || !buffer_floats))) return fail(SGR_EINVAL, "%s: bad buffer table", fn);
	std::vector<int64_t> used(num_buffers, 0);
	const bool splice = outs != nullptr;
	for (int i = 0; i < num_ranges; i++) {
		const SgrRebalanceRange &r = ranges[i];
		if (r.segment < 0 || r.segment >= num_segments) return fail(SGR_EINVAL, "%s: range %d names segment %d of %d", fn, i, r.segment, num_segments);
		if (r.buffer < (splice ? -1 : 0) || r.buffer >= num_buffers) return fail(SGR_EINVAL, "%s: range %d names buffer %d of %d", fn, i, r.buffer, num_buffers);
		const SgrDensifySegment &s = segments[r.segment];
		const bool from_old = !splice || r.buffer < 0;
		if (r.rows < 0 || (from_old && (r.src_row < 0 || (int64_t)r.src_row + r.rows > s.count)))
			return fail(SGR_EINVAL, "%s: range %d reads rows [%d, %lld) of segment %d, which has %d", fn, i, r.src_row, (long long)r.src_row + r.rows,
			            r.segment, s.count);
		if (splice && (r.dst_row < 0 || (int64_t)r.dst_row + r.rows > outs[r.segment].count))
			return fail(SGR_EINVAL, "%s: range %d writes rows [%d, %lld) of output %d, which has %d", fn, i, r.dst_row, (long long)r.dst_row + r.rows,
			            r.segment, outs[r.segment].count);
		const int64_t block = (int64_t)r.rows * rebalance_row_floats(s);
		int64_t at = 0;
		if (r.buffer >= 0) {
			at = used[r.buffer];
			used[r.buffer] += block;
			if (used[r.buffer] > buffer_floats[r.buffer])
				return fail(SGR_ENOMEM, "%s: buffer %d holds %lld floats, its blocks need %lld or more", fn, r.buffer, (long long)buffer_floats[r.buffer],
				            (long long)used[r.buffer]);
			if (!buffers[r.buffer] && block > 0) return fail(SGR_EINVAL, "%s: buffer %d is NULL", fn, r.buffer);
		}
		if (r.rows == 0) continue;
		float *src[kRebalanceTensors], *dst[kRebalanceTensors];
		int width[kRebalanceTensors];
		const int nt = rebalance_tensors(s, s.param, s.exp_avg, s.exp_avg_sq, s.max_radii2D, s.xyz_gradient_accum, s.denom, src, width);
		if (splice) {
			const SgrDensifyOutput &o = outs[r.segment];
			rebalance_tensors(s, o.param, o.exp_avg, o.exp_avg_sq, o.max_radii2D, o.xyz_gradient_accum, o.denom, dst, width);
		}
		float *buf = r.buffer >= 0 ? buffers[r.buffer] + at : nullptr;
		for (int t = 0; t < nt; t++) {
			const int64_t n = (int64_t)r.rows * width[t];
			float *old_rows = from_old ? src[t] + (int64_t)r.src_row * width[t] : nullptr;
			if (!splice) spans.push_back(RebalanceSpan{old_rows, buf, n});
			else spans.push_back(RebalanceSpan{from_old ? old_rows : buf, dst[t] + (int64_t)r.dst_row * width[t], n});
			if (buf) buf += n;
		}
	}
	return SGR_OK;
}

int64_t sgr_rebalance_row_floats(const SgrDensifySegment *segment) {
	if (!segment) {
		fail(SGR_EINVAL, "segment is NULL");
		return -1;
	}
	if (rebalance_format_ok(*segment, 0)) return -1;
	return rebalance_row_floats(*segment);
}

size_t sgr_rebalance_scratch_bytes(int32_t num_ranges) {
	return num_ranges >= 0 ? rebalance_scratch_bytes((long long)num_ranges * kRebalanceTensors) : 0;
}

static int rebalance_copy(const char *fn, const std::vector<RebalanceSpan> &spans, int32_t num_ranges, void *scratch, size_t scratch_bytes,
                          void *stream) {
	const size_t need = rebalance_scratch_bytes((long long)num_ranges * kRebalanceTensors);
	if (!spans.empty() && (!scratch || scratch_bytes < need)) return fail(SGR_ENOMEM, "%s: scratch too small: %zu < %zu", fn, scratch_bytes, need);
	if (rebalance_blocks(spans.data(), (int)spans.size()) > 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "%s: more than 2^31-1 blocks of floats to copy", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_rebalance_copy(spans.data(), (int)spans.size(), scratch, st), fn);
	return SGR_OK;
}

int sgr_rebalance_pack(const SgrDensifySegment *segments, int32_t num_segments, const SgrRebalanceRange *ranges, int32_t num_ranges,
                       float *const *buffers, const int64_t *buffer_floats, int32_t num_buffers, void *scratch, size_t scratch_bytes,
                       void *stream) {
	const char *fn = "sgr_rebalance_pack";
	int rc = check_rebalance_segments(fn, segments, num_segments);
	if (rc) return rc;
	std::vector<RebalanceSpan> spans;
	if ((rc = rebalance_spans(fn, segments, nullptr, num_segments, ranges, num_ranges, buffers, buffer_floats, num_buffers, spans))) return rc;
	return rebalance_copy(fn, spans, num_ranges, scratch, scratch_bytes, stream);
}

int sgr_rebalance_splice(const SgrDensifySegment *segments, const SgrDensifyOutput *outputs, int32_t num_segments, const SgrRebalanceRange *ranges,
                         int32_t num_ranges, const float *const *buffers, const int64_t *buffer_floats, int32_t num_buffers, void *scratch,
                         size_t scratch_bytes, void *stream) {
	const char *fn = "sgr_rebalance_splice";
	int rc = check_rebalance_segments(fn, segments, num_segments);
	if (rc) return rc;
	if (!outputs) return fail(SGR_EINVAL, "%s: output table is NULL", fn);
	for (int k = 0; k < num_segments; k++) {
		const SgrDensifySegment &s = segments[k];
		const SgrDensifyOutput &o = outputs[k];
		if (o.count < 0) return fail(SGR_EINVAL, "%s: output %d: count %d", fn, k, o.count);
		if (o.count == 0) continue;
		for (int a = 0; a < SGR_DENSIFY_TENSORS; a++) {
			const bool has = densify_width(s, a) > 0, mom = (s.moments >> a) & 1;
			if (has != (o.param[a] != nullptr)) return fail(SGR_EINVAL, "%s: output %d: %s is %s", fn, k, kDensifyTensor[a], has ? "NULL" : "given for a zero row width");
			if (mom != (o.exp_avg[a] != nullptr) || mom != (o.exp_avg_sq[a] != nullptr))
				return fail(SGR_EINVAL, "%s: output %d: the Adam moments of %s must be given exactly where its moment bit is set", fn, k, kDensifyTensor[a]);
		}
		if (!o.max_radii2D || !o.xyz_gradient_accum || !o.denom) return fail(SGR_EINVAL, "%s: output %d has a NULL statistics array", fn, k);
	}
	std::vector<RebalanceSpan> spans;
	if ((rc = rebalance_spans(fn, segments, outputs, num_segments, ranges, num_ranges, const_cast<float *const *>(buffers), buffer_floats, num_buffers,
	                          spans)))
		return rc;
	// every new row written exactly once: per segment, the ranges sorted by dst_row must tile [0, count)
	std::vector<std::pair<int64_t, int32_t>> cover;  // (segment << 32 | dst_row, rows)
	for (int i = 0; i < num_ranges; i++)
		if (ranges[i].rows > 0) cover.push_back({((int64_t)ranges[i].segment << 32) | (uint32_t)ranges[i].dst_row, ranges[i].rows});
	std::sort(cover.begin(), cover.end());
	size_t c = 0;
	for (int k = 0; k < num_segments; k++) {
		int64_t at = 0;
		for (; c < cover.size() && (cover[c].first >> 32) == k; c++) {
			if ((cover[c].first & 0xffffffffLL) != at) return fail(SGR_EINVAL, "%s: output %d: rows from %lld on are not written exactly once", fn, k, (long long)at);
			at += cover[c].second;
		}
		if (at != outputs[k].count) return fail(SGR_EINVAL, "%s: output %d: the ranges write %lld of its %d rows", fn, k, (long long)at, outputs[k].count);
	}
	return rebalance_copy(fn, spans, num_ranges, scratch, scratch_bytes, stream);
}

// the piece table of one side of sgr_peer_exchange_round: pieces checked against the staging regions, the empty ones dropped
static int peer_pieces(const char *fn, const char *side, const SgrPeers *peers, size_t staging_bytes, const SgrPeerPiece *pieces, int32_t num,
                       bool stage, PieceTable &t, long long &blocks) {
	t.n = 0;
	if (num < 0 || num > SGR_MAX_PEERS) return fail(SGR_EINVAL, "%s: %d %s pieces (at most %d)", fn, num, side, SGR_MAX_PEERS);
	if (num > 0 && !pieces) return fail(SGR_EINVAL, "%s: the %s pieces are NULL", fn, side);
	const long long cap = (long long)(staging_bytes / sizeof(float));
	for (int i = 0; i < num; i++) {
		const SgrPeerPiece &p = pieces[i];
		if (p.rank < 0 || p.rank >= peers->world || (stage && p.rank != peers->rank))
			return fail(SGR_EINVAL, "%s: %s piece %d names rank %d (this rank %d of %d)", fn, side, i, p.rank, peers->rank, peers->world);
		if (p.floats < 0 || p.offset < 0 || (p.offset & 3) || p.offset > cap - p.floats)
			return fail(SGR_EINVAL, "%s: %s piece %d: floats [%lld, +%lld) do not lie 16-byte aligned inside the %lld floats of a staging region", fn, side,
			            i, (long long)p.offset, (long long)p.floats, cap);
		if (p.floats == 0) continue;
		if (!p.local) return fail(SGR_EINVAL, "%s: %s piece %d has a NULL buffer", fn, side, i);
		if (int rc = check_aligned16("a piece's buffer", p.local)) return rc;
		float *region = reinterpret_cast<float *>(peers->records[p.rank]) + p.offset;
		t.src[t.n] = stage ? p.local : region;
		t.dst[t.n] = stage ? region : p.local;
		t.floats[t.n] = p.floats;
		blocks += peer_piece_blocks(p.floats);
		t.n++;
	}
	return SGR_OK;
}

int sgr_peer_exchange_round(const SgrPeers *peers, size_t staging_bytes, const SgrPeerPiece *stage, int32_t num_stage, const SgrPeerPiece *pull,
                            int32_t num_pull, void *stream) {
	const char *fn = "sgr_peer_exchange_round";
	if (!peers) return fail(SGR_EINVAL, "%s: peers is NULL", fn);
	if (peers->world < 1 || peers->world > SGR_MAX_PEERS || peers->rank < 0 || peers->rank >= peers->world)
		return fail(SGR_EINVAL, "%s: bad peer table: world=%d rank=%d (at most %d ranks)", fn, peers->world, peers->rank, SGR_MAX_PEERS);
	PeerTable pt = {};
	pt.world = peers->world;
	pt.rank = peers->rank;
	for (int p = 0; p < peers->world; p++) {
		if (!peers->records[p]) return fail(SGR_EINVAL, "%s: peer table entry %d has no staging region", fn, p);
		if (int rc = check_aligned16("a staging region", peers->records[p])) return rc;
		if (peers->world > 1 && !peers->flags[p]) return fail(SGR_EINVAL, "%s: peer table entry %d has no barrier pad", fn, p);
		pt.flags[p] = peers->flags[p];
	}
	PieceTable ts = {}, tp = {};
	long long blocks_stage = 0, blocks_pull = 0;
	if (int rc = peer_pieces(fn, "stage", peers, staging_bytes, stage, num_stage, true, ts, blocks_stage)) return rc;
	if (int rc = peer_pieces(fn, "pull", peers, staging_bytes, pull, num_pull, false, tp, blocks_pull)) return rc;
	if (blocks_stage > 0x7fffffffLL || blocks_pull > 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "%s: more than 2^31-1 blocks of floats to copy", fn);
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_peer_exchange_round(pt, ts, tp, st), fn);
	return SGR_OK;
}

int sgr_sparse_adam_step(const SgrSparseAdamSegment *segments, int32_t num_segments, const int32_t *radii, double beta1, double beta2,
                         double eps, void *stream) {
	if (!segments || num_segments <= 0) return fail(SGR_EINVAL, "segment table is empty");
	int64_t at = 0;
	for (int k = 0; k < num_segments; k++) {
		const SgrSparseAdamSegment &s = segments[k];
		if (s.start != at || s.count < 0) return fail(SGR_EINVAL, "segment %d: start %d (expected %lld), count %d", k, s.start, (long long)at, s.count);
		for (int a = 0; a < SGR_DENSIFY_TENSORS; a++) {
			const int w = s.width[a];
			if (w < 0) return fail(SGR_EINVAL, "segment %d: %s has width %d", k, kDensifyTensor[a], w);
			// the kernel indexes a 256-row tile's span [0, 256 w) with int
			if (w > SGR_SPARSE_ADAM_MAX_WIDTH)
				return fail(SGR_EUNSUPPORTED, "segment %d: %s has width %d > %d floats per row", k, kDensifyTensor[a], w, SGR_SPARSE_ADAM_MAX_WIDTH);
			if (w == 0) continue;
			if (s.count > 0 && (!s.param[a] || !s.grad[a] || !s.exp_avg[a] || !s.exp_avg_sq[a]))
				return fail(SGR_EINVAL, "segment %d: %s has a NULL pointer", k, kDensifyTensor[a]);
			if (s.step[a] < 1) return fail(SGR_EINVAL, "segment %d: %s has step %d (step counts from 1)", k, kDensifyTensor[a], s.step[a]);
			if (!std::isfinite(s.lr[a])) return fail(SGR_EINVAL, "segment %d: %s has a non-finite lr", k, kDensifyTensor[a]);
		}
		at += s.count;
	}
	if (at >= 0x7fffffffLL) return fail(SGR_EUNSUPPORTED, "%lld Gaussians in all exceed 2^31-2", (long long)at);
	if (!(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0)) return fail(SGR_EINVAL, "betas must lie in [0, 1)");
	if (at == 0) return SGR_OK;
	if (!radii) return fail(SGR_EINVAL, "radii is NULL");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_sparse_adam(segments, num_segments, radii, beta1, beta2, eps, st), "sparse_adam");
	return SGR_OK;
}

size_t sgr_knn_scratch_bytes(int32_t P) { return knn_scratch_bytes(P); }

int sgr_knn_mean_dist2(int32_t P, const float *points, float *mean_dist2, void *scratch, size_t scratch_bytes, void *stream) {
	if (P < 0) return fail(SGR_EINVAL, "P < 0");
	if (P == 0) return SGR_OK;
	if (!points || !mean_dist2) return fail(SGR_EINVAL, "NULL pointer passed to sgr_knn_mean_dist2");
	if (!scratch || scratch_bytes < knn_scratch_bytes(P)) return fail(SGR_ENOMEM, "knn scratch too small: %zu < %zu", scratch_bytes, knn_scratch_bytes(P));
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_knn(P, points, mean_dist2, scratch, scratch_bytes, st), "knn");
	return SGR_OK;
}

}  // extern "C"
