// capi.cu — the extern "C" surface of libsgr.so (include/sgr.h): argument validation, state carving, launch order.
// Host-side only; every device kernel lives in its own translation unit.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "sgr_common.cuh"

namespace sgr {

static thread_local char g_err[512] = "";
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
	g.ckey = take<uint32_t>(p, n);
	g.cval = take<uint32_t>(p, n);
	g.temp_bytes = memo_bytes((int64_t)P, [](int64_t n) { return geom_temp_bytes((int)n); });
	g.temp = take<char>(p, g.temp_bytes);
	g.total_bytes = (size_t)(p - reinterpret_cast<char *>(base));
	return g;
}
ImgView carve_img(void *base, int W, int H) {
	ImgView v;
	char *p = reinterpret_cast<char *>(base);
	const size_t gx = (W + SGR_TILE - 1) / SGR_TILE, gy = (H + SGR_TILE - 1) / SGR_TILE;
	v.ranges = take<uint2>(p, gx * gy + 1);
	v.tile_max_contrib = take<uint32_t>(p, gx * gy + 1);
	v.n_contrib = take<uint32_t>(p, (size_t)W * H + 1);
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
	b.sort_temp_bytes = memo_bytes(R, [](int64_t n) { return sort_temp_bytes(n); });
	b.sort_temp = take<char>(p, b.sort_temp_bytes);
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

// colour and covariance inputs of a projection: exactly one source of each, and SH coefficients only with M > 0
static int check_gaussian_inputs(const FrameDev &f, const float *shs, const float *colors_precomp, const float *scales,
                                 const float *rotations, const float *cov3D_precomp) {
	if ((shs == nullptr) == (colors_precomp == nullptr)) return fail(SGR_EINVAL, "provide exactly one of shs / colors_precomp");
	const bool sr = scales != nullptr && rotations != nullptr;
	if (sr == (cov3D_precomp != nullptr) || ((scales != nullptr) != (rotations != nullptr)))
		return fail(SGR_EINVAL, "provide exactly one of (scales, rotations) / cov3D_precomp");
	if (shs && f.M <= 0) return fail(SGR_EINVAL, "shs given but M == 0");
	return SGR_OK;
}

// pointers of the per-Gaussian chain rule; `inputs_ok` is the caller's check of its own input pointers
static int check_geom_grads(const char *fn, bool inputs_ok, const float *shs, const float *scales, const float *rotations,
                            const float *cov3D_precomp, const float *dL_dmeans3D, const float *dL_dmeans2D, const float *dL_dsh,
                            const float *dL_dopacity, const float *dL_dscales, const float *dL_drotations) {
	if (!inputs_ok || !dL_dmeans3D || !dL_dmeans2D || !dL_dopacity) return fail(SGR_EINVAL, "NULL pointer passed to %s", fn);
	if (shs && !dL_dsh) return fail(SGR_EINVAL, "shs given but dL_dsh is NULL");
	if (!cov3D_precomp && (!scales || !rotations || !dL_dscales || !dL_drotations))
		return fail(SGR_EINVAL, "scale/rotation path needs scales, rotations, dL_dscales, dL_drotations");
	return SGR_OK;
}

}  // namespace sgr

using namespace sgr;

extern "C" {

int sgr_abi_version(void) { return SGR_ABI_VERSION; }
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
	SGR_TRY(launch_project(f, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, radii,
	                       reinterpret_cast<GaussRec *>(records), st),
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

// FrameDev of the gathered problem (all world*chunk slots) seen through this rank's band
static int make_total_frame(const SgrFrame *frame, const SgrPeers *peers, FrameDev &fl, FrameDev &ft, PeerTable &pt, bool need_grad) {
	int rc = make_frame(frame, fl);
	if (rc) return rc;
	if ((rc = make_peers(peers, fl, need_grad, pt)) != SGR_OK) return rc;
	if (fl.S != 0) return fail(SGR_EUNSUPPORTED, "the fused Gaussian-sharded step supports S == 0 only (use the staged calls for feature channels)");
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

int sgr_sharded_forward(const SgrFrame *frame, const SgrPeers *peers, const float *means3D, const float *shs, const float *colors_precomp,
                        const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp, float *out_color,
                        float *out_depth, float *out_alpha, int32_t *radii_local, void *records_local, size_t geom_bytes, void *img_state,
                        size_t img_bytes, void *binning_state, size_t binning_bytes, int64_t capacity, int64_t gaussian_capacity,
                        uint32_t barrier_epoch, int32_t pre_barrier, void *stream) {
	FrameDev fl, ft;
	PeerTable pt = {};
	int rc = make_total_frame(frame, peers, fl, ft, pt, false);
	if (rc) return rc;
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
	const GeomView g = carve_geom(geom_state, ft.P);
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
	                               reinterpret_cast<GaussRec *>(records_local), g.depth_key,
	                               (size_t)(reinterpret_cast<char *>(g.iota) - reinterpret_cast<char *>(geom_state)), st),
	        "project+scatter");
	if (ft.P == 0) return SGR_OK;
	SGR_TRY(cudaMemsetAsync(g.big_count, 0, 64 * sizeof(uint32_t), st), "status reset");
	SGR_TRY(launch_peer_barrier(pt, barrier_epoch, g.big_count, st), "barrier");
	int n_order = ft.P;
	SGR_TRY(launch_count_and_order_runs(ft, g, pt.radii[pt.rank], pt.world, pt.chunk, st, gaussian_capacity, const_cast<float *>(pt.grad2d[pt.rank]), &n_order),
	        "count + depth_order");
	const BinView b = capacity > 0 ? carve_bin(binning_state, capacity) : carve_bin(nullptr, 0);
	SGR_TRY(launch_binning(ft, g, pt.radii[pt.rank], b, img, capacity, st, capacity, n_order), "binning");
	SGR_TRY(launch_blend_fwd(ft, g, b, img, nullptr, out_color, out_depth, out_alpha, nullptr, st), "blend_fwd");
	return SGR_OK;
}

int sgr_sharded_backward(const SgrFrame *frame, const SgrPeers *peers, int64_t capacity, const float *means3D, const float *shs,
                         const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                         const int32_t *radii_local, const void *records_local, const void *img_state, const void *binning_state,
                         const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                         float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                         float *dL_dscales, float *dL_drotations, float *dL_dcov3D, uint32_t barrier_epoch, void *stream) {
	FrameDev fl, ft;
	PeerTable pt = {};
	int rc = make_total_frame(frame, peers, fl, ft, pt, true);
	if (rc) return rc;
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = frame->debug != 0;
	if (!img_state || !out_alpha || !dL_dcolor || !dL_ddepth || !dL_dalpha) return fail(SGR_EINVAL, "NULL pointer passed to sgr_sharded_backward");
	if (capacity > 0 && !binning_state) return fail(SGR_EINVAL, "capacity > 0 but binning_state is NULL");
	if (fl.P > 0 && (rc = check_geom_grads("sgr_sharded_backward", means3D && radii_local && records_local, shs, scales, rotations, cov3D_precomp,
	                                       dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dopacity, dL_dscales, dL_drotations)) != SGR_OK)
		return rc;
	const GeomView g = carve_geom(pt.rec[pt.rank], ft.P);
	const ImgView img = carve_img(const_cast<void *>(img_state), ft.W, ft.H);
	const BinView b = carve_bin(const_cast<void *>(binning_state), capacity);
	float *grad2d = const_cast<float *>(pt.grad2d[pt.rank]);
	if (ft.P > 0)
		SGR_TRY(launch_blend_bwd(ft, g, b, img, nullptr, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, nullptr, grad2d, nullptr, st, true), "blend_bwd");
	SGR_TRY(launch_peer_barrier(pt, barrier_epoch, ft.P > 0 ? g.big_count : nullptr, st), "barrier");
	SGR_TRY(launch_preprocess_bwd(fl, &pt, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii_local,
	                              reinterpret_cast<const GaussRec *>(records_local), reinterpret_cast<const float *>(g.depth_key), dL_dmeans3D,
	                              dL_dmeans2D, shs ? dL_dsh : nullptr, dL_dcolors_precomp, dL_dopacity, cov3D_precomp ? nullptr : dL_dscales,
	                              cov3D_precomp ? nullptr : dL_drotations, dL_dcov3D, st),
	        "preprocess_bwd+gather");
	return SGR_OK;
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

int sgr_backward_blend(const SgrFrame *frame, int64_t num_instances, const float *semantics, const void *geom_state,
                       const void *binning_state, const void *img_state, const float *out_alpha, const float *dL_dcolor,
                       const float *dL_ddepth, const float *dL_dalpha, const float *dL_dsemantic, float *grad2d,
                       float *dL_dsemantics, void *stream) {
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
	SGR_TRY(launch_blend_bwd(f, g, b, img, semantics, out_alpha, dL_dcolor, dL_ddepth, dL_dalpha, dL_dsemantic, grad2d, dL_dsemantics, st),
	        "blend_bwd");
	return SGR_OK;
}

// shared body of sgr_backward_geom (no layer table) and sgr_backward_geom_layered; `fn` names the entry point in error messages.
// With a live layer (grad2d set, non-empty range) the layers' rows are merged into grad2d before the chain rule, and the main
// dL_dmeans2D of their range is restored from the pre-merge rows afterwards.
static int backward_geom(const char *fn, const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                         const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                         const void *geom_state, float *grad2d, const SgrLayerGrad *layers, int32_t num_layers, float *scratch,
                         float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                         float *dL_dscales, float *dL_drotations, float *dL_dcov3D, void *stream) {
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
	if ((rc = check_geom_grads(fn, means3D && radii && geom_state && grad2d, shs, scales, rotations, cov3D_precomp, dL_dmeans3D,
	                           dL_dmeans2D, dL_dsh, dL_dopacity, dL_dscales, dL_drotations)) != SGR_OK)
		return rc;
	if (hi > lo && !scratch) return fail(SGR_EINVAL, "scratch is NULL");
	const GeomView g = carve_geom(const_cast<void *>(geom_state), f.P);
	if (hi > lo) {
		SGR_TRY(launch_layer_stash(grad2d, lo, hi, scratch, false, nullptr, st), "layer stash");
		SGR_TRY(launch_layer_merge(grad2d, layers, num_layers, st), "layer merge");
	}
	SGR_TRY(launch_preprocess_bwd(f, nullptr, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii, g.rec, grad2d, dL_dmeans3D,
	                              dL_dmeans2D, shs ? dL_dsh : nullptr, dL_dcolors_precomp, dL_dopacity,
	                              cov3D_precomp ? nullptr : dL_dscales, cov3D_precomp ? nullptr : dL_drotations, dL_dcov3D, st),
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
	int rc = sgr_backward_blend(frame, num_instances, semantics, geom_state, binning_state, img_state, out_alpha, dL_dcolor, dL_ddepth,
	                            dL_dalpha, dL_dsemantic, grad2d_scratch, dL_dsemantics, stream);
	if (rc) return rc;
	return sgr_backward_geom(frame, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii, geom_state, grad2d_scratch,
	                         dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors_precomp, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D,
	                         stream);
}

// ---- render layers ----
// layer state: the img-state layout (ranges, tile_max_contrib, n_contrib) of the layer, then its tile lists u32[num_instances]
struct LayerView {
	ImgView img;
	uint32_t *list;
	size_t total_bytes;
};
static LayerView carve_layer(void *base, int W, int H, int64_t R) {
	LayerView v;
	v.img = carve_img(base, W, H);
	char *p = reinterpret_cast<char *>(base) + v.img.total_bytes;
	v.list = take<uint32_t>(p, R > 0 ? (size_t)R : 1);
	v.total_bytes = (size_t)(p - reinterpret_cast<char *>(base));
	return v;
}
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

int sgr_compose_forward(const SgrSegment *segments, int32_t num_segments, int32_t M, const float *poses, const float *idft,
                        const uint8_t *flip, const float *flip_quat, float *means3D, float *rotations, float *scales, float *opacities,
                        float *shs, void *stream) {
	int64_t P = 0;
	int rc = check_segments(segments, num_segments, M, P);
	if (rc) return rc;
	if (P == 0) return SGR_OK;
	if (!poses || !idft || !means3D || !rotations || !scales || !opacities || !shs) return fail(SGR_EINVAL, "NULL pointer passed to sgr_compose_forward");
	if (flip && !flip_quat) return fail(SGR_EINVAL, "flip mask given without flip_quat");
	cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
	const bool debug = false;
	SGR_TRY(launch_compose_fwd(segments, num_segments, M, poses, idft, flip, flip_quat, means3D, rotations, scales, opacities, shs, st), "compose_fwd");
	return SGR_OK;
}

int sgr_compose_backward(const SgrSegment *segments, const SgrSegmentGrads *grads, int32_t num_segments, int32_t M, const float *poses,
                         const float *idft, const uint8_t *flip, const float *flip_quat, const float *dL_dmeans3D,
                         const float *dL_drotations, const float *dL_dscales, const float *dL_dopacities, const float *dL_dshs,
                         float *dposes, float *pose_scratch, void *stream) {
	int64_t P = 0;
	int rc = check_segments(segments, num_segments, M, P);
	if (rc) return rc;
	if (!grads || !dposes || !pose_scratch || !poses || !idft) return fail(SGR_EINVAL, "NULL pointer passed to sgr_compose_backward");
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
	                           dL_dopacities, dL_dshs, pose_scratch, dposes, st),
	        "compose_bwd");
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
