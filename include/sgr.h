/*
 * sgr.h — C ABI of the H100-native (sm_90a) differentiable Gaussian rasterizer (libsgr.so).
 *
 * This is the drop-in boundary for the ONE hot path of zju3dv/street_gaussians that this repository
 * replaces (SURVEY.md §8b).  Each entry point names the reference interface it stands in for
 * (paths relative to /root/reference/submodules/diff-gaussian-rasterization = "DGR/",
 *  /root/reference/submodules/simple-knn = "KNN/").
 *
 * Conventions
 *  - plain C: pointers + sizes only; no torch / C++ types cross this boundary.
 *  - every pointer is a DEVICE pointer unless it is documented as host; all fp32 arrays are contiguous
 *    and laid out exactly like the tensors of the reference Python API
 *    (DGR/diff_gaussian_rasterization/__init__.py:197-233): means3D[P,3], shs[P,M,3], colors_precomp[P,3],
 *    semantics[P,S], opacities[P,1], scales[P,3], rotations[P,4] (w,x,y,z), cov3D_precomp[P,6],
 *    images [C,H,W].  A NULL pointer plays the role of the reference's empty tensor.
 *  - the CALLER owns all memory, including the forward->backward state buffers and scratch; the library is
 *    stateless between calls, re-entrant and thread-safe; every kernel is enqueued on `stream` (a cudaStream_t
 *    passed as void*).  The only host synchronisations are one 8-byte read-back of the instance count inside
 *    sgr_forward (the reference has the same one at DGR/cuda_rasterizer/rasterizer_impl.cu:283-284) and the read-back of the
 *    new sizes inside sgr_densify_plan.
 *  - return value: 0 on success, negative SGR_E* on failure; sgr_last_error() returns a thread-local message.
 *    With frame.debug != 0 every launch is followed by a stream synchronise + error check
 *    (the reference's CHECK_CUDA, DGR/cuda_rasterizer/auxiliary.h:166-173).
 */
#ifndef SGR_H_INCLUDED
#define SGR_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGR_ABI_VERSION 7

#define SGR_OK 0
#define SGR_EINVAL (-1)   /* bad argument combination / shape                     */
#define SGR_ECUDA (-2)    /* a CUDA runtime call or kernel failed                  */
#define SGR_ENOMEM (-3)   /* caller-provided buffer too small / allocator failed  */
#define SGR_EUNSUPPORTED (-4)

/* Maximum number of extra feature ("semantic") channels the BACKWARD pass accepts.  The reference has a
 * compile-time cap NUM_CLASSES = 20 (DGR/cuda_rasterizer/config.h:16) beyond which it is undefined behaviour;
 * this library returns SGR_EUNSUPPORTED above SGR_MAX_SEMANTIC_BWD instead.  Forward accepts any S. */
#define SGR_MAX_SEMANTIC_BWD 32

/* Per-call frame description == the 12 fields of GaussianRasterizationSettings
 * (DGR/diff_gaussian_rasterization/__init__.py:167-179) + problem sizes + the tile-row band this process owns. */
typedef struct SgrFrame {
	int32_t P;              /* number of Gaussians                                                       */
	int32_t D;              /* active SH degree (settings.sh_degree)                                     */
	int32_t M;              /* SH coefficients per Gaussian as stored (shs.shape[1]); 0 with colors_precomp */
	int32_t S;              /* extra feature channels (semantics.shape[1])                               */
	int32_t width, height;  /* image_width, image_height                                                 */
	float tan_fovx, tan_fovy;
	float scale_modifier;
	int32_t prefiltered;    /* accepted for API parity; a culled point is simply skipped (the reference traps) */
	int32_t debug;
	/* Multi-GPU tile-row sharding (no reference counterpart; SURVEY.md §8e): this call rasterises only the
	 * 16-pixel tile rows r with row_begin <= r < row_end and (r - row_begin) % row_step == 0.
	 * {0, 0, 0} or {0, ceil(H/16), 1} means the whole image.  Pixels of other rows are left untouched. */
	int32_t row_begin, row_end, row_step;
	const float *bg;         /* [3]  device                                                              */
	const float *viewmatrix; /* [16] device: world_view_transform  (W2C transposed, row-major)           */
	const float *projmatrix; /* [16] device: full_proj_transform                                         */
	const float *campos;     /* [3]  device                                                              */
} SgrFrame;

/* Caller-supplied device allocator, called at most once per sgr_forward with the size of the binning state once the
 * instance count is known.  Stands in for the reference's resize callbacks (std::function<char*(size_t)>,
 * DGR/rasterize_points.cu:27-33, DGR/cuda_rasterizer/rasterizer.h:36-38).  Must return a 256-byte aligned device
 * pointer valid until the matching sgr_backward_* calls have been enqueued, or NULL on failure. */
typedef void *(*sgr_alloc_fn)(void *user, size_t nbytes);

int sgr_abi_version(void);
const char *sgr_last_error(void);
/* Number of kernels of this library enqueued so far by the calling process (cub's internal sort / scan kernels are not
 * included).  Diagnostic only — bench.py reports the delta over its timed region as `gpu_launches`.  No reference counterpart. */
uint64_t sgr_launch_count(void);

/* Sizes (bytes) of the caller-owned forward state.  geom: per-Gaussian records (reference GeometryState,
 * DGR/cuda_rasterizer/rasterizer_impl.h:21-37); img: per-pixel / per-tile state (ImageState, :46-52).
 * binning (BinningState, :54-64) depends on the instance count R and is requested through sgr_alloc_fn;
 * sgr_binning_bytes(R) reports what will be asked for. */
int sgr_state_sizes(const SgrFrame *frame, size_t *geom_bytes, size_t *img_bytes);
size_t sgr_binning_bytes(int64_t num_instances);

/* Forward rasterisation.  Replaces RasterizeGaussiansCUDA -> CudaRasterizer::Rasterizer::forward
 * (DGR/rasterize_points.cu:35-124, DGR/cuda_rasterizer/rasterizer_impl.cu:197-343; pybind name
 * `rasterize_gaussians`, DGR/ext.cpp:16).
 *   exactly one of (shs, colors_precomp) and exactly one of ((scales, rotations), cov3D_precomp) must be non-NULL.
 *   out_color[3,H,W], out_depth[1,H,W], out_alpha[1,H,W], out_semantic[S,H,W] (may be NULL when S == 0), radii[P]:
 *   every element of the owned tile rows is written (no pre-zeroing needed for a whole-image band); radii is
 *   always fully written.
 *   *binning_state receives the pointer obtained from `alloc`; *num_instances the (Gaussian, tile) instance count
 *   of THIS library's binning (exact opacity-aware tile culling makes it <= the reference's num_rendered). */
int sgr_forward(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                const float *semantics, const float *opacities, const float *scales, const float *rotations,
                const float *cov3D_precomp, float *out_color, float *out_depth, float *out_alpha, float *out_semantic,
                int32_t *radii, void *geom_state, size_t geom_bytes, void *img_state, size_t img_bytes, sgr_alloc_fn alloc,
                void *alloc_user, void **binning_state, int64_t *num_instances, void *stream);

/* Forward without any host synchronisation ("R read back asynchronously or bounded", SURVEY.md §8b).  Identical to
 * sgr_forward except that the CALLER supplies the binning state, sized with sgr_binning_bytes(capacity), instead of the
 * library reading the instance count back to size it.  The count stays on the device: instances beyond `capacity` are
 * dropped (whole Gaussians, farthest first) and an overflow flag is raised in img_state — the frame is then incomplete,
 * and the caller must re-render with a larger capacity.  sgr_forward_status() fetches {instances, overflowed} when the
 * caller chooses to synchronise (e.g. once per N frames, or before the optimiser step).  Pass `capacity` as
 * num_instances to the sgr_backward_* calls.  No reference counterpart: the reference always blocks on a cudaMemcpy
 * (DGR/cuda_rasterizer/rasterizer_impl.cu:283-284). */
int sgr_forward_bounded(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                        const float *semantics, const float *opacities, const float *scales, const float *rotations,
                        const float *cov3D_precomp, float *out_color, float *out_depth, float *out_alpha, float *out_semantic,
                        int32_t *radii, void *geom_state, size_t geom_bytes, void *img_state, size_t img_bytes,
                        void *binning_state, size_t binning_bytes, int64_t capacity, void *stream);
/* Device->host copy of the status words of the last forward that used geom_state; synchronises `stream`.  `overflowed` is a bit
 * set: 1 = more instances than `capacity`, 2 = more Gaussians in the band than `gaussian_capacity` (sgr_sharded_forward). */
int sgr_forward_status(const SgrFrame *frame, const void *geom_state, int64_t *num_instances, int32_t *overflowed, void *stream);
/* Asynchronous variant: enqueues the copy of EIGHT uint32 {instances, overflow bits, instances emitted, Gaussians with instances
 * (compacted mode, else 0), epoch of a device barrier that TIMED OUT in this forward (0 = none; sgr_sharded_forward), 3 reserved}
 * into host_status (pinned host memory recommended) on `stream` and returns immediately; valid once the caller has observed
 * stream progress past this point. */
int sgr_forward_status_async(const SgrFrame *frame, const void *geom_state, uint32_t *host_status, void *stream);

/* Backward, stage 1 of 2: per-pixel backward blend.  Replaces BACKWARD::render
 * (DGR/cuda_rasterizer/backward.cu:415-641, called at rasterizer_impl.cu:454-477).
 *   grad2d[P,12] receives the per-Gaussian screen-space sums
 *     [0..2] dL/dmean2D (x, y NDC-scaled; z = sum |x|+|y|), [3..5] dL/dconic (xx, xy, yy), [6] dL/dopacity,
 *     [7..9] dL/dcolor, [10] dL/ddepth, [11] unused
 *   and dL_dsemantics[P,S] the feature-channel sums.  Both are ZEROED by this call and then accumulated, so with
 *   tile-row sharding each rank holds a partial sum that must be summed across ranks (one all-reduce) before
 *   stage 2.  S must be <= SGR_MAX_SEMANTIC_BWD. */
int sgr_backward_blend(const SgrFrame *frame, int64_t num_instances, const float *semantics, const void *geom_state,
                       const void *binning_state, const void *img_state, const float *out_alpha, const float *dL_dcolor,
                       const float *dL_ddepth, const float *dL_dalpha, const float *dL_dsemantic, float *grad2d,
                       float *dL_dsemantics, void *stream);

/* Backward, stage 2 of 2: per-Gaussian chain rule.  Replaces BACKWARD::preprocess = computeCov2DCUDA + preprocessCUDA
 * (DGR/cuda_rasterizer/backward.cu:643-709, 144-274, 346-412).  Every element of every non-NULL output is written
 * (zeros for Gaussians with radii <= 0), so outputs need no pre-zeroing:
 *   dL_dmeans3D[P,3], dL_dmeans2D[P,3], dL_dsh[P,M,3] (NULL when colors_precomp), dL_dcolors_precomp[P,3] (NULL with SH),
 *   dL_dopacity[P,1], dL_dscales[P,3], dL_drotations[P,4] (NULL with cov3D_precomp), dL_dcov3D[P,6] (may be NULL). */
int sgr_backward_geom(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                      const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                      const void *geom_state, const float *grad2d, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh,
                      float *dL_dcolors_precomp, float *dL_dopacity, float *dL_dscales, float *dL_drotations,
                      float *dL_dcov3D, void *stream);

/* Convenience: stage 1 + stage 2 on one device.  Replaces RasterizeGaussiansBackwardCUDA ->
 * CudaRasterizer::Rasterizer::backward (DGR/rasterize_points.cu:126-220, rasterizer_impl.cu:396-506; pybind name
 * `rasterize_gaussians_backward`, DGR/ext.cpp:17).  grad2d_scratch is P*12 floats of caller scratch. */
int sgr_backward(const SgrFrame *frame, int64_t num_instances, const float *means3D, const float *shs,
                 const float *colors_precomp, const float *semantics, const float *scales, const float *rotations,
                 const float *cov3D_precomp, const int32_t *radii, const void *geom_state, const void *binning_state,
                 const void *img_state, const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth,
                 const float *dL_dalpha, const float *dL_dsemantic, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh,
                 float *dL_dcolors_precomp, float *dL_dsemantics, float *dL_dopacity, float *dL_dscales,
                 float *dL_drotations, float *dL_dcov3D, float *grad2d_scratch, void *stream);

/* ---- Render layers: row ranges of the same call rendered alongside the full frame (whole image, one GPU) ----------------------
 * A layer is the half-open row range [begin, end) of the call's Gaussians plus a background colour; its images are bit-identical
 * to a separate sgr_forward on the sliced arrays with that background and S = 0 (colour, depth, alpha only).  That is the
 * reference's objects-only / background-only render with parse_camera_again=False (render_object / render_background,
 * lib/models/street_gaussian_renderer.py:13-40, train.py:114-122), which rasterises the actor rows [n_bkgd, P) of the tensors the
 * full render used.  Per tile the separate call's list is the subsequence of the main list with ids in the range (stable depth
 * pre-sort, stable tile sort), so the layer's list is compacted out of the main call's list and blended with the main call's
 * per-Gaussian records: nothing is projected, sorted or read back again, and the bounded mode stays free of host synchronisation.
 * An empty range (begin == end, also with P == 0) gives colour bg and zero depth and alpha, as render_kernel's empty branch
 * (street_gaussian_renderer.py:138-151) does — not the zero colour of sgr_forward's P == 0 short-circuit. */
typedef struct SgrLayer {
	int32_t begin, end;  /* 0 <= begin <= end <= frame.P */
	const float *bg;     /* [3] device */
} SgrLayer;
/* Bytes of one layer's caller-owned state (per-tile ranges, per-pixel contributor counts and the layer's tile lists) for a main call
 * whose sgr_backward_* calls take num_instances: the instance count of sgr_forward, or the capacity of sgr_forward_bounded. */
int sgr_layer_state_sizes(const SgrFrame *frame, int64_t num_instances, size_t *layer_bytes);
/* Renders `layer` from the state a whole-image sgr_forward / sgr_forward_bounded left in geom / binning / img state (frame == that
 * call's frame, num_instances == the value its backward takes).  out_color[3,H,W], out_depth[1,H,W], out_alpha[1,H,W]: every pixel
 * written.  With an empty range no state is read (geom / binning / img state may be NULL). */
int sgr_forward_layer(const SgrFrame *frame, const SgrLayer *layer, int64_t num_instances, const void *geom_state, const void *binning_state,
                      const void *img_state, void *layer_state, size_t layer_bytes, float *out_color, float *out_depth, float *out_alpha,
                      void *stream);
/* Backward blend of one layer (its sgr_forward_layer state): grad2d[end-begin, 12] (row r = Gaussian begin + r, same columns as
 * sgr_backward_blend) is ZEROED and accumulated.  Nothing is done for an empty range. */
int sgr_backward_blend_layer(const SgrFrame *frame, const SgrLayer *layer, const void *geom_state, const void *layer_state, const float *out_alpha,
                             const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha, float *grad2d, void *stream);
typedef struct SgrLayerGrad {
	int32_t begin, end;
	const float *grad2d;  /* [end-begin, 12] device (sgr_backward_blend_layer's output), or NULL: this layer has no gradient */
	float *dL_dmeans2D;   /* [end-begin, 3] device or NULL: receives this layer's own screen-space gradient ([0:3] of its grad2d) */
} SgrLayerGrad;
/* sgr_backward_geom for a layered call: the chain rule runs once on the main sums plus every layer's sums (all 12 columns), while
 * dL_dmeans2D receives the MAIN sums only, as a separate call would leave it (the densification statistics read it); each layer's
 * own [0:3] goes to its dL_dmeans2D sink.  grad2d[P,12] (the main sums) is CONSUMED: the layer rows are added into it in place.
 * layers: HOST array.  scratch: 3 floats per row of [lo, hi), the smallest range that covers every layer with a gradient (3 * P
 * floats always suffice).  Outputs and their rules as in sgr_backward_geom. */
int sgr_backward_geom_layered(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                              const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                              const void *geom_state, float *grad2d, const SgrLayerGrad *layers, int32_t num_layers, float *scratch,
                              float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                              float *dL_dscales, float *dL_drotations, float *dL_dcov3D, void *stream);

/* ---- Gaussian-sharded rendering (multi-GPU; no reference counterpart — the reference is single-GPU.  SURVEY.md §8e
 * "variant A": every rank owns P/N Gaussians AND a tile-row band) --------------------------------------------------
 * The forward of DGR/cuda_rasterizer/rasterizer_impl.cu:197-343 is split at the point where the per-Gaussian work
 * (FORWARD::preprocess, forward.cu:155-256) hands fixed-size screen-space records to the per-tile work:
 *   1. sgr_project          on the rank's own Gaussians -> records[P_local] (sgr_record_bytes() each) + radii[P_local]
 *   2. caller all-gathers records and radii (NCCL) into the first P_total*sgr_record_bytes() bytes of a geom_state
 *      sized for P_total, and a radii[P_total] array; padding slots must carry radii == 0
 *   3. sgr_forward_records  bins / sorts / blends the rank's tile-row band from the gathered records
 *   4. sgr_backward_blend   (frame.P = P_total) -> partial grad2d[P_total,12]; caller reduce-scatters it
 *   5. sgr_backward_geom    with frame.P = P_local, geom_state = the rank's own records, grad2d = its reduced slice.
 * Results are bit-identical to the single-GPU path for the forward images and agree to float summation order in the
 * gradients (tests/test_parity_gpu.py::test_gaussian_sharded_*). */
size_t sgr_record_bytes(void);
/* Step 1.  frame.P = number of local Gaussians; the tile-row band of `frame` is ignored.  Same input rules as
 * sgr_forward.  Writes records[P] (only slots with radii > 0 are meaningful) and radii[P] (all). */
int sgr_project(const SgrFrame *frame, const float *means3D, const float *shs, const float *colors_precomp,
                const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp,
                int32_t *radii, void *records, void *stream);
/* Step 3.  frame.P = P_total.  geom_state (sgr_state_sizes for P_total) must already hold the gathered records in its
 * first P_total*sgr_record_bytes() bytes; radii[P_total] is read, never written.  semantics[P_total,S] when S > 0.
 * capacity < 0: exact mode (instance count read back, binning state through `alloc`, like sgr_forward);
 * capacity >= 0: bounded mode (caller's binning_state of sgr_binning_bytes(capacity), like sgr_forward_bounded). */
int sgr_forward_records(const SgrFrame *frame, const int32_t *radii, const float *semantics, float *out_color,
                        float *out_depth, float *out_alpha, float *out_semantic, void *geom_state, size_t geom_bytes,
                        void *img_state, size_t img_bytes, sgr_alloc_fn alloc, void *alloc_user, void **binning_state_out,
                        int64_t *num_instances, void *binning_state, size_t binning_bytes, int64_t capacity, void *stream);

/* ---- Gaussian-sharded exchange over NVLink peer memory (replaces the two NCCL collectives of steps 2 and 4 above) -----
 * Requires every rank's gathered arrays to be mapped into every process (CUDA IPC / VMM; the Python host uses
 * torch.distributed._symmetric_memory) and the CYCLIC band layout: tile row r belongs to rank r % world.
 *   sgr_scatter_records : for every local slot i (global id g = rank*chunk + i) store the 48-B record into
 *                         peers.records[p][g] of each rank p whose band meets the Gaussian's tile rectangle, and
 *                         peers.radii[p][g] = radius for those ranks, 0 for all others (padding slots: 0 everywhere).
 *   sgr_gather_grad2d   : grad2d_local[i,0:12] = sum over the same ranks p of peers.grad2d[p][g,0:12]; rows of
 *                         invisible Gaussians are zero.
 * The caller must order them against the peers' kernels with a cross-rank barrier on the stream: one after
 * sgr_scatter_records (before any rank's sgr_forward_records) and one after sgr_backward_blend (before any rank's
 * sgr_gather_grad2d).  Traffic per Gaussian is 48 B x (#ranks it touches) + 4 B x world instead of 48 B x world. */
#define SGR_MAX_PEERS 16
typedef struct SgrPeers {
	int32_t world, rank;
	int64_t chunk;                      /* slots per rank */
	void *records[SGR_MAX_PEERS];       /* rank p's gathered record array (= start of its geom_state), world*chunk records */
	int32_t *radii[SGR_MAX_PEERS];      /* rank p's radii[world*chunk] */
	const float *grad2d[SGR_MAX_PEERS]; /* rank p's partial grad2d[world*chunk,12] (output of its sgr_backward_blend) */
	uint32_t *flags[SGR_MAX_PEERS];     /* rank p's barrier pad: uint32[SGR_MAX_PEERS], zero-initialised once by the caller and mapped
	                                       into every rank like the arrays above.  Only needed by sgr_peer_barrier / sgr_sharded_*. */
} SgrPeers;
int sgr_scatter_records(const SgrFrame *frame, const SgrPeers *peers, const void *records_local, const int32_t *radii_local,
                        void *stream);
int sgr_gather_grad2d(const SgrFrame *frame, const SgrPeers *peers, const void *records_local, const int32_t *radii_local,
                      float *grad2d_local, void *stream);

/* Device-side barrier across the ranks of `peers` on `stream` (no host involvement, no NCCL): each rank stores `epoch` into its
 * slot of every peer's pad (release, system scope, after fencing its earlier peer stores) and waits until every peer has stored
 * an epoch >= `epoch` into its own pad.  Every rank must issue the same sequence of barriers with epochs increasing by one
 * (first epoch 1).  epoch == 0 selects the device-side count: the library keeps the epoch in the rank's own pad (slot
 * SGR_MAX_PEERS) and increments it per barrier, so the call carries no per-step host value and a CUDA graph that captured a step
 * can be replayed.  Do not mix explicit and automatic epochs on one pad.  The wait is bounded (2 s): a rank that never arrives
 * cannot wedge the GPU. */
int sgr_peer_barrier(const SgrPeers *peers, uint32_t epoch, void *stream);

/* The Gaussian-sharded forward as ONE call (steps 1-3 above with the peer-memory exchange): project the rank's frame.P Gaussians and
 * deliver their records to the ranks whose band they meet (one kernel), device barrier, then bin / sort / blend the rank's band from
 * the delivered records — all launches issued back to back from C instead of six Python-level calls (a step split into
 * many Python-level calls is host-launch bound at N = 8).
 *   Delivery is by BLOCK RUNS, not by global index: the 256 consecutive Gaussians [256 b, 256 b + 256) of owner s that rank d needs
 *   are stored as one contiguous run into the first slots of [s*chunk + 256 b, +256) of rank d's record array (whole 128-B lines over
 *   NVLink), with the radius packed into the record; run lengths go to a table inside rank d's geom_state.  Ascending slot order
 *   equals ascending global-id order, so the depth order (ties included) and every pixel equal the single-GPU render.  In this mode
 *   peers->radii[rank] and the rows of peers->grad2d[rank] are indexed by SLOT; sgr_sharded_backward reads the rows back as the same runs.
 *   frame.P = local Gaussian count; frame.row_* = this rank's CYCLIC band (row_begin == rank, row_step == world); S must be 0.
 *   peers->records[rank] is this rank's geom_state (sgr_state_sizes for P = world*chunk, `geom_bytes` bytes) whose first
 *   world*chunk records are the delivery target; radii_local[chunk] / records_local[chunk] receive the rank's own results (kept
 *   for sgr_sharded_backward).  Bounded mode only: `capacity` instances (binning_state of sgr_binning_bytes(capacity)) and
 *   `gaussian_capacity` depth-order slots (< 0: world*chunk; the Gaussians delivered to this rank are compacted into them and
 *   sorted — sgr_forward_status reports both counts and both overflow bits).
 *   barrier_epoch: epoch of the barrier after the delivery (0 = device-side count, see sgr_peer_barrier); with pre_barrier != 0 a
 *   barrier with epoch barrier_epoch - 1 (or the next device-side count) is issued first (needed when the previous call on this
 *   workspace was a forward without a backward: peers may still be reading the records this call overwrites).  The rows of
 *   peers->grad2d[rank] that a backward can touch are zeroed by this call.  No array needs a particular content on entry. */
int sgr_sharded_forward(const SgrFrame *frame, const SgrPeers *peers, const float *means3D, const float *shs, const float *colors_precomp,
                        const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp, float *out_color,
                        float *out_depth, float *out_alpha, int32_t *radii_local, void *records_local, size_t geom_bytes, void *img_state,
                        size_t img_bytes, void *binning_state, size_t binning_bytes, int64_t capacity, int64_t gaussian_capacity,
                        uint32_t barrier_epoch, int32_t pre_barrier, void *stream);
/* The matching backward as ONE call (steps 4-5): blend_bwd of the band into peers->grad2d[rank], device barrier (barrier_epoch), then
 * the per-Gaussian chain rule of the rank's frame.P Gaussians, which sums each Gaussian's 12 screen-space values from the
 * ranks that rendered it while it runs: every thread block fetches its runs of rows from those ranks' partial grad2d (contiguous,
 * see sgr_sharded_forward) — no separate gather pass, no reduce-scatter.  Must follow the sgr_sharded_forward of the same frame on
 * the same workspace (it re-derives the run positions from the destination masks that call kept).  Outputs as in sgr_backward_geom. */
int sgr_sharded_backward(const SgrFrame *frame, const SgrPeers *peers, int64_t capacity, const float *means3D, const float *shs,
                         const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                         const int32_t *radii_local, const void *records_local, const void *img_state, const void *binning_state,
                         const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                         float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                         float *dL_dscales, float *dL_drotations, float *dL_dcov3D, uint32_t barrier_epoch, void *stream);

/* ---- Scene-graph composer (SURVEY.md §8 row f1; no native counterpart in the reference, which composes with ~40 PyTorch kernels) ----
 * One call builds the rasterizer's inputs from the raw parameters of every sub-model of the scene graph, as
 * StreetGaussianModel.get_xyz / get_rotation / get_scaling / get_opacity / get_features do
 * (lib/models/street_gaussian_model.py:287-449 with the activations of lib/models/gaussian_model.py:224-251 and the Fourier DC
 * colour of lib/models/gaussian_model_actor.py:71-80).  Segment s covers composed indices [start, start + count); segments must be
 * listed in ascending, gap-free order (background first, then the actors of the frame, as the reference concatenates them). */
#define SGR_MAX_FOURIER 8                 /* largest fourier_dim (cfg.model.gaussian.fourier_dim; 5 in the shipped configs) */
#define SGR_MAX_SEGMENTS_PER_LAUNCH 32    /* larger tables are processed in groups of this many segments */
typedef struct SgrSegment {
	int32_t start, count;   /* range in the composed arrays */
	int32_t fourier_dim;    /* rows of features_dc per Gaussian (1 for the background) */
	int32_t posed;          /* 0: world-space model (background); 1: actor, posed by poses[s] with optional mirroring */
	const float *xyz;            /* [count,3]      _xyz                                   (device) */
	const float *rotation;       /* [count,4]      _rotation, raw (w,x,y,z)                        */
	const float *scaling;        /* [count,3]      _scaling, log                                   */
	const float *opacity;        /* [count,1]      _opacity, logit                                 */
	const float *features_dc;    /* [count,C,3]    _features_dc                                    */
	const float *features_rest;  /* [count,M-1,3]  _features_rest (NULL when M == 1)               */
} SgrSegment;
typedef struct SgrSegmentGrads {   /* where sgr_compose_backward writes the gradient of each raw array (same shapes; fully written) */
	float *xyz, *rotation, *scaling, *opacity, *features_dc, *features_rest;
} SgrSegmentGrads;
/* segments: HOST array.  poses[num_segments,8] (device): actor -> world quaternion (w,x,y,z) as parse_camera leaves it in
 * obj_rots (street_gaussian_model.py:258-273; NOT required to be unit) + translation + 1 pad float; rows of unposed segments are
 * ignored.  idft[num_segments, SGR_MAX_FOURIER] (device): IDFT(t, C) row of each actor (lib/utils/sh_utils.py:120-130).
 * flip (device, uint8 [P] indexed by composed id, or NULL): 1 = mirror this Gaussian across the actor's local x-z plane (the
 * training-time symmetry augmentation, :275-284, 319-323, 347-349); flip_quat[4] (device) = the reference's flip_matrix.
 * Outputs (device, fully written): means3D[P,3], rotations[P,4], scales[P,3], opacities[P,1], shs[P,M,3]. */
int sgr_compose_forward(const SgrSegment *segments, int32_t num_segments, int32_t M, const float *poses, const float *idft,
                        const uint8_t *flip, const float *flip_quat, float *means3D, float *rotations, float *scales, float *opacities,
                        float *shs, void *stream);
/* Gradients of the five composed arrays -> gradients of every raw array (grads: HOST array parallel to segments) and of the
 * poses: dposes[num_segments,8] (device; rows of unposed segments are zero) — what autograd's expand / cat / einsum backward
 * accumulates for obj_rots and obj_trans in the reference.  pose_scratch: num_segments*16 floats of device scratch. */
int sgr_compose_backward(const SgrSegment *segments, const SgrSegmentGrads *grads, int32_t num_segments, int32_t M, const float *poses,
                         const float *idft, const uint8_t *flip, const float *flip_quat, const float *dL_dmeans3D,
                         const float *dL_drotations, const float *dL_dscales, const float *dL_dopacities, const float *dL_dshs,
                         float *dposes, float *pose_scratch, void *stream);

/* ---- Image-space losses with their gradient (SURVEY.md §8 row f2) ----
 * value = w_l1 * L1(image, gt, mask) + w_ssim * SSIM(image, gt, mask)  and  dL_dimage = d value / d image  in two kernels.
 * Replaces l1_loss (lib/utils/loss_utils.py:21-37), ssim / _ssim (:91-126: 11x11 Gaussian window, sigma 1.5, zero padding, C1 = 0.01^2,
 * C2 = 0.03^2, both images zeroed outside the mask, mean over ALL pixels) and the autograd replay of both.  The training loss of
 * train.py:103-104 is  w_l1 = (1 - lambda_dssim) * lambda_l1,  w_ssim = -lambda_dssim,  plus the constant lambda_dssim.
 *   image, gt: [C,H,W] device; mask: uint8 [H*W] device or NULL; dL_dimage: [C,H,W] device or NULL (value only).
 *   scalars (device, 4 floats): {value, L1, SSIM, number of masked pixels}.  scratch: sgr_image_loss_scratch_bytes(C,H,W) bytes. */
size_t sgr_image_loss_scratch_bytes(int32_t C, int32_t H, int32_t W);
int sgr_image_loss(int32_t C, int32_t H, int32_t W, const float *image, const float *gt, const uint8_t *mask, float w_l1, float w_ssim,
                   float *dL_dimage, float *scalars, void *scratch, size_t scratch_bytes, void *stream);
/* Sky / accumulation loss (train.py:107-113): acc clamped to [1e-6, 1-1e-6], mean over the N pixels of sky ? -log(1-acc) : -log(acc).
 * scalars (device, 2 floats): {weight * mean, mean}; dL_dacc[N] (or NULL) = weight * d mean / d acc.  scratch: >= 8 bytes. */
int sgr_sky_loss(int64_t N, const float *acc, const uint8_t *sky_mask, float weight, float *dL_dacc, float *scalars, void *scratch,
                 void *stream);
/* Object-accumulation loss (train.py:114-122, on the acc of the objects-only render): acc clamped to [1e-6, 1-1e-6], mean over the
 * N pixels of obj_bound ? -(acc log acc + (1-acc) log(1-acc)) : -log(1-acc).  scalars (device, 2 floats): {weight * mean, mean};
 * dL_dacc[N] (or NULL) = weight * d mean / d acc, zero where the clamp is active.  scratch: >= 8 bytes. */
int sgr_obj_acc_loss(int64_t N, const float *acc, const uint8_t *obj_bound, float weight, float *dL_dacc, float *scalars, void *scratch,
                     void *stream);
/* LiDAR depth loss (train.py:124-132): on the valid pixels (lidar_depth > 0 and mask, mask uint8 [N] or NULL = all),
 * err = |depth / (acc + 1e-10) - lidar_depth|; value = mean of the k = int(keep * n) smallest err (n = valid pixels, k formed in
 * double and truncated like Python's int(0.95 * n)).  acc is the UNCLAMPED accumulation (render_pkg['acc']), not the sky loss's
 * clamped copy.  The k smallest are found on the device by an exact radix select, so nothing is read back to the host and the grid
 * sizes depend on N only (the call can be captured in a CUDA graph).  NaN errors order above every number, like torch.topk.
 * Gradients (either pointer may be NULL): the k selected pixels get g = weight * sign(e - lidar_depth) / k with sign(0) = 0,
 * dL_ddepth = g / (acc + 1e-10), dL_dacc = -g * e / (acc + 1e-10); all other pixels 0.  Of the pixels tied at the k-th value, those
 * with the lowest flat index are taken.  k == 0 (n <= 1 at keep = 0.95) gives a NaN value and all-zero gradients.
 *   depth, acc, lidar_depth: [N] fp32 device; 0 < keep <= 1; N < 2^31.
 *   scalars (device, 4 floats): {weight * mean, mean, n, k}.  scratch: sgr_lidar_depth_loss_scratch_bytes(N) bytes. */
size_t sgr_lidar_depth_loss_scratch_bytes(int64_t N);
int sgr_lidar_depth_loss(int64_t N, const float *depth, const float *acc, const float *lidar_depth, const uint8_t *mask, double keep,
                         float weight, float *dL_ddepth, float *dL_dacc, float *scalars, void *scratch, size_t scratch_bytes, void *stream);

/* ---- Post-backward bookkeeping of a training iteration (SURVEY.md §8 row f3) ----
 * Densification statistics of StreetGaussianModel.set_max_radii2D + add_densification_stats
 * (lib/models/street_gaussian_model.py:551-571), all sub-models in one pass over the composed index space: for every Gaussian
 * with radii > 0:  max_radii2D = max(max_radii2D, radii);  xyz_gradient_accum[:,0] += |grad.xy|;  [:,1] += |grad.z|;  denom += 1.
 * segments: HOST array, ascending and gap-free like SgrSegment; radii[P] int32 and means2D_grad[P,3] (viewspace_points.grad) device. */
typedef struct SgrStatSegment {
	int32_t start, count;
	float *max_radii2D;         /* [count]    */
	float *xyz_gradient_accum;  /* [count,2]  */
	float *denom;               /* [count,1]  */
} SgrStatSegment;
int sgr_densify_stats(const SgrStatSegment *segments, int32_t num_segments, const int32_t *radii, const float *means2D_grad, void *stream);
/* One multi-tensor Adam step (GaussianModel.update_optimizer -> torch.optim.Adam.step, lib/models/gaussian_model.py:300-303, 316-318:
 * no weight decay, no amsgrad): for each tensor  m <- m + (g - m)(1 - beta1);  v <- beta2 v + (1 - beta2) g^2;
 * param <- param - lr / (1 - beta1^step) * m / (sqrt(v) / sqrt(1 - beta2^step) + eps).  `step` is the 1-based step count AFTER
 * this update (torch increments before use).  betas / eps are doubles because torch forms 1 - beta in Python floats before it
 * rounds to fp32 (1 - 0.999f differs from 0.001f by 1.3e-5 relative).  tensors: HOST array; every pointer device, fp32, `numel` elements. */
typedef struct SgrAdamTensor {
	float *param;
	const float *grad;
	float *exp_avg, *exp_avg_sq;
	int64_t numel;
	float lr;
	int32_t step;
} SgrAdamTensor;
int sgr_adam_step(const SgrAdamTensor *tensors, int32_t num_tensors, double beta1, double beta2, double eps, void *stream);

/* ---- Densification: clone / split / prune with the Adam state, and the opacity reset (SURVEY.md §8 row f3) ----
 * GaussianModelBkgd.densify_and_prune (lib/models/gaussian_model_bkgd.py:74-114) and GaussianModelActor.densify_and_prune
 * (lib/models/gaussian_model_actor.py:204-261) with GaussianModel.densify_and_clone / _split / prune_points / densification_postfix
 * (lib/models/gaussian_model.py:416-520), for every sub-model at once.  Per parent Gaussian of a segment:
 *   g = xyz_gradient_accum[:, grad_col] / denom (NaN -> 0);  s = exp(_scaling);
 *   clone  = |g| >= grad_threshold and max(s) <= dense_threshold  -> appends a copy of the parent's raw rows;
 *   split  =  g  >= grad_threshold and max(s) >  dense_threshold  -> the parent is replaced by 2 children,
 *            xyz = quaternion_to_matrix(_rotation) (z_c * s) + _xyz,  scaling = log(s / 1.6), everything else copied;
 *   prune  (over the rows after clone and split) sigmoid(_opacity) < min_opacity, or with prune_big:
 *            background: max(s_row) > big_threshold unless ||xyz_row - center|| > diameter;
 *            actor:      max(s_row) > big_threshold, or either sample R(normalize(q)) (z (*) s_row) + xyz_row leaves [min_xyz, max_xyz].
 * Output rows of a segment: [kept originals that were not split, kept clones, kept child 0, kept child 1], each section in parent
 * order (the reference's stable order).  Kept originals carry their exp_avg / exp_avg_sq; clones and children get zero moments;
 * the three statistics are zero at the new size.  The thresholds are the fp32 values torch forms (fp32 tensor x Python float).
 * Normal draws: SGR_DENSIFY_DRAWS floats per parent: [0,3) child 0, [3,6) child 1, [6 + 3 (2 r + j), +3) box sample j of row
 * slot r (slot 0: the parent itself or child 0; slot 1: its clone or child 1).  draws == NULL: generated by Philox from
 * (seed, composed parent index); otherwise read from draws[P, SGR_DENSIFY_DRAWS] (device; a test seam). */
#define SGR_DENSIFY_BACKGROUND 0
#define SGR_DENSIFY_ACTOR 1
#define SGR_DENSIFY_TENSORS 7   /* _xyz, _features_dc, _features_rest, _opacity, _scaling, _rotation, _semantic */
#define SGR_DENSIFY_DRAWS 18
#define SGR_DENSIFY_RESULT 8    /* int64 per segment read back by sgr_densify_plan, see below */
typedef struct SgrDensifySegment {
	int32_t kind;            /* SGR_DENSIFY_BACKGROUND / SGR_DENSIFY_ACTOR */
	int32_t count;           /* Gaussians of this sub-model */
	int32_t dc_width;        /* floats per row of _features_dc   (fourier_dim * 3)             */
	int32_t rest_width;      /* floats per row of _features_rest ((M - 1) * 3; 0 -> param NULL)  */
	int32_t semantic_width;  /* floats per row of _semantic      (0 -> param NULL)              */
	int32_t grad_col;        /* column of xyz_gradient_accum: 0, or 1 with densify_grad_abs      */
	int32_t prune_big;
	int32_t reserved;
	float *param[SGR_DENSIFY_TENSORS];       /* device, rows of width 3, dc, rest, 1, 3, 4, semantic */
	float *exp_avg[SGR_DENSIFY_TENSORS];     /* NULL (both moments) when the tensor has no optimizer state */
	float *exp_avg_sq[SGR_DENSIFY_TENSORS];
	float *max_radii2D, *xyz_gradient_accum, *denom;   /* [count], [count,2], [count,1] */
	float grad_threshold, dense_threshold, big_threshold, min_opacity;
	float sphere_center[3], sphere_diameter;  /* background: sphere_center, 2 * sphere_radius */
	float min_xyz[3], max_xyz[3];             /* actor: tracking box */
} SgrDensifySegment;
typedef struct SgrDensifyOutput {     /* the new tensors of one segment, sized by sgr_densify_plan's result */
	int32_t count, reserved;
	float *param[SGR_DENSIFY_TENSORS];
	float *exp_avg[SGR_DENSIFY_TENSORS];      /* NULL exactly where the input's moment is NULL */
	float *exp_avg_sq[SGR_DENSIFY_TENSORS];
	float *max_radii2D, *xyz_gradient_accum, *denom;
} SgrDensifyOutput;
/* Device scratch for a table of num_segments segments holding P Gaussians in all.  plan and apply must get the same scratch. */
size_t sgr_densify_scratch_bytes(int32_t num_segments, int64_t P);
/* Decide every parent's rows, scan them, and copy result[num_segments, SGR_DENSIFY_RESULT] (HOST int64) back in one transfer:
 * {new count, points_total, points_clone, points_split, points_below_min_opacity, points_big_ws, points_pruned, 0}.  This is
 * the only host synchronisation of a densification.  segments: HOST array, every segment's tensors left untouched. */
int sgr_densify_plan(const SgrDensifySegment *segments, int32_t num_segments, uint64_t seed, const float *draws, void *scratch,
                     size_t scratch_bytes, int64_t *result, void *stream);
/* Write the new tensors: same segments, seed, draws and scratch as the plan; outputs: HOST array, outputs[k].count == result[k][0]. */
int sgr_densify_apply(const SgrDensifySegment *segments, const SgrDensifyOutput *outputs, int32_t num_segments, uint64_t seed,
                      const float *draws, void *scratch, size_t scratch_bytes, void *stream);
/* GaussianModel.reset_opacity (lib/models/gaussian_model.py:410-414) in place: _opacity = inverse_sigmoid(min(sigmoid(_opacity), 0.01))
 * and the opacity tensor's exp_avg / exp_avg_sq (when non-NULL) zeroed.  Reads count, param[3], exp_avg[3], exp_avg_sq[3] only. */
int sgr_reset_opacity(const SgrDensifySegment *segments, int32_t num_segments, void *stream);

/* ---- Visibility-masked ("sparse") Adam: an OPT-IN deviation from the reference (no counterpart there) ----
 * One Adam step that updates only the rows of the Gaussians this frame rendered.  Segments are the sub-models in composition order
 * (ascending, gap-free, as for sgr_densify_stats); row l of segment k is VISIBLE iff radii[start_k + l] > 0 (the reference's
 * visibility_filter, street_gaussian_renderer.py:274).  For each tensor a with width[a] > 0:
 *   visible rows:   exactly sgr_adam_step's update (same arithmetic, same rounding: bit-equal), with that tensor's lr and step;
 *   invisible rows: param, exp_avg and exp_avg_sq are not written and grad is not read.
 * `step` is the tensor's 1-based step count after this update, as for sgr_adam_step; there are no per-row step counts.  A tensor with
 * width 0 is not touched (pointers may be NULL); widths above SGR_SPARSE_ADAM_MAX_WIDTH return SGR_EUNSUPPORTED.  Traffic: 4 B per row of radii + 28 B per element of a visible row, rounded up to
 * 32-B sectors; a 256-row tile with no visible row costs only its radii.  No host synchronisation.
 * segments: HOST array; every pointer device, fp32, rows of `width` floats; radii[sum of counts] int32 device.
 * betas / eps are doubles for the same reason as in sgr_adam_step. */
#define SGR_SPARSE_ADAM_MAX_WIDTH 8388607   /* 2^23 - 1 floats per row: a 256-row tile spans fewer than 2^31 floats */
typedef struct SgrSparseAdamSegment {
	int32_t start, count;                       /* range in the composed index space                      */
	float *param[SGR_DENSIFY_TENSORS];          /* _xyz, _features_dc, _features_rest, _opacity, _scaling, _rotation, _semantic */
	const float *grad[SGR_DENSIFY_TENSORS];
	float *exp_avg[SGR_DENSIFY_TENSORS];
	float *exp_avg_sq[SGR_DENSIFY_TENSORS];
	int32_t width[SGR_DENSIFY_TENSORS];         /* floats per row; 0 = not updated by this call           */
	float lr[SGR_DENSIFY_TENSORS];
	int32_t step[SGR_DENSIFY_TENSORS];
	int32_t reserved;
} SgrSparseAdamSegment;
int sgr_sparse_adam_step(const SgrSparseAdamSegment *segments, int32_t num_segments, const int32_t *radii, double beta1, double beta2,
                         double eps, void *stream);

/* present[P] (uint8 0/1) = view-space z > 0.2.  Replaces markVisible -> checkFrustum
 * (DGR/rasterize_points.cu:222-241, rasterizer_impl.cu:54-66, 141-153; pybind `mark_visible`, DGR/ext.cpp:18). */
int sgr_mark_visible(int32_t P, const float *means3D, const float *viewmatrix, const float *projmatrix, uint8_t *present,
                     void *stream);

/* radii[P] and means2D[P,2] only.  Replaces RasterizeGaussiansfilterCUDA -> Rasterizer::visible_filter ->
 * filter_preprocessCUDA (DGR/rasterize_points.cu:243-307, rasterizer_impl.cu:345-392, forward.cu:259-334;
 * pybind `rasterize_gaussians_filter`, DGR/ext.cpp:19).  Both outputs are fully written (zeros when culled). */
int sgr_visible_filter(const SgrFrame *frame, const float *means3D, const float *scales, const float *rotations,
                       const float *cov3D_precomp, int32_t *radii, float *means2D, void *stream);

/* mean squared distance to the 3 nearest neighbours.  Replaces distCUDA2 -> SimpleKNN::knn
 * (KNN/spatial.cu:14-26, KNN/simple_knn.cu:185-220; pybind `distCUDA2`, KNN/ext.cpp:15-17).
 * scratch: sgr_knn_scratch_bytes(P) bytes of caller scratch. */
size_t sgr_knn_scratch_bytes(int32_t P);
int sgr_knn_mean_dist2(int32_t P, const float *points, float *mean_dist2, void *scratch, size_t scratch_bytes,
                       void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SGR_H_INCLUDED */
