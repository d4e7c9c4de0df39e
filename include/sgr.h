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
 *  - shs, rotations and their gradients dL_dsh, dL_drotations must be 16-byte aligned (the kernels move those rows with
 *    16-byte vector accesses); every entry point that takes them returns SGR_EINVAL otherwise.  A fresh allocation is;
 *    a view at an odd float offset into a larger buffer may not be.
 *  - with shs, M >= (D + 1)^2: the active degree never evaluates coefficients that are not stored (SGR_EINVAL otherwise;
 *    the reference reads past the row).  Coefficients beyond (D + 1)^2 are never read and get zero gradient.
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

/* Saturation split of sgr_forward / sgr_forward_bounded (whole-image frames of at most 16384 tiles without semantic channels; other
 * forwards bin in one pass).  The Gaussians whose depth-order instance offsets stay within a budget of B instances are binned and
 * blended first; the farther ones are then binned only into the tiles where some pixel has not saturated (T >= 1e-4), so their
 * instances behind saturated pixels are never emitted.  Images, radii, n_contrib and the tile lists the backward reads do not depend
 * on B; the instances emitted (status word 3) do.  Per calling thread, like sgr_last_error: sgr_set_near_budget sets B for the
 * forwards the thread enqueues from then on and returns the previous setting.  SGR_NEAR_BUDGET_AUTO (any negative value) is the
 * library's rule, a fixed fraction of the frame's instance count; a budget of at least the instance count (SGR_NEAR_BUDGET_ALL)
 * is the one-pass binning, whose tile lists hold every instance — sgr_forward_layer needs those.  A bounded frame overflows only when
 * the instances it emits exceed the capacity; it then keeps the Gaussians whose whole instance counts fit, as the one-pass binning. */
#define SGR_NEAR_BUDGET_AUTO (-1)
#define SGR_NEAR_BUDGET_ALL INT64_MAX
int64_t sgr_set_near_budget(int64_t budget);

/* Sizes (bytes) of the caller-owned forward state.  geom: per-Gaussian records (reference GeometryState,
 * DGR/cuda_rasterizer/rasterizer_impl.h:21-37); img: per-pixel / per-tile state (ImageState, :46-52).
 * binning (BinningState, :54-64) depends on the instance count R and is requested through sgr_alloc_fn;
 * sgr_binning_bytes(R) reports what will be asked for. */
int sgr_state_sizes(const SgrFrame *frame, size_t *geom_bytes, size_t *img_bytes);
size_t sgr_binning_bytes(int64_t num_instances);

/* Byte offsets of the sections of the three forward states, as the library carves them for `frame` and a binning state of
 * num_instances slots (sgr_forward's instance count, or the capacity of a bounded forward: bounded != 0).  Every section starts
 * 256-byte aligned; geom_bytes / img_bytes / binning_bytes are what sgr_state_sizes and sgr_binning_bytes report.  key_bytes is the
 * width of the tile ids in keys_in (2 or 4).  Diagnostic only, like sgr_launch_count: it lets tests and tools read a state without
 * restating its layout (DESIGN.md §3 gives each section's contents).  No reference counterpart. */
typedef struct SgrStateLayout {
	size_t rec, tiles_touched, depth_key, iota, depth_sorted, perm, offsets, big_list, status, jac, ckey, cval, geom_bytes;
	size_t ranges, tile_max_contrib, n_contrib, blend_T, far_ranges, split, img_bytes;
	size_t keys_in, keys_out, vals_in, vals_out, sort_temp, bucket, binning_bytes;
	int32_t key_bytes;
} SgrStateLayout;
int sgr_state_layout(const SgrFrame *frame, int64_t num_instances, int32_t bounded, SgrStateLayout *out);
/* Indices of the u32[64] status words (section `status` of the geom state; zeroed by every forward, words 1-8 are what
 * sgr_forward_status_async copies). */
#define SGR_STATUS_INSTANCES 1    /* instance count R of the frame */
#define SGR_STATUS_OVERFLOW 2     /* overflow bits, as sgr_forward_status reports them */
#define SGR_STATUS_EMITTED 3      /* instances emitted E: the emitted sequence is [0, E) of keys_in / vals_in */
#define SGR_STATUS_NEAR 8         /* saturation split: the near pass's block of four words, laid out like words 0-3 */
#define SGR_STATUS_NEAR_END (SGR_STATUS_NEAR + 3)  /* end E_near of the near pass in the emitted sequence */
#define SGR_STATUS_SPLIT_K 12     /* Gaussians of the near pass, in depth order */
#define SGR_STATUS_SPLIT_FIT 13   /* Gaussians whose whole instance counts fit the capacity */
#define SGR_STATUS_FAR_END 14     /* instances the far pass emitted (E = E_near + this) */

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
 * call's frame, num_instances == the value its backward takes).  That call must have binned every instance: enqueue it with
 * sgr_set_near_budget(SGR_NEAR_BUDGET_ALL).  out_color[3,H,W], out_depth[1,H,W], out_alpha[1,H,W]: every pixel
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
 *   1. sgr_project          on the rank's own Gaussians -> a geom_state for P_local (sgr_state_sizes bytes, NOT P_local *
 *                           sgr_record_bytes()): records[P_local] at its head, the colour Jacobian further in + radii[P_local]
 *   2. caller all-gathers the records (the first P_local*sgr_record_bytes() bytes of that state, padded to chunk) and radii
 *      (NCCL) into the first P_total*sgr_record_bytes() bytes of a geom_state
 *      sized for P_total, and a radii[P_total] array; padding slots must carry radii == 0
 *   3. sgr_forward_records  bins / sorts / blends the rank's tile-row band from the gathered records
 *   4. sgr_backward_blend   (frame.P = P_total) -> partial grad2d[P_total,12]; caller reduce-scatters it
 *   5. sgr_backward_geom    with frame.P = P_local, geom_state = the state step 1 wrote, unchanged (it reads the colour Jacobian
 *                           there), grad2d = its reduced slice.
 * Results are bit-identical to the single-GPU path for the forward images and agree to float summation order in the
 * gradients (tests/test_parity_gpu.py::test_gaussian_sharded_*). */
size_t sgr_record_bytes(void);
/* Step 1.  frame.P = number of local Gaussians; the tile-row band of `frame` is ignored.  Same input rules as
 * sgr_forward.  `records` must be a geom state for frame.P: at least the geom_bytes sgr_state_sizes reports for this frame.  The
 * call writes records[P] at its head (only slots with radii > 0 are meaningful), and with shs the SH colour's direction Jacobian
 * (48 B per visible Gaussian) BEYOND the first P*sgr_record_bytes() bytes, where sgr_backward_geom (step 5) reads it; and
 * radii[P] (all).  A buffer of only P*sgr_record_bytes() bytes is too small. */
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
	float *sem[SGR_MAX_PEERS];          /* feature channels of the fused step (sgr_sharded_*_features only; may be NULL otherwise):  */
	float *gsem[SGR_MAX_PEERS];         /* rank p's sem[world*chunk, S] (delivered semantics) and gsem[world*chunk, S] (its partial
	                                       dL/dsemantics), rows by slot like records and grad2d, mapped into every rank */
	float *pose_acc[SGR_MAX_PEERS];     /* rank p's composer accumulator section: SGR_POSE_ACC_ROWS rows of 16 floats, mapped into every
	                                       rank (sgr_compose_pose_reduce_peers only; may be NULL otherwise) */
	void *loss[SGR_MAX_PEERS];          /* rank p's loss section: loss_bytes bytes, mapped into every rank (sgr_band_halo_exchange_peers /
	                                       sgr_band_peer_sum only; may be NULL otherwise) */
	size_t loss_bytes;                  /* size of every rank's loss section (sgr_band_peer_bytes) */
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
/* The same two calls with feature channels: frame->S in [1, SGR_MAX_SEMANTIC_BWD] and peers->sem / peers->gsem set for every rank.
 * Forward: semantics [frame.P, S] (this rank's own rows) travel with the records — the same block runs, the same slots, in rank d's
 * sem section — and the blend reads them by slot; out_semantic [S, H, W] receives the band's rows (the caller zeroes the others).
 * Backward: the blend writes this band's partial dL/dsemantics rows by slot into the rank's gsem section (which it zeroes first);
 * after the barrier each rank fetches its own Gaussians' rows from the ranks that rendered them, as the same runs, and adds them in
 * ascending rank order into dL_dsemantics [frame.P, S].  No NCCL, no host read-back; the arguments before them are those of
 * sgr_sharded_forward / sgr_sharded_backward. */
int sgr_sharded_forward_features(const SgrFrame *frame, const SgrPeers *peers, const float *means3D, const float *shs, const float *colors_precomp,
                                 const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp,
                                 float *out_color, float *out_depth, float *out_alpha, int32_t *radii_local, void *records_local,
                                 size_t geom_bytes, void *img_state, size_t img_bytes, void *binning_state, size_t binning_bytes,
                                 int64_t capacity, int64_t gaussian_capacity, uint32_t barrier_epoch, int32_t pre_barrier,
                                 const float *semantics, float *out_semantic, void *stream);
int sgr_sharded_backward_features(const SgrFrame *frame, const SgrPeers *peers, int64_t capacity, const float *means3D, const float *shs,
                                  const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                                  const int32_t *radii_local, const void *records_local, const void *img_state, const void *binning_state,
                                  const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                                  float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                                  float *dL_dscales, float *dL_drotations, float *dL_dcov3D, uint32_t barrier_epoch,
                                  const float *dL_dsemantic, float *dL_dsemantics, void *stream);

/* Render layers in the fused Gaussian-sharded step: row ranges of THIS rank's Gaussians rendered on this rank's band from the tile lists
 * of the same call, as sgr_forward_layer does on one GPU.  The tile lists hold slots, which do not give back an owner's row, so layer
 * membership travels with the record: the owner writes one byte per Gaussian (bit k = layer k) by the same block runs into the same
 * slot of layer_peers->layer_mask[d], before the forward's barrier.  Each layer's lists are compacted out of the main lists by that bit, so a
 * rank's layer image equals the band rows of one GPU's separate call on the rank-major concatenation of every rank's layer rows (a
 * layer empty on this rank still shows the other ranks' rows; empty everywhere: colour bg, zero depth and alpha).  Every rank passes
 * the same number of layers (at most SGR_MAX_SHARDED_LAYERS) with the same bg; S must be 0.
 *   sgr_sharded_layer_state_sizes : bytes of ONE layer's caller-owned state (frame.P = local count, `capacity` as in sgr_sharded_forward):
 *                                   its tile lists and contributor counts, and room for the backward's scratch rows (60 B per local
 *                                   Gaussian, used in the first layer's state).  Kept from the forward to its backward.
 *   sgr_sharded_forward_layers    : sgr_sharded_forward plus the layers' images: the band's rows are written, the others left alone.
 *   sgr_sharded_backward_layers   : sgr_sharded_backward plus the layers' gradients.  Each layer with a gradient is blended backward by
 *                                   slot into its part of this rank's layer_grad2d section (the rows of the slots delivered here are
 *                                   zeroed first); after the backward's barrier each owner sums its rows of the main section and of every
 *                                   layer's from the ranks that rendered them, in ascending rank order, as the same runs, and the chain
 *                                   rule runs once on main + layers (as sgr_backward_geom_layered), while dL_dmeans2D gets the main sums
 *                                   only and each layer's sink its own [0:3].  With no layer gradient the call is sgr_sharded_backward.
 * layers: HOST table.  No NCCL, no host read-back, no extra barrier; grids depend on the tile count and chunk only, so the layered step
 * captures in a CUDA graph.  Every argument is checked before anything is enqueued.
 * Every rank must give the same layers an upstream gradient (or none): an owner gathers the layer rows of the other ranks only for the
 * layers that have a gradient on its own call, so a layer with a gradient on one rank and none on another loses that rank's share. */
#define SGR_MAX_SHARDED_LAYERS 2
typedef struct SgrLayerPeers {        /* the layer sections of every rank of the SgrPeers table, mapped into every rank like its arrays */
	int32_t layers;                     /* L: layers every rank's layer_grad2d section holds (SGR_EINVAL when num_layers > L)       */
	int32_t reserved;
	uint8_t *layer_mask[SGR_MAX_PEERS]; /* rank p's layer_mask[world*chunk]: bit k = layer k, rows by slot like the records           */
	float *layer_grad2d[SGR_MAX_PEERS]; /* rank p's layer_grad2d[L, world*chunk, 12] (L >= num_layers): its partial layer rows by slot,
	                                       layer k at k*world*chunk*12 floats                                                           */
} SgrLayerPeers;
typedef struct SgrShardedLayer {
	int32_t begin, end;           /* 0 <= begin <= end <= frame.P (this rank's rows)                                          */
	const float *bg;              /* [3] device                                                                                */
	void *state;                  /* sgr_sharded_layer_state_sizes bytes, device                                               */
	size_t state_bytes;
	float *color, *depth, *alpha; /* [3,H,W], [1,H,W], [1,H,W] device: forward outputs (the backward reads alpha)              */
	const float *dL_dcolor, *dL_ddepth, *dL_dalpha;  /* backward: upstream gradients of the three images, all NULL = none          */
	float *dL_dmeans2D;           /* backward: [end-begin, 3] device or NULL: the layer's own screen-space gradient             */
} SgrShardedLayer;
int sgr_sharded_layer_state_sizes(const SgrFrame *frame, int64_t capacity, size_t *layer_bytes);
int sgr_sharded_forward_layers(const SgrFrame *frame, const SgrPeers *peers, const float *means3D, const float *shs, const float *colors_precomp,
                               const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp, float *out_color,
                               float *out_depth, float *out_alpha, int32_t *radii_local, void *records_local, size_t geom_bytes, void *img_state,
                               size_t img_bytes, void *binning_state, size_t binning_bytes, int64_t capacity, int64_t gaussian_capacity,
                               uint32_t barrier_epoch, int32_t pre_barrier, const SgrLayerPeers *layer_peers, const SgrShardedLayer *layers,
                               int32_t num_layers, void *stream);
int sgr_sharded_backward_layers(const SgrFrame *frame, const SgrPeers *peers, int64_t capacity, const float *means3D, const float *shs,
                                const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                                const int32_t *radii_local, const void *records_local, const void *img_state, const void *binning_state,
                                const float *out_alpha, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                                float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                                float *dL_dscales, float *dL_drotations, float *dL_dcov3D, uint32_t barrier_epoch, const SgrLayerPeers *layer_peers,
                                const SgrShardedLayer *layers, int32_t num_layers, void *stream);

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
/* The same two calls with the learned background pose correction of lib/models/camera_pose.py:89-114
 * (cfg.model.use_pose_correction; street_gaussian_model.py:311-312, 340-341) applied to every segment with posed == 0.
 * bkgd_correction (device, 8 floats): qw qx qy qz tx ty tz pad — the caller's rows pose_correction_rots[id] / pose_correction_trans[id].
 * With q = c / max(|c|, 1e-12) (F.normalize) and R = quaternion_to_matrix(q) (which normalises q once more, with no clamp, so a zero
 * correction gives NaN like the reference): xyz' = R xyz + t and rotation' = q (x) normalize(_rotation), NOT normalised again.
 * Backward: dcorrection (device, 8 floats: d q, d t, 0) receives the gradient of every unposed row, through both normalisations on
 * the matrix path and through F.normalize alone on the rotation path; pose_scratch must hold (num_segments + 1) * 16 floats. */
int sgr_compose_forward_corrected(const SgrSegment *segments, int32_t num_segments, int32_t M, const float *poses, const float *idft,
                                  const uint8_t *flip, const float *flip_quat, const float *bkgd_correction, float *means3D, float *rotations,
                                  float *scales, float *opacities, float *shs, void *stream);
int sgr_compose_backward_corrected(const SgrSegment *segments, const SgrSegmentGrads *grads, int32_t num_segments, int32_t M,
                                   const float *poses, const float *idft, const uint8_t *flip, const float *flip_quat,
                                   const float *bkgd_correction, const float *dL_dmeans3D, const float *dL_drotations, const float *dL_dscales,
                                   const float *dL_dopacities, const float *dL_dshs, float *dposes, float *dcorrection, float *pose_scratch,
                                   void *stream);
/* The composer under Gaussian sharding: each rank composes its own rows of every sub-model (a segment may have count 0) with the
 * replicated poses and correction, so its backward sees one share of the frame's pose and correction terms.  The backward above is
 * split in two around a sum over the ranks:
 *   sgr_compose_backward_rows : the per-row gradients exactly as sgr_compose_backward (bkgd_correction NULL) or
 *                               sgr_compose_backward_corrected write them, and this rank's accumulator rows
 *                               pose_acc[sgr_compose_pose_rows(num_segments, bkgd_correction != NULL), 16] (device, fully written): per
 *                               segment (then one row for the correction) the 16 sums sum g_xyz (x) x_local (9), the rotation path (4),
 *                               sum g_xyz (3) of its rows.
 *   sgr_compose_pose_finalize : dposes[num_segments, 8] and, with bkgd_correction, dcorrection[8] from accumulator rows that already
 *                               hold the frame's sums.  The map is linear in the rows with coefficients from poses / bkgd_correction
 *                               only, so finalizing summed rows equals finalizing the rows of the whole frame up to the order of the
 *                               fp32 additions (which the single-GPU call takes from its atomics).
 *   sgr_compose_pose_reduce_peers : pose_acc on entry holds this rank's rows, on return the frame's sums, added from 0 in ascending rank
 *                               order from every rank's peers->pose_acc section (so every rank computes the same bytes), and dposes /
 *                               dcorrection are finalized from them.  Per group of SGR_POSE_ACC_ROWS rows: the rank's rows are copied
 *                               into its section, device barrier, sum, device barrier (no rank overwrites its section while a peer may
 *                               still read it).  The barriers take the device-side count of sgr_peer_barrier (the fused step's pad).
 *                               No NCCL, no host read-back; every rank must make the call with the same segment table.
 * pose_acc_bytes: the size of pose_acc (SGR_ENOMEM below 64 bytes per row).  Arguments are checked before anything is enqueued. */
#define SGR_POSE_ACC_ROWS 256
int32_t sgr_compose_pose_rows(int32_t num_segments, int32_t corrected);
int sgr_compose_backward_rows(const SgrSegment *segments, const SgrSegmentGrads *grads, int32_t num_segments, int32_t M, const float *poses,
                              const float *idft, const uint8_t *flip, const float *flip_quat, const float *bkgd_correction,
                              const float *dL_dmeans3D, const float *dL_drotations, const float *dL_dscales, const float *dL_dopacities,
                              const float *dL_dshs, float *pose_acc, size_t pose_acc_bytes, void *stream);
int sgr_compose_pose_finalize(const SgrSegment *segments, int32_t num_segments, const float *poses, const float *bkgd_correction,
                              const float *pose_acc, size_t pose_acc_bytes, float *dposes, float *dcorrection, void *stream);
int sgr_compose_pose_reduce_peers(const SgrPeers *peers, const SgrSegment *segments, int32_t num_segments, const float *poses,
                                  const float *bkgd_correction, float *pose_acc, size_t pose_acc_bytes, float *dposes, float *dcorrection,
                                  void *stream);

/* ---- Colour correction (lib/models/color_correction.py:129-140, cfg.model.use_color_correction) ----
 * out[i] = A[i,0] image[0] + A[i,1] image[1] + A[i,2] image[2] + A[i,3] per pixel: the products in einsum's order, then the bias.
 * image, out, dL_dout, dL_dimage: [3,H,W] fp32 device; affine, dL_daffine: [3,4] fp32 device (row-major).
 * Backward: dL_dimage = A^T dL_dout per pixel (may be NULL), dL_daffine[i,j] = sum over pixels of dL_dout[i] [image[j], 1], reduced in
 * a fixed order, so repeated calls give bit-identical results; grid sizes depend on H*W only (no host synchronisation).
 * scratch: sgr_color_correct_scratch_bytes(H, W) bytes. */
int sgr_color_correct_forward(int32_t H, int32_t W, const float *image, const float *affine, float *out, void *stream);
size_t sgr_color_correct_scratch_bytes(int32_t H, int32_t W);
int sgr_color_correct_backward(int32_t H, int32_t W, const float *image, const float *affine, const float *dL_dout, float *dL_dimage,
                               float *dL_daffine, void *scratch, size_t scratch_bytes, void *stream);
/* Regularisation of the colour correction (color_correction.py:134-140 as train.py:135-138 uses it):
 * value (device, 1 float) = weight * mean(|A - I| + |A_sky - I|) over the 12 entries (|A_sky - I| left out when affine_sky is NULL);
 * g_affine / g_affine_sky (device, 12 floats, either may be NULL) = weight / 12 * sign(A - I), 0 where A == I. */
int sgr_color_correction_reg(const float *affine, const float *affine_sky, float weight, float *value, float *g_affine, float *g_affine_sky,
                             void *stream);

/* ---- Sky cube map composite (lib/models/sky_cubemap.py:77-123 at street_gaussian_renderer.py:107-111, model.nsg.include_sky) ----
 * rgb_out = rgb + sky (1 - acc) per pixel.  A pixel of column i, row j looks along Rm^T K^-1 (i + jitter_x, j + jitter_y, 1)
 * (Rm = w2c[:3, :3]; both jitters NULL: 0.5 each).  Pixels the mode selects take the cube map's bilinear lookup with edge wrap
 * (a tap past a cube corner takes the mean of the three taps that exist; DESIGN.md §2), clamped to [0, 1]; the others take `fill`.
 *   SGR_SKY_MASK_ACC    pixels with 1 - acc > 1e-3 (fp32)
 *   SGR_SKY_MASK_GIVEN  pixels with sky_mask != 0, and every pixel of rows 0-49; sky_mask is only read
 * rgb, rgb_out, dL_dout: [3,H,W]; acc, dL_dacc, jitter_x, jitter_y: [H,W]; sky_mask: [H,W] bytes (NULL for SGR_SKY_MASK_ACC);
 * cube_map, dL_dcube: [6,R,R,3] (face 0:+x 1:-x 2:+y 3:-y 4:+z 5:-z, then row, column, channel); K: [3,3]; w2c: [4,4] row-major.
 * All fp32 device memory.  Backward: dL_dacc = -sum_c sky_c dL_dout_c (may be NULL); dL_dcube is ADDED to (the caller zeroes it;
 * may be NULL); dL/drgb is dL_dout itself.  One kernel each way, grid sizes depend on H*W only (no host synchronisation). */
#define SGR_SKY_MASK_ACC 0
#define SGR_SKY_MASK_GIVEN 1
int sgr_sky_composite_forward(int32_t H, int32_t W, int32_t R, int32_t mode, float fill, const float *rgb, const float *acc,
                              const uint8_t *sky_mask, const float *cube_map, const float *K, const float *w2c, const float *jitter_x,
                              const float *jitter_y, float *rgb_out, void *stream);
int sgr_sky_composite_backward(int32_t H, int32_t W, int32_t R, int32_t mode, float fill, const float *acc, const uint8_t *sky_mask,
                               const float *cube_map, const float *K, const float *w2c, const float *jitter_x, const float *jitter_y,
                               const float *dL_dout, float *dL_dacc, float *dL_dcube, void *stream);

/* ---- Tracked actor poses (lib/models/actor_pose.py as StreetGaussianModel.parse_camera uses it, street_gaussian_model.py:257-271) ----
 * poses[a] = (qw, qx, qy, qz, tx, ty, tz) of visible actor a on one camera, the rows sgr_compose_forward takes:
 * matrix_to_quaternion(R_ego) (x) rot and R_ego trans + t_ego, with rot / trans interpolated between the two tracklet entries of the
 * actor's track nearest `timestamp` (ties: the entry first in the track's order), each entry's translation plus opt_trans and its
 * rotation turned by opt_rots about z; with opt_trans / opt_rots given and is_val set, interpolated again between the poses at the two
 * training timestamps of camera `cam` nearest `timestamp` inside the track's span (DESIGN.md §5 lists the reference's quirks kept).
 * idft[a, fourier_dim] (may be NULL) = IDFT(fourier_scale (frame - start_frame) / (end_frame - start_frame), fourier_dim).
 * The track table (device, built once): track t owns entries [track_off[t], track_off[t+1]) of entry_fc [E, 2] int32 (frame, column:
 * the track's argwhere order) and entry_ts [E] float64 (the frame's tracklet timestamp); track_span [T, 2] float64 (start, end
 * timestamp); track_frames [T, 2] int32 (start, end frame); camera c owns cam_ts[cam_off[c], cam_off[c+1]) float64, its training
 * timestamps in order (may be NULL with num_cams == 0).  input_trans [F, K, 3], input_rots [F, K, 4] (w, x, y, z) fp32 device.
 * Per call: tracks (HOST, n_act int32 in [0, num_tracks)); ego_pose [4, 4] row-major fp32 device; opt_trans [F, K, 3] and opt_rots
 * [F, K] fp32 device, both or neither (model.nsg.opt_track); poses [n_act, 7] fp32 device.  Every track used must have >= 2 entries.
 * Backward: dL_dopt_trans / dL_dopt_rots are ADDED to (the caller zeroes them); each actor touches at most 4 rows of each (8 on the
 * validation path), summed per row in actor order so repeated calls agree bit for bit.  scratch: sgr_actor_pose_scratch_bytes(n_act).
 * Grid sizes depend on n_act only and nothing is read back to the host. */
int sgr_actor_pose_forward(int32_t num_tracks, int32_t K, const int32_t *track_off, const int32_t *entry_fc, const double *entry_ts,
                           const double *track_span, const int32_t *track_frames, int32_t num_cams, const int32_t *cam_off, const double *cam_ts,
                           const float *input_trans, const float *input_rots, int32_t n_act, const int32_t *tracks, double timestamp, int32_t cam,
                           int32_t is_val, const float *ego_pose, const float *opt_trans, const float *opt_rots, int32_t frame, double fourier_scale,
                           int32_t fourier_dim, float *poses, float *idft, void *stream);
size_t sgr_actor_pose_scratch_bytes(int32_t n_act);
int sgr_actor_pose_backward(int32_t num_tracks, int32_t K, const int32_t *track_off, const int32_t *entry_fc, const double *entry_ts,
                            const double *track_span, const int32_t *track_frames, int32_t num_cams, const int32_t *cam_off, const double *cam_ts,
                            const float *input_trans, const float *input_rots, int32_t n_act, const int32_t *tracks, double timestamp, int32_t cam,
                            int32_t is_val, const float *ego_pose, const float *opt_trans, const float *opt_rots, const float *dL_dposes,
                            float *dL_dopt_trans, float *dL_dopt_rots, void *scratch, size_t scratch_bytes, void *stream);

/* ---- Feature channels (street_gaussian_renderer.py:206-264: cfg.render.render_normal, cfg.data.use_semantic) ----
 * Per-Gaussian normals (GaussianModel.get_normals, gaussian_model.py:256-269) of the COMPOSED rows sgr_compose_forward writes:
 * n = quaternion_to_matrix(rotations[i])[:, argmin(scales[i])] (the matrix with its own normalisation by sqrt(q.q); the lowest index
 * wins ties, a NaN scale counts as the minimum), kept if sum(-d n) >= 0 with d = (means3D[i] - camera_center) / |...|, else -n (a NaN
 * dot product takes -n).  means3D, scales, normals: [P,3]; rotations, dL_drotations: [P,4] (16-B aligned); camera_center: [3]; all fp32
 * device.  decision: [P] bytes device, written by the forward (bits 0-1 the column, bit 2 the negation) and applied by the backward,
 * which writes dL_drotations (fully written) through both of the matrix's normalisation and the column; the column and the sign
 * pass no gradient, and nothing reaches means3D or scales.  One kernel each way; grids depend on P only. */
int sgr_gaussian_normals_forward(int32_t P, const float *means3D, const float *rotations, const float *scales, const float *camera_center,
                                 float *normals, uint8_t *decision, void *stream);
int sgr_gaussian_normals_backward(int32_t P, const float *rotations, const uint8_t *decision, const float *dL_dnormals, float *dL_drotations,
                                  void *stream);
/* Composed semantics (StreetGaussianModel.get_semantic, street_gaussian_model.py:417-431) over [background, actor_0, ...]:
 *   background rows (bg_semantic [n_bg,K]):   'logits' the rows;  'probabilities' softmax over each row
 *   actor a's rows (actor_semantic[a] [n,1]):  zeros except column class_label[a] = the value ('logits') or its sigmoid
 * Rows come out in compose's order into semantics [n_bg + sum counts, K].  actor_count, class_label (in [0, K)) and the pointer
 * arrays actor_semantic / dL_dactor_semantic are HOST arrays of n_act entries; every tensor is fp32 device.  The backward reads the
 * forward's output `semantics`; dL_dbg (may be NULL) and each dL_dactor_semantic[a] are fully written (dL_dactor_semantic may be NULL).
 * Grids depend on the row counts only. */
#define SGR_SEMANTIC_LOGITS 0
#define SGR_SEMANTIC_PROBABILITIES 1
int sgr_compose_semantics_forward(int32_t K, int32_t mode, int32_t n_bg, const float *bg_semantic, int32_t n_act, const int32_t *actor_count,
                                  const int32_t *class_label, const float *const *actor_semantic, float *semantics, void *stream);
int sgr_compose_semantics_backward(int32_t K, int32_t mode, int32_t n_bg, int32_t n_act, const int32_t *actor_count, const int32_t *class_label,
                                   const float *semantics, const float *dL_dsemantics, float *dL_dbg, float *const *dL_dactor_semantic,
                                   void *stream);
/* Finishing of the rendered feature image rendered [S,H,W] (street_gaussian_renderer.py:245-264), channels [0, normal_channels) the
 * normals (normal_channels 0 or 3) and the K = S - normal_channels others the semantics:
 *   normals [3,H,W]  = x / max(|x|, 1e-12) per pixel (F.normalize(dim=0))
 *   semantic [K,H,W] = 'probabilities' log(x / (sum_c x_c + 1e-8) + 1e-8);  'logits' x
 * normals / semantic may be NULL only where they have no channel.  Backward: dL_drendered [S,H,W] fully written; dL_dnormals and
 * dL_dsemantic may be NULL (zero).  One thread per pixel, one kernel each way. */
int sgr_finish_features_forward(int32_t S, int32_t H, int32_t W, int32_t normal_channels, int32_t mode, const float *rendered, float *normals,
                                float *semantic, void *stream);
int sgr_finish_features_backward(int32_t S, int32_t H, int32_t W, int32_t normal_channels, int32_t mode, const float *rendered,
                                 const float *dL_dnormals, const float *dL_dsemantic, float *dL_drendered, void *stream);

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

/* ---- The same four losses on a tile-row band (multi-GPU: each rank holds the rendered rows of its band, DESIGN.md §8) ----
 * The band is row_begin / row_end / row_step as in SgrFrame (16-pixel tile rows r with row_begin <= r < row_end, (r - row_begin) %
 * row_step == 0; row_begin == row_end is an empty band).  The rendered inputs (image, acc, depth) are [.., H, W] frames of which the
 * band's rows are read (and, for the image, the halo rows); gt, the masks and lidar_depth are whole frames.  Each loss runs in stages
 * with a collective of the caller in between: kernels -> SUM of the partial buffers over the ranks -> kernels.  Every rank then holds
 * the value of the whole frame, and the gradient rows of its band equal those of the single-GPU call bit for bit; the calls write only
 * the band's rows of the gradients (the caller zeroes the rest).
 *
 * Halo: the photometric loss reads the image rows within 10 px of the band.  A rank sends, for each of its tile rows whose neighbour
 * is owned by another rank, 10 rows to that owner: SEND_UP the first rows of the tile row (to the owner of the tile row above),
 * SEND_DOWN its last rows (to the owner of the row below).  It receives RECV_UP, the 10 rows above (the SEND_DOWN of the rank above),
 * and RECV_DOWN, the 10 rows below (the SEND_UP of the rank below); rows past H are dropped.  A buffer is [C][rows][W] fp32, rows =
 * sgr_band_halo_rows(...) (-1 for a bad band or side).  An empty band sends and receives nothing. */
#define SGR_HALO_SEND_UP 0
#define SGR_HALO_SEND_DOWN 1
#define SGR_HALO_RECV_UP 2
#define SGR_HALO_RECV_DOWN 3
int64_t sgr_band_halo_rows(int32_t H, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t side);
int sgr_band_halo_pack(int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t side, const float *image,
                       float *buffer, void *stream);
int sgr_band_halo_unpack(int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t side,
                         const float *buffer, float *image, void *stream);
/* Photometric loss (sgr_image_loss) on a band, image holding the band's rows and its halo.  partials (device, 3 doubles): {sum of the SSIM
 * map, sum of |image - gt| over the masked elements, number of masked pixels} over the band's pixels; stats zeroes and fills them, the
 * caller sums them over the ranks, grad reads the sums.  scratch: sgr_image_loss_scratch_bytes(C, H, W), the same buffer in both calls.
 * scalars: as sgr_image_loss's, of the whole frame. */
int sgr_band_image_loss_stats(int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *image,
                              const float *gt, const uint8_t *mask, double *partials, void *scratch, size_t scratch_bytes, void *stream);
int sgr_band_image_loss_grad(int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *image,
                             const float *gt, const uint8_t *mask, float w_l1, float w_ssim, const double *partials, float *dL_dimage,
                             float *scalars, void *scratch, size_t scratch_bytes, void *stream);
/* Sky and object-accumulation losses on a band: the band's dL_dacc rows (weight / (H W) times the derivative; or NULL) and
 * partial[0] = the sum of the per-pixel losses over the band (device double, zeroed by the call).  After the caller's sum,
 * sgr_band_acc_loss_value writes {weight * mean, mean} with mean = sum / N, N = H W. */
int sgr_band_sky_loss(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *acc, const uint8_t *sky_mask,
                      float weight, float *dL_dacc, double *partial, void *stream);
int sgr_band_obj_acc_loss(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *acc, const uint8_t *obj_bound,
                          float weight, float *dL_dacc, double *partial, void *stream);
int sgr_band_acc_loss_value(int64_t N, float weight, const double *sum, float *scalars, void *stream);
/* LiDAR depth loss on a band: the radix select of sgr_lidar_depth_loss with every histogram summed over the ranks.
 *   keys                      the band's keys, n and the level-0 histogram into *state (zeroed first);  caller sums words
 *                             [0, SGR_LIDAR_LEVEL0_WORDS) of *state: n, the select fields (still zero) and hist[0];
 *   select level 1, 2         select on the summed level l - 1, the band's level-l histogram;  caller sums hist[l];
 *   select level 3            select on the summed level 2 (k, t and the ties to take are now the same on every rank), then
 *                             sums[0] = sum of the errors < t and sums[1 + r] = number of errors == t in tile row r, over the band
 *                             (device doubles [1 + ceil(H / 16)], zeroed by the call);  caller sums `sums`;
 *   grad                      the band's gradient rows (either may be NULL) and scalars {weight * mean, mean, n, k} of the frame.
 * The ties taken are those of lowest flat index over the whole frame: a rank's come after the summed ties of the tile rows above.
 * scratch: sgr_band_lidar_scratch_bytes(H, W), the same buffer in every stage.  H W < 2^31. */
#define SGR_LIDAR_BINS 2048
typedef struct SgrLidarState {
	uint32_t n, k, prefix, rank; /* valid pixels; int(keep n); the selected digits, in the end t; rank of t among them, in the end the ties taken */
	double sum_lt;               /* used by sgr_lidar_depth_loss only */
	uint32_t hist[3][SGR_LIDAR_BINS];
} SgrLidarState;
#define SGR_LIDAR_LEVEL0_WORDS (6 + SGR_LIDAR_BINS)
size_t sgr_band_lidar_scratch_bytes(int32_t H, int32_t W);
int sgr_band_lidar_keys(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *depth, const float *acc,
                        const float *lidar_depth, const uint8_t *mask, SgrLidarState *state, void *scratch, size_t scratch_bytes, void *stream);
int sgr_band_lidar_select(int32_t level, double keep, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step,
                          SgrLidarState *state, double *sums, void *scratch, size_t scratch_bytes, void *stream);
int sgr_band_lidar_grad(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *depth, const float *acc,
                        const float *lidar_depth, float weight, const SgrLidarState *state, const double *sums, float *dL_ddepth,
                        float *dL_dacc, float *scalars, void *scratch, size_t scratch_bytes, void *stream);
/* The band losses' two exchanges over peer memory (the Gaussian-sharded step's SgrPeers, its loss sections and its barrier pad): no NCCL,
 * no host read-back.  Every rank of `peers` makes the same sequence of calls with the same C, H, W (and the same type and count).
 *   sgr_band_halo_exchange_peers : this rank's SEND_UP and SEND_DOWN messages of `image` (sgr_band_halo_pack's [C][rows][W] layout) go
 *                           into its own loss section (SEND_UP at offset 0, SEND_DOWN at half the section's halo part), device barrier,
 *                           then RECV_UP is read from the SEND_DOWN message in the section of rank (rank - 1) % world and RECV_DOWN from
 *                           the SEND_UP message of rank (rank + 1) % world (the neighbours of cyclic and contiguous bands) and written
 *                           into `out` with sgr_band_halo_unpack's mapping, device barrier.  Only the RECV rows of `out` are written;
 *                           `out` may be `image`.  An empty band, or world 1, sends and receives nothing but takes both barriers.
 *   sgr_band_peer_sum      : out[i] = sum over ranks p = 0, 1, .., world - 1 (in that order, from 0) of rank p's local[i]: the local
 *                           array is copied into the rank's loss section, device barrier, every rank adds the sections, device
 *                           barrier.  Every rank computes the same bytes; int32 sums are exact (two's complement), fp64 ones take
 *                           that fixed order.  `out` may be `local`.  count == 0 takes the barriers only.
 * The barriers are sgr_peer_barrier's with the device-side count (epoch 0): two per call, as sgr_compose_pose_reduce_peers takes them.  The
 * second keeps a rank from overwriting its section while a peer may still read it, so the calls may follow each other on a stream.
 * sgr_band_peer_bytes(C, H, W): the loss section both need: the largest pair of halo messages of any band of an image of H rows (two
 * slots of C x 10 ceil(ceil(H / 16) / 2) x W floats) and the largest array the band losses sum (SGR_LIDAR_LEVEL0_WORDS int32, one
 * level of SGR_LIDAR_BINS, 1 + ceil(H / 16) doubles, 5 doubles); 0 for bad sizes.  peers->loss_bytes below it: SGR_ENOMEM.  Arguments
 * are checked before anything is enqueued. */
#define SGR_PEER_SUM_INT32 0
#define SGR_PEER_SUM_FLOAT64 1
size_t sgr_band_peer_bytes(int32_t C, int32_t H, int32_t W);
int sgr_band_halo_exchange_peers(const SgrPeers *peers, int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step,
                                 const float *image, float *out, void *stream);
int sgr_band_peer_sum(const SgrPeers *peers, int32_t type, int64_t count, const void *local, void *out, void *stream);

/* ---- The sky composite and the colour correction on a tile-row band (the stages between the rasterizer and the losses) ----
 * The band and the buffers as in the band losses above: every image argument is a whole [.., H, W] frame of which only the band's pixels
 * are read and written (the caller zeroes the other rows where it needs zeros); sky_mask and the jitters are whole frames.  Each pixel is
 * indexed by its global row and column, so the band's rows of every output equal those of the whole-frame call bit for bit.  Grid sizes
 * depend on H, W (and R) and the band only; nothing is read back to the host.
 * Sky: the arguments of sgr_sky_composite_forward / _backward.  dL_dcube is ADDED to and receives this band's partial sum; the caller
 * sums it over the ranks (its texels' float atomics make it equal to the whole-frame dL_dcube up to their order).
 * Colour correction: the backward writes the band's dL_dimage rows (may be NULL) and partials[12] (device doubles, row-major like the
 * affine) = the band's sums dL_dout_i [image_j, 1], accumulated in double in a fixed order.  The caller sums partials over the ranks,
 * then sgr_band_color_correct_affine_grad rounds the sums to the fp32 dL_daffine[3,4].  scratch: sgr_band_color_correct_scratch_bytes(H, W)
 * bytes (0 for a bad size).  H W < 2^31. */
int sgr_band_sky_composite_forward(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t R, int32_t mode, float fill,
                                   const float *rgb, const float *acc, const uint8_t *sky_mask, const float *cube_map, const float *K,
                                   const float *w2c, const float *jitter_x, const float *jitter_y, float *rgb_out, void *stream);
int sgr_band_sky_composite_backward(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t R, int32_t mode, float fill,
                                    const float *acc, const uint8_t *sky_mask, const float *cube_map, const float *K, const float *w2c,
                                    const float *jitter_x, const float *jitter_y, const float *dL_dout, float *dL_dacc, float *dL_dcube,
                                    void *stream);
int sgr_band_color_correct_forward(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *image, const float *affine,
                                   float *out, void *stream);
size_t sgr_band_color_correct_scratch_bytes(int32_t H, int32_t W);
int sgr_band_color_correct_backward(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, const float *image, const float *affine,
                                    const float *dL_dout, float *dL_dimage, double *partials, void *scratch, size_t scratch_bytes, void *stream);
int sgr_band_color_correct_affine_grad(const double *sums, float *dL_daffine, void *stream);
/* The sky's cube gradient summed over peer memory (the Gaussian-sharded step's SgrPeers for world, rank and the barrier pad, plus every
 * rank's sky section): no NCCL, no host read-back, and only the cube blocks some rank's band touched cross between ranks.  A block is
 * 32 x 32 texels of one face (clipped at the face's last rows and columns when R is not a multiple of 32): sgr_sky_grad_blocks(R) =
 * 6 ceil(R / 32)^2 of them, block b = (face * ceil(R / 32) + row / 32) * ceil(R / 32) + column / 32.
 *   sgr_band_sky_composite_backward_marked : sgr_band_sky_composite_backward (dL_dcube required) that also fills block_map
 *                           [sgr_sky_grad_blocks(R)] bytes: block_map is cleared, then set to 1 at the block of every texel the
 *                           band's atomics add into (taps wrapped onto a neighbouring face included).  Same grid as the unmarked call.
 *   sgr_sky_grad_peer_sum  : in place on this rank's dense partial dL_dcube, which must be zero outside the blocks its block_map marks
 *                           (as the marking backward leaves it on a zeroed dL_dcube).  Stage: the marked blocks and the map go into the
 *                           rank's own section, device barrier.  Owner sum: block b belongs to rank b % world, which adds, for p = 0,
 *                           1, .., world - 1, the block of every rank p that marked it (fp32, from 0.0f) into its own section, device
 *                           barrier.  Gather: every rank copies each block some rank marked from its owner's section into dL_dcube,
 *                           device barrier.  So every rank ends with the same bytes, blocks no rank marked stay zero, and section
 *                           bytes no rank staged in this call are never read.  Three launches of one 256-thread CTA per block (grids
 *                           depend on R only) and three sgr_peer_barrier barriers with the device-side count (epoch 0).
 *   sgr_sky_peer_bytes(R)  : bytes of one rank's sky section: [6 R^2 3 fp32, padded to 256 B | sgr_sky_grad_blocks(R) map bytes],
 *                           padded to 256 B; 0 for a bad R.  sky_peers->bytes below it: SGR_ENOMEM.
 * Every rank of `peers` makes the same calls with the same R.  Sections and dL_dcube must be 16-byte aligned (16-byte loads and
 * stores).  Arguments are checked before anything is enqueued. */
typedef struct SgrSkyPeers {
	void *sec[SGR_MAX_PEERS];           /* rank p's sky section, mapped into every rank */
	size_t bytes;                       /* size of every rank's sky section (sgr_sky_peer_bytes) */
} SgrSkyPeers;
int64_t sgr_sky_grad_blocks(int32_t R);
size_t sgr_sky_peer_bytes(int32_t R);
int sgr_band_sky_composite_backward_marked(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t R, int32_t mode,
                                           float fill, const float *acc, const uint8_t *sky_mask, const float *cube_map, const float *K,
                                           const float *w2c, const float *jitter_x, const float *jitter_y, const float *dL_dout, float *dL_dacc,
                                           float *dL_dcube, uint8_t *block_map, void *stream);
int sgr_sky_grad_peer_sum(const SgrPeers *peers, const SgrSkyPeers *sky_peers, int32_t R, const uint8_t *block_map, float *dL_dcube, void *stream);
/* The marks the block-masked cube Adam (sgr_cube_sparse_adam_step below) consumes, accumulated over backward passes:
 *   sgr_band_sky_composite_backward_or_marks : sgr_band_sky_composite_backward_marked without the clearing: the band's blocks are
 *                           set to 1 in block_map and every other byte keeps its value (the same kernel and grid as the marking call).
 *                           With the band of every tile row (0, ceil(H / 16), 1) its dL_dacc equals sgr_sky_composite_backward's bit
 *                           for bit and its dL_dcube equals it up to the order of the texels' float atomics.
 *   sgr_sky_grad_peer_sum_union : sgr_sky_grad_peer_sum that also sets union_map[b] = 1 (other bytes kept) for every block some rank's
 *                           staged map marks.  The gather reads the union from the staged maps in the ranks' sky sections, so every
 *                           rank writes the same bytes into its own union_map, a [sgr_sky_grad_blocks(R)]-byte device buffer distinct
 *                           from block_map.  No rank can re-mark a staged map before every peer has read it: a section's map is written
 *                           only by its rank's stage launch, the next one comes after this call's last barrier, and every rank reaches
 *                           that barrier only after its gather has read all the maps.  A caller's union_map is never read by a peer. */
int sgr_band_sky_composite_backward_or_marks(int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step, int32_t R, int32_t mode,
                                             float fill, const float *acc, const uint8_t *sky_mask, const float *cube_map, const float *K,
                                             const float *w2c, const float *jitter_x, const float *jitter_y, const float *dL_dout, float *dL_dacc,
                                             float *dL_dcube, uint8_t *block_map, void *stream);
int sgr_sky_grad_peer_sum_union(const SgrPeers *peers, const SgrSkyPeers *sky_peers, int32_t R, const uint8_t *block_map, float *dL_dcube,
                                uint8_t *union_map, void *stream);
/* The cube map as a lat-long image: cubemap_to_latlong (lib/models/sky_cubemap.py:178-191), which SkyCubeMap.save_state_dict
 * (:36-46) writes as sky_latlong.png, without nvdiffrast.  Pixel (row i, column j) of the H x W image samples cube_map [6, R, R, 3] with
 * the composite's lookup (the same taps, weights, edge wrap and corner rule as sgr_sky_composite_forward) along
 *   (sin t sin p, cos t, -sin t cos p),  t = pi gy_i,  p = pi gx_j,  gy = linspace(1/H, 1 - 1/H, H),  gx = linspace(-1 + 1/W, 1 - 1/W, W),
 * every step in fp32 as torch forms the reference's tensors.  latlong [H, W, 3] fp32 (may be NULL) takes the samples unclamped, as the
 * reference returns them; latlong_u8 [H, W, 3] uint8 (may be NULL) takes (uint8)(clamp(v, 0, 1) * 255), the fp32 product truncated, as
 * the reference's astype(np.uint8) (a NaN sample gives 0).  At least one output; no gradient.  One launch, one thread per pixel;
 * 0 < R <= 16384, H, W > 0, H W <= (2^31 - 1) 256.  Device pointers; cube_map is read with 4-byte loads. */
int sgr_sky_cube_to_latlong(int32_t R, const float *cube_map, int32_t H, int32_t W, float *latlong, uint8_t *latlong_u8, void *stream);
/* The feature maps' finishing (sgr_finish_features_forward / _backward) on a tile-row band: the whole-frame calls' arguments plus the
 * band.  rendered, normals, semantic, dL_dnormals, dL_dsemantic and dL_drendered are whole [C, H, W] frames; only the band's pixels are
 * read and written (the caller zeroes the other rows where it needs zeros), each at its frame index, so the band's rows equal the
 * whole-frame call's bit for bit.  The operation is per pixel: no partial sums, nothing for the ranks to exchange.  An empty band
 * launches nothing.  H W < 2^31. */
int sgr_band_finish_features_forward(int32_t S, int32_t H, int32_t W, int32_t normal_channels, int32_t mode, int32_t row_begin, int32_t row_end,
                                     int32_t row_step, const float *rendered, float *normals, float *semantic, void *stream);
int sgr_band_finish_features_backward(int32_t S, int32_t H, int32_t W, int32_t normal_channels, int32_t mode, int32_t row_begin, int32_t row_end,
                                      int32_t row_step, const float *rendered, const float *dL_dnormals, const float *dL_dsemantic,
                                      float *dL_drendered, void *stream);

/* ---- Evaluation metrics: masked L1, PSNR and SSIM of rendered views, value only ----
 * Replaces the scoring of training_report (train.py:274-303: l1_loss and psnr of the clamped render, lib/utils/loss_utils.py:21-37,
 * 61-78) and of metrics.py:76-81 (ssim and psnr of the saved 8-bit PNGs).  Per view, over C channels of H x W:
 *   abs_diff, sq_diff   sum of |x - y| and (x - y)^2 over the masked elements (C x the pixels whose mask byte is non-zero; every
 *                       pixel when mask is NULL), the difference formed in fp64;
 *   masked              the number of masked elements (an integer, exact below 2^53);
 *   ssim                sum of the SSIM map over all C H W elements: the reference's ssim / _ssim (11x11 Gaussian window, sigma 1.5,
 *                       zero padding, C1 = 0.01^2, C2 = 0.03^2, sigma = E[x^2] - mu^2) in fp32, the arithmetic of sgr_image_loss;
 *   elements            C H W (of the band, for the band call).
 * flags (per call):
 *   SGR_EVAL_CLAMP        image and gt clamped to [0, 1] first (training_report); NaN stays NaN;
 *   SGR_EVAL_QUANT8       then the round trip of the PNGs metrics.py reads: torchvision.utils.save_image stores
 *                         uint8(clamp(255 x + 0.5, 0, 255)) (255 x and + 0.5 each rounded in fp32: the nearest level, halves up) and
 *                         to_tensor reads it back as / 255 in fp32 (needs CLAMP);
 *   SGR_EVAL_SSIM_MASKED  SSIM of the images zeroed outside the mask, as ssim(mask=) does; without it SSIM runs on the unmasked images;
 *   SGR_EVAL_NO_SSIM      the SSIM map is not formed (the L1 / PSNR sums only): ssim and elements get nothing added.
 * sgr_eval_metrics_accumulate scores V views (image, gt: [V][C][H][W] fp32 device; mask: uint8 [V][H][W] device or NULL) and ADDS view
 * v's sums to sums[v] (device; the caller zeroes a fresh slot).  No float atomics: each 16 x 16 tile's partial sums are formed in a
 * fixed order and the tiles summed in a fixed order in fp64, so identical calls give identical bits and V views in one call give the
 * bits of V calls of one view.  Nothing is read back to the host; the grids depend on V, C, H, W (and the band) only.
 * scratch: sgr_eval_metrics_scratch_bytes(V, C, H, W) bytes (0 for bad sizes).  V C <= 65535, H W < 2^31.
 *
 * sgr_band_eval_metrics_accumulate: the same sums over the pixels of a tile-row band (as for the band losses above), image holding the
 * band's rows and the rows within 5 px of them (the photometric loss's halo, sgr_band_halo_pack / _unpack, carries them); gt and mask
 * are whole frames.  A tile gives the partials of the whole-frame call's block for that tile, so the sums over the ranks equal the
 * whole-frame sums up to the fp64 regrouping of the tile partials: |difference| <= 2 (T - 1) 2^-53 sum |partials| for T tiles.
 *
 * sgr_eval_metrics_finish: out[V + 1][4] fp32 device: out[v] = {psnr, ssim, l1, n} with mse = sq_diff / masked,
 * psnr = 20 log10(1 / sqrt(mse)), ssim = ssim / elements, l1 = abs_diff / masked, n = masked; out[V] = {the means over the views of
 * the fp32 psnr, ssim and l1 values (summed in fp64), V}.  The reference's edge results are kept: mse = 0 gives psnr = +inf, and an
 * empty mask gives NaN psnr and l1 (0 / 0), which make their means NaN as well.  A view scored only with SGR_EVAL_NO_SSIM has ssim NaN. */
#define SGR_EVAL_CLAMP 1
#define SGR_EVAL_QUANT8 2
#define SGR_EVAL_SSIM_MASKED 4
#define SGR_EVAL_NO_SSIM 8
typedef struct SgrEvalSums {
	double abs_diff, sq_diff, ssim, masked, elements;
} SgrEvalSums;
size_t sgr_eval_metrics_scratch_bytes(int32_t V, int32_t C, int32_t H, int32_t W);
int sgr_eval_metrics_accumulate(int32_t V, int32_t C, int32_t H, int32_t W, int32_t flags, const float *image, const float *gt,
                                const uint8_t *mask, SgrEvalSums *sums, void *scratch, size_t scratch_bytes, void *stream);
int sgr_band_eval_metrics_accumulate(int32_t V, int32_t C, int32_t H, int32_t W, int32_t row_begin, int32_t row_end, int32_t row_step,
                                     int32_t flags, const float *image, const float *gt, const uint8_t *mask, SgrEvalSums *sums,
                                     void *scratch, size_t scratch_bytes, void *stream);
int sgr_eval_metrics_finish(int32_t V, const SgrEvalSums *sums, float *out, void *stream);

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
	int32_t moments;         /* bit a: tensor a carries Adam moments in the rebalance row format (read by sgr_rebalance_* only) */
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

/* ---- Rebalancing Gaussian ownership across ranks (Gaussian-sharded training; no reference counterpart) ----
 * Moves row ranges of every sub-model between ranks together with their Adam moments and densification statistics.  The row
 * format of a segment's tensors, in this order:
 *   param[0..6] (widths 3, dc, rest, 1, 3, 4, semantic; a zero width is skipped), exp_avg[0..6] then exp_avg_sq[0..6] of the
 *   tensors whose bit is set in `moments`, then max_radii2D (1), xyz_gradient_accum (2), denom (1);
 * one range's block holds its `rows` rows tensor after tensor (each tensor's rows contiguous, so every copy is one flat span), i.e.
 * rows x sgr_rebalance_row_floats(segment) floats.  A buffer holds the blocks of the ranges that name it, in table order, from
 * float 0.  Segments: SgrDensifySegment with count, the widths, `moments` and, for count > 0, the pointers of every tensor carried
 * (exp_avg[a] / exp_avg_sq[a] non-NULL exactly where bit a of `moments` is set); kind and the thresholds are not read.  Ranges,
 * segments, buffers and buffer_floats are HOST arrays; the buffers and tensors are device memory.  Each call is ONE kernel that
 * copies every span (none when no range has rows), after one host-to-device copy of its span table into `scratch`.  Traffic: 2 x 4 B
 * per float moved (a read and a write). */
typedef struct SgrRebalanceRange {
	int32_t segment;   /* index into the segment table                                                        */
	int32_t buffer;    /* index into the buffer table; sgr_rebalance_splice only: -1 = the segment's old tensors */
	int32_t src_row;   /* first row read from the segment's old tensors (pack, and splice with buffer -1)      */
	int32_t dst_row;   /* first row written into the new tensors (splice; not read by pack)                    */
	int32_t rows;
	int32_t reserved;
} SgrRebalanceRange;
/* Floats per row of `segment` in a buffer; -1 (and sgr_last_error) for bad widths or moment bits. */
int64_t sgr_rebalance_row_floats(const SgrDensifySegment *segment);
/* Device scratch for the span table of a call with num_ranges ranges. */
size_t sgr_rebalance_scratch_bytes(int32_t num_ranges);
/* Copy rows [src_row, src_row + rows) of every tensor of ranges[i].segment into the block of range i in buffers[ranges[i].buffer].
 * Every range must lie inside its segment's rows and every buffer must hold its blocks (buffer_floats[b] floats). */
int sgr_rebalance_pack(const SgrDensifySegment *segments, int32_t num_segments, const SgrRebalanceRange *ranges, int32_t num_ranges,
                       float *const *buffers, const int64_t *buffer_floats, int32_t num_buffers, void *scratch, size_t scratch_bytes,
                       void *stream);
/* Write the new tensors outputs[k] (count = the segment's new row count; pointers as sgr_densify_apply's outputs, with moments
 * exactly where bit a of segments[k].moments is set): range i fills new rows [dst_row, dst_row + rows) of its segment from its block
 * in buffers[buffer], or with buffer -1 from the segment's old rows [src_row, src_row + rows).  The ranges of each segment must cover
 * its new rows exactly once.  The caller orders them [received from lower ranks | kept | received from higher ranks]. */
int sgr_rebalance_splice(const SgrDensifySegment *segments, const SgrDensifyOutput *outputs, int32_t num_segments, const SgrRebalanceRange *ranges,
                         int32_t num_ranges, const float *const *buffers, const int64_t *buffer_floats, int32_t num_buffers, void *scratch,
                         size_t scratch_bytes, void *stream);

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

/* ---- Block-masked Adam of the sky cube map: an OPT-IN deviation from the reference (whose torch.optim.Adam steps every texel) ----
 * One Adam step of cube->param [6, R, R, 3] (cube->numel must be 6 R^2 3) over the 32 x 32-texel blocks block_map marks, numbered as for
 * sgr_sky_grad_blocks (block_map holds sgr_sky_grad_blocks(R) bytes, any non-zero byte marks):
 *   marked blocks:   exactly sgr_adam_step's update of their texels (same arithmetic, same rounding: bit-equal), with cube->lr and
 *                    cube->step; then the block's byte is set to 0, so the map comes back empty;
 *   unmarked blocks: param, exp_avg and exp_avg_sq are not written and grad is not read.
 * `step` is the 1-based step count after this update, as for sgr_adam_step; there are no per-block step counts.  One launch of one
 * 256-thread CTA per block: the grid depends on R only and nothing is read back, so the call can be captured in a CUDA graph.  Traffic:
 * 1 B per block plus 28 B per float of a marked block.  0 < R <= 16384; pointers are device memory, fp32 (scalar accesses: no alignment
 * beyond 4 B); betas / eps are doubles for the same reason as in sgr_adam_step.  Arguments are checked before anything is enqueued. */
int sgr_cube_sparse_adam_step(int32_t R, const SgrAdamTensor *cube, uint8_t *block_map, double beta1, double beta2, double eps, void *stream);

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
