"""ctypes loader for libsgr.so (include/sgr.h), and how the package calls it: `call` (device guard, current stream, error
check) and `f32` (the contiguous fp32 form the entries read).  The product path has NO fallback: if the CUDA library is
missing or does not export the ABI, importing / calling raises — it never routes through a CPU implementation.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
from typing import Optional

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsgr.so")
ABI_VERSION = 7

SYMBOLS = ["sgr_abi_version", "sgr_last_error", "sgr_launch_count", "sgr_set_near_budget", "sgr_state_sizes", "sgr_binning_bytes", "sgr_state_layout", "sgr_forward", "sgr_forward_bounded",
           "sgr_forward_status", "sgr_forward_status_async", "sgr_backward_blend",
           "sgr_backward_geom", "sgr_backward", "sgr_mark_visible", "sgr_visible_filter", "sgr_knn_scratch_bytes",
           "sgr_knn_mean_dist2", "sgr_record_bytes", "sgr_project", "sgr_forward_records",
           "sgr_scatter_records", "sgr_gather_grad2d", "sgr_peer_barrier", "sgr_sharded_forward", "sgr_sharded_backward",
           "sgr_sharded_forward_features", "sgr_sharded_backward_features",
           "sgr_sharded_layer_state_sizes", "sgr_sharded_forward_layers", "sgr_sharded_backward_layers",
           "sgr_compose_forward", "sgr_compose_backward", "sgr_image_loss_scratch_bytes", "sgr_image_loss", "sgr_sky_loss",
           "sgr_obj_acc_loss", "sgr_lidar_depth_loss_scratch_bytes", "sgr_lidar_depth_loss", "sgr_densify_stats", "sgr_adam_step",
           "sgr_densify_scratch_bytes", "sgr_densify_plan", "sgr_densify_apply", "sgr_reset_opacity", "sgr_rebalance_row_floats",
           "sgr_rebalance_scratch_bytes", "sgr_rebalance_pack", "sgr_rebalance_splice", "sgr_sparse_adam_step",
           "sgr_layer_state_sizes", "sgr_forward_layer", "sgr_backward_blend_layer", "sgr_backward_geom_layered",
           "sgr_compose_forward_corrected", "sgr_compose_backward_corrected", "sgr_compose_pose_rows", "sgr_compose_backward_rows",
           "sgr_compose_pose_finalize", "sgr_compose_pose_reduce_peers", "sgr_color_correct_forward", "sgr_color_correct_scratch_bytes",
           "sgr_color_correct_backward", "sgr_color_correction_reg", "sgr_sky_composite_forward", "sgr_sky_composite_backward",
           "sgr_actor_pose_forward", "sgr_actor_pose_scratch_bytes", "sgr_actor_pose_backward", "sgr_gaussian_normals_forward",
           "sgr_gaussian_normals_backward", "sgr_compose_semantics_forward", "sgr_compose_semantics_backward", "sgr_finish_features_forward",
           "sgr_finish_features_backward", "sgr_band_halo_rows", "sgr_band_halo_pack", "sgr_band_halo_unpack", "sgr_band_image_loss_stats",
           "sgr_band_image_loss_grad", "sgr_band_sky_loss", "sgr_band_obj_acc_loss", "sgr_band_acc_loss_value", "sgr_band_lidar_scratch_bytes",
           "sgr_band_lidar_keys", "sgr_band_lidar_select", "sgr_band_lidar_grad", "sgr_band_peer_bytes", "sgr_band_halo_exchange_peers",
           "sgr_band_peer_sum", "sgr_band_sky_composite_forward",
           "sgr_band_sky_composite_backward", "sgr_sky_grad_blocks", "sgr_sky_peer_bytes", "sgr_band_sky_composite_backward_marked",
           "sgr_sky_grad_peer_sum", "sgr_band_color_correct_forward", "sgr_band_color_correct_scratch_bytes",
           "sgr_band_color_correct_backward", "sgr_band_color_correct_affine_grad", "sgr_band_finish_features_forward",
           "sgr_band_finish_features_backward", "sgr_eval_metrics_scratch_bytes",
           "sgr_eval_metrics_accumulate", "sgr_band_eval_metrics_accumulate", "sgr_eval_metrics_finish",
           "sgr_band_sky_composite_backward_or_marks", "sgr_sky_grad_peer_sum_union", "sgr_cube_sparse_adam_step",
           "sgr_sky_cube_to_latlong", "sgr_peer_exchange_round"]

SKY_MASK_ACC, SKY_MASK_GIVEN = 0, 1
SEMANTIC_LOGITS, SEMANTIC_PROBABILITIES = 0, 1
MAX_SEMANTIC_BWD = 32  # SGR_MAX_SEMANTIC_BWD: feature channels a backward (and the fused Gaussian-sharded step) takes


class SgrFrame(C.Structure):
    _fields_ = [("P", C.c_int32), ("D", C.c_int32), ("M", C.c_int32), ("S", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("scale_modifier", C.c_float), ("prefiltered", C.c_int32),
                ("debug", C.c_int32), ("row_begin", C.c_int32), ("row_end", C.c_int32), ("row_step", C.c_int32),
                ("bg", C.c_void_p), ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("campos", C.c_void_p)]


# sgr_state_layout: the byte offset of each section of the geom, img and binning states, in carve order, and each state's size
GEOM_SECTIONS = ("rec", "tiles_touched", "depth_key", "iota", "depth_sorted", "perm", "offsets", "big_list", "status", "jac", "ckey", "cval")
IMG_SECTIONS = ("ranges", "tile_max_contrib", "n_contrib", "blend_T", "far_ranges", "split")
BIN_SECTIONS = ("keys_in", "keys_out", "vals_in", "vals_out", "sort_temp", "bucket")


class SgrStateLayout(C.Structure):
    _fields_ = ([(k, C.c_size_t) for k in GEOM_SECTIONS + ("geom_bytes",) + IMG_SECTIONS + ("img_bytes",) + BIN_SECTIONS + ("binning_bytes",)]
                + [("key_bytes", C.c_int32)])


# indices of the status words (SGR_STATUS_*, include/sgr.h)
STATUS_INSTANCES, STATUS_OVERFLOW, STATUS_EMITTED = 1, 2, 3
STATUS_NEAR, STATUS_NEAR_END, STATUS_SPLIT_K, STATUS_SPLIT_FIT, STATUS_FAR_END = 8, 11, 12, 13, 14


MAX_PEERS = 16


class SgrPeers(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32), ("chunk", C.c_int64), ("records", C.c_void_p * MAX_PEERS),
                ("radii", C.c_void_p * MAX_PEERS), ("grad2d", C.c_void_p * MAX_PEERS), ("flags", C.c_void_p * MAX_PEERS),
                ("sem", C.c_void_p * MAX_PEERS), ("gsem", C.c_void_p * MAX_PEERS), ("pose_acc", C.c_void_p * MAX_PEERS),
                ("loss", C.c_void_p * MAX_PEERS), ("loss_bytes", C.c_size_t)]


POSE_ACC_ROWS = 256  # SGR_POSE_ACC_ROWS: rows of 16 floats in a rank's composer accumulator section


MAX_FOURIER = 8


class SgrSegment(C.Structure):
    _fields_ = [("start", C.c_int32), ("count", C.c_int32), ("fourier_dim", C.c_int32), ("posed", C.c_int32), ("xyz", C.c_void_p),
                ("rotation", C.c_void_p), ("scaling", C.c_void_p), ("opacity", C.c_void_p), ("features_dc", C.c_void_p),
                ("features_rest", C.c_void_p)]


class SgrSegmentGrads(C.Structure):
    _fields_ = [("xyz", C.c_void_p), ("rotation", C.c_void_p), ("scaling", C.c_void_p), ("opacity", C.c_void_p), ("features_dc", C.c_void_p),
                ("features_rest", C.c_void_p)]


class SgrStatSegment(C.Structure):
    _fields_ = [("start", C.c_int32), ("count", C.c_int32), ("max_radii2D", C.c_void_p), ("xyz_gradient_accum", C.c_void_p), ("denom", C.c_void_p)]


class SgrAdamTensor(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("numel", C.c_int64),
                ("lr", C.c_float), ("step", C.c_int32)]


DENSIFY_TENSORS = 7   # _xyz, _features_dc, _features_rest, _opacity, _scaling, _rotation, _semantic
DENSIFY_DRAWS = 18
DENSIFY_RESULT = 8
DENSIFY_BACKGROUND, DENSIFY_ACTOR = 0, 1


class SgrDensifySegment(C.Structure):
    _fields_ = [("kind", C.c_int32), ("count", C.c_int32), ("dc_width", C.c_int32), ("rest_width", C.c_int32), ("semantic_width", C.c_int32),
                ("grad_col", C.c_int32), ("prune_big", C.c_int32), ("moments", C.c_int32), ("param", C.c_void_p * DENSIFY_TENSORS),
                ("exp_avg", C.c_void_p * DENSIFY_TENSORS), ("exp_avg_sq", C.c_void_p * DENSIFY_TENSORS), ("max_radii2D", C.c_void_p),
                ("xyz_gradient_accum", C.c_void_p), ("denom", C.c_void_p), ("grad_threshold", C.c_float), ("dense_threshold", C.c_float),
                ("big_threshold", C.c_float), ("min_opacity", C.c_float), ("sphere_center", C.c_float * 3), ("sphere_diameter", C.c_float),
                ("min_xyz", C.c_float * 3), ("max_xyz", C.c_float * 3)]


class SgrDensifyOutput(C.Structure):
    _fields_ = [("count", C.c_int32), ("reserved", C.c_int32), ("param", C.c_void_p * DENSIFY_TENSORS), ("exp_avg", C.c_void_p * DENSIFY_TENSORS),
                ("exp_avg_sq", C.c_void_p * DENSIFY_TENSORS), ("max_radii2D", C.c_void_p), ("xyz_gradient_accum", C.c_void_p), ("denom", C.c_void_p)]


class SgrRebalanceRange(C.Structure):
    _fields_ = [("segment", C.c_int32), ("buffer", C.c_int32), ("src_row", C.c_int32), ("dst_row", C.c_int32), ("rows", C.c_int32),
                ("reserved", C.c_int32)]


SPARSE_ADAM_MAX_WIDTH = 8388607   # floats per row


class SgrPeerPiece(C.Structure):
    _fields_ = [("rank", C.c_int32), ("reserved", C.c_int32), ("offset", C.c_int64), ("floats", C.c_int64), ("local", C.c_void_p)]


class SgrSparseAdamSegment(C.Structure):
    _fields_ = [("start", C.c_int32), ("count", C.c_int32), ("param", C.c_void_p * DENSIFY_TENSORS), ("grad", C.c_void_p * DENSIFY_TENSORS),
                ("exp_avg", C.c_void_p * DENSIFY_TENSORS), ("exp_avg_sq", C.c_void_p * DENSIFY_TENSORS), ("width", C.c_int32 * DENSIFY_TENSORS),
                ("lr", C.c_float * DENSIFY_TENSORS), ("step", C.c_int32 * DENSIFY_TENSORS), ("reserved", C.c_int32)]


class SgrLayer(C.Structure):
    _fields_ = [("begin", C.c_int32), ("end", C.c_int32), ("bg", C.c_void_p)]


MAX_SHARDED_LAYERS = 2  # SGR_MAX_SHARDED_LAYERS: render layers of the fused Gaussian-sharded step


class SgrLayerPeers(C.Structure):
    _fields_ = [("layers", C.c_int32), ("reserved", C.c_int32), ("layer_mask", C.c_void_p * MAX_PEERS), ("layer_grad2d", C.c_void_p * MAX_PEERS)]


class SgrSkyPeers(C.Structure):
    _fields_ = [("sec", C.c_void_p * MAX_PEERS), ("bytes", C.c_size_t)]


class SgrShardedLayer(C.Structure):
    _fields_ = [("begin", C.c_int32), ("end", C.c_int32), ("bg", C.c_void_p), ("state", C.c_void_p), ("state_bytes", C.c_size_t),
                ("color", C.c_void_p), ("depth", C.c_void_p), ("alpha", C.c_void_p), ("dL_dcolor", C.c_void_p), ("dL_ddepth", C.c_void_p),
                ("dL_dalpha", C.c_void_p), ("dL_dmeans2D", C.c_void_p)]


class SgrLayerGrad(C.Structure):
    _fields_ = [("begin", C.c_int32), ("end", C.c_int32), ("grad2d", C.c_void_p), ("dL_dmeans2D", C.c_void_p)]


HALO_SEND_UP, HALO_SEND_DOWN, HALO_RECV_UP, HALO_RECV_DOWN = 0, 1, 2, 3
LIDAR_BINS = 2048
LIDAR_LEVEL0_WORDS = 6 + LIDAR_BINS
PEER_SUM_INT32, PEER_SUM_FLOAT64 = 0, 1  # element types of sgr_band_peer_sum


class SgrLidarState(C.Structure):
    _fields_ = [("n", C.c_uint32), ("k", C.c_uint32), ("prefix", C.c_uint32), ("rank", C.c_uint32), ("sum_lt", C.c_double),
                ("hist", (C.c_uint32 * LIDAR_BINS) * 3)]


EVAL_CLAMP, EVAL_QUANT8, EVAL_SSIM_MASKED, EVAL_NO_SSIM = 1, 2, 4, 8
EVAL_SUMS = 5  # doubles of an SgrEvalSums: abs_diff, sq_diff, ssim, masked, elements


ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)

_lib = None


class SgrError(RuntimeError):
    pass


def lib():
    """Load libsgr.so (once).  Raises if the extension has not been built — there is deliberately no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SgrError(f"{LIB_PATH} not found: build it with `python -m street_gaussians_b200.build` "
                       "(or __graft_entry__.build()); street_gaussians_b200 has no non-CUDA fallback")
    L = C.CDLL(LIB_PATH)
    for s in SYMBOLS:
        if not hasattr(L, s):
            raise SgrError(f"libsgr.so does not export {s}")
    L.sgr_abi_version.restype = C.c_int
    if L.sgr_abi_version() != ABI_VERSION:
        raise SgrError(f"libsgr.so ABI version {L.sgr_abi_version()} != expected {ABI_VERSION}; rebuild")
    L.sgr_last_error.restype = C.c_char_p
    L.sgr_launch_count.restype = C.c_uint64
    L.sgr_launch_count.argtypes = []
    L.sgr_state_sizes.restype = C.c_int
    L.sgr_state_sizes.argtypes = [C.POINTER(SgrFrame), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.sgr_binning_bytes.restype = C.c_size_t
    L.sgr_binning_bytes.argtypes = [C.c_int64]
    L.sgr_state_layout.restype = C.c_int
    L.sgr_state_layout.argtypes = [C.POINTER(SgrFrame), C.c_int64, C.c_int32, C.POINTER(SgrStateLayout)]
    vp = C.c_void_p
    L.sgr_forward.restype = C.c_int
    L.sgr_forward.argtypes = [C.POINTER(SgrFrame)] + [vp] * 8 + [vp] * 5 + [vp, C.c_size_t, vp, C.c_size_t, ALLOC_FN, vp,
                                                                         C.POINTER(vp), C.POINTER(C.c_int64), vp]
    L.sgr_forward_bounded.restype = C.c_int
    L.sgr_forward_bounded.argtypes = [C.POINTER(SgrFrame)] + [vp] * 8 + [vp] * 5 + [vp, C.c_size_t, vp, C.c_size_t, vp, C.c_size_t, C.c_int64, vp]
    L.sgr_forward_status.restype = C.c_int
    L.sgr_forward_status.argtypes = [C.POINTER(SgrFrame), vp, C.POINTER(C.c_int64), C.POINTER(C.c_int32), vp]
    L.sgr_forward_status_async.restype = C.c_int
    L.sgr_forward_status_async.argtypes = [C.POINTER(SgrFrame), vp, vp, vp]
    L.sgr_record_bytes.restype = C.c_size_t
    L.sgr_record_bytes.argtypes = []
    L.sgr_project.restype = C.c_int
    L.sgr_project.argtypes = [C.POINTER(SgrFrame)] + [vp] * 7 + [vp, vp, vp]
    L.sgr_forward_records.restype = C.c_int
    L.sgr_forward_records.argtypes = [C.POINTER(SgrFrame), vp, vp] + [vp] * 4 + [vp, C.c_size_t, vp, C.c_size_t, ALLOC_FN, vp,
                                                                                  C.POINTER(vp), C.POINTER(C.c_int64), vp, C.c_size_t,
                                                                                  C.c_int64, vp]
    L.sgr_scatter_records.restype = C.c_int
    L.sgr_scatter_records.argtypes = [C.POINTER(SgrFrame), C.POINTER(SgrPeers), vp, vp, vp]
    L.sgr_gather_grad2d.restype = C.c_int
    L.sgr_gather_grad2d.argtypes = [C.POINTER(SgrFrame), C.POINTER(SgrPeers), vp, vp, vp, vp]
    L.sgr_peer_barrier.restype = C.c_int
    L.sgr_peer_barrier.argtypes = [C.POINTER(SgrPeers), C.c_uint32, vp]
    L.sgr_sharded_forward.restype = C.c_int
    L.sgr_sharded_forward.argtypes = [C.POINTER(SgrFrame), C.POINTER(SgrPeers)] + [vp] * 7 + [vp] * 3 + [vp, vp, C.c_size_t, vp, C.c_size_t, vp,
                                                                                                C.c_size_t, C.c_int64, C.c_int64, C.c_uint32,
                                                                                                C.c_int32, vp]
    L.sgr_sharded_backward.restype = C.c_int
    L.sgr_sharded_backward.argtypes = [C.POINTER(SgrFrame), C.POINTER(SgrPeers), C.c_int64] + [vp] * 6 + [vp] * 4 + [vp] * 4 + [vp] * 8 + [C.c_uint32, vp]
    L.sgr_sharded_forward_features.restype = C.c_int
    L.sgr_sharded_forward_features.argtypes = L.sgr_sharded_forward.argtypes[:-1] + [vp, vp, vp]
    L.sgr_sharded_backward_features.restype = C.c_int
    L.sgr_sharded_backward_features.argtypes = L.sgr_sharded_backward.argtypes[:-1] + [vp, vp, vp]
    L.sgr_sharded_layer_state_sizes.restype = C.c_int
    L.sgr_sharded_layer_state_sizes.argtypes = [C.POINTER(SgrFrame), C.c_int64, C.POINTER(C.c_size_t)]
    L.sgr_sharded_forward_layers.restype = C.c_int
    L.sgr_sharded_forward_layers.argtypes = L.sgr_sharded_forward.argtypes[:-1] + [C.POINTER(SgrLayerPeers), C.POINTER(SgrShardedLayer), C.c_int32, vp]
    L.sgr_sharded_backward_layers.restype = C.c_int
    L.sgr_sharded_backward_layers.argtypes = L.sgr_sharded_backward.argtypes[:-1] + [C.POINTER(SgrLayerPeers), C.POINTER(SgrShardedLayer), C.c_int32, vp]
    L.sgr_compose_forward.restype = C.c_int
    L.sgr_compose_forward.argtypes = [C.POINTER(SgrSegment), C.c_int32, C.c_int32] + [vp] * 10
    L.sgr_compose_backward.restype = C.c_int
    L.sgr_compose_backward.argtypes = [C.POINTER(SgrSegment), C.POINTER(SgrSegmentGrads), C.c_int32, C.c_int32] + [vp] * 12
    L.sgr_compose_forward_corrected.restype = C.c_int
    L.sgr_compose_forward_corrected.argtypes = [C.POINTER(SgrSegment), C.c_int32, C.c_int32] + [vp] * 11
    L.sgr_compose_backward_corrected.restype = C.c_int
    L.sgr_compose_backward_corrected.argtypes = [C.POINTER(SgrSegment), C.POINTER(SgrSegmentGrads), C.c_int32, C.c_int32] + [vp] * 14
    L.sgr_compose_pose_rows.restype = C.c_int32
    L.sgr_compose_pose_rows.argtypes = [C.c_int32, C.c_int32]
    L.sgr_compose_backward_rows.restype = C.c_int
    L.sgr_compose_backward_rows.argtypes = [C.POINTER(SgrSegment), C.POINTER(SgrSegmentGrads), C.c_int32, C.c_int32] + [vp] * 11 + [C.c_size_t, vp]
    L.sgr_compose_pose_finalize.restype = C.c_int
    L.sgr_compose_pose_finalize.argtypes = [C.POINTER(SgrSegment), C.c_int32] + [vp] * 3 + [C.c_size_t, vp, vp, vp]
    L.sgr_compose_pose_reduce_peers.restype = C.c_int
    L.sgr_compose_pose_reduce_peers.argtypes = [C.POINTER(SgrPeers), C.POINTER(SgrSegment), C.c_int32] + [vp] * 3 + [C.c_size_t, vp, vp, vp]
    L.sgr_color_correct_forward.restype = C.c_int
    L.sgr_color_correct_forward.argtypes = [C.c_int32, C.c_int32, vp, vp, vp, vp]
    L.sgr_color_correct_scratch_bytes.restype = C.c_size_t
    L.sgr_color_correct_scratch_bytes.argtypes = [C.c_int32, C.c_int32]
    L.sgr_color_correct_backward.restype = C.c_int
    L.sgr_color_correct_backward.argtypes = [C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.sgr_color_correction_reg.restype = C.c_int
    L.sgr_color_correction_reg.argtypes = [vp, vp, C.c_float, vp, vp, vp, vp]
    L.sgr_sky_composite_forward.restype = C.c_int
    L.sgr_sky_composite_forward.argtypes = [C.c_int32] * 4 + [C.c_float] + [vp] * 10
    L.sgr_sky_composite_backward.restype = C.c_int
    L.sgr_sky_composite_backward.argtypes = [C.c_int32] * 4 + [C.c_float] + [vp] * 11
    track_table = [C.c_int32, C.c_int32, vp, vp, vp, vp, vp, C.c_int32, vp, vp, vp, vp]
    pose_call = [C.c_int32, vp, C.c_double, C.c_int32, C.c_int32, vp, vp, vp]
    L.sgr_actor_pose_forward.restype = C.c_int
    L.sgr_actor_pose_forward.argtypes = track_table + pose_call + [C.c_int32, C.c_double, C.c_int32, vp, vp, vp]
    L.sgr_actor_pose_scratch_bytes.restype = C.c_size_t
    L.sgr_actor_pose_scratch_bytes.argtypes = [C.c_int32]
    L.sgr_actor_pose_backward.restype = C.c_int
    L.sgr_actor_pose_backward.argtypes = track_table + pose_call + [vp, vp, vp, vp, C.c_size_t, vp]
    L.sgr_gaussian_normals_forward.restype = C.c_int
    L.sgr_gaussian_normals_forward.argtypes = [C.c_int32] + [vp] * 7
    L.sgr_gaussian_normals_backward.restype = C.c_int
    L.sgr_gaussian_normals_backward.argtypes = [C.c_int32] + [vp] * 5
    i32p = C.POINTER(C.c_int32)
    L.sgr_compose_semantics_forward.restype = C.c_int
    L.sgr_compose_semantics_forward.argtypes = [C.c_int32, C.c_int32, C.c_int32, vp, C.c_int32, i32p, i32p, C.POINTER(vp), vp, vp]
    L.sgr_compose_semantics_backward.restype = C.c_int
    L.sgr_compose_semantics_backward.argtypes = [C.c_int32] * 4 + [i32p, i32p, vp, vp, vp, C.POINTER(vp), vp]
    L.sgr_finish_features_forward.restype = C.c_int
    L.sgr_finish_features_forward.argtypes = [C.c_int32] * 5 + [vp] * 4
    L.sgr_finish_features_backward.restype = C.c_int
    L.sgr_finish_features_backward.argtypes = [C.c_int32] * 5 + [vp] * 5
    L.sgr_image_loss_scratch_bytes.restype = C.c_size_t
    L.sgr_image_loss_scratch_bytes.argtypes = [C.c_int32] * 3
    L.sgr_image_loss.restype = C.c_int
    L.sgr_image_loss.argtypes = [C.c_int32] * 3 + [vp, vp, vp, C.c_float, C.c_float, vp, vp, vp, C.c_size_t, vp]
    L.sgr_sky_loss.restype = C.c_int
    L.sgr_sky_loss.argtypes = [C.c_int64, vp, vp, C.c_float, vp, vp, vp, vp]
    L.sgr_obj_acc_loss.restype = C.c_int
    L.sgr_obj_acc_loss.argtypes = [C.c_int64, vp, vp, C.c_float, vp, vp, vp, vp]
    L.sgr_lidar_depth_loss_scratch_bytes.restype = C.c_size_t
    L.sgr_lidar_depth_loss_scratch_bytes.argtypes = [C.c_int64]
    L.sgr_lidar_depth_loss.restype = C.c_int
    L.sgr_lidar_depth_loss.argtypes = [C.c_int64, vp, vp, vp, vp, C.c_double, C.c_float, vp, vp, vp, vp, C.c_size_t, vp]
    band = [C.c_int32] * 3
    L.sgr_band_halo_rows.restype = C.c_int64
    L.sgr_band_halo_rows.argtypes = [C.c_int32] + band + [C.c_int32]
    L.sgr_band_halo_pack.restype = C.c_int
    L.sgr_band_halo_pack.argtypes = [C.c_int32] * 3 + band + [C.c_int32, vp, vp, vp]
    L.sgr_band_halo_unpack.restype = C.c_int
    L.sgr_band_halo_unpack.argtypes = [C.c_int32] * 3 + band + [C.c_int32, vp, vp, vp]
    L.sgr_band_image_loss_stats.restype = C.c_int
    L.sgr_band_image_loss_stats.argtypes = [C.c_int32] * 3 + band + [vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.sgr_band_image_loss_grad.restype = C.c_int
    L.sgr_band_image_loss_grad.argtypes = [C.c_int32] * 3 + band + [vp, vp, vp, C.c_float, C.c_float, vp, vp, vp, vp, C.c_size_t, vp]
    for name in ("sgr_band_sky_loss", "sgr_band_obj_acc_loss"):
        getattr(L, name).restype = C.c_int
        getattr(L, name).argtypes = [C.c_int32] * 2 + band + [vp, vp, C.c_float, vp, vp, vp]
    L.sgr_band_acc_loss_value.restype = C.c_int
    L.sgr_band_acc_loss_value.argtypes = [C.c_int64, C.c_float, vp, vp, vp]
    L.sgr_band_lidar_scratch_bytes.restype = C.c_size_t
    L.sgr_band_lidar_scratch_bytes.argtypes = [C.c_int32] * 2
    L.sgr_band_lidar_keys.restype = C.c_int
    L.sgr_band_lidar_keys.argtypes = [C.c_int32] * 2 + band + [vp] * 5 + [vp, C.c_size_t, vp]
    L.sgr_band_lidar_select.restype = C.c_int
    L.sgr_band_lidar_select.argtypes = [C.c_int32, C.c_double] + [C.c_int32] * 2 + band + [vp, vp, vp, C.c_size_t, vp]
    L.sgr_band_lidar_grad.restype = C.c_int
    L.sgr_band_lidar_grad.argtypes = [C.c_int32] * 2 + band + [vp] * 3 + [C.c_float] + [vp] * 5 + [vp, C.c_size_t, vp]
    L.sgr_band_peer_bytes.restype = C.c_size_t
    L.sgr_band_peer_bytes.argtypes = [C.c_int32] * 3
    L.sgr_band_halo_exchange_peers.restype = C.c_int
    L.sgr_band_halo_exchange_peers.argtypes = [C.POINTER(SgrPeers)] + [C.c_int32] * 3 + band + [vp, vp, vp]
    L.sgr_band_peer_sum.restype = C.c_int
    L.sgr_band_peer_sum.argtypes = [C.POINTER(SgrPeers), C.c_int32, C.c_int64, vp, vp, vp]
    L.sgr_band_sky_composite_forward.restype = C.c_int
    L.sgr_band_sky_composite_forward.argtypes = [C.c_int32] * 2 + band + [C.c_int32] * 2 + [C.c_float] + [vp] * 10
    L.sgr_band_sky_composite_backward.restype = C.c_int
    L.sgr_band_sky_composite_backward.argtypes = [C.c_int32] * 2 + band + [C.c_int32] * 2 + [C.c_float] + [vp] * 11
    L.sgr_sky_grad_blocks.restype = C.c_int64
    L.sgr_sky_grad_blocks.argtypes = [C.c_int32]
    L.sgr_sky_peer_bytes.restype = C.c_size_t
    L.sgr_sky_peer_bytes.argtypes = [C.c_int32]
    L.sgr_band_sky_composite_backward_marked.restype = C.c_int
    L.sgr_band_sky_composite_backward_marked.argtypes = [C.c_int32] * 2 + band + [C.c_int32] * 2 + [C.c_float] + [vp] * 12
    L.sgr_sky_grad_peer_sum.restype = C.c_int
    L.sgr_sky_grad_peer_sum.argtypes = [C.POINTER(SgrPeers), C.POINTER(SgrSkyPeers), C.c_int32, vp, vp, vp]
    L.sgr_band_sky_composite_backward_or_marks.restype = C.c_int
    L.sgr_band_sky_composite_backward_or_marks.argtypes = L.sgr_band_sky_composite_backward_marked.argtypes
    L.sgr_sky_grad_peer_sum_union.restype = C.c_int
    L.sgr_sky_grad_peer_sum_union.argtypes = [C.POINTER(SgrPeers), C.POINTER(SgrSkyPeers), C.c_int32, vp, vp, vp, vp]
    L.sgr_sky_cube_to_latlong.restype = C.c_int
    L.sgr_sky_cube_to_latlong.argtypes = [C.c_int32, vp, C.c_int32, C.c_int32, vp, vp, vp]
    L.sgr_band_color_correct_forward.restype = C.c_int
    L.sgr_band_color_correct_forward.argtypes = [C.c_int32] * 2 + band + [vp] * 4
    L.sgr_band_color_correct_scratch_bytes.restype = C.c_size_t
    L.sgr_band_color_correct_scratch_bytes.argtypes = [C.c_int32] * 2
    L.sgr_band_color_correct_backward.restype = C.c_int
    L.sgr_band_color_correct_backward.argtypes = [C.c_int32] * 2 + band + [vp] * 6 + [C.c_size_t, vp]
    L.sgr_band_color_correct_affine_grad.restype = C.c_int
    L.sgr_band_color_correct_affine_grad.argtypes = [vp] * 3
    L.sgr_band_finish_features_forward.restype = C.c_int
    L.sgr_band_finish_features_forward.argtypes = [C.c_int32] * 5 + band + [vp] * 4
    L.sgr_band_finish_features_backward.restype = C.c_int
    L.sgr_band_finish_features_backward.argtypes = [C.c_int32] * 5 + band + [vp] * 5
    L.sgr_eval_metrics_scratch_bytes.restype = C.c_size_t
    L.sgr_eval_metrics_scratch_bytes.argtypes = [C.c_int32] * 4
    L.sgr_eval_metrics_accumulate.restype = C.c_int
    L.sgr_eval_metrics_accumulate.argtypes = [C.c_int32] * 5 + [vp] * 4 + [vp, C.c_size_t, vp]
    L.sgr_band_eval_metrics_accumulate.restype = C.c_int
    L.sgr_band_eval_metrics_accumulate.argtypes = [C.c_int32] * 4 + band + [C.c_int32] + [vp] * 4 + [vp, C.c_size_t, vp]
    L.sgr_eval_metrics_finish.restype = C.c_int
    L.sgr_eval_metrics_finish.argtypes = [C.c_int32, vp, vp, vp]
    L.sgr_densify_stats.restype = C.c_int
    L.sgr_densify_stats.argtypes = [C.POINTER(SgrStatSegment), C.c_int32, vp, vp, vp]
    L.sgr_adam_step.restype = C.c_int
    L.sgr_adam_step.argtypes = [C.POINTER(SgrAdamTensor), C.c_int32, C.c_double, C.c_double, C.c_double, vp]
    L.sgr_densify_scratch_bytes.restype = C.c_size_t
    L.sgr_densify_scratch_bytes.argtypes = [C.c_int32, C.c_int64]
    L.sgr_densify_plan.restype = C.c_int
    L.sgr_densify_plan.argtypes = [C.POINTER(SgrDensifySegment), C.c_int32, C.c_uint64, vp, vp, C.c_size_t, C.POINTER(C.c_int64), vp]
    L.sgr_densify_apply.restype = C.c_int
    L.sgr_densify_apply.argtypes = [C.POINTER(SgrDensifySegment), C.POINTER(SgrDensifyOutput), C.c_int32, C.c_uint64, vp, vp, C.c_size_t, vp]
    L.sgr_reset_opacity.restype = C.c_int
    L.sgr_reset_opacity.argtypes = [C.POINTER(SgrDensifySegment), C.c_int32, vp]
    L.sgr_rebalance_row_floats.restype = C.c_int64
    L.sgr_rebalance_row_floats.argtypes = [C.POINTER(SgrDensifySegment)]
    L.sgr_rebalance_scratch_bytes.restype = C.c_size_t
    L.sgr_rebalance_scratch_bytes.argtypes = [C.c_int32]
    rebalance_tables = [C.POINTER(SgrRebalanceRange), C.c_int32, C.POINTER(vp), C.POINTER(C.c_int64), C.c_int32, vp, C.c_size_t, vp]
    L.sgr_rebalance_pack.restype = C.c_int
    L.sgr_rebalance_pack.argtypes = [C.POINTER(SgrDensifySegment), C.c_int32] + rebalance_tables
    L.sgr_rebalance_splice.restype = C.c_int
    L.sgr_rebalance_splice.argtypes = [C.POINTER(SgrDensifySegment), C.POINTER(SgrDensifyOutput), C.c_int32] + rebalance_tables
    L.sgr_peer_exchange_round.restype = C.c_int
    L.sgr_peer_exchange_round.argtypes = [C.POINTER(SgrPeers), C.c_size_t, C.POINTER(SgrPeerPiece), C.c_int32, C.POINTER(SgrPeerPiece), C.c_int32, vp]
    L.sgr_sparse_adam_step.restype = C.c_int
    L.sgr_sparse_adam_step.argtypes = [C.POINTER(SgrSparseAdamSegment), C.c_int32, vp, C.c_double, C.c_double, C.c_double, vp]
    L.sgr_cube_sparse_adam_step.restype = C.c_int
    L.sgr_cube_sparse_adam_step.argtypes = [C.c_int32, C.POINTER(SgrAdamTensor), vp, C.c_double, C.c_double, C.c_double, vp]
    L.sgr_layer_state_sizes.restype = C.c_int
    L.sgr_layer_state_sizes.argtypes = [C.POINTER(SgrFrame), C.c_int64, C.POINTER(C.c_size_t)]
    L.sgr_forward_layer.restype = C.c_int
    L.sgr_forward_layer.argtypes = [C.POINTER(SgrFrame), C.POINTER(SgrLayer), C.c_int64, vp, vp, vp, vp, C.c_size_t, vp, vp, vp, vp]
    L.sgr_backward_blend_layer.restype = C.c_int
    L.sgr_backward_blend_layer.argtypes = [C.POINTER(SgrFrame), C.POINTER(SgrLayer)] + [vp] * 8
    L.sgr_backward_geom_layered.restype = C.c_int
    L.sgr_backward_geom_layered.argtypes = [C.POINTER(SgrFrame)] + [vp] * 9 + [C.POINTER(SgrLayerGrad), C.c_int32, vp] + [vp] * 8 + [vp]
    L.sgr_backward_blend.restype = C.c_int
    L.sgr_backward_blend.argtypes = [C.POINTER(SgrFrame), C.c_int64] + [vp] * 12
    L.sgr_backward_geom.restype = C.c_int
    L.sgr_backward_geom.argtypes = [C.POINTER(SgrFrame)] + [vp] * 18
    L.sgr_backward.restype = C.c_int
    L.sgr_backward.argtypes = [C.POINTER(SgrFrame), C.c_int64] + [vp] * 27
    L.sgr_mark_visible.restype = C.c_int
    L.sgr_mark_visible.argtypes = [C.c_int32, vp, vp, vp, vp, vp]
    L.sgr_visible_filter.restype = C.c_int
    L.sgr_visible_filter.argtypes = [C.POINTER(SgrFrame)] + [vp] * 7
    L.sgr_knn_scratch_bytes.restype = C.c_size_t
    L.sgr_knn_scratch_bytes.argtypes = [C.c_int32]
    L.sgr_knn_mean_dist2.restype = C.c_int
    L.sgr_knn_mean_dist2.argtypes = [C.c_int32, vp, vp, vp, C.c_size_t, vp]
    _lib = L
    return L


# sgr_set_near_budget: the library's rule / every instance in one binning pass (the full tile lists render layers are compacted from)
NEAR_BUDGET_AUTO, NEAR_BUDGET_ALL = -1, (1 << 63) - 1


@contextlib.contextmanager
def near_budget(budget: int):
    """The forwards this thread enqueues inside the block use `budget` as the near budget of the saturation split (include/sgr.h,
    sgr_set_near_budget); the previous setting is restored on exit.  Their results do not depend on it."""
    fn = (_lib or lib()).sgr_set_near_budget
    fn.restype, fn.argtypes = C.c_int64, [C.c_int64]
    prev = fn(int(budget))
    try:
        yield
    finally:
        fn(prev)


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().sgr_last_error()
        raise SgrError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")


def ptr(t: Optional[torch.Tensor]):
    """The tensor's device address for a `void*` argument; NULL for None or an empty tensor."""
    if t is None or t.numel() == 0:
        return None
    return C.c_void_p(t.data_ptr())


def stream(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def call(name: str, device, *args) -> None:
    """Call the entry `name` with `args` and raise SgrError if it fails.  With a `device`, the call runs with that device current
    (work the library enqueues and the ALLOC_FN callbacks it makes target it) and gets the device's current stream as its last
    argument.  device=None is for the entries that take no stream (sgr_state_sizes, sgr_state_layout, sgr_layer_state_sizes)."""
    fn = getattr(_lib or lib(), name)
    if device is None:
        rc = fn(*args)
    else:
        with torch.cuda.device(device):
            rc = fn(*args, stream(device))
    check(rc, name)


def f32(t: torch.Tensor, device=None, align16: bool = False) -> torch.Tensor:
    """`t` as a contiguous fp32 tensor, on `device` if one is given; copied only when it has to be.  align16: also copy a view
    whose address is not 16-byte aligned (a contiguous view keeps its storage offset, e.g. a slice of a flat parameter buffer),
    for the arguments the library reads with 16-byte loads (rotation and SH rows, include/sgr.h)."""
    if t.dtype != torch.float32 or (device is not None and t.device != device):
        t = t.to(device=device, dtype=torch.float32)
    t = t.contiguous()
    return t.clone() if align16 and t.data_ptr() % 16 else t
