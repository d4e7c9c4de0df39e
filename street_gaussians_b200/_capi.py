"""ctypes loader for libsgr.so (include/sgr.h).  The product path has NO fallback: if the CUDA library is missing or
does not export the ABI, importing / calling raises — it never routes through a CPU implementation.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsgr.so")
ABI_VERSION = 7

SYMBOLS = ["sgr_abi_version", "sgr_last_error", "sgr_launch_count", "sgr_state_sizes", "sgr_binning_bytes", "sgr_forward", "sgr_forward_bounded",
           "sgr_forward_status", "sgr_forward_status_async", "sgr_backward_blend",
           "sgr_backward_geom", "sgr_backward", "sgr_mark_visible", "sgr_visible_filter", "sgr_knn_scratch_bytes",
           "sgr_knn_mean_dist2", "sgr_record_bytes", "sgr_project", "sgr_forward_records",
           "sgr_scatter_records", "sgr_gather_grad2d", "sgr_peer_barrier", "sgr_sharded_forward", "sgr_sharded_backward",
           "sgr_compose_forward", "sgr_compose_backward", "sgr_image_loss_scratch_bytes", "sgr_image_loss", "sgr_sky_loss",
           "sgr_obj_acc_loss", "sgr_lidar_depth_loss_scratch_bytes", "sgr_lidar_depth_loss", "sgr_densify_stats", "sgr_adam_step",
           "sgr_densify_scratch_bytes", "sgr_densify_plan", "sgr_densify_apply", "sgr_reset_opacity", "sgr_sparse_adam_step",
           "sgr_layer_state_sizes", "sgr_forward_layer", "sgr_backward_blend_layer", "sgr_backward_geom_layered"]


class SgrFrame(C.Structure):
    _fields_ = [("P", C.c_int32), ("D", C.c_int32), ("M", C.c_int32), ("S", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("scale_modifier", C.c_float), ("prefiltered", C.c_int32),
                ("debug", C.c_int32), ("row_begin", C.c_int32), ("row_end", C.c_int32), ("row_step", C.c_int32),
                ("bg", C.c_void_p), ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("campos", C.c_void_p)]


MAX_PEERS = 16


class SgrPeers(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32), ("chunk", C.c_int64), ("records", C.c_void_p * MAX_PEERS),
                ("radii", C.c_void_p * MAX_PEERS), ("grad2d", C.c_void_p * MAX_PEERS), ("flags", C.c_void_p * MAX_PEERS)]


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
                ("grad_col", C.c_int32), ("prune_big", C.c_int32), ("reserved", C.c_int32), ("param", C.c_void_p * DENSIFY_TENSORS),
                ("exp_avg", C.c_void_p * DENSIFY_TENSORS), ("exp_avg_sq", C.c_void_p * DENSIFY_TENSORS), ("max_radii2D", C.c_void_p),
                ("xyz_gradient_accum", C.c_void_p), ("denom", C.c_void_p), ("grad_threshold", C.c_float), ("dense_threshold", C.c_float),
                ("big_threshold", C.c_float), ("min_opacity", C.c_float), ("sphere_center", C.c_float * 3), ("sphere_diameter", C.c_float),
                ("min_xyz", C.c_float * 3), ("max_xyz", C.c_float * 3)]


class SgrDensifyOutput(C.Structure):
    _fields_ = [("count", C.c_int32), ("reserved", C.c_int32), ("param", C.c_void_p * DENSIFY_TENSORS), ("exp_avg", C.c_void_p * DENSIFY_TENSORS),
                ("exp_avg_sq", C.c_void_p * DENSIFY_TENSORS), ("max_radii2D", C.c_void_p), ("xyz_gradient_accum", C.c_void_p), ("denom", C.c_void_p)]


SPARSE_ADAM_MAX_WIDTH = 8388607   # floats per row


class SgrSparseAdamSegment(C.Structure):
    _fields_ = [("start", C.c_int32), ("count", C.c_int32), ("param", C.c_void_p * DENSIFY_TENSORS), ("grad", C.c_void_p * DENSIFY_TENSORS),
                ("exp_avg", C.c_void_p * DENSIFY_TENSORS), ("exp_avg_sq", C.c_void_p * DENSIFY_TENSORS), ("width", C.c_int32 * DENSIFY_TENSORS),
                ("lr", C.c_float * DENSIFY_TENSORS), ("step", C.c_int32 * DENSIFY_TENSORS), ("reserved", C.c_int32)]


class SgrLayer(C.Structure):
    _fields_ = [("begin", C.c_int32), ("end", C.c_int32), ("bg", C.c_void_p)]


class SgrLayerGrad(C.Structure):
    _fields_ = [("begin", C.c_int32), ("end", C.c_int32), ("grad2d", C.c_void_p), ("dL_dmeans2D", C.c_void_p)]


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
    L.sgr_compose_forward.restype = C.c_int
    L.sgr_compose_forward.argtypes = [C.POINTER(SgrSegment), C.c_int32, C.c_int32] + [vp] * 10
    L.sgr_compose_backward.restype = C.c_int
    L.sgr_compose_backward.argtypes = [C.POINTER(SgrSegment), C.POINTER(SgrSegmentGrads), C.c_int32, C.c_int32] + [vp] * 12
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
    L.sgr_sparse_adam_step.restype = C.c_int
    L.sgr_sparse_adam_step.argtypes = [C.POINTER(SgrSparseAdamSegment), C.c_int32, vp, C.c_double, C.c_double, C.c_double, vp]
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


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().sgr_last_error()
        raise SgrError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")
