"""ctypes binding of libb2v.so (the C ABI declared in include/b2v.h).

The product path has NO CPU fallback: if the CUDA library is missing or fails to load, every
entry point raises.  (`pyslam_b200.build.build()` compiles it in-tree with nvcc.)
"""

from __future__ import annotations

import ctypes as C
import os

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_DIR, "libb2v.so")

B2V_OK = 0
B2V_SEM_VOTING, B2V_SEM_PROBABILISTIC, B2V_SEM_MAX_LABELS = 0, 1, 8
B2V_ERR_INVALID_ARGUMENT = 1
B2V_ERR_CUDA = 2
B2V_ERR_CAPACITY = 3
B2V_ERR_UNSUPPORTED = 4
B2V_ASSOC_PENDING = -(1 << 31)   # object id of a pending vote triple (b2v_sgrid_assoc_votes)

BLOCK_SIZE = 8
BLOCK_VOXELS = 512
VOXEL_PLANES = 5

#: every symbol include/b2v.h declares (tests check the library exports all of them)
EXPORTED_SYMBOLS = [
    "b2v_create", "b2v_destroy", "b2v_reset", "b2v_last_error",
    "b2v_integrate_batch", "b2v_integrate_batch_u16", "b2v_synchronize", "b2v_capacity",
    "b2v_num_blocks", "b2v_last_frame_stats", "b2v_last_mesh_stats",
    "b2v_counters", "b2v_set_overlap", "b2v_set_fusion", "b2v_set_group_size", "b2v_set_input_event", "b2v_set_rectification", "b2v_remap", "b2v_profile_enable", "b2v_profile_read", "b2v_export_blocks", "b2v_upload_blocks", "b2v_last_touched_keys", "b2v_block_key_hashes", "b2v_extract_mesh", "b2v_copy_mesh",
    "b2v_extract_points", "b2v_export_halo_device", "b2v_extract_mesh_with_halo",
    "b2v_extract_points_with_halo", "b2v_weld_mesh_device", "b2v_weld_last_error", "b2v_grid_create_ex", "b2v_grid_capacity",
    "b2v_grid_destroy", "b2v_grid_clear",
    "b2v_grid_last_error", "b2v_grid_integrate_ex", "b2v_grid_integrate_rgbd", "b2v_filter_shadow_points", "b2v_grid_synchronize", "b2v_grid_num_blocks",
    "b2v_grid_size", "b2v_grid_get_voxels", "b2v_grid_copy_voxels",
    "b2v_grid_remove_low_count_voxels", "b2v_grid_export_blocks", "b2v_grid_carve",
    "b2v_grid_get_voxels_in_frustum", "b2v_grid_get_voxels_in_bb", "b2v_version", "b2v_device_sm_count", "b2v_selftest_division",
    "b2v_sgrid_create_ex", "b2v_sgrid_capacity", "b2v_sgrid_destroy", "b2v_sgrid_last_error", "b2v_sgrid_clear",
    "b2v_sgrid_set_depth_threshold", "b2v_sgrid_set_depth_decay_rate", "b2v_sgrid_integrate",
    "b2v_sgrid_integrate_rgbd",
    "b2v_sgrid_num_blocks", "b2v_sgrid_get_voxels", "b2v_sgrid_copy_voxels", "b2v_sgrid_get_voxels_in_bb",
    "b2v_sgrid_get_voxels_in_frustum",
    "b2v_sgrid_remove_low_count_voxels", "b2v_sgrid_remove_low_confidence_segments", "b2v_sgrid_merge_segments",
    "b2v_sgrid_remove_segment", "b2v_sgrid_label_overflows", "b2v_sgrid_carve",
    "b2v_sgrid_assign_object_ids_to_instance_ids", "b2v_sgrid_copy_instance_map", "b2v_sgrid_set_next_object_id",
    "b2v_sgrid_get_next_object_id", "b2v_grid_set_rectification", "b2v_grid_set_frame", "b2v_sgrid_set_rectification",
    "b2v_sgrid_set_frame", "b2v_sgrid_remap_instance_ids", "b2v_grid_set_shard", "b2v_sgrid_set_shard",
    "b2v_sgrid_assoc_votes", "b2v_sgrid_copy_assoc_votes", "b2v_sgrid_assoc_resolve",
    "b2v_grid_upload_blocks", "b2v_sgrid_export_blocks", "b2v_sgrid_upload_blocks",
    "b2v_sgrid_set_label_overflow", "b2v_sgrid_label_storage", "b2v_sgrid_export_labels", "b2v_sgrid_upload_labels",
    "b2v_grid_set_input_order_sums",
    "b2v_set_frame_store", "b2v_frame_store_clear", "b2v_frame_store_last", "b2v_frame_store_stats",
    "b2v_integrate_stored",
    *(f"{g}_{n}" for g in ("b2v_grid", "b2v_sgrid")
      for n in ("set_frame_store", "frame_store_clear", "frame_store_last", "frame_store_stats", "stage_stored")),
]


class B2VFrame(C.Structure):
    """`b2v_frame`: the staged images of one frame (device pointers)."""
    _fields_ = [
        ("depth", C.c_void_p),
        ("filtered_depth", C.c_void_p),
        ("color", C.c_void_p),
        ("class_image", C.c_void_p),
        ("instance_image", C.c_void_p),
        ("height", C.c_int32),
        ("width", C.c_int32),
    ]


class B2VConfig(C.Structure):
    _fields_ = [
        ("voxel_size", C.c_float),
        ("block_size", C.c_int32),
        ("sdf_trunc", C.c_float),
        ("depth_trunc", C.c_float),
        ("depth_stride", C.c_int32),
        ("capacity_blocks", C.c_uint32),
        ("device", C.c_int32),
        ("shard_rank", C.c_int32),
        ("shard_count", C.c_int32),
        ("unit_resolution", C.c_int32),
        ("voxel_length", C.c_double),
        ("sdf_trunc_d", C.c_double),
        ("max_capacity_blocks", C.c_uint32),
    ]


class B2VConfigEx(C.Structure):
    """b2v_config with its last field, color_f64 (b2v_version() >= 112).  The field sits in what is B2VConfig's tail
    padding, so both have the header's size, and a B2VConfig (ctypes zero-fills it) creates a float32-colour volume."""
    _fields_ = B2VConfig._fields_ + [("color_f64", C.c_int32)]


_lib = None


def load() -> C.CDLL:
    """Load libb2v.so and declare the prototypes.  Raises RuntimeError when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: the CUDA extension was not built "
            "(run `python -m pyslam_b200.build`); there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, u32 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32
    p_i64 = C.POINTER(C.c_int64)

    L.b2v_version.restype = C.c_int
    L.b2v_device_sm_count.restype = C.c_int
    L.b2v_device_sm_count.argtypes = [i32]
    L.b2v_selftest_division.restype = C.c_int
    L.b2v_selftest_division.argtypes = [i32, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]

    L.b2v_create.restype = C.c_int
    L.b2v_create.argtypes = [C.POINTER(B2VConfigEx), C.POINTER(vp)]
    L.b2v_destroy.restype = C.c_int
    L.b2v_destroy.argtypes = [vp]
    L.b2v_reset.restype = C.c_int
    L.b2v_reset.argtypes = [vp]
    L.b2v_last_error.restype = C.c_char_p
    L.b2v_last_error.argtypes = [vp]
    L.b2v_integrate_batch.restype = C.c_int
    L.b2v_integrate_batch.argtypes = [vp, i32, vp, vp, i32, i32, vp, vp, vp]
    L.b2v_synchronize.restype = C.c_int
    L.b2v_synchronize.argtypes = [vp]
    L.b2v_capacity.restype = C.c_int
    L.b2v_capacity.argtypes = [vp, p_i64, p_i64]
    L.b2v_num_blocks.restype = i64
    L.b2v_num_blocks.argtypes = [vp]
    L.b2v_last_mesh_stats.restype = C.c_int
    L.b2v_last_mesh_stats.argtypes = [vp, vp]
    L.b2v_last_frame_stats.restype = C.c_int
    L.b2v_last_frame_stats.argtypes = [vp, p_i64, p_i64]
    L.b2v_counters.restype = C.c_int
    L.b2v_counters.argtypes = [vp, p_i64, p_i64, p_i64]
    L.b2v_set_overlap.restype = C.c_int
    L.b2v_set_overlap.argtypes = [vp, i32]
    L.b2v_profile_enable.restype = C.c_int
    L.b2v_profile_enable.argtypes = [vp, i32]
    L.b2v_profile_read.restype = C.c_int
    L.b2v_profile_read.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), p_i64, p_i64]
    L.b2v_sgrid_create_ex.restype = C.c_int
    L.b2v_sgrid_create_ex.argtypes = [C.c_double, i32, C.c_uint32, C.c_uint32, i32, i32, C.POINTER(vp)]
    L.b2v_sgrid_capacity.restype = C.c_int
    L.b2v_sgrid_capacity.argtypes = [vp, p_i64, p_i64]
    L.b2v_sgrid_destroy.argtypes = [vp]
    L.b2v_sgrid_last_error.restype = C.c_char_p
    L.b2v_sgrid_last_error.argtypes = [vp]
    L.b2v_sgrid_clear.argtypes = [vp]
    L.b2v_sgrid_set_depth_threshold.argtypes = [vp, C.c_float]
    L.b2v_sgrid_set_depth_decay_rate.argtypes = [vp, C.c_float]
    L.b2v_sgrid_integrate.restype = C.c_int
    L.b2v_sgrid_integrate.argtypes = [vp, C.c_int64, vp, i32, vp, i32, vp, vp, vp]
    L.b2v_sgrid_integrate_rgbd.restype = C.c_int
    L.b2v_sgrid_integrate_rgbd.argtypes = [vp, vp, vp, vp, vp, i32, i32, vp, vp, C.c_float, C.c_float, i32, i32]
    L.b2v_sgrid_carve.restype = C.c_int
    L.b2v_sgrid_carve.argtypes = [vp, vp, i32, i32, vp, C.c_float, C.c_float, vp, C.c_float]
    L.b2v_sgrid_assign_object_ids_to_instance_ids.restype = C.c_int64
    L.b2v_sgrid_assign_object_ids_to_instance_ids.argtypes = [vp, vp, i32, i32, vp, C.c_float, C.c_float, vp, vp, vp,
                                                             C.c_float, i32, C.c_float, i32]
    L.b2v_sgrid_copy_instance_map.argtypes = [vp, vp, vp]
    L.b2v_sgrid_assoc_votes.restype = C.c_int64
    L.b2v_sgrid_assoc_votes.argtypes = [vp, vp, i32, i32, vp, C.c_float, C.c_float, vp, vp, vp, C.c_float, i32]
    L.b2v_sgrid_copy_assoc_votes.restype = C.c_int
    L.b2v_sgrid_copy_assoc_votes.argtypes = [vp, vp]
    L.b2v_sgrid_assoc_resolve.restype = C.c_int64
    L.b2v_sgrid_assoc_resolve.argtypes = [vp, vp, i64, i32, i32, vp, vp, C.c_float, i32]
    L.b2v_sgrid_set_next_object_id.argtypes = [vp, i32]
    L.b2v_sgrid_get_next_object_id.restype = i32
    L.b2v_sgrid_get_next_object_id.argtypes = [vp]
    L.b2v_sgrid_num_blocks.restype = C.c_int64
    L.b2v_sgrid_num_blocks.argtypes = [vp]
    L.b2v_sgrid_get_voxels.restype = C.c_int64
    L.b2v_sgrid_get_voxels.argtypes = [vp, i32, C.c_float]
    L.b2v_sgrid_copy_voxels.argtypes = [vp] * 6
    L.b2v_sgrid_get_voxels_in_bb.restype = C.c_int64
    L.b2v_sgrid_get_voxels_in_bb.argtypes = [vp, vp, i32, C.c_float]
    L.b2v_sgrid_get_voxels_in_frustum.restype = C.c_int64
    L.b2v_sgrid_get_voxels_in_frustum.argtypes = [vp, vp, i32, i32, vp, C.c_float, C.c_float, i32, C.c_float]
    L.b2v_sgrid_remove_low_count_voxels.argtypes = [vp, i32]
    L.b2v_sgrid_remove_low_confidence_segments.argtypes = [vp, i32]
    L.b2v_sgrid_merge_segments.argtypes = [vp, i32, i32]
    L.b2v_sgrid_remove_segment.argtypes = [vp, i32]
    L.b2v_sgrid_label_overflows.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.b2v_sgrid_set_label_overflow.restype = C.c_int
    L.b2v_sgrid_set_label_overflow.argtypes = [vp, C.c_uint64, C.c_uint64]
    L.b2v_sgrid_label_storage.restype = C.c_int
    L.b2v_sgrid_label_storage.argtypes = [vp, p_i64, p_i64, p_i64, p_i64]
    L.b2v_sgrid_export_labels.restype = i64
    L.b2v_sgrid_export_labels.argtypes = [vp] * 5
    L.b2v_sgrid_upload_labels.restype = C.c_int
    L.b2v_sgrid_upload_labels.argtypes = [vp, i64] + [vp] * 5
    L.b2v_integrate_batch_u16.restype = C.c_int
    L.b2v_integrate_batch_u16.argtypes = [vp, i32, vp, C.c_float, vp, i32, i32, vp, vp, vp]
    L.b2v_set_rectification.restype = C.c_int
    L.b2v_set_rectification.argtypes = [vp, vp, vp, i32, i32, i32]
    L.b2v_remap.restype = C.c_int
    L.b2v_remap.argtypes = [vp, i32, i32, i32, vp, vp, vp, i32, i32]
    L.b2v_set_fusion.restype = C.c_int
    L.b2v_set_fusion.argtypes = [vp, i32]
    L.b2v_set_input_event.restype = C.c_int
    L.b2v_set_input_event.argtypes = [vp, vp]
    L.b2v_set_group_size.restype = C.c_int
    L.b2v_set_group_size.argtypes = [vp, i32]
    L.b2v_set_frame_store.restype = C.c_int
    L.b2v_set_frame_store.argtypes = [vp, i32]
    L.b2v_frame_store_clear.restype = C.c_int
    L.b2v_frame_store_clear.argtypes = [vp]
    L.b2v_frame_store_last.restype = C.c_int
    L.b2v_frame_store_last.argtypes = [vp, vp, i32]
    L.b2v_frame_store_stats.restype = C.c_int
    L.b2v_frame_store_stats.argtypes = [vp, p_i64, p_i64]
    L.b2v_integrate_stored.restype = C.c_int
    L.b2v_integrate_stored.argtypes = [vp, i32, vp, vp, vp, vp]
    L.b2v_export_blocks.restype = i64
    L.b2v_export_blocks.argtypes = [vp, vp, vp, i64]
    L.b2v_upload_blocks.restype = C.c_int
    L.b2v_upload_blocks.argtypes = [vp, i64, vp, vp]
    L.b2v_last_touched_keys.restype = i64
    L.b2v_last_touched_keys.argtypes = [vp, vp, i64]
    L.b2v_block_key_hashes.restype = C.c_int
    L.b2v_block_key_hashes.argtypes = [vp, i64, vp]
    L.b2v_extract_mesh.restype = C.c_int
    L.b2v_extract_mesh.argtypes = [vp, p_i64, p_i64]
    L.b2v_copy_mesh.restype = C.c_int
    L.b2v_copy_mesh.argtypes = [vp, vp, vp, vp, vp]
    L.b2v_extract_points.restype = C.c_int
    L.b2v_extract_points.argtypes = [vp, p_i64]
    L.b2v_export_halo_device.restype = C.c_int
    L.b2v_export_halo_device.argtypes = [vp, i32, vp, vp, vp, vp, i64, i64]
    L.b2v_extract_mesh_with_halo.restype = C.c_int
    L.b2v_extract_mesh_with_halo.argtypes = [vp, i64, vp, vp, p_i64, p_i64]
    L.b2v_extract_points_with_halo.restype = C.c_int
    L.b2v_extract_points_with_halo.argtypes = [vp, i64, vp, vp, p_i64]
    L.b2v_weld_mesh_device.restype = C.c_int
    L.b2v_weld_mesh_device.argtypes = [i32, i32, vp, vp] + [vp] * 8 + [p_i64]
    L.b2v_weld_last_error.restype = C.c_char_p
    L.b2v_weld_last_error.argtypes = []

    L.b2v_grid_create_ex.restype = C.c_int
    L.b2v_grid_create_ex.argtypes = [C.c_float, i32, u32, u32, i32, C.POINTER(vp)]
    L.b2v_grid_capacity.restype = C.c_int
    L.b2v_grid_capacity.argtypes = [vp, p_i64, p_i64]
    L.b2v_grid_destroy.restype = C.c_int
    L.b2v_grid_destroy.argtypes = [vp]
    L.b2v_grid_clear.restype = C.c_int
    L.b2v_grid_clear.argtypes = [vp]
    L.b2v_grid_last_error.restype = C.c_char_p
    L.b2v_grid_last_error.argtypes = [vp]
    L.b2v_grid_integrate_ex.restype = C.c_int
    L.b2v_grid_integrate_ex.argtypes = [vp, vp, i32, vp, i32, i64]
    L.b2v_grid_set_input_order_sums.restype = C.c_int
    L.b2v_grid_set_input_order_sums.argtypes = [vp, i32]
    L.b2v_grid_integrate_rgbd.restype = C.c_int
    L.b2v_grid_integrate_rgbd.argtypes = [vp, vp, vp, i32, i32, vp, vp, C.c_float, C.c_float, i32]
    L.b2v_filter_shadow_points.restype = C.c_int
    L.b2v_filter_shadow_points.argtypes = [vp, i32, i32, i32, i32, C.c_float, vp, i32]
    L.b2v_grid_synchronize.restype = C.c_int
    L.b2v_grid_synchronize.argtypes = [vp]
    L.b2v_grid_num_blocks.restype = i64
    L.b2v_grid_num_blocks.argtypes = [vp]
    L.b2v_grid_size.restype = i64
    L.b2v_grid_size.argtypes = [vp]
    L.b2v_grid_get_voxels.restype = i64
    L.b2v_grid_get_voxels.argtypes = [vp, i32]
    L.b2v_grid_copy_voxels.restype = C.c_int
    L.b2v_grid_copy_voxels.argtypes = [vp, vp, vp]
    L.b2v_grid_remove_low_count_voxels.restype = C.c_int
    L.b2v_grid_remove_low_count_voxels.argtypes = [vp, i32]
    L.b2v_grid_carve.restype = C.c_int
    L.b2v_grid_carve.argtypes = [vp, vp, i32, i32, vp, C.c_float, C.c_float, vp, C.c_float]
    L.b2v_grid_get_voxels_in_frustum.restype = i64
    L.b2v_grid_get_voxels_in_frustum.argtypes = [vp, vp, i32, i32, vp, C.c_float, C.c_float, i32]
    L.b2v_grid_get_voxels_in_bb.restype = i64
    L.b2v_grid_get_voxels_in_bb.argtypes = [vp, vp, i32]
    L.b2v_grid_export_blocks.restype = i64
    L.b2v_grid_export_blocks.argtypes = [vp, vp, vp]
    L.b2v_grid_upload_blocks.restype = C.c_int
    L.b2v_grid_upload_blocks.argtypes = [vp, i64, vp, vp]
    L.b2v_sgrid_export_blocks.restype = i64
    L.b2v_sgrid_export_blocks.argtypes = [vp] * 13
    L.b2v_sgrid_upload_blocks.restype = C.c_int
    L.b2v_sgrid_upload_blocks.argtypes = [vp, i64] + [vp] * 12
    for prefix in ("b2v_grid", "b2v_sgrid"):
        fn = getattr(L, prefix + "_set_rectification")
        fn.restype = C.c_int
        fn.argtypes = [vp, vp, vp, i32, i32, i32]
        fn = getattr(L, prefix + "_set_shard")
        fn.restype = C.c_int
        fn.argtypes = [vp, i32, i32]
    L.b2v_grid_set_frame.restype = C.c_int
    L.b2v_grid_set_frame.argtypes = [vp, vp, i32, C.c_float, vp, i32, i32, i32, C.POINTER(B2VFrame)]
    L.b2v_sgrid_set_frame.restype = C.c_int
    L.b2v_sgrid_set_frame.argtypes = [vp, vp, i32, C.c_float, vp, vp, vp, i32, i32, i32, C.POINTER(B2VFrame)]
    for g in ("b2v_grid", "b2v_sgrid"):
        for name, args in (("set_frame_store", [vp, i32]), ("frame_store_clear", [vp]),
                           ("frame_store_last", [vp, C.POINTER(i32)]), ("frame_store_stats", [vp, p_i64, p_i64]),
                           ("stage_stored", [vp, i32, C.POINTER(B2VFrame)])):
            fn = getattr(L, f"{g}_{name}")
            fn.restype = C.c_int
            fn.argtypes = args
    L.b2v_sgrid_remap_instance_ids.restype = C.c_int
    L.b2v_sgrid_remap_instance_ids.argtypes = [vp, C.POINTER(vp)]
    _lib = L
    return L
