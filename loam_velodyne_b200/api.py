"""ctypes binding of libloam_b200.so (include/loam_b200.h and include/loam_b200_host.h).

Two layers, both thin:
  * ``Ctx``           -- the kernel-level C ABI (feature extraction, BVH k-NN, LM iterations, voxel grid, transforms)
  * ``ScanRegistration`` / ``LaserOdometry`` / ``LaserMapping`` / ``Pipeline`` -- handles over the C++ drop-in classes
    loam::BasicScanRegistration / BasicLaserOdometry / BasicLaserMapping (same method names as the reference classes).

There is no CPU implementation behind any of this: without the built library the import fails, and without an H100 every
compute call raises ``LoamB200Error``.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# LOAM_B200_LIB: development aid (A/B builds of the same ABI); the product library sits next to this file
LIB_PATH = os.environ.get("LOAM_B200_LIB") or os.path.join(HERE, "libloam_b200.so")

_F = C.POINTER(C.c_float)
_I = C.POINTER(C.c_int)
_B = C.POINTER(C.c_int8)
_D = C.POINTER(C.c_double)


class LoamB200Error(RuntimeError):
    pass


class RegParams(C.Structure):
    _fields_ = [("nFeatureRegions", C.c_int), ("curvatureRegion", C.c_int), ("maxCornerSharp", C.c_int),
                ("maxCornerLessSharp", C.c_int), ("maxSurfaceFlat", C.c_int), ("lessFlatFilterSize", C.c_float),
                ("surfaceCurvatureThreshold", C.c_float)]

    @staticmethod
    def default():
        return RegParams(6, 5, 2, 20, 4, np.float32(0.2), np.float32(0.1))


class Features(C.Structure):
    _fields_ = [("sharp_idx", _I), ("sharp_cap", C.c_int), ("n_sharp", C.c_int),
                ("less_sharp_idx", _I), ("less_sharp_cap", C.c_int), ("n_less_sharp", C.c_int),
                ("flat_idx", _I), ("flat_cap", C.c_int), ("n_flat", C.c_int),
                ("label", _B),
                ("less_flat_ds", _F), ("less_flat_cap", C.c_int), ("n_less_flat", C.c_int)]


class Pose(C.Structure):
    _fields_ = [("rot", C.c_float * 3), ("sin_", C.c_float * 3), ("cos_", C.c_float * 3), ("pos", C.c_float * 3)]


class OdomPose(C.Structure):
    _fields_ = [("rot", C.c_float * 3), ("sin_", C.c_float * 3), ("cos_", C.c_float * 3), ("pos", C.c_float * 3),
                ("inv_scan_period", C.c_float), ("iter", C.c_int)]


class LmResult(C.Structure):
    _fields_ = [("rot", C.c_float * 3), ("pos", C.c_float * 3), ("iterations", C.c_int), ("converged", C.c_int)]


class AlignResult(C.Structure):
    _fields_ = [("rot", C.c_float * 3), ("pos", C.c_float * 3), ("iterations", C.c_int), ("n_selected", C.c_int),
                ("rms", C.c_float), ("degenerate", C.c_int), ("converged", C.c_int)]


class RelocParams(C.Structure):
    """loam_b200_reloc_params; default(): the recommended parameters (LOAM_B200_RELOC_PARAMS_DEFAULT)."""
    _fields_ = [("score_radius", C.c_int), ("coarse_radius", C.c_int), ("fine_radius", C.c_int), ("keep", C.c_int),
                ("max_iterations", C.c_int), ("dedup_m", C.c_float), ("dedup_deg", C.c_float)]

    @staticmethod
    def default():
        return RelocParams(3, 3, 1, 16, 30, np.float32(0.5), np.float32(5.0))


class RelocCandidate(C.Structure):
    _fields_ = [("hypothesis", C.c_int), ("score_selected", C.c_int), ("coarse", AlignResult), ("fine", AlignResult),
                ("selected", C.c_int), ("rms", C.c_float)]


# recommended relocalisation grid (include/loam_b200.h): full circle at 2 deg, 0.4 m steps four to each side of the prior
RELOC_YAW_STEP_DEG, RELOC_XZ_STEP, RELOC_XZ_STEPS = 2.0, 0.4, 4


class PlaceParams(C.Structure):
    """loam_b200_place_params; default(): the recommended parameters (LOAM_B200_PLACE_PARAMS_DEFAULT)."""
    _fields_ = [("rings", C.c_int), ("sectors", C.c_int), ("max_radius", C.c_float), ("height_offset", C.c_float),
                ("min_range", C.c_float), ("max_range", C.c_float)]

    @staticmethod
    def default():
        return PlaceParams(20, 60, np.float32(80.0), np.float32(2.0), np.float32(0.0), np.float32(100.0))


class PlaceMatch(C.Structure):
    _fields_ = [("candidate", C.c_int), ("shift", C.c_int), ("yaw", C.c_float), ("pos", C.c_float * 3),
                ("dist", C.c_double)]


# recommended place spacing and global relocalisation grid (include/loam_b200.h LOAM_B200_PLACE_*)
PLACE_SPACING, PLACE_TOP_M = 4.0, 5
PLACE_YAW_STEP_DEG, PLACE_YAW_STEPS, PLACE_XZ_STEP, PLACE_XZ_STEPS = 2.0, 3, 0.4, 5


# loam_b200_segment as a numpy record (the segment array of dense_segment / segment_cloud is filled in place)
SEGMENT_DTYPE = np.dtype([("size", "<i4"), ("first", "<i4"), ("lo", "<f4", 3), ("hi", "<f4", 3),
                          ("centroid", "<f4", 3)])


class Segment(C.Structure):
    _fields_ = [("size", C.c_int32), ("first", C.c_int32), ("lo", C.c_float * 3), ("hi", C.c_float * 3),
                ("centroid", C.c_float * 3)]


class GroundParams(C.Structure):
    """loam_b200_ground_params; default(): the recommended starting point (DESIGN.md "Ground patches")."""
    _fields_ = [("max_slope_deg", C.c_float), ("max_curvature", C.c_float), ("tol", C.c_float),
                ("max_step", C.c_float), ("min_size", C.c_int)]

    @staticmethod
    def default():
        return GroundParams(np.float32(15.0), np.float32(0.05), np.float32(0.3), np.float32(0.2), 200)


class NormalEq(C.Structure):
    _fields_ = [("AtA", C.c_float * 36), ("AtB", C.c_float * 6), ("n_selected", C.c_int),
                ("n_corner_selected", C.c_int)]


class MapWindow(C.Structure):
    _fields_ = [("cen", C.c_int * 3), ("valid_cubes", _I), ("n_valid", C.c_int), ("corner_leaf", C.c_float),
                ("surf_leaf", C.c_float)]


TREE_ODOM_CORNER, TREE_ODOM_SURF, TREE_MAP_CORNER, TREE_MAP_SURF = range(4)
BUILD_NONE, BUILD_CLUSTER_PAIR, BUILD_CLUSTER, BUILD_MULTI_LAUNCH = range(4)
# cloud slots of the registration and odometry stages (include/loam_b200.h)
(C_REG_FULL, C_REG_SHARP, C_REG_LESS_SHARP, C_REG_FLAT, C_REG_LESS_FLAT, C_ODOM_SHARP, C_ODOM_LESS_SHARP, C_ODOM_FLAT,
 C_ODOM_LESS_FLAT, C_ODOM_FULL, C_ODOM_LAST_CORNER, C_ODOM_LAST_SURF) = range(12)
# cloud slots of the mapping stage (include/loam_b200.h)
(C_MAP_CORNER_LAST, C_MAP_SURF_LAST, C_MAP_FULL, C_MAP_CORNER_STACK_DS, C_MAP_SURF_STACK_DS, C_MAP_CORNER_FROM_MAP,
 C_MAP_SURF_FROM_MAP, C_MAP_SURROUND_DS, C_MAP_CORNER_POOL, C_MAP_SURF_POOL) = range(12, 22)
K_FEATURES, K_TREE_BUILD, K_KNN, K_MAP_ITER, K_ODOM_ITER, K_TRANSFORM, K_VOXEL, K_DENSE = range(8)
KERNEL_FAMILIES = ["features", "tree_build", "knn", "map_iter", "odom_iter", "transform", "voxel", "dense"]
_U = C.POINTER(C.c_uint32)
_U16 = C.POINTER(C.c_uint16)
_LL = C.POINTER(C.c_longlong)
DENSE_MAX_VOXELS = 2**31 - 1  # default cap of the whole-run voxel map: none below the export's int32 count
# recommended carve mode parameters (DESIGN.md "Carve mode"): margin in metres, maximum range in metres
DENSE_CARVE_MARGIN, DENSE_CARVE_MAX_RANGE = 2.0, 100.0

_lib = None


def lib():
    """Load libloam_b200.so (built by ``__graft_entry__.build()`` / ``make -C loam_velodyne_b200/csrc``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LoamB200Error(f"{LIB_PATH} is missing: build it with `make -C loam_velodyne_b200/csrc` "
                            "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    sig = {
        "loam_b200_strerror": (C.c_char_p, [C.c_int]),
        "loam_b200_last_error": (C.c_char_p, [vp]),
        "loam_b200_version": (C.c_int, []),
        "loam_b200_create": (C.c_int, [C.POINTER(vp), C.c_int]),
        "loam_b200_destroy": (C.c_int, [vp]),
        "loam_b200_sync": (C.c_int, [vp]),
        "loam_b200_bind_thread": (C.c_int, [C.c_int]),
        "loam_b200_set_priority": (C.c_int, [vp, C.c_int]),
        "loam_b200_allow_async_capture": (C.c_int, [vp, C.c_int]),
        "loam_b200_stream": (vp, [vp]),
        "loam_b200_extract_features": (C.c_int, [vp, _F, C.c_int, _I, _I, C.c_int, C.POINTER(RegParams),
                                                 C.POINTER(Features)]),
        "loam_b200_tree_build": (C.c_int, [vp, C.c_int, _F, C.c_int]),
        "loam_b200_tree_size": (C.c_int, [vp, C.c_int]),
        "loam_b200_tree_knn": (C.c_int, [vp, C.c_int, _F, C.c_int, C.c_int, C.c_float, _I, _F]),
        "loam_b200_map_set_queries": (C.c_int, [vp, _F, C.c_int, _F, C.c_int]),
        "loam_b200_map_iterate": (C.c_int, [vp, C.POINTER(Pose), C.POINTER(NormalEq)]),
        "loam_b200_map_iterate_debug": (C.c_int, [vp, C.POINTER(Pose), C.POINTER(NormalEq), _F, _B]),
        "loam_b200_map_iterate_stats": (C.c_int, [vp, C.POINTER(Pose), C.POINTER(NormalEq), C.POINTER(C.c_ulonglong),
                                          C.POINTER(C.c_ulonglong)]),
        "loam_b200_odom_set_last": (C.c_int, [vp, _F, C.c_int, _F, C.c_int]),
        "loam_b200_odom_set_current": (C.c_int, [vp, _F, C.c_int, _F, C.c_int]),
        "loam_b200_odom_solve": (C.c_int, [vp, _F, _F, C.c_float, C.c_int, C.c_float, C.c_float, C.POINTER(LmResult)]),
        "loam_b200_map_solve": (C.c_int, [vp, _F, _F, C.c_int, C.c_float, C.c_float, C.POINTER(LmResult)]),
        "loam_b200_odom_iterate": (C.c_int, [vp, C.POINTER(OdomPose), C.POINTER(NormalEq)]),
        "loam_b200_odom_iterate_debug": (C.c_int, [vp, C.POINTER(OdomPose), C.POINTER(NormalEq), _F, _B, _I]),
        "loam_b200_debug_gn_solve": (C.c_int, [vp, _F, C.c_int, C.c_int, C.c_float, _F, _I]),
        "loam_b200_debug_sort_pairs": (C.c_int, [vp, _U, _I, C.c_int, C.c_int, C.c_int, C.c_int, _U, _I, _I]),
        "loam_b200_transform_to_end": (C.c_int, [vp, _F, C.c_int, C.POINTER(OdomPose)]),
        "loam_b200_transform_to_map": (C.c_int, [vp, _F, C.c_int, C.POINTER(Pose)]),
        "loam_b200_voxel_grid": (C.c_int, [vp, _F, C.c_int, C.c_float, _F, C.c_int, _I]),
        "loam_b200_cloud_upload": (C.c_int, [vp, C.c_int, _F, C.c_int]),
        "loam_b200_cloud_upload_device": (C.c_int, [vp, C.c_int, vp, C.c_int]),
        "loam_b200_cloud_download": (C.c_int, [vp, C.c_int, _F, C.c_int, _I]),
        "loam_b200_cloud_size": (C.c_int, [vp, C.c_int]),
        "loam_b200_cloud_swap": (C.c_int, [vp, C.c_int, C.c_int]),
        "loam_b200_cloud_copy_many": (C.c_int, [vp, _I, vp, _I, C.c_int]),
        "loam_b200_cloud_copy": (C.c_int, [vp, C.c_int, vp, C.c_int]),
        "loam_b200_reg_bin": (C.c_int, [vp, _F, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float, _I, _I]),
        "loam_b200_reg_run": (C.c_int, [vp, _I, _I, C.c_int, C.POINTER(RegParams), _I]),
        "loam_b200_reg_indices": (C.c_int, [vp, C.c_int, _I, C.c_int, _I]),
        "loam_b200_reg_labels": (C.c_int, [vp, _B, C.c_int]),
        "loam_b200_odom_prepare": (C.c_int, [vp]),
        "loam_b200_odom_adopt": (C.c_int, [vp, vp, _I]),
        "loam_b200_cloud_transform_to_end2": (C.c_int, [vp, C.c_int, C.c_int, C.POINTER(OdomPose)]),
        "loam_b200_odom_rebuild_last": (C.c_int, [vp]),
        "loam_b200_cloud_transform_to_end": (C.c_int, [vp, C.c_int, C.POINTER(OdomPose)]),
        "loam_b200_cloud_transform_to_map": (C.c_int, [vp, C.c_int, C.POINTER(Pose)]),
        "loam_b200_map_pool_append": (C.c_int, [vp, C.c_int, _F, C.c_int]),
        "loam_b200_map_begin_sweep": (C.c_int, [vp, C.POINTER(Pose), C.POINTER(MapWindow), _I]),
        "loam_b200_map_end_sweep": (C.c_int, [vp, C.POINTER(Pose)]),
        "loam_b200_map_end_sweep_async": (C.c_int, [vp, C.POINTER(Pose)]),
        "loam_b200_map_surround": (C.c_int, [vp, _I, _I, C.c_int, C.c_float]),
        "loam_b200_map_surround_async": (C.c_int, [vp, _I, _I, C.c_int, C.c_float]),
        "loam_b200_map_debug_from_map": (C.c_int, [vp, C.c_int]),
        "loam_b200_debug_map_prune": (C.c_int, [vp, C.c_int]),
        "loam_b200_debug_odom_ring_ranges": (C.c_int, [vp, C.c_int]),
        "loam_b200_debug_tree_build_path": (C.c_int, [vp, C.c_int]),
        "loam_b200_dense_enable": (C.c_int, [vp, C.c_float, C.c_longlong]),
        "loam_b200_dense_insert": (C.c_int, [vp, C.c_int]),
        "loam_b200_dense_stats": (C.c_int, [vp, _LL]),
        "loam_b200_dense_export": (C.c_int, [vp, _F, _U, C.c_int, _I]),
        "loam_b200_dense_clear": (C.c_int, [vp]),
        "loam_b200_dense_visibility": (C.c_int, [vp, C.c_double, C.c_double, C.c_double]),
        "loam_b200_dense_observe": (C.c_int, [vp, C.c_int, C.POINTER(Pose)]),
        "loam_b200_dense_carving": (C.c_int, [vp, C.c_double, C.c_double]),
        "loam_b200_dense_export_filtered": (C.c_int, [vp, C.c_double, _F, _U, _U16, _U16, C.c_int, _I]),
        "loam_b200_dense_export_normals": (C.c_int, [vp, C.c_double, C.c_int, _D, _F, _U, _F, C.c_int, _I]),
        "loam_b200_debug_dense_table_slots": (C.c_int, [vp, _LL]),
        "loam_b200_debug_dense_carve_index": (C.c_int, [vp, C.POINTER(C.c_uint64), C.c_longlong, _LL]),
        "loam_b200_dense_snapshot": (C.c_int, [vp, C.POINTER(C.c_uint64), _U, _U16, _U16, _D, C.c_int, _I]),
        "loam_b200_dense_merge": (C.c_int, [vp, _U, _U16, _U16, _D, C.c_int, C.POINTER(Pose)]),
        "loam_b200_dense_target_build": (C.c_int, [vp, C.c_double, C.c_int, _D, _I]),
        "loam_b200_dense_target_load": (C.c_int, [vp, C.c_float, _F, _F, C.c_int]),
        "loam_b200_dense_align_iterate": (C.c_int, [vp, _F, C.c_int, C.c_int, C.POINTER(Pose), C.c_int,
                                                    C.POINTER(NormalEq), _F, _I, _F, _B]),
        "loam_b200_dense_align": (C.c_int, [vp, _F, C.c_int, C.c_int, C.POINTER(Pose), C.c_int, C.c_int,
                                            C.POINTER(AlignResult)]),
        "loam_b200_dense_score": (C.c_int, [vp, _F, C.c_int, C.c_int, C.POINTER(Pose), C.c_int, C.c_int, _I, _F]),
        "loam_b200_dense_align_batch": (C.c_int, [vp, _F, C.c_int, C.c_int, C.POINTER(Pose), C.c_int, C.c_int, C.c_int,
                                                  C.POINTER(AlignResult)]),
        "loam_b200_reloc_grid": (C.c_int, [C.POINTER(Pose), C.c_float, C.c_int, C.c_float, C.c_int, C.POINTER(Pose),
                                           C.c_int, _I]),
        "loam_b200_dense_relocalize": (C.c_int, [vp, _F, C.c_int, C.c_int, C.POINTER(Pose), C.c_int,
                                                 C.POINTER(RelocParams), C.POINTER(RelocCandidate), C.c_int, _I]),
        "loam_b200_dense_raycast": (C.c_int, [vp, _F, C.c_int, C.c_int, C.POINTER(Pose), C.c_float, C.c_float, _F, _I]),
        "loam_b200_debug_dense_ray_index_bytes": (C.c_int, [vp, _LL]),
        "loam_b200_dense_distance_build": (C.c_int, [vp, _I, _I, C.c_float, _F, _I]),
        "loam_b200_dense_distance_query": (C.c_int, [vp, _F, C.c_int, C.c_int, _F, _F]),
        "loam_b200_debug_dense_distance_bytes": (C.c_int, [vp, _LL]),
        "loam_b200_place_descriptor": (C.c_int, [vp, _F, C.c_int, C.c_int, C.POINTER(PlaceParams), _F]),
        "loam_b200_dense_place_build": (C.c_int, [vp, _F, C.c_int, _F, C.c_int, C.POINTER(PlaceParams)]),
        "loam_b200_dense_place_query": (C.c_int, [vp, _F, C.c_int, C.c_int, C.c_int, C.POINTER(PlaceMatch), _I]),
        "loam_b200_place_grid": (C.c_int, [C.POINTER(PlaceMatch), C.c_int, C.c_float, C.c_int, C.c_float, C.c_int,
                                           C.POINTER(Pose), C.c_int, _I]),
        "loam_b200_dense_relocalize_global": (C.c_int, [vp, _F, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int,
                                                        C.c_float, C.c_int, C.POINTER(RelocParams),
                                                        C.POINTER(RelocCandidate), C.c_int, _I]),
        "loam_b200_debug_dense_place_descriptors": (C.c_int, [vp, _F, C.c_longlong, _LL]),
        "loam_b200_dense_target_size": (C.c_int, [vp, _I]),
        "loam_b200_dense_segment": (C.c_int, [vp, C.c_float, C.c_int, C.c_int, _I, C.POINTER(Segment), C.c_int, _I]),
        "loam_b200_cloud_segment": (C.c_int, [vp, _F, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, _I,
                                              C.POINTER(Segment), C.c_int, _I]),
        "loam_b200_dense_ground": (C.c_int, [vp, C.POINTER(GroundParams), _I, C.POINTER(Segment), C.c_int, _I]),
        "loam_b200_dense_segment_above_ground": (C.c_int, [vp, C.c_float, C.c_int, C.c_int, _I, C.POINTER(Segment),
                                                           C.c_int, _I]),
        "loam_b200_dense_ground_cloud": (C.c_int, [vp, _F, C.c_int, C.c_int, C.POINTER(Pose), C.c_int, C.c_float, _B,
                                                   _F, _I]),
        "loam_b200_comm_unique_id": (C.c_int, [C.POINTER(C.c_ubyte)]),
        "loam_b200_comm_init": (C.c_int, [vp, C.c_int, C.c_int, C.POINTER(C.c_ubyte)]),
        "loam_b200_comm_destroy": (C.c_int, [vp]),
        "loam_b200_map_set_shard": (C.c_int, [vp, C.c_int, C.c_int]),
        "loam_b200_profile_enable": (C.c_int, [vp, C.c_int]),
        "loam_b200_profile_reset": (C.c_int, [vp]),
        "loam_b200_profile_get": (C.c_int, [vp, C.c_int, _D, C.POINTER(C.c_longlong)]),
        "loam_b200_launch_count": (C.c_longlong, [vp]),
        "loam_b200_total_launch_count": (C.c_longlong, []),
        # host handles
        "loam_b200_host_last_error": (C.c_char_p, []),
        "loam_b200_host_set_device": (None, [C.c_int]),
        "loam_b200_scanreg_create": (vp, []),
        "loam_b200_scanreg_destroy": (None, [vp]),
        "loam_b200_scanreg_configure": (C.c_int, [vp, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float]),
        "loam_b200_transform_maintenance": (C.c_int, [_F, _F, _F, _F]),
        "loam_b200_host_gn_solve": (C.c_int, [_F, _F, C.c_int, C.c_float, _F, _I]),
        "loam_b200_scanreg_process_unordered": (C.c_int, [vp, _F, C.c_int, C.c_float, C.c_float, C.c_int]),
        "loam_b200_scanreg_process": (C.c_int, [vp, _F, _I, C.c_int]),
        "loam_b200_scanreg_cloud_size": (C.c_int, [vp, C.c_int]),
        "loam_b200_scanreg_cloud_copy": (C.c_int, [vp, C.c_int, _F]),
        "loam_b200_scanreg_index_size": (C.c_int, [vp, C.c_int]),
        "loam_b200_scanreg_index_copy": (C.c_int, [vp, C.c_int, _I]),
        "loam_b200_odom_create": (vp, [C.c_float, C.c_int]),
        "loam_b200_odom_destroy": (None, [vp]),
        "loam_b200_odom_set_inputs": (C.c_int, [vp, _F, C.c_int, _F, C.c_int, _F, C.c_int, _F, C.c_int, _F, C.c_int]),
        "loam_b200_odom_process": (C.c_int, [vp]),
        "loam_b200_odom_full_to_end": (C.c_int, [vp]),
        "loam_b200_odom_get_twist": (C.c_int, [vp, C.c_int, _F]),
        "loam_b200_odom_cloud_size": (C.c_int, [vp, C.c_int]),
        "loam_b200_odom_cloud_copy": (C.c_int, [vp, C.c_int, _F]),
        "loam_b200_odom_last_iterations": (C.c_int, [vp]),
        "loam_b200_map_create": (vp, [C.c_float, C.c_int]),
        "loam_b200_map_destroy": (None, [vp]),
        "loam_b200_map_seed": (C.c_int, [vp, _F, C.c_int, _F, C.c_int]),
        "loam_b200_map_set_inputs": (C.c_int, [vp, _F, C.c_int, _F, C.c_int, _F, C.c_int]),
        "loam_b200_map_update_odometry": (C.c_int, [vp, _F]),
        "loam_b200_map_process": (C.c_int, [vp]),
        "loam_b200_map_get_twist": (C.c_int, [vp, C.c_int, _F]),
        "loam_b200_map_cloud_size": (C.c_int, [vp, C.c_int]),
        "loam_b200_map_cloud_copy": (C.c_int, [vp, C.c_int, _F]),
        "loam_b200_map_last_iterations": (C.c_int, [vp]),
        "loam_b200_map_last_phase_seconds": (C.c_int, [vp, _D]),
        "loam_b200_map_retain_from_map": (C.c_int, [vp, C.c_int]),
        "loam_b200_map_dense_enable": (C.c_int, [vp, C.c_float, C.c_longlong]),
        "loam_b200_map_dense_stats": (C.c_int, [vp, _LL]),
        "loam_b200_map_dense_export": (C.c_int, [vp, _F, _U, C.c_int, _I]),
        "loam_b200_map_dense_clear": (C.c_int, [vp]),
        "loam_b200_map_dense_visibility": (C.c_int, [vp, C.c_double, C.c_double, C.c_double]),
        "loam_b200_map_dense_carving": (C.c_int, [vp, C.c_double, C.c_double]),
        "loam_b200_map_dense_export_filtered": (C.c_int, [vp, C.c_double, _F, _U, _U16, _U16, C.c_int, _I]),
        "loam_b200_map_dense_export_normals": (C.c_int, [vp, C.c_double, C.c_int, _D, _F, _U, _F, C.c_int, _I]),
        "loam_b200_map_debug_dense_table_slots": (C.c_int, [vp, _LL]),
        "loam_b200_map_dense_snapshot": (C.c_int, [vp, C.POINTER(C.c_uint64), _U, _U16, _U16, _D, C.c_int, _I]),
        "loam_b200_map_dense_merge": (C.c_int, [vp, _U, _U16, _U16, _D, C.c_int, _F]),
        "loam_b200_map_dense_target_build": (C.c_int, [vp, C.c_double, C.c_int, _D, _I]),
        "loam_b200_map_dense_target_load": (C.c_int, [vp, C.c_float, _F, _F, C.c_int]),
        "loam_b200_map_dense_align": (C.c_int, [vp, _F, C.c_int, _F, C.c_int, C.c_int, _F, _I, _F]),
        "loam_b200_map_dense_score": (C.c_int, [vp, _F, C.c_int, _F, C.c_int, C.c_int, _I, _F]),
        "loam_b200_map_dense_align_batch": (C.c_int, [vp, _F, C.c_int, _F, C.c_int, C.c_int, C.c_int, _F, _I, _F]),
        "loam_b200_map_dense_relocalize": (C.c_int, [vp, _F, C.c_int, _F, C.c_int, C.POINTER(RelocParams),
                                                     C.POINTER(RelocCandidate), C.c_int, _I]),
        "loam_b200_map_dense_raycast": (C.c_int, [vp, _F, C.c_int, _F, C.c_float, C.c_float, _F, _I]),
        "loam_b200_map_dense_distance_build": (C.c_int, [vp, _I, _I, C.c_float, _F, _I]),
        "loam_b200_map_dense_distance_query": (C.c_int, [vp, _F, C.c_int, _F, _F]),
        "loam_b200_map_dense_place_build": (C.c_int, [vp, _F, C.c_int, _F, C.c_int, C.POINTER(PlaceParams)]),
        "loam_b200_map_dense_place_query": (C.c_int, [vp, _F, C.c_int, C.c_int, C.POINTER(PlaceMatch), _I]),
        "loam_b200_map_dense_relocalize_global": (C.c_int, [vp, _F, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float,
                                                            C.c_int, C.POINTER(RelocParams),
                                                            C.POINTER(RelocCandidate), C.c_int, _I]),
        "loam_b200_map_dense_target_size": (C.c_int, [vp, _I]),
        "loam_b200_map_dense_segment": (C.c_int, [vp, C.c_float, C.c_int, C.c_int, _I, C.POINTER(Segment), C.c_int,
                                                  _I]),
        "loam_b200_map_dense_ground": (C.c_int, [vp, C.POINTER(GroundParams), _I, C.POINTER(Segment), C.c_int, _I]),
        "loam_b200_map_dense_segment_above_ground": (C.c_int, [vp, C.c_float, C.c_int, C.c_int, _I,
                                                               C.POINTER(Segment), C.c_int, _I]),
        "loam_b200_map_dense_ground_cloud": (C.c_int, [vp, _F, C.c_int, _F, C.c_int, C.c_float, _F, _I, _F, _I]),
        "loam_b200_host_nccl_unique_id": (C.c_int, [C.POINTER(C.c_ubyte)]),
        "loam_b200_map_enable_sharding": (C.c_int, [vp, C.c_int, C.c_int, C.POINTER(C.c_ubyte)]),
        "loam_b200_map_kernel_profile": (C.c_int, [vp, C.c_int, _D]),
        "loam_b200_map_kernel_profile_queries": (C.c_int, [vp, _F, C.c_int, C.c_int, _D]),
        "loam_b200_map_peer_export": (C.c_int, [vp, C.POINTER(C.c_ubyte)]),
        "loam_b200_map_enable_cube_sharding": (C.c_int, [vp, C.c_int, C.c_int, C.POINTER(C.c_ubyte), C.c_int]),
        "loam_b200_map_enable_cube_sharding_local": (C.c_int, [C.POINTER(vp), C.c_int, C.c_int]),
        "loam_b200_map_disable_cube_sharding": (C.c_int, [vp]),
        "loam_b200_peer_export": (C.c_int, [vp, C.POINTER(C.c_ubyte)]),
        "loam_b200_peer_connect": (C.c_int, [vp, C.c_int, C.c_int, C.POINTER(C.c_ubyte), C.c_int]),
        "loam_b200_peer_connect_local": (C.c_int, [C.POINTER(vp), C.c_int, C.c_int]),
        "loam_b200_peer_disconnect": (C.c_int, [vp]),
        "loam_b200_shard_owner": (C.c_int, [C.c_int, C.c_int, C.c_int]),
        "loam_b200_shard_stores": (C.c_int, [C.c_float, C.c_int, C.c_int, C.c_int]),
        "loam_b200_pipeline_create": (vp, [C.c_float, C.c_int, C.c_int]),
        "loam_b200_pipeline_destroy": (None, [vp]),
        "loam_b200_pipeline_seed_map": (C.c_int, [vp, _F, C.c_int, _F, C.c_int]),
        "loam_b200_pipeline_sweep": (C.c_int, [vp, _F, _I, C.c_int, _F, _F, _D]),
        "loam_b200_pipeline_sweep_device": (C.c_int, [vp, vp, _I, C.c_int, _F, _F, _D]),
        "loam_b200_pipeline_sweep_hostclouds": (C.c_int, [vp, _F, _I, C.c_int, _F, _F, _D]),
        "loam_b200_pipeline_submit": (C.c_int, [vp, _F, vp, _I, C.c_int]),
        "loam_b200_pipeline_collect": (C.c_int, [vp, C.c_int, _F, _F, _I]),
        "loam_b200_pipeline_sync": (C.c_int, [vp]),
        "loam_b200_pipeline_stage_seconds": (C.c_int, [vp, _D, C.c_int]),
        "loam_b200_pipeline_scanreg": (vp, [vp]),
        "loam_b200_pipeline_odom": (vp, [vp]),
        "loam_b200_pipeline_map": (vp, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    L._signatures = sig
    _lib = L
    return L


def _fp(a):
    return a.ctypes.data_as(_F)


def _ip(a):
    return a.ctypes.data_as(_I)


def _pts(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a.reshape(-1, 4)


_libm = None


def sincos_f32(angle):
    """(sinf(angle), cosf(angle)) from the C math library, as loam::Angle caches them (std::sin / std::cos of a float).
    numpy's float32 sin / cos round differently for a good share of angles beyond a few tenths of a radian."""
    global _libm
    if _libm is None:
        import ctypes.util
        _libm = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
        for fn in (_libm.sinf, _libm.cosf):
            fn.restype = C.c_float
            fn.argtypes = [C.c_float]
    a = float(np.float32(angle))
    return np.float32(_libm.sinf(a)), np.float32(_libm.cosf(a))


def make_pose(twist6) -> Pose:
    """Pose struct from (rot_x, rot_y, rot_z, x, y, z) with float sin/cos like loam::Angle caches them."""
    t = np.asarray(twist6, dtype=np.float32)
    p = Pose()
    for i in range(3):
        p.rot[i] = t[i]
        p.sin_[i], p.cos_[i] = sincos_f32(t[i])
        p.pos[i] = t[3 + i]
    return p


def make_odom_pose(twist6, scan_period=0.1, it=0) -> OdomPose:
    t = np.asarray(twist6, dtype=np.float32)
    p = OdomPose()
    for i in range(3):
        p.rot[i] = t[i]
        p.sin_[i], p.cos_[i] = sincos_f32(t[i])
        p.pos[i] = t[3 + i]
    p.inv_scan_period = np.float32(1.0) / np.float32(scan_period)
    p.iter = it
    return p


def ring_ranges(ring_sizes):
    """Inclusive (start, end) per ring exactly as processScanlines builds _scanIndices (BasicScanRegistration.cpp:38-41)."""
    sizes = np.asarray(ring_sizes, dtype=np.int64)
    ends = np.cumsum(sizes)
    starts = ends - sizes
    e = np.where(ends > 0, ends - 1, 0)
    return starts.astype(np.int32), e.astype(np.int32)


class Ctx:
    """Kernel-level context (include/loam_b200.h)."""

    def __init__(self, device: int = 0):
        self.L = lib()
        h = C.c_void_p()
        rc = self.L.loam_b200_create(C.byref(h), device)
        if rc != 0:
            raise LoamB200Error(f"loam_b200_create: {self.L.loam_b200_strerror(rc).decode()}")
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.loam_b200_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _ck(self, rc, what):
        if rc != 0:
            detail = self.L.loam_b200_last_error(self.h).decode()
            raise LoamB200Error(f"{what}: {self.L.loam_b200_strerror(rc).decode()} {detail}")

    def reg_bin(self, xyz, lower_deg, upper_deg, n_rings, scan_period=0.1):
        """Ring-binning front end (loam_b200_reg_bin) -> (ring-ordered n_kept x 4 cloud, ring sizes)."""
        a = np.ascontiguousarray(xyz, dtype=np.float32)
        sizes = np.zeros(n_rings, np.int32)
        kept = C.c_int(0)
        self._ck(self.L.loam_b200_reg_bin(self.h, _fp(a), a.shape[0], 0, lower_deg, upper_deg, n_rings, scan_period,
                                          _ip(sizes), C.byref(kept)), "reg_bin")
        out = np.empty((max(kept.value, 1), 4), np.float32)
        got = C.c_int(0)
        self._ck(self.L.loam_b200_cloud_download(self.h, 0, _fp(out), out.shape[0], C.byref(got)), "cloud_download")  # C_REG_FULL
        return out[:got.value].copy(), sizes

    def extract_features(self, pts, ring_sizes, params: RegParams | None = None):
        pts = _pts(pts)
        n = pts.shape[0]
        rs, re = ring_ranges(ring_sizes)
        R = rs.shape[0]
        prm = params or RegParams.default()
        cs, cl, cf = R * prm.nFeatureRegions * prm.maxCornerSharp, R * prm.nFeatureRegions * prm.maxCornerLessSharp, \
            R * prm.nFeatureRegions * prm.maxSurfaceFlat
        sharp = np.empty(cs + 1, np.int32)
        less = np.empty(cl + 1, np.int32)
        flat = np.empty(cf + 1, np.int32)
        label = np.empty(n + 1, np.int8)
        lf = np.empty((n + 1, 4), np.float32)
        out = Features(_ip(sharp), cs, 0, _ip(less), cl, 0, _ip(flat), cf, 0, label.ctypes.data_as(_B), _fp(lf), n, 0)
        self._ck(self.L.loam_b200_extract_features(self.h, _fp(pts), n, _ip(rs), _ip(re), R, C.byref(prm), C.byref(out)),
                 "extract_features")
        return {"sharp": sharp[:out.n_sharp].copy(), "less_sharp": less[:out.n_less_sharp].copy(),
                "flat": flat[:out.n_flat].copy(), "label": label[:n].copy(),
                "less_flat_ds": lf[:out.n_less_flat].copy()}

    def tree_build(self, slot, pts):
        pts = _pts(pts)
        self._ck(self.L.loam_b200_tree_build(self.h, slot, _fp(pts), pts.shape[0]), "tree_build")

    def tree_knn(self, slot, queries, k, max_d2=np.inf):
        q = _pts(queries)
        idx = np.empty((q.shape[0], k), np.int32)
        d2 = np.empty((q.shape[0], k), np.float32)
        self._ck(self.L.loam_b200_tree_knn(self.h, slot, _fp(q), q.shape[0], k, np.float32(max_d2), _ip(idx), _fp(d2)),
                 "tree_knn")
        return idx, d2

    def map_set_shard(self, rank, world):
        self._ck(self.L.loam_b200_map_set_shard(self.h, rank, world), "map_set_shard")

    def map_set_queries(self, corner, surf):
        c, s = _pts(corner), _pts(surf)
        self._ck(self.L.loam_b200_map_set_queries(self.h, _fp(c), c.shape[0], _fp(s), s.shape[0]), "map_set_queries")
        self._nq = c.shape[0] + s.shape[0]

    # ---- mapping stage (device-resident map; include/loam_b200.h "Mapping stage")
    def cloud_upload(self, slot, pts):
        a = _pts(pts)
        self._ck(self.L.loam_b200_cloud_upload(self.h, slot, _fp(a), a.shape[0]), "cloud_upload")

    def cloud_download(self, slot):
        n = self.L.loam_b200_cloud_size(self.h, slot)
        if n < 0:
            self._ck(n, "cloud_size")
        out = np.empty((max(n, 1), 4), np.float32)
        got = C.c_int(0)
        self._ck(self.L.loam_b200_cloud_download(self.h, slot, _fp(out), out.shape[0], C.byref(got)), "cloud_download")
        return out[:got.value].copy()

    def cloud_swap(self, a, b):
        self._ck(self.L.loam_b200_cloud_swap(self.h, a, b), "cloud_swap")

    def map_pool_append(self, kind, pts):
        a = _pts(pts)
        self._ck(self.L.loam_b200_map_pool_append(self.h, kind, _fp(a), a.shape[0]), "map_pool_append")

    def map_begin_sweep(self, twist6, cen, valid_cubes, corner_leaf=0.2, surf_leaf=0.4):
        """Window + stacks of one sweep -> sizes_out[4] (from-map corner / surface counts, corner / surface stack sizes);
        map_iterate then runs over the persistent map with the down-sized stacks as queries."""
        p = make_pose(twist6)
        cubes = np.ascontiguousarray(valid_cubes, dtype=np.int32).reshape(-1)
        win = MapWindow()
        for i in range(3):
            win.cen[i] = int(cen[i])
        win.valid_cubes = _ip(cubes) if cubes.size else None
        win.n_valid = cubes.size
        win.corner_leaf = corner_leaf
        win.surf_leaf = surf_leaf
        sizes = np.zeros(4, np.int32)
        self._ck(self.L.loam_b200_map_begin_sweep(self.h, C.byref(p), C.byref(win), _ip(sizes)), "map_begin_sweep")
        self._nq = int(sizes[2]) + int(sizes[3])
        return sizes

    def map_end_sweep(self, twist6, asynchronous=False):
        p = make_pose(twist6)
        fn = self.L.loam_b200_map_end_sweep_async if asynchronous else self.L.loam_b200_map_end_sweep
        self._ck(fn(self.h, C.byref(p)), "map_end_sweep")

    def map_debug_from_map(self, on=True):
        self._ck(self.L.loam_b200_map_debug_from_map(self.h, 1 if on else 0), "map_debug_from_map")

    def debug_map_prune(self, mode):
        """-1 automatic (from the L2 size), 0 off, 1 on."""
        self._ck(self.L.loam_b200_debug_map_prune(self.h, mode), "debug_map_prune")

    # ---- odometry stage (include/loam_b200.h "Odometry stage"): last clouds and queries from the cloud slots
    def odom_adopt(self, src: "Ctx", src5):
        """The registration -> odometry hand-off from `src`'s slots src5 (sharp, less sharp, flat, less flat, full)."""
        s = np.ascontiguousarray(src5, dtype=np.int32).reshape(5)
        self._ck(self.L.loam_b200_odom_adopt(self.h, src.h, _ip(s)), "odom_adopt")

    def odom_prepare(self):
        """This sweep's queries from the ODOM_SHARP / ODOM_FLAT slots; odom_iterate / odom_solve then search them."""
        self._ck(self.L.loam_b200_odom_prepare(self.h), "odom_prepare")
        self._noq = (self.L.loam_b200_cloud_size(self.h, C_ODOM_SHARP) + self.L.loam_b200_cloud_size(self.h, C_ODOM_FLAT))

    def odom_rebuild_last(self):
        """Trees and ring offsets of the ODOM_LAST_CORNER / ODOM_LAST_SURF slots (built asynchronously)."""
        self._ck(self.L.loam_b200_odom_rebuild_last(self.h), "odom_rebuild_last")

    def cloud_transform_to_end2(self, slot_a, slot_b, twist6, scan_period=0.1):
        p = make_odom_pose(twist6, scan_period, 0)
        self._ck(self.L.loam_b200_cloud_transform_to_end2(self.h, slot_a, slot_b, C.byref(p)), "cloud_transform_to_end2")

    def debug_odom_ring_ranges(self, mode):
        """1 automatic (index ranges on ring-ordered last clouds), 0 always the serial scan."""
        self._ck(self.L.loam_b200_debug_odom_ring_ranges(self.h, mode), "debug_odom_ring_ranges")

    def debug_tree_build_path(self, slot):
        """BUILD_CLUSTER_PAIR, BUILD_CLUSTER or BUILD_MULTI_LAUNCH: how tree `slot` was last built."""
        rc = self.L.loam_b200_debug_tree_build_path(self.h, slot)
        if rc < 0:
            self._ck(rc, "debug_tree_build_path")
        return rc

    def map_iterate(self, twist6, debug=False):
        p = make_pose(twist6)
        ne = NormalEq()
        if debug:
            coeff = np.zeros((self._nq, 4), np.float32)
            sel = np.zeros(self._nq, np.int8)
            self._ck(self.L.loam_b200_map_iterate_debug(self.h, C.byref(p), C.byref(ne), _fp(coeff),
                                                        sel.ctypes.data_as(_B)), "map_iterate_debug")
            return _ne(ne), coeff, sel
        self._ck(self.L.loam_b200_map_iterate(self.h, C.byref(p), C.byref(ne)), "map_iterate")
        return _ne(ne)

    def map_iterate_stats(self, twist6):
        """(normal equations, BVH nodes visited, leaves visited) of one instrumented launch."""
        p = make_pose(twist6)
        ne = NormalEq()
        nodes = C.c_ulonglong(0)
        leaves = C.c_ulonglong(0)
        self._ck(self.L.loam_b200_map_iterate_stats(self.h, C.byref(p), C.byref(ne), C.byref(nodes), C.byref(leaves)),
                 "map_iterate_stats")
        return _ne(ne), nodes.value, leaves.value

    def odom_set_last(self, corner, surf):
        c, s = _pts(corner), _pts(surf)
        self._ck(self.L.loam_b200_odom_set_last(self.h, _fp(c), c.shape[0], _fp(s), s.shape[0]), "odom_set_last")

    def odom_set_current(self, sharp, flat):
        c, s = _pts(sharp), _pts(flat)
        self._ck(self.L.loam_b200_odom_set_current(self.h, _fp(c), c.shape[0], _fp(s), s.shape[0]), "odom_set_current")
        self._noq = c.shape[0] + s.shape[0]

    def odom_iterate(self, twist6, it, scan_period=0.1, debug=False):
        p = make_odom_pose(twist6, scan_period, it)
        ne = NormalEq()
        if debug:
            coeff = np.zeros((self._noq, 4), np.float32)
            sel = np.zeros(self._noq, np.int8)
            ind = np.zeros((self._noq, 3), np.int32)
            self._ck(self.L.loam_b200_odom_iterate_debug(self.h, C.byref(p), C.byref(ne), _fp(coeff),
                                                         sel.ctypes.data_as(_B), _ip(ind)), "odom_iterate_debug")
            return _ne(ne), coeff, sel, ind
        self._ck(self.L.loam_b200_odom_iterate(self.h, C.byref(p), C.byref(ne)), "odom_iterate")
        return _ne(ne)

    def debug_gn_solve(self, AtA, AtB, first_iteration=True, eigen_threshold=10.0):
        """The device loops' warp-parallel 6 x 6 step on n systems (AtA n x 6 x 6, AtB n x 6) -> (x n x 6, degenerate n)."""
        A = np.ascontiguousarray(AtA, dtype=np.float32).reshape(-1, 36)
        b = np.ascontiguousarray(AtB, dtype=np.float32).reshape(-1, 6)
        packed = np.ascontiguousarray(np.concatenate([A, b], axis=1), dtype=np.float32)
        n = packed.shape[0]
        x = np.zeros((n, 6), np.float32)
        deg = np.zeros(n, np.int32)
        self._ck(self.L.loam_b200_debug_gn_solve(self.h, _fp(packed), n, 1 if first_iteration else 0, eigen_threshold,
                                                 _fp(x), _ip(deg)), "debug_gn_solve")
        return x, deg

    def debug_sort_pairs(self, keys, vals, key_bits, live=None, out_params=True):
        """The shared radix sort on (keys uint32, vals int32) -> (keys, vals, path): only the first min(n, live) entries
        are sorted (live=None: all); path 0 one-cluster sort, 1 onesweep with 4 items per thread, 2 with 16, -1 none."""
        k = np.ascontiguousarray(keys, dtype=np.uint32).reshape(-1)
        v = np.ascontiguousarray(vals, dtype=np.int32).reshape(-1)
        if k.shape != v.shape:
            raise ValueError("keys and vals differ in length")
        n = k.shape[0]
        ko = np.zeros(max(n, 1), np.uint32)
        vo = np.zeros(max(n, 1), np.int32)
        path = C.c_int(-1)
        kin = k if n else np.zeros(1, np.uint32)  # never a NULL pointer
        vin = v if n else np.zeros(1, np.int32)
        self._ck(self.L.loam_b200_debug_sort_pairs(self.h, kin.ctypes.data_as(_U), _ip(vin), n,
                                                   -1 if live is None else int(live), int(key_bits),
                                                   1 if out_params else 0, ko.ctypes.data_as(_U), _ip(vo),
                                                   C.byref(path)), "debug_sort_pairs")
        return ko[:n].copy(), vo[:n].copy(), path.value

    def odom_solve(self, twist6, scan_period=0.1, max_iter=25, delta_t=0.1, delta_r=0.1):
        """Whole scan-to-scan Gauss-Newton loop on the device -> (twist6, iterations)."""
        t = np.ascontiguousarray(twist6, dtype=np.float32)
        rot, pos = t[:3].copy(), t[3:].copy()
        res = LmResult()
        self._ck(self.L.loam_b200_odom_solve(self.h, _fp(rot), _fp(pos), np.float32(1.0) / np.float32(scan_period), max_iter,
                                             delta_t, delta_r, C.byref(res)), "odom_solve")
        return np.array(list(res.rot) + list(res.pos), np.float32), res.iterations

    def map_solve(self, twist6, max_iter=10, delta_t=0.05, delta_r=0.05):
        """Whole scan-to-map Gauss-Newton loop on the device -> (twist6, iterations)."""
        t = np.ascontiguousarray(twist6, dtype=np.float32)
        rot, pos = t[:3].copy(), t[3:].copy()
        res = LmResult()
        self._ck(self.L.loam_b200_map_solve(self.h, _fp(rot), _fp(pos), max_iter, delta_t, delta_r, C.byref(res)),
                 "map_solve")
        return np.array(list(res.rot) + list(res.pos), np.float32), res.iterations

    def transform_to_end(self, pts, twist6, scan_period=0.1):
        a = _pts(pts).copy()
        p = make_odom_pose(twist6, scan_period, 0)
        self._ck(self.L.loam_b200_transform_to_end(self.h, _fp(a), a.shape[0], C.byref(p)), "transform_to_end")
        return a

    def transform_to_map(self, pts, twist6):
        a = _pts(pts).copy()
        p = make_pose(twist6)
        self._ck(self.L.loam_b200_transform_to_map(self.h, _fp(a), a.shape[0], C.byref(p)), "transform_to_map")
        return a

    def voxel_grid(self, pts, leaf):
        a = _pts(pts)
        out = np.empty_like(a)
        n = C.c_int(0)
        self._ck(self.L.loam_b200_voxel_grid(self.h, _fp(a), a.shape[0], np.float32(leaf), _fp(out), a.shape[0],
                                             C.byref(n)), "voxel_grid")
        return out[:n.value].copy()

    # ---- whole-run voxel map (include/loam_b200.h "Whole-run voxel map")
    def dense_enable(self, leaf, max_voxels=DENSE_MAX_VOXELS):
        self._ck(self.L.loam_b200_dense_enable(self.h, np.float32(leaf), int(max_voxels)), "dense_enable")
        self.dense_leaf = np.float32(leaf)

    def dense_insert(self, slot):
        """Accumulate the cloud in `slot` (fill it with cloud_upload)."""
        self._ck(self.L.loam_b200_dense_insert(self.h, slot), "dense_insert")

    def dense_stats(self):
        """{"voxels", "skipped", "dropped"} (synchronises)."""
        out = np.zeros(3, np.int64)
        self._ck(self.L.loam_b200_dense_stats(self.h, out.ctypes.data_as(_LL)), "dense_stats")
        return _dense_stats(out)

    def dense_export(self, max_miss_ratio=None, evidence=False):
        """(centroids N x 4 float32, counts N uint32) in ascending voxel order.  With max_miss_ratio only the voxels with
        misses <= max_miss_ratio * hits; with evidence=True also (hits N uint16, misses N uint16)."""
        if max_miss_ratio is None and not evidence:
            return _dense_export(lambda pts, cnt, cap, n: self.L.loam_b200_dense_export(self.h, pts, cnt, cap, n),
                                 self.dense_stats()["voxels"], lambda rc: self._ck(rc, "dense_export"))
        return _dense_export_filtered(
            lambda *a: self.L.loam_b200_dense_export_filtered(self.h, *a), max_miss_ratio, evidence,
            self.dense_stats()["voxels"], lambda rc: self._ck(rc, "dense_export_filtered"))

    def dense_export_normals(self, max_miss_ratio=None, radius=1, viewpoint=(0.0, 0.0, 0.0)):
        """(centroids N x 4 float32, counts N uint32, normals N x 4 float32: nx, ny, nz, curvature) of the voxels
        dense_export(max_miss_ratio) returns (None: every voxel).  Neighbourhood: the exported voxels within `radius`
        (1..3) voxels on every axis; normals flipped towards `viewpoint` (map frame); NaN where fewer than 3 neighbours."""
        return _dense_export_normals(lambda *a: self.L.loam_b200_dense_export_normals(self.h, *a), max_miss_ratio,
                                     radius, viewpoint, self.dense_stats()["voxels"],
                                     lambda rc: self._ck(rc, "dense_export_normals"))

    def dense_table_slots(self):
        """Test query: slots of the whole-run map's hash table (0 while the map is off)."""
        out = C.c_longlong(0)
        self._ck(self.L.loam_b200_debug_dense_table_slots(self.h, C.byref(out)), "dense_table_slots")
        return out.value

    def dense_visibility(self, h_res_deg, v_res_deg, margin):
        """Visibility pass of every later insert by the mapping stage (h_res_deg = 0: off); see dense_observe."""
        self._ck(self.L.loam_b200_dense_visibility(self.h, float(h_res_deg), float(v_res_deg), float(margin)),
                 "dense_visibility")

    def dense_observe(self, slot, twist6):
        """The visibility pass over the cloud in `slot` (map frame) seen from the pose (rot_x, rot_y, rot_z, x, y, z):
        one miss for every stored voxel the cloud sees through."""
        p = make_pose(twist6)
        self._ck(self.L.loam_b200_dense_observe(self.h, slot, C.byref(p)), "dense_observe")

    def dense_carving(self, margin=DENSE_CARVE_MARGIN, max_range=DENSE_CARVE_MAX_RANGE):
        """Carve mode of the visibility pass instead of the range image (max_range = 0: off): every point's ray is walked
        from the pose through the map, and each stored voxel it crosses up to min(r - margin, max_range), and that no
        point of the cloud falls into, gets one miss per observed cloud.  See dense_observe."""
        self._ck(self.L.loam_b200_dense_carving(self.h, float(margin), float(max_range)), "dense_carving")

    def dense_carve_index(self):
        """Test query: carve mode's occupancy index -> (brick keys B uint64 ascending, masks B x 8 uint64)."""
        n = C.c_longlong(0)
        rc = self.L.loam_b200_debug_dense_carve_index(self.h, None, 0, C.byref(n))
        if rc not in (0, -5):  # LOAM_B200_ERR_CAPACITY: the count is in n
            self._ck(rc, "dense_carve_index")
        rows = np.zeros((n.value, 9), np.uint64)
        self._ck(self.L.loam_b200_debug_dense_carve_index(self.h, rows.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                          n.value, C.byref(n)), "dense_carve_index")
        return rows[:, 0].copy(), rows[:, 1:].copy()

    def dense_clear(self):
        self._ck(self.L.loam_b200_dense_clear(self.h), "dense_clear")

    # ---- snapshots and merging (include/loam_b200.h "Whole-run voxel map snapshots and merging")
    def dense_snapshot(self):
        """The exact state of every stored voxel in ascending key order: a dict of "keys" (N uint64), "counts" (N
        uint32), "hits", "misses" (N uint16), "sums" (N x 4 float64: x, y, z, intensity) and "leaf" (the map's leaf)."""
        return _dense_snapshot(lambda *a: self.L.loam_b200_dense_snapshot(self.h, *a), self.dense_stats()["voxels"],
                               getattr(self, "dense_leaf", None), lambda rc: self._ck(rc, "dense_snapshot"))

    def dense_merge(self, snap, twist6=None):
        """Add a snapshot's entries into the map, as stored (twist6 None) or under the rigid transform twist6 = (rot_x,
        rot_y, rot_z, x, y, z); each entry's voxel is that of its transformed centroid at this map's leaf."""
        a = _merge_arrays(snap)
        p = make_pose(twist6) if twist6 is not None else None
        self._ck(self.L.loam_b200_dense_merge(self.h, *_merge_ptrs(a), C.byref(p) if p is not None else None),
                 "dense_merge")

    # ---- alignment against the whole-run voxel map (include/loam_b200.h "Alignment against the whole-run voxel map")
    def dense_target_build(self, max_miss_ratio=None, radius=1, viewpoint=(0.0, 0.0, 0.0)):
        """Snapshot dense_export_normals(max_miss_ratio, radius, viewpoint) on the device as the alignment target ->
        its voxel count."""
        ratio = math.inf if max_miss_ratio is None else float(max_miss_ratio)
        vp = np.ascontiguousarray(viewpoint, np.float64).reshape(3)
        n = C.c_int(0)
        self._ck(self.L.loam_b200_dense_target_build(self.h, ratio, int(radius), vp.ctypes.data_as(_D), C.byref(n)),
                 "dense_target_build")
        return n.value

    def dense_target_load(self, leaf, centroids, normals):
        """The alignment target from host arrays (N x 4 centroids, N x 4 normals as dense_export_normals returns them;
        a NaN nx: no normal), e.g. a map saved from an earlier session."""
        c, nr = _pts(centroids), _pts(normals)
        if c.shape[0] != nr.shape[0]:
            raise ValueError("dense_target_load: centroids and normals differ in length")
        self._ck(self.L.loam_b200_dense_target_load(self.h, np.float32(leaf), _fp(c), _fp(nr), c.shape[0]),
                 "dense_target_load")

    def dense_align_iterate(self, pts, twist6, search_radius=1, debug=False):
        """One point-to-plane iteration of sensor-frame pts at twist6 against the target -> (normal equations,
        sum of pd2^2 over the selected rows); with debug=True also (match N int32, coeff N x 4, selected N int8)."""
        a = _pts(pts)
        n = a.shape[0]
        p = make_pose(twist6)
        ne = NormalEq()
        ss = np.zeros(1, np.float32)
        if debug:
            match = np.zeros(max(n, 1), np.int32)
            coeff = np.zeros((max(n, 1), 4), np.float32)
            sel = np.zeros(max(n, 1), np.int8)
            self._ck(self.L.loam_b200_dense_align_iterate(self.h, _fp(a), n, 0, C.byref(p), int(search_radius),
                                                          C.byref(ne), _fp(ss), _ip(match), _fp(coeff),
                                                          sel.ctypes.data_as(_B)), "dense_align_iterate")
            return _ne(ne), ss[0], match[:n].copy(), coeff[:n].copy(), sel[:n].copy()
        self._ck(self.L.loam_b200_dense_align_iterate(self.h, _fp(a), n, 0, C.byref(p), int(search_radius),
                                                      C.byref(ne), _fp(ss), None, None, None), "dense_align_iterate")
        return _ne(ne), ss[0]

    def dense_align(self, pts, twist6, search_radius=1, max_iterations=10):
        """Gauss-Newton of sensor-frame pts against the target from twist6 -> (twist6 float32, {"iterations",
        "n_selected", "rms", "degenerate", "converged"}).  Coarse to fine: search_radius 3, then 1 from the result."""
        a = _pts(pts)
        p = make_pose(twist6)
        r = AlignResult()
        self._ck(self.L.loam_b200_dense_align(self.h, _fp(a), a.shape[0], 0, C.byref(p), int(search_radius),
                                              int(max_iterations), C.byref(r)), "dense_align")
        return _align_out(list(r.rot) + list(r.pos), r.iterations, r.n_selected, r.rms, r.degenerate, r.converged)

    # ---- relocalisation (include/loam_b200.h "Relocalisation against the whole-run voxel map")
    def dense_score(self, pts, twists, search_radius=3):
        """Per pose of twists (K x 6) what dense_align_iterate returns there in n_selected and sum_pd2_sq, all poses in
        one launch per chunk -> (n_selected int32[K], sum_pd2_sq float32[K])."""
        a = _pts(pts)
        poses, k = _poses(twists)
        sel = np.zeros(max(k, 1), np.int32)
        ss = np.zeros(max(k, 1), np.float32)
        self._ck(self.L.loam_b200_dense_score(self.h, _fp(a), a.shape[0], 0, poses, k, int(search_radius), _ip(sel),
                                              _fp(ss)), "dense_score")
        return sel[:k].copy(), ss[:k].copy()

    def dense_align_batch(self, pts, twists, search_radius=1, max_iterations=10):
        """One dense_align per initial pose of twists (K x 6), each equal to the single call -> (K x 6 float32, list of
        K info dicts as dense_align)."""
        a = _pts(pts)
        poses, k = _poses(twists)
        res = (AlignResult * max(k, 1))()
        self._ck(self.L.loam_b200_dense_align_batch(self.h, _fp(a), a.shape[0], 0, poses, k, int(search_radius),
                                                    int(max_iterations), res), "dense_align_batch")
        outs = [_align_out(list(r.rot) + list(r.pos), r.iterations, r.n_selected, r.rms, r.degenerate, r.converged)
                for r in res[:k]]
        return np.array([o[0] for o in outs], np.float32).reshape(k, 6), [o[1] for o in outs]

    def dense_relocalize(self, pts, hypotheses, params=None, cap=16):
        """Relocalise pts among the hypotheses (K x 6 twists, e.g. reloc_grid) -> ranked candidates (at most cap), each
        a dict: hypothesis, score_selected, coarse / fine (twist, info) as dense_align, selected, rms."""
        a = _pts(pts)
        poses, k = _poses(hypotheses)
        prm = params if params is not None else RelocParams.default()
        out = (RelocCandidate * max(int(cap), 1))()
        n = C.c_int(0)
        self._ck(self.L.loam_b200_dense_relocalize(self.h, _fp(a), a.shape[0], 0, poses, k, C.byref(prm), out,
                                                   int(cap), C.byref(n)), "dense_relocalize")
        return [_candidate(r) for r in out[:n.value]]

    # ---- ray casting (include/loam_b200.h "Ray casting the whole-run voxel map")
    def dense_raycast(self, rays, twist6, min_range=0.0, max_range=100.0, on_device=False, n=None):
        """Cast sensor-frame rays (N x 4, w ignored: lidar_rays() or a sweep's own points) from twist6 into the target
        -> (range float32[N]: the surfel-refined distance to the first target voxel met within (min_range, max_range],
        +inf when none; index int32[N]: its position in the target's ascending key order, -1 when none).  With
        on_device=True, rays is the address of n float[4] in device memory."""
        p = make_pose(twist6)
        if on_device:
            ptr, k = C.cast(C.c_void_p(int(rays)), _F), int(n)
        else:
            a = _pts(rays)
            ptr, k = _fp(a), a.shape[0]
        rng = np.zeros(max(k, 1), np.float32)
        idx = np.zeros(max(k, 1), np.int32)
        self._ck(self.L.loam_b200_dense_raycast(self.h, ptr, k, 1 if on_device else 0, C.byref(p), np.float32(min_range),
                                                np.float32(max_range), _fp(rng), _ip(idx)), "dense_raycast")
        return rng[:k].copy(), idx[:k].copy()

    def dense_ray_index_bytes(self):
        """Test query: device bytes of the target's ray index (0 until the first cast after a build or load)."""
        out = C.c_longlong(0)
        self._ck(self.L.loam_b200_debug_dense_ray_index_bytes(self.h, C.byref(out)), "dense_ray_index_bytes")
        return out.value

    # ---- distance field (include/loam_b200.h "Distance field of the whole-run voxel map")
    def dense_distance_field(self, lo, dims, max_distance, download=True):
        """Build the distance field of the target over the box of voxels lo + [0, dims) (3 ints each, x y z; see
        voxel_box) -> (dist float32, sq int32), each shaped (nz, ny, nx): the distance in metres to the nearest target
        voxel (+inf beyond max_distance) and its square in voxel units (-1 beyond).  download=False keeps the field on
        the device only and returns (None, None)."""
        lo_a, dims_a, shape = _box_args(lo, dims)
        dist = np.zeros(shape, np.float32) if download else None
        sq = np.zeros(shape, np.int32) if download else None
        self._ck(self.L.loam_b200_dense_distance_build(self.h, _ip(lo_a), _ip(dims_a), np.float32(max_distance),
                                                       _fp(dist) if download else None,
                                                       _ip(sq) if download else None), "dense_distance_field")
        return dist, sq

    def dense_distance_query(self, pts, on_device=False, n=None, gradient=False):
        """The last distance field at map-frame pts (N x 4, w ignored), trilinear between cell centres (NaN outside
        them) -> dist float32[N], or (dist, grad float32[N, 3]) with gradient=True.  With on_device=True, pts is the
        address of n float[4] in device memory."""
        ptr, k = _pts_or_device(pts, on_device, n)
        dist = np.zeros(max(k, 1), np.float32)
        grad = np.zeros((max(k, 1), 3), np.float32) if gradient else None
        self._ck(self.L.loam_b200_dense_distance_query(self.h, ptr, k, 1 if on_device else 0, _fp(dist),
                                                       _fp(grad) if gradient else None), "dense_distance_query")
        return (dist[:k].copy(), grad[:k].copy()) if gradient else dist[:k].copy()

    def dense_distance_bytes(self):
        """Test query: device bytes of the distance field (4 per cell of the box; 0 without a field)."""
        out = C.c_longlong(0)
        self._ck(self.L.loam_b200_debug_dense_distance_bytes(self.h, C.byref(out)), "dense_distance_bytes")
        return out.value

    # ---- Euclidean segmentation (include/loam_b200.h "Euclidean segmentation of the whole-run voxel map and of clouds")
    def dense_segment(self, tolerance, min_size=1, max_size=None):
        """Euclidean segments of the target's voxels (centroids within tolerance metres, at most 4 leaves) with
        min_size <= size <= max_size -> (labels int32[N]: per target voxel in key order, its segment's rank or -1;
        segments: dict of arrays size, first, lo, hi, centroid), ranked by size descending, ties by first."""
        n = C.c_int(0)
        self._ck(self.L.loam_b200_dense_target_size(self.h, C.byref(n)), "dense_segment")
        return _segment_call(lambda lab, seg, cap, k: self.L.loam_b200_dense_segment(
            self.h, np.float32(tolerance), int(min_size), _max_size(max_size), lab, seg, cap, k), n.value,
            lambda rc: self._ck(rc, "dense_segment"))

    def dense_target_size(self):
        """Voxels of the current target (the length of dense_segment's labels); raises without a target."""
        n = C.c_int(0)
        self._ck(self.L.loam_b200_dense_target_size(self.h, C.byref(n)), "dense_target_size")
        return n.value

    def segment_cloud(self, pts, tolerance, min_size=1, max_size=None, on_device=False, n=None):
        """Euclidean segments of a cloud's points (N x 4, w ignored; with on_device=True the address of n float[4] in
        device memory); needs no map and no target -> (labels int32[N] in input order, -1 for points not kept or not
        finite; segments as dense_segment, first = the smallest input index)."""
        ptr, k = _pts_or_device(pts, on_device, n)
        return _segment_call(lambda lab, seg, cap, kk: self.L.loam_b200_cloud_segment(
            self.h, ptr, k, 1 if on_device else 0, np.float32(tolerance), int(min_size), _max_size(max_size), lab,
            seg, cap, kk), k, lambda rc: self._ck(rc, "segment_cloud"))

    # ---- ground (include/loam_b200.h "Ground of the whole-run voxel map"; y is up)
    def dense_ground(self, params=None):
        """Ground patches of the target (params: GroundParams, default GroundParams.default()) -> (labels int32[N]:
        per target voxel in key order, its patch's rank or -1; patches: dict of arrays as dense_segment).  The ground
        flags stay with the target for dense_segment_above_ground and dense_ground_cloud."""
        prm = params if params is not None else GroundParams.default()
        n = C.c_int(0)
        self._ck(self.L.loam_b200_dense_target_size(self.h, C.byref(n)), "dense_ground")
        return _segment_call(lambda lab, seg, cap, k: self.L.loam_b200_dense_ground(
            self.h, C.byref(prm), lab, seg, cap, k), n.value, lambda rc: self._ck(rc, "dense_ground"))

    def dense_segment_above_ground(self, tolerance, min_size=1, max_size=None):
        """dense_segment over the target voxels that are not ground (after dense_ground) -> as dense_segment, labels
        over the whole target with -1 on the ground."""
        n = C.c_int(0)
        self._ck(self.L.loam_b200_dense_target_size(self.h, C.byref(n)), "dense_segment_above_ground")
        return _segment_call(lambda lab, seg, cap, k: self.L.loam_b200_dense_segment_above_ground(
            self.h, np.float32(tolerance), int(min_size), _max_size(max_size), lab, seg, cap, k), n.value,
            lambda rc: self._ck(rc, "dense_segment_above_ground"))

    def dense_ground_cloud(self, pts, twist6, search_radius=1, max_height=0.1, on_device=False, n=None, out=None):
        """Ground points of sensor-frame pts (N x 4) at twist6 against the target's ground -> (labels int8[N]: 1
        ground, 0 not ground, -1 not finite or outside the key range; the points labelled 0 in input order, K x 4).
        With on_device=True, pts is the address of n float[4] in device memory and out that of room for n float[4]
        in device memory (or None): the second value is then K, the points being at out."""
        ptr, k = _pts_or_device(pts, on_device, n)
        p = make_pose(twist6)
        labels = np.zeros(max(k, 1), np.int8)
        if on_device:
            dst = None if out is None else C.cast(C.c_void_p(int(out)), _F)
        else:
            ng = np.zeros((max(k, 1), 4), np.float32)
            dst = _fp(ng)
        kk = C.c_int(0)
        self._ck(self.L.loam_b200_dense_ground_cloud(self.h, ptr, k, 1 if on_device else 0, C.byref(p),
                                                     int(search_radius), np.float32(max_height),
                                                     labels.ctypes.data_as(_B), dst, C.byref(kk)),
                 "dense_ground_cloud")
        return labels[:k].copy(), (kk.value if on_device else ng[:kk.value].copy())

    # ---- place recognition (include/loam_b200.h "Place recognition and global relocalisation")
    def place_descriptor(self, pts, params=None, on_device=False, n=None):
        """Polar height descriptor of sensor-frame pts (N x 4, w ignored) -> float32 (rings, sectors).  With
        on_device=True, pts is the address of n float[4] in device memory."""
        prm = params if params is not None else PlaceParams.default()
        ptr, k = _pts_or_device(pts, on_device, n)
        out = np.zeros((prm.rings, prm.sectors), np.float32)
        self._ck(self.L.loam_b200_place_descriptor(self.h, ptr, k, 1 if on_device else 0, C.byref(prm), _fp(out)),
                 "place_descriptor")
        return out

    def dense_place_build(self, positions, rays, params=None):
        """The place database of the target: one descriptor per position (K x 3, map frame), rendered through
        dense_raycast of rays (N x 4, e.g. lidar_rays) from that position with rot = 0."""
        prm = params if params is not None else PlaceParams.default()
        p = np.ascontiguousarray(positions, np.float32).reshape(-1, 3)
        r = _pts(rays)
        self._ck(self.L.loam_b200_dense_place_build(self.h, _fp(p), p.shape[0], _fp(r), r.shape[0], C.byref(prm)),
                 "dense_place_build")

    def dense_place_query(self, pts, top_m=PLACE_TOP_M, on_device=False, n=None):
        """The top_m places for sensor-frame pts -> list of dicts: candidate, shift, yaw, pos (float32[3]), dist."""
        ptr, k = _pts_or_device(pts, on_device, n)
        out = (PlaceMatch * max(int(top_m), 1))()
        got = C.c_int(0)
        self._ck(self.L.loam_b200_dense_place_query(self.h, ptr, k, 1 if on_device else 0, int(top_m), out,
                                                    C.byref(got)), "dense_place_query")
        return [_place_match(m) for m in out[:got.value]]

    def dense_relocalize_global(self, pts, top_m=PLACE_TOP_M, yaw_step_deg=PLACE_YAW_STEP_DEG,
                                yaw_steps=PLACE_YAW_STEPS, xz_step=PLACE_XZ_STEP, xz_steps=PLACE_XZ_STEPS,
                                params=None, cap=16):
        """Relocalise pts with no prior: dense_place_query(top_m), then dense_relocalize over place_grid of its
        matches -> what dense_relocalize returns; a candidate's hypothesis indexes that grid."""
        a = _pts(pts)
        prm = params if params is not None else RelocParams.default()
        out = (RelocCandidate * max(int(cap), 1))()
        got = C.c_int(0)
        self._ck(self.L.loam_b200_dense_relocalize_global(self.h, _fp(a), a.shape[0], 0, int(top_m),
                                                          np.float32(yaw_step_deg), int(yaw_steps),
                                                          np.float32(xz_step), int(xz_steps), C.byref(prm), out,
                                                          int(cap), C.byref(got)), "dense_relocalize_global")
        return [_candidate(r) for r in out[:got.value]]

    def dense_place_descriptors(self):
        """Test query: the database's descriptors -> float32 (K, rings, sectors) (K = 0 without a database)."""
        n = C.c_longlong(0)
        rc = self.L.loam_b200_debug_dense_place_descriptors(self.h, None, 0, C.byref(n))
        if rc not in (0, -5):
            self._ck(rc, "dense_place_descriptors")
        out = np.zeros(max(n.value, 1), np.float32)
        self._ck(self.L.loam_b200_debug_dense_place_descriptors(self.h, _fp(out), n.value, C.byref(n)),
                 "dense_place_descriptors")
        return out[:n.value].copy()

    def profile(self, on=True):
        self.L.loam_b200_profile_enable(self.h, 1 if on else 0)
        self.L.loam_b200_profile_reset(self.h)

    def profile_get(self):
        out = {}
        for i, name in enumerate(KERNEL_FAMILIES):
            ms = C.c_double(0)
            n = C.c_longlong(0)
            self.L.loam_b200_profile_get(self.h, i, C.byref(ms), C.byref(n))
            out[name] = (ms.value, n.value)
        return out

    def launch_count(self):
        return self.L.loam_b200_launch_count(self.h)


def _dense_stats(out):
    return {"voxels": int(out[0]), "skipped": int(out[1]), "dropped": int(out[2])}


def _dense_export(fn, n, ck):
    pts = np.zeros((max(n, 1), 4), np.float32)
    cnt = np.zeros(max(n, 1), np.uint32)
    got = C.c_int(0)
    ck(fn(_fp(pts), cnt.ctypes.data_as(_U), n, C.byref(got)))
    return pts[:got.value].copy(), cnt[:got.value].copy()


def _dense_export_filtered(fn, max_miss_ratio, evidence, n, ck):
    ratio = math.inf if max_miss_ratio is None else float(max_miss_ratio)
    pts = np.zeros((max(n, 1), 4), np.float32)
    cnt = np.zeros(max(n, 1), np.uint32)
    hits = np.zeros(max(n, 1), np.uint16)
    misses = np.zeros(max(n, 1), np.uint16)
    got = C.c_int(0)
    ck(fn(ratio, _fp(pts), cnt.ctypes.data_as(_U), hits.ctypes.data_as(_U16) if evidence else None,
          misses.ctypes.data_as(_U16) if evidence else None, n, C.byref(got)))
    k = got.value
    out = (pts[:k].copy(), cnt[:k].copy())
    return out + (hits[:k].copy(), misses[:k].copy()) if evidence else out


def _dense_export_normals(fn, max_miss_ratio, radius, viewpoint, n, ck):
    ratio = math.inf if max_miss_ratio is None else float(max_miss_ratio)
    vp = np.ascontiguousarray(viewpoint, np.float64).reshape(3)
    pts = np.zeros((max(n, 1), 4), np.float32)
    cnt = np.zeros(max(n, 1), np.uint32)
    nrm = np.zeros((max(n, 1), 4), np.float32)
    got = C.c_int(0)
    ck(fn(ratio, int(radius), vp.ctypes.data_as(_D), _fp(pts), cnt.ctypes.data_as(_U), _fp(nrm), n, C.byref(got)))
    k = got.value
    return pts[:k].copy(), cnt[:k].copy(), nrm[:k].copy()


def _dense_snapshot(fn, n, leaf, ck):
    keys = np.zeros(max(n, 1), np.uint64)
    cnt = np.zeros(max(n, 1), np.uint32)
    hits = np.zeros(max(n, 1), np.uint16)
    misses = np.zeros(max(n, 1), np.uint16)
    sums = np.zeros((max(n, 1), 4), np.float64)
    got = C.c_int(0)
    ck(fn(keys.ctypes.data_as(C.POINTER(C.c_uint64)), cnt.ctypes.data_as(_U), hits.ctypes.data_as(_U16),
          misses.ctypes.data_as(_U16), sums.ctypes.data_as(_D), n, C.byref(got)))
    k = got.value
    return {"leaf": None if leaf is None else np.float32(leaf), "keys": keys[:k].copy(), "counts": cnt[:k].copy(),
            "hits": hits[:k].copy(), "misses": misses[:k].copy(), "sums": sums[:k].copy()}


def _merge_arrays(snap):
    """(counts uint32, hits uint16, misses uint16, sums N x 4 float64) of a snapshot dict, contiguous."""
    cnt = np.ascontiguousarray(snap["counts"], np.uint32).reshape(-1)
    hits = np.ascontiguousarray(snap["hits"], np.uint16).reshape(-1)
    misses = np.ascontiguousarray(snap["misses"], np.uint16).reshape(-1)
    sums = np.ascontiguousarray(snap["sums"], np.float64).reshape(-1, 4)
    if not hits.shape[0] == misses.shape[0] == sums.shape[0] == cnt.shape[0]:
        raise ValueError("dense_merge: the snapshot's arrays differ in length")
    return cnt, hits, misses, sums


def _merge_ptrs(arrays):
    cnt, hits, misses, sums = arrays
    return (cnt.ctypes.data_as(_U), hits.ctypes.data_as(_U16), misses.ctypes.data_as(_U16), sums.ctypes.data_as(_D),
            cnt.shape[0])


DENSE_SNAPSHOT_FORMAT = 1  # version of the .npz layout of save_dense_snapshot


def save_dense_snapshot(path, snap):
    """Write a snapshot (Ctx.dense_snapshot / LaserMapping.dense_map_snapshot) to a plain .npz file: the five arrays,
    the leaf and a format version; no pickled objects."""
    leaf = snap.get("leaf")
    np.savez(path, format=np.int64(DENSE_SNAPSHOT_FORMAT), leaf=np.float32(np.nan if leaf is None else leaf),
             keys=np.asarray(snap["keys"], np.uint64), counts=np.asarray(snap["counts"], np.uint32),
             hits=np.asarray(snap["hits"], np.uint16), misses=np.asarray(snap["misses"], np.uint16),
             sums=np.asarray(snap["sums"], np.float64).reshape(-1, 4))


def load_dense_snapshot(path):
    """Read a file written by save_dense_snapshot -> the snapshot dict (ValueError on another format version)."""
    with np.load(path, allow_pickle=False) as z:
        version = int(z["format"])
        if version != DENSE_SNAPSHOT_FORMAT:
            raise ValueError(f"load_dense_snapshot: format {version}, expected {DENSE_SNAPSHOT_FORMAT}")
        leaf = np.float32(z["leaf"])
        return {"leaf": None if np.isnan(leaf) else leaf, "keys": z["keys"].astype(np.uint64),
                "counts": z["counts"].astype(np.uint32), "hits": z["hits"].astype(np.uint16),
                "misses": z["misses"].astype(np.uint16), "sums": z["sums"].astype(np.float64).reshape(-1, 4)}


def _align_out(twist, iterations, n_selected, rms, degenerate, converged):
    return np.array(twist, np.float32), {"iterations": int(iterations), "n_selected": int(n_selected),
                                         "rms": np.float32(rms), "degenerate": bool(degenerate),
                                         "converged": bool(converged)}


def _poses(twists):
    """K x 6 twists -> (ctypes Pose array of at least one element, K)."""
    t = np.ascontiguousarray(twists, np.float32).reshape(-1, 6)
    poses = (Pose * max(t.shape[0], 1))()
    for i in range(t.shape[0]):
        poses[i] = make_pose(t[i])
    return poses, t.shape[0]


def _candidate(r):
    return {"hypothesis": int(r.hypothesis), "score_selected": int(r.score_selected),
            "coarse": _align_out(list(r.coarse.rot) + list(r.coarse.pos), r.coarse.iterations, r.coarse.n_selected,
                                 r.coarse.rms, r.coarse.degenerate, r.coarse.converged),
            "fine": _align_out(list(r.fine.rot) + list(r.fine.pos), r.fine.iterations, r.fine.n_selected, r.fine.rms,
                               r.fine.degenerate, r.fine.converged),
            "selected": int(r.selected), "rms": np.float32(r.rms)}


def _pts_or_device(pts, on_device, n):
    """(float pointer, count) of a host N x 4 array, or of a device address of n float[4]."""
    if on_device:
        return C.cast(C.c_void_p(int(pts)), _F), int(n)
    a = _pts(pts)
    return _fp(a), a.shape[0]


def _max_size(max_size):
    return 2147483647 if max_size is None else int(max_size)


def _segment_call(call, n, ck):
    """call(labels, segments, cap, n_out) with room for n entries (K <= n) -> (labels int32[n], dict of the K
    segments' fields)."""
    labels = np.zeros(max(n, 1), np.int32)
    seg = np.zeros(max(n, 1), SEGMENT_DTYPE)
    k = C.c_int(0)
    ck(call(_ip(labels), seg.ctypes.data_as(C.POINTER(Segment)), n, C.byref(k)))
    return labels[:n].copy(), {f: seg[f][:k.value].copy() for f in SEGMENT_DTYPE.names}


def _box_args(lo, dims):
    """(lo int32[3], dims int32[3], numpy shape (nz, ny, nx)) of a distance field's box."""
    lo_a = np.ascontiguousarray(lo, np.int32).reshape(3)
    dims_a = np.ascontiguousarray(dims, np.int32).reshape(3)
    shape = tuple(int(d) for d in dims_a[::-1]) if (dims_a >= 1).all() else (0,)
    return lo_a, dims_a, shape


def _place_match(m):
    return {"candidate": int(m.candidate), "shift": int(m.shift), "yaw": np.float32(m.yaw),
            "pos": np.array(m.pos, np.float32), "dist": float(m.dist)}


def _ne(ne: NormalEq):
    return {"AtA": np.array(ne.AtA, dtype=np.float32).reshape(6, 6), "AtB": np.array(ne.AtB, dtype=np.float32),
            "n_selected": ne.n_selected, "n_corner_selected": ne.n_corner_selected}


# ---------------------------------------------------------------------------------------------------------------------
# handles over the C++ drop-in classes
class _Handle:
    def _ck(self, rc, what):
        if rc < 0:
            raise LoamB200Error(f"{what}: {self.L.loam_b200_host_last_error().decode()}")
        return rc

    def _cloud(self, size_fn, copy_fn, which):
        n = size_fn(self.h, which)
        out = np.empty((n, 4), np.float32)
        if n:
            copy_fn(self.h, which, _fp(out))
        return out


class ScanRegistration(_Handle):
    """loam::BasicScanRegistration (reference: include/loam_velodyne/BasicScanRegistration.h:135-164)."""
    NAMES = {"full": 0, "sharp": 1, "less_sharp": 2, "flat": 3, "less_flat": 4}

    def __init__(self, handle=None):
        self.L = lib()
        self.own = handle is None
        self.h = handle if handle is not None else self.L.loam_b200_scanreg_create()

    def __del__(self):
        if getattr(self, "own", False) and self.h:
            self.L.loam_b200_scanreg_destroy(self.h)
            self.h = None

    def configure(self, scan_period=0.1, n_regions=6, curv_region=5, max_sharp=2, max_flat=4, less_flat_leaf=0.2,
                  curv_thr=0.1):
        self._ck(self.L.loam_b200_scanreg_configure(self.h, scan_period, n_regions, curv_region, max_sharp, max_flat,
                                                    less_flat_leaf, curv_thr), "configure")

    def process(self, pts, ring_sizes):
        pts = _pts(pts)
        rs = np.ascontiguousarray(ring_sizes, dtype=np.int32)
        self._ck(self.L.loam_b200_scanreg_process(self.h, _fp(pts), _ip(rs), rs.shape[0]), "processScanlines")

    def process_unordered(self, xyz, lower_deg, upper_deg, n_rings):
        """MultiScanRegistration::process: unordered sensor-frame xyz (n x 3) -> ring binning on the GPU -> extraction."""
        a = np.ascontiguousarray(xyz, dtype=np.float32)
        self._ck(self.L.loam_b200_scanreg_process_unordered(self.h, _fp(a), a.shape[0], lower_deg, upper_deg, n_rings),
                 "processUnorderedSweep")

    def cloud(self, name):
        return self._cloud(self.L.loam_b200_scanreg_cloud_size, self.L.loam_b200_scanreg_cloud_copy, self.NAMES[name])

    def indices(self, name):
        w = self.NAMES[name]
        n = self.L.loam_b200_scanreg_index_size(self.h, w)
        out = np.empty(n, np.int32)
        if n:
            self.L.loam_b200_scanreg_index_copy(self.h, w, _ip(out))
        return out


class LaserOdometry(_Handle):
    """loam::BasicLaserOdometry (reference: include/loam_velodyne/BasicLaserOdometry.h:13-48)."""
    NAMES = {"last_corner": 0, "last_surf": 1, "full": 2}

    def __init__(self, scan_period=0.1, max_iter=25, handle=None):
        self.L = lib()
        self.own = handle is None
        self.h = handle if handle is not None else self.L.loam_b200_odom_create(scan_period, max_iter)

    def __del__(self):
        if getattr(self, "own", False) and self.h:
            self.L.loam_b200_odom_destroy(self.h)
            self.h = None

    def set_inputs(self, sharp, less_sharp, flat, less_flat, full):
        a = [_pts(x) for x in (sharp, less_sharp, flat, less_flat, full)]
        self._ck(self.L.loam_b200_odom_set_inputs(self.h, _fp(a[0]), a[0].shape[0], _fp(a[1]), a[1].shape[0],
                                                  _fp(a[2]), a[2].shape[0], _fp(a[3]), a[3].shape[0], _fp(a[4]),
                                                  a[4].shape[0]), "set_inputs")

    def process(self):
        self._ck(self.L.loam_b200_odom_process(self.h), "BasicLaserOdometry::process")

    def full_to_end(self):
        self._ck(self.L.loam_b200_odom_full_to_end(self.h), "transformToEnd")

    def twist(self, which):
        out = np.empty(6, np.float32)
        self.L.loam_b200_odom_get_twist(self.h, {"transform": 0, "sum": 1}[which], _fp(out))
        return out

    def cloud(self, name):
        return self._cloud(self.L.loam_b200_odom_cloud_size, self.L.loam_b200_odom_cloud_copy, self.NAMES[name])

    def last_iterations(self):
        return self.L.loam_b200_odom_last_iterations(self.h)


class LaserMapping(_Handle):
    """loam::BasicLaserMapping (reference: include/loam_velodyne/BasicLaserMapping.h:77-111)."""
    NAMES = {"full": 0, "surround_ds": 1, "corner_from_map": 2, "surf_from_map": 3, "corner_stack_ds": 4,
             "surf_stack_ds": 5, "corner_cubes": 6, "surf_cubes": 7}

    def __init__(self, scan_period=0.1, max_iter=10, handle=None):
        self.L = lib()
        self.own = handle is None
        self.h = handle if handle is not None else self.L.loam_b200_map_create(scan_period, max_iter)

    def __del__(self):
        if getattr(self, "own", False) and self.h:
            self.L.loam_b200_map_destroy(self.h)
            self.h = None

    def retain_from_map(self, on=True):
        """Test hook: keep the reference's internal from-map clouds ("corner_from_map" / "surf_from_map") every sweep."""
        self._ck(self.L.loam_b200_map_retain_from_map(self.h, 1 if on else 0), "retainFromMapClouds")

    def seed(self, corner, surf):
        c, s = _pts(corner), _pts(surf)
        self._ck(self.L.loam_b200_map_seed(self.h, _fp(c), c.shape[0], _fp(s), s.shape[0]), "seedMap")

    def set_inputs(self, corner_last, surf_last, full):
        a = [_pts(x) for x in (corner_last, surf_last, full)]
        self._ck(self.L.loam_b200_map_set_inputs(self.h, _fp(a[0]), a[0].shape[0], _fp(a[1]), a[1].shape[0], _fp(a[2]),
                                                 a[2].shape[0]), "set_inputs")

    def update_odometry(self, sum6):
        s = np.ascontiguousarray(sum6, dtype=np.float32)
        self.L.loam_b200_map_update_odometry(self.h, _fp(s))

    def process(self):
        return bool(self._ck(self.L.loam_b200_map_process(self.h), "BasicLaserMapping::process"))

    def twist(self, which):
        out = np.empty(6, np.float32)
        self.L.loam_b200_map_get_twist(self.h, {"aft": 0, "bef": 1, "tobe": 2}[which], _fp(out))
        return out

    def cloud(self, name):
        return self._cloud(self.L.loam_b200_map_cloud_size, self.L.loam_b200_map_cloud_copy, self.NAMES[name])

    def last_iterations(self):
        return self.L.loam_b200_map_last_iterations(self.h)

    def last_phase_ms(self):
        out = np.zeros(4, np.float64)
        self.L.loam_b200_map_last_phase_seconds(self.h, out.ctypes.data_as(_D))
        return dict(zip(["begin_sweep", "lm_loop", "end_sweep", "surround"], np.round(out * 1e3, 3)))

    # ---- whole-run voxel map (BasicLaserMapping::enableDenseMap & co.)
    def enable_dense_map(self, leaf, max_voxels=DENSE_MAX_VOXELS):
        """Accumulate every mapped sweep's registered full-resolution cloud into a voxel map on the GPU (off by default)."""
        self._ck(self.L.loam_b200_map_dense_enable(self.h, np.float32(leaf), int(max_voxels)), "enableDenseMap")
        self.dense_leaf = np.float32(leaf)

    def dense_stats(self):
        """{"voxels", "skipped", "dropped"} of the whole-run voxel map."""
        out = np.zeros(3, np.int64)
        self._ck(self.L.loam_b200_map_dense_stats(self.h, out.ctypes.data_as(_LL)), "denseMapStats")
        return _dense_stats(out)

    def dense_map(self, max_miss_ratio=None, evidence=False):
        """(centroids N x 4 float32: x, y, z, intensity; counts N uint32) in ascending voxel order (x fastest).  With
        max_miss_ratio only the voxels with misses <= max_miss_ratio * hits; with evidence=True also (hits N uint16,
        misses N uint16)."""
        if max_miss_ratio is None and not evidence:
            return _dense_export(lambda pts, cnt, cap, n: self.L.loam_b200_map_dense_export(self.h, pts, cnt, cap, n),
                                 self.dense_stats()["voxels"], lambda rc: self._ck(rc, "denseMap"))
        return _dense_export_filtered(
            lambda *a: self.L.loam_b200_map_dense_export_filtered(self.h, *a), max_miss_ratio, evidence,
            self.dense_stats()["voxels"], lambda rc: self._ck(rc, "denseMap"))

    def dense_map_normals(self, max_miss_ratio=None, radius=1, viewpoint=(0.0, 0.0, 0.0)):
        """(centroids N x 4, counts N, normals N x 4: nx, ny, nz, curvature) of the voxels dense_map(max_miss_ratio)
        returns; see Ctx.dense_export_normals.  The default viewpoint, the origin, is the first sweep's sensor position."""
        return _dense_export_normals(lambda *a: self.L.loam_b200_map_dense_export_normals(self.h, *a), max_miss_ratio,
                                     radius, viewpoint, self.dense_stats()["voxels"],
                                     lambda rc: self._ck(rc, "denseMapNormals"))

    def dense_table_slots(self):
        """Test query: slots of the whole-run map's hash table (0 while the map is off)."""
        out = C.c_longlong(0)
        self._ck(self.L.loam_b200_map_debug_dense_table_slots(self.h, C.byref(out)), "denseTableSlots")
        return out.value

    def dense_map_snapshot(self):
        """BasicLaserMapping::denseMapSnapshot; returns what Ctx.dense_snapshot returns."""
        return _dense_snapshot(lambda *a: self.L.loam_b200_map_dense_snapshot(self.h, *a), self.dense_stats()["voxels"],
                               getattr(self, "dense_leaf", None), lambda rc: self._ck(rc, "denseMapSnapshot"))

    def merge_dense_map(self, snap, twist6=None):
        """BasicLaserMapping::mergeDenseMap; as Ctx.dense_merge."""
        a = _merge_arrays(snap)
        t = np.ascontiguousarray(twist6, np.float32).reshape(6) if twist6 is not None else None
        self._ck(self.L.loam_b200_map_dense_merge(self.h, *_merge_ptrs(a), _fp(t) if t is not None else None),
                 "mergeDenseMap")

    def build_dense_target(self, max_miss_ratio=None, radius=1, viewpoint=(0.0, 0.0, 0.0)):
        """BasicLaserMapping::buildDenseTarget: snapshot dense_map_normals(...) as the alignment target -> voxels."""
        ratio = math.inf if max_miss_ratio is None else float(max_miss_ratio)
        vp = np.ascontiguousarray(viewpoint, np.float64).reshape(3)
        n = C.c_int(0)
        self._ck(self.L.loam_b200_map_dense_target_build(self.h, ratio, int(radius), vp.ctypes.data_as(_D),
                                                         C.byref(n)), "buildDenseTarget")
        return n.value

    def load_dense_target(self, leaf, centroids, normals):
        """BasicLaserMapping::loadDenseTarget from host arrays; see Ctx.dense_target_load."""
        c, nr = _pts(centroids), _pts(normals)
        if c.shape[0] != nr.shape[0]:
            raise ValueError("load_dense_target: centroids and normals differ in length")
        self._ck(self.L.loam_b200_map_dense_target_load(self.h, np.float32(leaf), _fp(c), _fp(nr), c.shape[0]),
                 "loadDenseTarget")

    def align_to_dense_target(self, pts, twist6, search_radius=1, max_iterations=10):
        """BasicLaserMapping::alignToDenseTarget; returns what Ctx.dense_align returns."""
        a = _pts(pts)
        t = np.ascontiguousarray(twist6, np.float32).reshape(6)
        out = np.zeros(6, np.float32)
        st = np.zeros(4, np.int32)
        rms = np.zeros(1, np.float32)
        self._ck(self.L.loam_b200_map_dense_align(self.h, _fp(a), a.shape[0], _fp(t), int(search_radius),
                                                  int(max_iterations), _fp(out), _ip(st), _fp(rms)),
                 "alignToDenseTarget")
        return _align_out(out, st[0], st[1], rms[0], st[2], st[3])

    def score_dense_target(self, pts, twists, search_radius=3):
        """BasicLaserMapping::scoreDenseTarget; returns what Ctx.dense_score returns."""
        a = _pts(pts)
        t = np.ascontiguousarray(twists, np.float32).reshape(-1, 6)
        k = t.shape[0]
        sel = np.zeros(max(k, 1), np.int32)
        ss = np.zeros(max(k, 1), np.float32)
        self._ck(self.L.loam_b200_map_dense_score(self.h, _fp(a), a.shape[0], _fp(t), k, int(search_radius), _ip(sel),
                                                  _fp(ss)), "scoreDenseTarget")
        return sel[:k].copy(), ss[:k].copy()

    def align_to_dense_target_batch(self, pts, twists, search_radius=1, max_iterations=10):
        """BasicLaserMapping::alignToDenseTarget over a vector of twists; returns what Ctx.dense_align_batch returns."""
        a = _pts(pts)
        t = np.ascontiguousarray(twists, np.float32).reshape(-1, 6)
        k = t.shape[0]
        out = np.zeros((max(k, 1), 6), np.float32)
        st = np.zeros((max(k, 1), 4), np.int32)
        rms = np.zeros(max(k, 1), np.float32)
        self._ck(self.L.loam_b200_map_dense_align_batch(self.h, _fp(a), a.shape[0], _fp(t), k, int(search_radius),
                                                        int(max_iterations), _fp(out), _ip(st), _fp(rms)),
                 "alignToDenseTarget")
        infos = [_align_out(out[i], st[i, 0], st[i, 1], rms[i], st[i, 2], st[i, 3])[1] for i in range(k)]
        return out[:k].copy(), infos

    def relocalize_in_dense_target(self, pts, hypotheses, params=None, cap=16):
        """BasicLaserMapping::relocalizeInDenseTarget; returns what Ctx.dense_relocalize returns."""
        a = _pts(pts)
        t = np.ascontiguousarray(hypotheses, np.float32).reshape(-1, 6)
        prm = params if params is not None else RelocParams.default()
        out = (RelocCandidate * max(int(cap), 1))()
        n = C.c_int(0)
        self._ck(self.L.loam_b200_map_dense_relocalize(self.h, _fp(a), a.shape[0], _fp(t), t.shape[0], C.byref(prm), out,
                                                       int(cap), C.byref(n)), "relocalizeInDenseTarget")
        return [_candidate(r) for r in out[:n.value]]

    def raycast_dense_target(self, rays, twist6, min_range=0.0, max_range=100.0):
        """BasicLaserMapping::raycastDenseTarget; returns what Ctx.dense_raycast returns."""
        a = _pts(rays)
        t = np.ascontiguousarray(twist6, np.float32).reshape(6)
        k = a.shape[0]
        rng = np.zeros(max(k, 1), np.float32)
        idx = np.zeros(max(k, 1), np.int32)
        self._ck(self.L.loam_b200_map_dense_raycast(self.h, _fp(a), k, _fp(t), np.float32(min_range),
                                                    np.float32(max_range), _fp(rng), _ip(idx)), "raycastDenseTarget")
        return rng[:k].copy(), idx[:k].copy()

    def segment_dense_target(self, tolerance, min_size=1, max_size=None):
        """BasicLaserMapping::segmentDenseTarget; returns what Ctx.dense_segment returns."""
        n = C.c_int(0)
        self._ck(self.L.loam_b200_map_dense_target_size(self.h, C.byref(n)), "segmentDenseTarget")
        return _segment_call(lambda lab, seg, cap, k: self.L.loam_b200_map_dense_segment(
            self.h, np.float32(tolerance), int(min_size), _max_size(max_size), lab, seg, cap, k), n.value,
            lambda rc: self._ck(rc, "segmentDenseTarget"))

    def ground_dense_target(self, params=None):
        """BasicLaserMapping::groundDenseTarget; returns what Ctx.dense_ground returns."""
        prm = params if params is not None else GroundParams.default()
        n = C.c_int(0)
        self._ck(self.L.loam_b200_map_dense_target_size(self.h, C.byref(n)), "groundDenseTarget")
        return _segment_call(lambda lab, seg, cap, k: self.L.loam_b200_map_dense_ground(
            self.h, C.byref(prm), lab, seg, cap, k), n.value, lambda rc: self._ck(rc, "groundDenseTarget"))

    def segment_dense_target_above_ground(self, tolerance, min_size=1, max_size=None):
        """BasicLaserMapping::segmentDenseTargetAboveGround; returns what Ctx.dense_segment_above_ground returns."""
        n = C.c_int(0)
        self._ck(self.L.loam_b200_map_dense_target_size(self.h, C.byref(n)), "segmentDenseTargetAboveGround")
        return _segment_call(lambda lab, seg, cap, k: self.L.loam_b200_map_dense_segment_above_ground(
            self.h, np.float32(tolerance), int(min_size), _max_size(max_size), lab, seg, cap, k), n.value,
            lambda rc: self._ck(rc, "segmentDenseTargetAboveGround"))

    def split_ground(self, pts, twist6, search_radius=1, max_height=0.1):
        """BasicLaserMapping::splitGround -> (ground points, other finite points), each K x 4 in input order: the
        points Ctx.dense_ground_cloud labels 1 and 0."""
        a = _pts(pts)
        t = np.ascontiguousarray(twist6, np.float32).reshape(6)
        k = a.shape[0]
        g = np.zeros((max(k, 1), 4), np.float32)
        ng = np.zeros((max(k, 1), 4), np.float32)
        kg, kn = C.c_int(0), C.c_int(0)
        self._ck(self.L.loam_b200_map_dense_ground_cloud(self.h, _fp(a), k, _fp(t), int(search_radius),
                                                         np.float32(max_height), _fp(g), C.byref(kg), _fp(ng),
                                                         C.byref(kn)), "splitGround")
        return g[:kg.value].copy(), ng[:kn.value].copy()

    def build_dense_distance_field(self, lo, dims, max_distance, download=True):
        """BasicLaserMapping::buildDenseDistanceField; as Ctx.dense_distance_field."""
        lo_a, dims_a, shape = _box_args(lo, dims)
        dist = np.zeros(shape, np.float32) if download else None
        sq = np.zeros(shape, np.int32) if download else None
        self._ck(self.L.loam_b200_map_dense_distance_build(self.h, _ip(lo_a), _ip(dims_a), np.float32(max_distance),
                                                           _fp(dist) if download else None,
                                                           _ip(sq) if download else None), "buildDenseDistanceField")
        return dist, sq

    def query_dense_distance(self, pts, gradient=False):
        """BasicLaserMapping::queryDenseDistance; returns what Ctx.dense_distance_query returns."""
        a = _pts(pts)
        k = a.shape[0]
        dist = np.zeros(max(k, 1), np.float32)
        grad = np.zeros((max(k, 1), 3), np.float32) if gradient else None
        self._ck(self.L.loam_b200_map_dense_distance_query(self.h, _fp(a), k, _fp(dist), _fp(grad) if gradient else None),
                 "queryDenseDistance")
        return (dist[:k].copy(), grad[:k].copy()) if gradient else dist[:k].copy()

    def build_dense_places(self, positions, rays, params=None):
        """BasicLaserMapping::buildDensePlaces; as Ctx.dense_place_build."""
        prm = params if params is not None else PlaceParams.default()
        p = np.ascontiguousarray(positions, np.float32).reshape(-1, 3)
        r = _pts(rays)
        self._ck(self.L.loam_b200_map_dense_place_build(self.h, _fp(p), p.shape[0], _fp(r), r.shape[0],
                                                        C.byref(prm)), "buildDensePlaces")

    def query_dense_places(self, pts, top_m=PLACE_TOP_M):
        """BasicLaserMapping::queryDensePlaces; returns what Ctx.dense_place_query returns."""
        a = _pts(pts)
        out = (PlaceMatch * max(int(top_m), 1))()
        got = C.c_int(0)
        self._ck(self.L.loam_b200_map_dense_place_query(self.h, _fp(a), a.shape[0], int(top_m), out, C.byref(got)),
                 "queryDensePlaces")
        return [_place_match(m) for m in out[:got.value]]

    def relocalize_global_in_dense_target(self, pts, top_m=PLACE_TOP_M, yaw_step_deg=PLACE_YAW_STEP_DEG,
                                          yaw_steps=PLACE_YAW_STEPS, xz_step=PLACE_XZ_STEP, xz_steps=PLACE_XZ_STEPS,
                                          params=None, cap=16):
        """BasicLaserMapping::relocalizeGlobalInDenseTarget; returns what Ctx.dense_relocalize_global returns."""
        a = _pts(pts)
        prm = params if params is not None else RelocParams.default()
        out = (RelocCandidate * max(int(cap), 1))()
        got = C.c_int(0)
        self._ck(self.L.loam_b200_map_dense_relocalize_global(self.h, _fp(a), a.shape[0], int(top_m),
                                                              np.float32(yaw_step_deg), int(yaw_steps),
                                                              np.float32(xz_step), int(xz_steps), C.byref(prm), out,
                                                              int(cap), C.byref(got)),
                 "relocalizeGlobalInDenseTarget")
        return [_candidate(r) for r in out[:got.value]]

    def enable_dense_visibility(self, h_res_deg, v_res_deg, margin):
        """Count, per voxel of the whole-run map, the mapped sweeps that see through it (h_res_deg = 0: off); filter
        with dense_map(max_miss_ratio=...)."""
        self._ck(self.L.loam_b200_map_dense_visibility(self.h, float(h_res_deg), float(v_res_deg), float(margin)),
                 "enableDenseVisibility")

    def enable_dense_carving(self, margin=DENSE_CARVE_MARGIN, max_range=DENSE_CARVE_MAX_RANGE):
        """The visibility pass in carve mode: each mapped sweep's rays give one miss to every stored voxel they cross
        (max_range = 0: off; the range-image mode must be off); filter with dense_map(max_miss_ratio=...)."""
        self._ck(self.L.loam_b200_map_dense_carving(self.h, float(margin), float(max_range)), "enableDenseCarving")

    def clear_dense_map(self):
        self._ck(self.L.loam_b200_map_dense_clear(self.h), "clearDenseMap")

    def enable_sharding(self, rank, world, nccl_id: bytes | None):
        """Evaluate the rank-th of `world` query slices; with nccl_id (128 bytes, same on every rank) the normal
        equations are all-reduced over NCCL each iteration."""
        if nccl_id is None:
            self._ck(self.L.loam_b200_map_enable_sharding(self.h, rank, world, None), "enableSharding")
        else:
            buf = (C.c_ubyte * 128).from_buffer_copy(nccl_id)
            self._ck(self.L.loam_b200_map_enable_sharding(self.h, rank, world, buf), "enableSharding")


    def kernel_profile(self, reps=50):
        """The scan-to-map iteration kernel as this object launches it, timed with CUDA events (see the header)."""
        out = np.zeros(5, np.float64)
        self._ck(self.L.loam_b200_map_kernel_profile(self.h, reps, out.ctypes.data_as(_D)), "map_kernel_profile")
        return {"avg_us": float(out[0]), "queries": int(out[1]), "probes_per_query": float(out[2]),
                "candidates_per_query": float(out[3]), "n_selected": int(out[4])}

    def kernel_profile_queries(self, queries, reps=10):
        """... on caller-supplied surface queries in the map frame (k-NN bandwidth stress)."""
        q = _pts(queries)
        out = np.zeros(5, np.float64)
        self._ck(self.L.loam_b200_map_kernel_profile_queries(self.h, _fp(q), q.shape[0], reps, out.ctypes.data_as(_D)),
                 "map_kernel_profile_queries")
        return {"avg_us": float(out[0]), "queries": int(out[1]), "probes_per_query": float(out[2]),
                "candidates_per_query": float(out[3]), "n_selected": int(out[4])}

    # ---- multi-GPU with the map sharded by cube slabs (include/loam_b200_host.h)
    def peer_export(self) -> bytes:
        buf = (C.c_ubyte * 64)()
        self._ck(self.L.loam_b200_map_peer_export(self.h, buf), "exportPeerHandle")
        return bytes(buf)

    def enable_cube_sharding(self, rank, world, handles: bytes, slab_metres=10):
        """handles: world x 64 bytes (peer_export of every rank, in rank order)."""
        buf = (C.c_ubyte * (64 * world)).from_buffer_copy(handles)
        self._ck(self.L.loam_b200_map_enable_cube_sharding(self.h, rank, world, buf, slab_metres), "enableCubeSharding")


    def disable_cube_sharding(self):
        """Unmap the peers' inboxes; every rank calls it, then the ranks synchronise, then the objects may be destroyed."""
        self._ck(self.L.loam_b200_map_disable_cube_sharding(self.h), "disableCubeSharding")


def enable_cube_sharding_local(mappings, slab_metres=10):
    """Several LaserMapping objects of this process become the ranks 0..n-1 of one cube-sharded map."""
    L = lib()
    arr = (C.c_void_p * len(mappings))(*[m.h for m in mappings])
    if L.loam_b200_map_enable_cube_sharding_local(arr, len(mappings), slab_metres) < 0:
        raise LoamB200Error(f"enableCubeShardingLocal: {L.loam_b200_host_last_error().decode()}")


def shard_stores(x, rank, world, slab_metres=10):
    return lib().loam_b200_shard_stores(float(x), rank, world, slab_metres) == 1


def shard_owner(cell_x, world, slab_metres=10):
    return lib().loam_b200_shard_owner(int(cell_x), slab_metres, world)


class Pipeline(_Handle):
    """registration -> odometry -> mapping chained in-process on one sweep (SURVEY.md §8b "who calls it")."""

    def __init__(self, scan_period=0.1, odom_iter=25, map_iter=10):
        self.L = lib()
        self.h = self.L.loam_b200_pipeline_create(scan_period, odom_iter, map_iter)
        self.scanreg = ScanRegistration(self.L.loam_b200_pipeline_scanreg(self.h))
        self.odom = LaserOdometry(handle=self.L.loam_b200_pipeline_odom(self.h))
        self.mapping = LaserMapping(handle=self.L.loam_b200_pipeline_map(self.h))

    def __del__(self):
        if getattr(self, "h", None):
            self.L.loam_b200_pipeline_destroy(self.h)
            self.h = None

    def seed_map(self, corner, surf):
        c, s = _pts(corner), _pts(surf)
        self._ck(self.L.loam_b200_pipeline_seed_map(self.h, _fp(c), c.shape[0], _fp(s), s.shape[0]), "seed_map")

    def sweep(self, pts, ring_sizes, mode="fused"):
        """mode "fused": clouds stay in HBM between the three stages; "hostclouds": every hand-off goes through the
        reference's own entry points and host pcl clouds (as separate ROS nodes would use the classes)."""
        pts = _pts(pts)
        rs = np.ascontiguousarray(ring_sizes, dtype=np.int32)
        odom = np.empty(6, np.float32)
        aft = np.empty(6, np.float32)
        st = np.zeros(5, np.float64)
        fn = self.L.loam_b200_pipeline_sweep if mode == "fused" else self.L.loam_b200_pipeline_sweep_hostclouds
        ok = self._ck(fn(self.h, _fp(pts), _ip(rs), rs.shape[0], _fp(odom), _fp(aft), st.ctypes.data_as(_D)),
                      "pipeline_sweep")
        return bool(ok), odom, aft, st

    def sweep_device(self, device_ptr, ring_sizes):
        """Sweep already resident in GPU memory (device_ptr: address of n x 4 float32, e.g. tensor.data_ptr())."""
        rs = np.ascontiguousarray(ring_sizes, dtype=np.int32)
        odom = np.empty(6, np.float32)
        aft = np.empty(6, np.float32)
        st = np.zeros(5, np.float64)
        ok = self._ck(self.L.loam_b200_pipeline_sweep_device(self.h, C.c_void_p(device_ptr), _ip(rs), rs.shape[0],
                                                             _fp(odom), _fp(aft), st.ctypes.data_as(_D)),
                      "pipeline_sweep_device")
        return bool(ok), odom, aft, st


    def sync(self):
        """Everything enqueued by the three stages (helper threads included) has finished on the GPU."""
        self._ck(self.L.loam_b200_pipeline_sync(self.h), "pipeline_sync")

    def stage_seconds(self, reset=False):
        """Streaming mode: seconds per stage thread (registration, odometry, mapping) spent working / waiting / in hand-offs."""
        out = np.zeros(9, np.float64)
        self.L.loam_b200_pipeline_stage_seconds(self.h, out.ctypes.data_as(_D), 1 if reset else 0)
        return {"busy": out[0:3].copy(), "idle": out[3:6].copy(), "handoff": out[6:9].copy()}

    # ---- streaming form: the three stages run concurrently on consecutive sweeps (include/loam_b200_host.h)
    def submit(self, pts=None, ring_sizes=None, device_ptr=None):
        """Queue one sweep (host array `pts` or `device_ptr`); the buffer must stay alive until collected."""
        rs = np.ascontiguousarray(ring_sizes, dtype=np.int32)
        if device_ptr is None:
            pts = _pts(pts)
            self._keep = getattr(self, "_keep", [])
            self._keep.append(pts)
            rc = self.L.loam_b200_pipeline_submit(self.h, _fp(pts), None, _ip(rs), rs.shape[0])
        else:
            rc = self.L.loam_b200_pipeline_submit(self.h, None, C.c_void_p(device_ptr), _ip(rs), rs.shape[0])
        self._ck(rc, "pipeline_submit")

    def collect(self, wait=True):
        """Oldest finished sweep -> (ok, odom_sum6, map_aft6), or None when nothing is pending / ready."""
        odom = np.empty(6, np.float32)
        aft = np.empty(6, np.float32)
        ok = C.c_int(0)
        rc = self._ck(self.L.loam_b200_pipeline_collect(self.h, 1 if wait else 0, _fp(odom), _fp(aft), C.byref(ok)),
                      "pipeline_collect")
        if rc == 0:
            return None
        if getattr(self, "_keep", None):
            self._keep.pop(0)
        return bool(ok.value), odom, aft

    def run_stream(self, sweeps=None, device_ptrs=None):
        """Submit every sweep, collect every result (in order) -> list of (ok, odom_sum6, map_aft6)."""
        res = []
        n = len(sweeps)
        for i in range(n):
            if device_ptrs is not None:
                self.submit(ring_sizes=sweeps[i][1], device_ptr=device_ptrs[i])
            else:
                self.submit(sweeps[i][0], sweeps[i][1])
            r = self.collect(wait=False)
            if r is not None:
                res.append(r)
        while len(res) < n:
            r = self.collect(wait=True)
            if r is None:
                break
            res.append(r)
        self.sync()  # the last sweep's asynchronous map update has been issued and has finished
        return res


def transform_maintenance(sum6, bef6, aft6):
    """loam::BasicTransformMaintenance: updateOdometry + updateMappingTransform + transformAssociateToMap -> mapped pose."""
    a = [np.ascontiguousarray(v, dtype=np.float32).reshape(6) for v in (sum6, bef6, aft6)]
    out = np.zeros(6, np.float32)
    if lib().loam_b200_transform_maintenance(_fp(a[0]), _fp(a[1]), _fp(a[2]), _fp(out)) != 0:
        raise LoamB200Error("transform_maintenance: invalid arguments")
    return out


def gn_solve(AtA, AtB, first_iteration=True, eigen_threshold=10.0):
    """The library's 6 x 6 Gauss-Newton step (host arithmetic, same source as the device loop) -> (x, degenerate)."""
    L = lib()
    a = np.ascontiguousarray(AtA, dtype=np.float32).reshape(36)
    b = np.ascontiguousarray(AtB, dtype=np.float32).reshape(6)
    x = np.zeros(6, np.float32)
    deg = C.c_int(0)
    if L.loam_b200_host_gn_solve(_fp(a), _fp(b), 1 if first_iteration else 0, eigen_threshold, _fp(x), C.byref(deg)) != 0:
        raise LoamB200Error("gn_solve: invalid arguments")
    return x, bool(deg.value)


def reloc_grid(prior6, yaw_step_deg=RELOC_YAW_STEP_DEG, yaw_steps=None, xz_step=RELOC_XZ_STEP,
               xz_steps=RELOC_XZ_STEPS, sincos=False):
    """loam_b200_reloc_grid (host only): the relocalisation grid around prior6 -> K x 6 float32 twists, j (yaw) outer,
    then iz, then ix; yaw_steps None: a full circle, ceil(180 / yaw_step_deg).  sincos=True also returns the poses'
    cached sin and cos (K x 3 each)."""
    L = lib()
    if yaw_steps is None:
        yaw_steps = int(math.ceil(180.0 / float(np.float32(yaw_step_deg))))
    prior = make_pose(prior6)
    n = C.c_int(0)
    args = (C.byref(prior), np.float32(yaw_step_deg), int(yaw_steps), np.float32(xz_step), int(xz_steps))
    rc = L.loam_b200_reloc_grid(*args, None, 0, C.byref(n))
    if rc not in (0, -5):  # LOAM_B200_ERR_CAPACITY: the count is in n
        raise LoamB200Error(f"reloc_grid: {L.loam_b200_strerror(rc).decode()}")
    out = (Pose * n.value)()
    if L.loam_b200_reloc_grid(*args, out, n.value, C.byref(n)) != 0:
        raise LoamB200Error("reloc_grid failed")
    tw = np.array([list(p.rot) + list(p.pos) for p in out], np.float32).reshape(-1, 6)
    if not sincos:
        return tw
    return tw, np.array([list(p.sin_) for p in out], np.float32), np.array([list(p.cos_) for p in out], np.float32)


def lidar_rays(elevations_deg, n_az):
    """Unit directions of a spinning lidar in the LOAM frame, synth's convention: per elevation e (ring-major), n_az
    azimuths theta = 2 pi a / n_az, x = -sin(theta) cos(e), y = sin(e), z = cos(theta) cos(e) -> N x 4 float32 (w = 0),
    the rays of Ctx.dense_raycast."""
    e = np.radians(np.asarray(elevations_deg, np.float64).reshape(-1))[:, None]
    theta = 2.0 * math.pi * np.arange(int(n_az), dtype=np.float64)[None, :] / int(n_az)
    d = np.stack([-np.sin(theta) * np.cos(e), np.broadcast_to(np.sin(e), (e.shape[0], int(n_az))),
                  np.cos(theta) * np.cos(e), np.zeros((e.shape[0], int(n_az)))], axis=-1)
    return np.ascontiguousarray(d.reshape(-1, 4), np.float32)


def voxel_box(min_xyz, max_xyz, leaf):
    """The box of voxels (lo int32[3], dims int32[3]) that covers the map-frame corners min_xyz .. max_xyz (metres,
    x y z) by the map's voxel rule v = floorf(c * (1.0f / leaf)) in float32: lo = the voxel of min_xyz, dims = the
    voxel of max_xyz - lo + 1 (at least 1 per axis).  The argument of Ctx.dense_distance_field."""
    inv = np.float32(1.0) / np.float32(leaf)
    a = np.floor(np.asarray(min_xyz, np.float32).reshape(3) * inv).astype(np.int64)
    b = np.floor(np.asarray(max_xyz, np.float32).reshape(3) * inv).astype(np.int64)
    return a.astype(np.int32), np.maximum(b - a + 1, 1).astype(np.int32)


def place_grid(matches, yaw_step_deg=PLACE_YAW_STEP_DEG, yaw_steps=PLACE_YAW_STEPS, xz_step=PLACE_XZ_STEP,
               xz_steps=PLACE_XZ_STEPS):
    """loam_b200_place_grid (host only): the hypothesis list of dense_relocalize_global for the matches of
    dense_place_query (dicts) -> K x 6 float32 twists, reloc_grid around each match in order."""
    L = lib()
    ms = (PlaceMatch * max(len(matches), 1))()
    for i, m in enumerate(matches):
        ms[i].candidate, ms[i].shift, ms[i].yaw, ms[i].dist = m["candidate"], m["shift"], m["yaw"], m["dist"]
        for e in range(3):
            ms[i].pos[e] = m["pos"][e]
    n = C.c_int(0)
    args = (ms, len(matches), np.float32(yaw_step_deg), int(yaw_steps), np.float32(xz_step), int(xz_steps))
    rc = L.loam_b200_place_grid(*args, None, 0, C.byref(n))
    if rc not in (0, -5):  # LOAM_B200_ERR_CAPACITY: the count is in n
        raise LoamB200Error(f"place_grid: {L.loam_b200_strerror(rc).decode()}")
    out = (Pose * max(n.value, 1))()
    if L.loam_b200_place_grid(*args, out, n.value, C.byref(n)) != 0:
        raise LoamB200Error("place_grid failed")
    return np.array([list(p.rot) + list(p.pos) for p in out[:n.value]], np.float32).reshape(-1, 6)


def thin_trajectory(positions, spacing=PLACE_SPACING):
    """Places for dense_place_build from a trajectory (K x 3, in driving order): the first position, then every
    position at least `spacing` metres (straight line) from the last one kept -> M x 3 float32."""
    p = np.ascontiguousarray(positions, np.float32).reshape(-1, 3)
    keep = []
    for i in range(p.shape[0]):
        if not keep or np.linalg.norm(p[i].astype(np.float64) - p[keep[-1]].astype(np.float64)) >= spacing:
            keep.append(i)
    return p[keep].copy()


def nccl_unique_id() -> bytes:
    """128-byte NCCL id (call on rank 0, broadcast to the others)."""
    buf = (C.c_ubyte * 128)()
    if lib().loam_b200_host_nccl_unique_id(buf) != 0:
        raise LoamB200Error(lib().loam_b200_host_last_error().decode())
    return bytes(buf)


def shard_slice(n: int, rank: int, world: int):
    """Contiguous slice [lo, hi) of n queries evaluated by `rank` (mirror of map_iterate_impl in csrc/loam_b200.cu)."""
    return n * rank // world, n * (rank + 1) // world


def set_device(device: int):
    lib().loam_b200_host_set_device(device)
