"""laser_slam_b200 -- H100-native scan-to-local-map ICP + pose-graph hot path of ethz-asl/laser_slam.

This package is a thin ctypes front-end over the C ABI in include/ls_b200.h (libls_b200.so, built by
laser_slam_b200/csrc/Makefile for sm_90a).  The compute path is the CUDA library; there is NO CPU
fallback: loading fails loudly when the shared library is missing and ls_b200_init fails when no
CUDA device is usable.
"""
import collections
import ctypes
import math
import os
import struct
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "libls_b200.so")
_lib = None

LS_OK, LS_ERR_CONVERGENCE = 0, 1
LS_ERR_ARG = -1


class ConvergenceError(RuntimeError):
    """Mirror of PointMatcher::ConvergenceError (reference laser_slam/src/laser_track.cpp:499)."""


class LsError(RuntimeError):
    pass


class IcpParams(ctypes.Structure):
    _fields_ = [("max_iterations", ctypes.c_int), ("trim_ratio", ctypes.c_float),
                ("use_differential", ctypes.c_int), ("min_diff_rot", ctypes.c_float),
                ("min_diff_trans", ctypes.c_float), ("smooth_length", ctypes.c_int),
                ("cell_size", ctypes.c_float), ("leaf_split", ctypes.c_int), ("max_cells", ctypes.c_int),
                ("reading_sampling_prob", ctypes.c_float), ("reference_normals_knn", ctypes.c_int),
                ("reference_sampling_ratio", ctypes.c_float), ("unapplied_modules", ctypes.c_int)]


class IcpStats(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_int), ("converged", ctypes.c_int), ("max_iter_reached", ctypes.c_int),
                ("last_kept", ctypes.c_int), ("last_limit", ctypes.c_float), ("used_ratio", ctypes.c_float),
                ("device_ms", ctypes.c_float), ("build_ms", ctypes.c_float), ("grid_cells", ctypes.c_int),
                ("grid_tables", ctypes.c_int), ("grid_overflow", ctypes.c_int), ("icp_ms", ctypes.c_float)]


class Factor(ctypes.Structure):
    _fields_ = [("type", ctypes.c_int32), ("robust", ctypes.c_int32), ("fix_a", ctypes.c_int32),
                ("reserved", ctypes.c_int32), ("key_a", ctypes.c_uint64), ("key_b", ctypes.c_uint64),
                ("meas", ctypes.c_double * 7), ("sigma", ctypes.c_double * 6), ("fixed_a", ctypes.c_double * 7)]


class PgStats(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_int), ("n_poses", ctypes.c_int), ("n_factors", ctypes.c_int),
                ("n_border", ctypes.c_int), ("cost_first", ctypes.c_double), ("cost_last", ctypes.c_double),
                ("last_step_max", ctypes.c_double), ("device_ms", ctypes.c_float)]


FACTOR_PRIOR, FACTOR_BETWEEN = 0, 1


class PointFilter(ctypes.Structure):
    """ls_point_filter: one filter of a per-scan input chain (include/ls_b200.h, LS_PF_*)."""
    _fields_ = [("type", ctypes.c_int32), ("dim", ctypes.c_int32), ("knn", ctypes.c_int32), ("step", ctypes.c_int32),
                ("remove_inside", ctypes.c_int32), ("reserved", ctypes.c_int32), ("dist", ctypes.c_float),
                ("prob", ctypes.c_float), ("box", ctypes.c_float * 6), ("leaf", ctypes.c_float * 3),
                ("reserved_f", ctypes.c_float)]


PF_REMOVE_NAN, PF_MAX_DIST, PF_MIN_DIST, PF_BOUNDING_BOX, PF_RANDOM_SAMPLING = 1, 2, 3, 4, 5
PF_FIX_STEP_SAMPLING, PF_VOXEL_GRID, PF_SURFACE_NORMAL, PF_SAMPLING_SURFACE_NORMAL = 6, 7, 8, 9


class LocalMapParams(ctypes.Structure):
    """ls_local_map_params: the map fields of LaserSlamWorkerParams (reference laser_slam_ros/include/laser_slam_ros/
    common.hpp:20-31) plus the first buffer size."""
    _fields_ = [("distance_to_consider_fixed", ctypes.c_double), ("separate_distant_map", ctypes.c_int),
                ("voxel_size_m", ctypes.c_double), ("minimum_point_number_per_voxel", ctypes.c_int),
                ("remove_ground_from_local_map", ctypes.c_int), ("ground_distance_to_robot_center_m", ctypes.c_double),
                ("initial_capacity_points", ctypes.c_int)]


LM_LOCAL, LM_LOCAL_FILTERED, LM_DISTANT, LM_FILTERED_MAP, LM_QUEUE = 0, 1, 2, 3, 4


class OccupancyParams(ctypes.Structure):
    """ls_occupancy_params: laser_to_octomap's resolution, hit, miss and max range, volumetric_mapping's clamping and
    occupancy threshold, and the first number of 8x8x8 bricks."""
    _fields_ = [("resolution", ctypes.c_double), ("prob_hit", ctypes.c_double), ("prob_miss", ctypes.c_double),
                ("clamp_min", ctypes.c_double), ("clamp_max", ctypes.c_double), ("occupancy_threshold", ctypes.c_double),
                ("max_range", ctypes.c_double), ("initial_capacity", ctypes.c_int)]


class OccupancyStats(ctypes.Structure):
    _fields_ = [("rays_cast", ctypes.c_int64), ("rays_skipped", ctypes.c_int64), ("free_updates", ctypes.c_int64),
                ("occupied_updates", ctypes.c_int64), ("known_voxels", ctypes.c_int64), ("bricks", ctypes.c_int64),
                ("device_bytes", ctypes.c_int64), ("device_ms", ctypes.c_float)]


class OctreeStats(ctypes.Structure):
    _fields_ = [("nodes", ctypes.c_int64), ("payload_bytes", ctypes.c_int64), ("occupied_leaves", ctypes.c_int64),
                ("device_ms", ctypes.c_float)]


class FullOctreeStats(ctypes.Structure):
    _fields_ = [("nodes", ctypes.c_int64), ("leaves", ctypes.c_int64), ("payload_bytes", ctypes.c_int64),
                ("device_ms", ctypes.c_float)]


class OctomapReadStats(ctypes.Structure):
    """ls_octomap_read_stats: the file's node counts, the map's known voxels, bricks and resolution after the read."""
    _fields_ = [("nodes", ctypes.c_int64), ("inner_nodes", ctypes.c_int64), ("free_leaves", ctypes.c_int64),
                ("occupied_leaves", ctypes.c_int64), ("known_voxels", ctypes.c_int64), ("bricks", ctypes.c_int64),
                ("resolution", ctypes.c_double), ("device_ms", ctypes.c_float)]


class OccupancyEditStats(ctypes.Structure):
    """ls_occupancy_edit_stats: loop points set, voxels newly known, and the map's known voxels, bricks and device bytes
    after the call."""
    _fields_ = [("voxels_set", ctypes.c_int64), ("new_known", ctypes.c_int64), ("known_voxels", ctypes.c_int64),
                ("bricks", ctypes.c_int64), ("device_bytes", ctypes.c_int64), ("device_ms", ctypes.c_float)]


class OccupancyChangeStats(ctypes.Structure):
    """ls_occupancy_change_stats: bricks compared (the map's plus the baseline's), voxels changed, the baseline's bricks
    after the call, device bytes change detection holds and the call's device ms."""
    _fields_ = [("bricks_compared", ctypes.c_int64), ("changed", ctypes.c_int64), ("baseline_bricks", ctypes.c_int64),
                ("device_bytes", ctypes.c_int64), ("device_ms", ctypes.c_float)]


class LeafStats(ctypes.Structure):
    """ls_leaf_stats: the listed leaves per state, and per state and depth 0..16, and the call's device ms."""
    _fields_ = [("free_leaves", ctypes.c_int64), ("occupied_leaves", ctypes.c_int64),
                ("free_by_depth", ctypes.c_int64 * 17), ("occupied_by_depth", ctypes.c_int64 * 17),
                ("device_ms", ctypes.c_float)]


class GridInfo(ctypes.Structure):
    """ls_grid_info: the 2D projection's width and height in cells, resolution, origin (the lower corner of cell (0, 0)),
    the cells of -1, 0 and 100, and the call's device ms."""
    _fields_ = [("width", ctypes.c_int64), ("height", ctypes.c_int64), ("resolution", ctypes.c_double),
                ("origin_x", ctypes.c_double), ("origin_y", ctypes.c_double), ("unknown_cells", ctypes.c_int64),
                ("free_cells", ctypes.c_int64), ("occupied_cells", ctypes.c_int64), ("device_ms", ctypes.c_float)]


class OccupancyQueryStats(ctypes.Structure):
    _fields_ = [("keys_visited", ctypes.c_int64), ("device_ms", ctypes.c_float)]


class DistanceMapParams(ctypes.Structure):
    _fields_ = [("max_dist", ctypes.c_float), ("bbx_min", ctypes.c_float * 3), ("bbx_max", ctypes.c_float * 3),
                ("treat_unknown_as_occupied", ctypes.c_int)]


class DistanceMapStats(ctypes.Structure):
    """ls_distance_map_stats: the box (first key and cells per axis), cells, obstacles, the map's resolution, M, getMaxDist,
    the handle's device bytes and the update's device ms."""
    _fields_ = [("min_key", ctypes.c_int32 * 3), ("size", ctypes.c_int32 * 3), ("cells", ctypes.c_int64),
                ("obstacles", ctypes.c_int64), ("resolution", ctypes.c_double), ("max_sqdist_cells", ctypes.c_int32),
                ("max_dist", ctypes.c_float), ("device_bytes", ctypes.c_int64), ("device_ms", ctypes.c_float)]


class DistanceMapQueryStats(ctypes.Structure):
    _fields_ = [("outside", ctypes.c_int64), ("device_ms", ctypes.c_float)]


OCC_KNOWN, OCC_OCCUPIED = 1, 2
LEAVES_FREE, LEAVES_OCCUPIED, LEAVES_ALL = 1, 2, 3
CELL_FREE, CELL_OCCUPIED, CELL_UNKNOWN = 0, 1, 2
RAY_INVALID, RAY_HIT, RAY_UNKNOWN, RAY_MAX_RANGE, RAY_KEY_BOUND = 0, 1, 2, 3, 4
LS_ERR_NOMEM, LS_ERR_STATE = -3, -4


def build(force=False):
    """Compile libls_b200.so in-tree (nvcc cross-compiles sm_90a without a GPU)."""
    src_dir = os.path.join(_HERE, "csrc")
    srcs = [os.path.join(src_dir, f) for f in os.listdir(src_dir)] + [os.path.join(_HERE, "..", "include", "ls_b200.h")]
    stale = (not os.path.exists(LIB_PATH)) or os.path.getmtime(LIB_PATH) < max(os.path.getmtime(s) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-C", src_dir, "-s"])
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LsError(f"{LIB_PATH} is missing: build it with laser_slam_b200.build() "
                          "(there is no CPU fallback for this path)")
        L = ctypes.CDLL(LIB_PATH)
        vp, ci, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64
        PP, PS = ctypes.POINTER(IcpParams), ctypes.POINTER(IcpStats)
        L.ls_b200_init.argtypes = [ci, ctypes.POINTER(vp)]
        L.ls_b200_destroy.argtypes = [vp]
        L.ls_b200_destroy.restype = None
        L.ls_b200_last_error.argtypes = [vp]
        L.ls_b200_last_error.restype = ctypes.c_char_p
        L.ls_b200_launch_count.argtypes = [vp]
        L.ls_b200_launch_count.restype = u64
        L.ls_icp_default_params.argtypes = [PP]
        L.ls_icp_default_params.restype = None
        L.ls_icp_params_from_yaml.argtypes = [ctypes.c_char_p, PP]
        L.ls_icp_register.argtypes = [vp, PP, vp, ci, vp, vp, ci, ci, vp, vp, PS, vp, vp, vp]
        L.ls_nn_query.argtypes = [vp, PP, vp, ci, vp, ci, vp, vp, vp]
        L.ls_transform_cloud.argtypes = [vp, vp, vp, vp, ci, ci, vp, vp]
        L.ls_check_rigid.argtypes = [vp]
        L.ls_correct_rigid.argtypes = [vp, vp]
        L.ls_correct_rigid.restype = None
        L.ls_map_create.argtypes = [vp, ci, ci, ctypes.POINTER(vp)]
        L.ls_map_destroy.argtypes = [vp]
        L.ls_map_destroy.restype = None
        L.ls_map_push_scan.argtypes = [vp, vp, vp, ci, ci, ctypes.POINTER(u64)]
        L.ls_map_push_scan_async.argtypes = [vp, vp, vp, ci, ci, ctypes.POINTER(u64)]
        L.ls_map_sync.argtypes = [vp]
        L.ls_host_is_pinned.argtypes = [vp]
        L.ls_map_scan_size.argtypes = [vp, u64]
        L.ls_icp_register_submap.argtypes = [vp, PP, vp, u64, ci, vp, vp, vp, vp, PS, vp, vp, vp]
        L.ls_map_assemble.argtypes = [vp, vp, ci, vp, vp, vp, vp, ctypes.POINTER(ci)]
        L.ls_shard_exchange_create.argtypes = [vp, ci, ci, vp]
        L.ls_shard_exchange_connect.argtypes = [vp, vp]
        L.ls_shard_exchange_close.argtypes = [vp]
        L.ls_shard_exchange_close.restype = None
        L.ls_icp_register_submap_sharded.argtypes = [vp, PP, vp, u64, ci, vp, vp, vp, vp, PS]
        L.ls_icp_register_submaps.argtypes = [vp, PP, vp, ci, vp, vp, vp, ci, vp, vp, vp, vp, PS]
        L.ls_estimate_normals.argtypes = [vp, vp, ci, ci, vp]
        L.ls_map_push_scan_estimate_normals.argtypes = [vp, vp, ci, ci, ctypes.POINTER(u64)]
        L.ls_icp_register_submap_batch.argtypes = [vp, PP, vp, ci, vp, vp, vp, vp, vp, vp, vp, vp]
        L.ls_icp_register_submap_batch_begin.argtypes = [vp, PP, vp, ci, vp, vp, vp, vp, vp]
        L.ls_icp_register_submap_batch_end.argtypes = [vp, vp, vp, vp]
        L.ls_pg_create.argtypes = [ci, ctypes.POINTER(vp)]
        L.ls_pg_destroy.argtypes = [vp]
        L.ls_pg_destroy.restype = None
        L.ls_pg_last_error.argtypes = [vp]
        L.ls_pg_last_error.restype = ctypes.c_char_p
        L.ls_pg_launch_count.argtypes = [vp]
        L.ls_pg_launch_count.restype = u64
        L.ls_pg_num_poses.argtypes = [vp]
        L.ls_pg_num_factors.argtypes = [vp]
        L.ls_pg_add_poses.argtypes = [vp, vp, vp, vp, ci]
        L.ls_pg_set_poses.argtypes = [vp, vp, vp, ci]
        L.ls_pg_add_factors.argtypes = [vp, ctypes.POINTER(Factor), ci, vp]
        L.ls_pg_remove_factors.argtypes = [vp, vp, ci]
        L.ls_pg_optimize.argtypes = [vp, ci, ctypes.POINTER(PgStats)]
        L.ls_pg_get_poses.argtypes = [vp, vp, vp, ctypes.POINTER(ci)]
        L.ls_pg_marginals.argtypes = [vp, vp, ci, vp]
        L.ls_keep_point.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_float]
        L.ls_ingest_pointcloud2.argtypes = [ci, vp, ci, ci, ci, ci, ci, vp]
        L.ls_filter_cylinder.argtypes = [ci, vp, ci, vp, ctypes.c_double, ctypes.c_double, ci, vp, ctypes.POINTER(ci)]
        L.ls_voxel_grid.argtypes = [ci, vp, ci, vp, vp, ctypes.POINTER(ci)]
        L.ls_deskew_revolution.argtypes = [ci, vp, vp, ci, vp, vp, vp]
        L.ls_point_filters_from_yaml.argtypes = [ctypes.c_char_p, vp, ci, ctypes.POINTER(ci)]
        L.ls_filter_cloud.argtypes = [vp, vp, ci, vp, vp, ci, ci, vp, vp, ctypes.POINTER(ci)]
        L.ls_map_push_scan_filtered.argtypes = [vp, vp, ci, vp, vp, ci, ci, ctypes.POINTER(u64), ctypes.POINTER(ci)]
        L.ls_local_map_create.argtypes = [vp, ctypes.POINTER(LocalMapParams), ctypes.POINTER(vp)]
        L.ls_local_map_destroy.argtypes = [vp]
        L.ls_local_map_destroy.restype = None
        L.ls_local_map_add_scan.argtypes = [vp, vp, u64, vp, ctypes.c_double, ctypes.POINTER(ci)]
        L.ls_local_map_filter.argtypes = [vp, vp, ctypes.POINTER(ci)]
        L.ls_local_map_size.argtypes = [vp, ci]
        L.ls_local_map_download.argtypes = [vp, ci, vp, ci, ctypes.POINTER(ci)]
        L.ls_local_map_take_queue.argtypes = [vp, vp, ci, vp, ci, ctypes.POINTER(ci)]
        L.ls_local_map_transform.argtypes = [vp, vp]
        L.ls_local_map_clear.argtypes = [vp]
        i64p = ctypes.POINTER(ctypes.c_int64)
        L.ls_occupancy_default_params.argtypes = [ctypes.POINTER(OccupancyParams)]
        L.ls_occupancy_default_params.restype = None
        L.ls_occupancy_create.argtypes = [vp, ctypes.POINTER(OccupancyParams), ctypes.POINTER(vp)]
        L.ls_occupancy_destroy.argtypes = [vp]
        L.ls_occupancy_destroy.restype = None
        L.ls_occupancy_insert_scan.argtypes = [vp, vp, u64, vp, ctypes.POINTER(OccupancyStats)]
        L.ls_occupancy_size.argtypes = [vp, ci, i64p]
        L.ls_occupancy_download.argtypes = [vp, ci, vp, vp, vp, ctypes.c_int64, i64p]
        L.ls_occupancy_build_octree.argtypes = [vp, ctypes.POINTER(OctreeStats)]
        L.ls_occupancy_download_octree.argtypes = [vp, vp, ctypes.c_int64, vp, vp, ctypes.c_int64]
        L.ls_occupancy_write_octomap.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(OctreeStats)]
        L.ls_occupancy_read_octree.argtypes = [vp, vp, ctypes.c_int64, ctypes.c_int64, ctypes.c_double,
                                               ctypes.POINTER(OctomapReadStats)]
        L.ls_occupancy_read_octomap.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(OctomapReadStats)]
        L.ls_occupancy_build_full_octree.argtypes = [vp, ctypes.POINTER(FullOctreeStats)]
        L.ls_occupancy_download_full_octree.argtypes = [vp, vp, ctypes.c_int64]
        L.ls_occupancy_write_octomap_full.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(FullOctreeStats)]
        L.ls_occupancy_read_full_octree.argtypes = [vp, vp, ctypes.c_int64, ctypes.c_int64, ctypes.c_double,
                                                    ctypes.POINTER(OctomapReadStats)]
        L.ls_occupancy_read_octomap_full.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(OctomapReadStats)]
        QS = ctypes.POINTER(OccupancyQueryStats)
        L.ls_occupancy_cell_status.argtypes = [vp, vp, ci, vp, vp, QS]
        L.ls_occupancy_line_status.argtypes = [vp, vp, vp, ci, vp, ci, vp, vp, QS]
        L.ls_occupancy_cast_rays.argtypes = [vp, vp, vp, ci, ci, ctypes.c_double, vp, vp, QS]
        L.ls_occupancy_box_status.argtypes = [vp, vp, vp, ci, vp, QS]
        L.ls_occupancy_check_paths.argtypes = [vp, vp, vp, ci, vp, ci, vp, QS]
        L.ls_occupancy_set_boxes.argtypes = [vp, vp, vp, vp, ci, ctypes.POINTER(OccupancyEditStats)]
        L.ls_occupancy_clear.argtypes = [vp]
        L.ls_occupancy_box_voxels.argtypes = [vp, vp, vp, ci, vp, vp, vp, ctypes.c_int64, i64p]
        L.ls_occupancy_bounds.argtypes = [vp, vp, vp]
        L.ls_occupancy_track_changes.argtypes = [vp, ci]
        L.ls_occupancy_changes.argtypes = [vp, vp, vp, vp, vp, ctypes.c_int64, i64p, ci,
                                           ctypes.POINTER(OccupancyChangeStats)]
        L.ls_occupancy_build_leaves.argtypes = [vp, vp, vp, ctypes.POINTER(LeafStats)]
        L.ls_occupancy_download_leaves.argtypes = [vp, ci, vp, vp, vp, ctypes.c_int64, i64p]
        L.ls_occupancy_marker_cubes.argtypes = [vp, ctypes.c_double, ctypes.c_double, ctypes.c_double, vp, vp, vp, vp,
                                                ctypes.c_int64, i64p]
        L.ls_occupancy_build_projection.argtypes = [vp, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                                    ctypes.POINTER(GridInfo)]
        L.ls_occupancy_download_projection.argtypes = [vp, vp, ctypes.c_int64]
        L.ls_distance_map_create.argtypes = [vp, ctypes.POINTER(DistanceMapParams), ctypes.POINTER(vp)]
        L.ls_distance_map_destroy.argtypes = [vp]
        L.ls_distance_map_destroy.restype = None
        L.ls_distance_map_update.argtypes = [vp, vp, ctypes.POINTER(DistanceMapStats)]
        L.ls_distance_map_query.argtypes = [vp, vp, ci, vp, vp, vp, ctypes.POINTER(DistanceMapQueryStats)]
        L.ls_distance_map_download.argtypes = [vp, vp, vp, ctypes.c_int64, i64p]
        _lib = L
    return _lib


def default_params(**kw):
    p = IcpParams()
    lib().ls_icp_default_params(ctypes.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def params_from_yaml(text):
    p = IcpParams()
    rc = lib().ls_icp_params_from_yaml(text.encode(), ctypes.byref(p))
    if rc != 0:
        raise LsError(f"unsupported ICP chain configuration (rc={rc})")
    return p


def keep_mask(n, salt, prob):
    """ls_keep_point for indices 0..n-1: the deterministic RandomSamplingDataPointsFilter rule (host side of the C ABI)."""
    f = lib().ls_keep_point
    return np.fromiter((f(i, salt, prob) for i in range(n)), dtype=bool, count=n)


def point_filters_from_yaml(text):
    """Parse a DataPointsFilters YAML list (LaserTrackParams::icp_input_filters_file) into a chain of PointFilter records
    (ls_point_filters_from_yaml).  Host code, no GPU needed.  Raises LsError naming the index of a refused filter."""
    n = ctypes.c_int(0)
    rc = lib().ls_point_filters_from_yaml(text.encode(), None, 0, ctypes.byref(n))
    if rc != 0:
        raise LsError(f"unsupported input filter #{n.value} (rc={rc})")
    arr = (PointFilter * max(n.value, 1))()
    rc = lib().ls_point_filters_from_yaml(text.encode(), ctypes.cast(arr, ctypes.c_void_p), n.value, ctypes.byref(n))
    if rc != 0:
        raise LsError(f"unsupported input filter #{n.value} (rc={rc})")
    return list(arr[:n.value])


def _chain(filters):
    if isinstance(filters, str):
        filters = point_filters_from_yaml(filters)
    filters = list(filters)
    arr = (PointFilter * max(len(filters), 1))(*filters)
    return arr, len(filters)


READING_SALT, REFERENCE_SALT = 0x7e11, 0x5a17   # the salts PointMatcher::DataPointsFilters uses (compat.hpp)


def _rc(rc, what):
    if rc != 0:
        raise LsError(f"{what}: rc={rc}")


def ingest_pointcloud2(data, point_step, off_x, off_y, off_z, n, device=0):
    """sensor_msgs/PointCloud2 payload (bytes / uint8 array) -> (n,4) float32 features {x,y,z,1} on the device."""
    buf = np.frombuffer(data, np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data.view(np.uint8))
    out = np.empty((max(n, 1), 4), np.float32)
    _rc(lib().ls_ingest_pointcloud2(device, buf.ctypes.data, point_step, off_x, off_y, off_z, n, out.ctypes.data), "ls_ingest_pointcloud2")
    return out[:n]


def filter_cylinder(pts4, center, radius_m, height_m, remove_points_inside=False, device=0):
    """applyCylindricalFilter (reference laser_slam_ros/include/laser_slam_ros/common.hpp:194-223) on the device."""
    p = np.ascontiguousarray(pts4, np.float32)
    c = np.ascontiguousarray(center, np.float64)
    out = np.empty((max(len(p), 1), 4), np.float32)
    n = ctypes.c_int(0)
    _rc(lib().ls_filter_cylinder(device, p.ctypes.data, len(p), c.ctypes.data, float(radius_m), float(height_m),
                                 int(bool(remove_points_inside)), out.ctypes.data, ctypes.byref(n)), "ls_filter_cylinder")
    return out[:n.value].copy()


def voxel_grid(pts4, leaf_size, device=0):
    """pcl::VoxelGrid centroids (reference laser_slam_ros/src/laser_slam_worker.cpp:434-441) on the device."""
    p = np.ascontiguousarray(pts4, np.float32)
    leaf = np.ascontiguousarray(np.broadcast_to(np.asarray(leaf_size, np.float32), (3,)), np.float32)
    out = np.empty((max(len(p), 1), 4), np.float32)
    n = ctypes.c_int(0)
    _rc(lib().ls_voxel_grid(device, p.ctypes.data, len(p), leaf.ctypes.data, out.ctypes.data, ctypes.byref(n)), "ls_voxel_grid")
    return out[:n.value].copy()


def deskew_revolution(points4, packet_offsets, T_packets, T_final, device=0):
    """The point arithmetic of the Velodyne assembler (reference sensor_drivers/velodyne_assembler/src/
    velodyne_assembler_ros.cpp:57-143) on the device: packet k = points[packet_offsets[k]:packet_offsets[k+1]] is moved by
    T_packets[k] and then everything by T_final (4x4 row-major numpy matrices here; ls_deskew_revolution)."""
    p = np.ascontiguousarray(points4, np.float32)
    offs = np.ascontiguousarray(packet_offsets, np.int32)
    K = len(offs) - 1
    tp = np.ascontiguousarray(np.stack([colmajor(T) for T in T_packets]), np.float32) if K > 0 else np.zeros((1, 16), np.float32)
    tf = colmajor(T_final)
    out = np.empty((max(len(p), 1), 4), np.float32)
    _rc(lib().ls_deskew_revolution(device, p.ctypes.data, offs.ctypes.data, K, tp.ctypes.data, tf.ctypes.data, out.ctypes.data),
        "ls_deskew_revolution")
    return out[:len(p)].copy()


def apply_chain_filters(ctx, reading4, ref4, ref_normals3, params):
    """The reading / reference DataPointsFilters of an ICP chain (icp_default.yaml:1-7) as PointMatcher::ICP::compute runs
    them before matching, in their deterministic form: RandomSampling of the reading (ls_keep_point), surface normals of
    the reference on the device (ls_estimate_normals, exact k-NN) and its sampling.  Returns (reading, ref, ref_normals)."""
    reading4 = np.ascontiguousarray(reading4, np.float32)
    ref4 = np.ascontiguousarray(ref4, np.float32)
    if params.reading_sampling_prob < 1.0:
        reading4 = np.ascontiguousarray(reading4[keep_mask(len(reading4), READING_SALT, params.reading_sampling_prob)])
    if params.reference_normals_knn > 0:
        ref_normals3 = ctx.estimate_normals(ref4, knn=max(3, min(16, params.reference_normals_knn)))
        if params.reference_sampling_ratio < 1.0:
            keep = keep_mask(len(ref4), REFERENCE_SALT, params.reference_sampling_ratio)
            ref4, ref_normals3 = np.ascontiguousarray(ref4[keep]), np.ascontiguousarray(ref_normals3[keep])
    return reading4, ref4, ref_normals3


def colmajor(T):
    return np.ascontiguousarray(np.asarray(T, np.float32).T).ravel()


def from_colmajor(t16):
    return np.asarray(t16).reshape(4, 4).T.copy()


def _ptr(a):
    return a.ctypes.data if a is not None else None


def _f32c(a, cols):
    a = np.asarray(a)
    if a.dtype != np.float32 or not a.flags.c_contiguous:
        a = np.ascontiguousarray(a, np.float32)
    assert a.ndim == 2 and a.shape[1] == cols, f"expected (N,{cols}) float32"
    return a


class Context:
    """One ls_ctx: one CUDA device, one stream; calls are synchronous (results on the host at return)."""

    def __init__(self, device=0):
        self._h = ctypes.c_void_p()
        rc = lib().ls_b200_init(device, ctypes.byref(self._h))
        if rc != 0:
            raise LsError(f"ls_b200_init(device={device}) failed with {rc}: no usable CUDA device "
                          "(this path has no CPU fallback)")

    def close(self):
        if self._h:
            lib().ls_b200_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc == LS_ERR_CONVERGENCE:
            raise ConvergenceError(lib().ls_b200_last_error(self._h).decode())
        if rc != 0:
            raise LsError(f"rc={rc}: {lib().ls_b200_last_error(self._h).decode()}")

    @property
    def launch_count(self):
        return int(lib().ls_b200_launch_count(self._h))

    def set_icp_cta_budget(self, ctas):
        """ls_b200_set_icp_cta_budget: cap the persistent ICP kernel's CTAs (0 = all); returns the budget in force."""
        self._check(lib().ls_b200_set_icp_cta_budget(self._h, int(ctas)))
        return int(lib().ls_b200_icp_cta_budget(self._h))

    def shard_exchange_create(self, shard_rank, shard_count):
        """Query-sharded registration, step 1 on every shard: allocate this GPU's exchange buffer; returns its 64 IPC
        handle bytes (ls_shard_exchange_create)."""
        h = np.zeros(64, np.uint8)
        self._check(lib().ls_shard_exchange_create(self._h, int(shard_rank), int(shard_count), h.ctypes.data))
        return h.tobytes()

    def shard_exchange_connect(self, handles):
        """Step 2 on every shard: map the peers' buffers; `handles` = every shard's handle bytes in rank order."""
        h = np.frombuffer(b"".join(bytes(x) for x in handles), np.uint8).copy()
        self._check(lib().ls_shard_exchange_connect(self._h, h.ctypes.data))

    def icp_register(self, reading4, ref4, ref_normals3, T0, params=None, want_ids=False, want_hist=False,
                     raise_on_convergence=True):
        """PointMatcher::ICP::compute(reading, reference, T0).  Returns dict(T, stats, rc[, ids, d2, T_iter_hist])."""
        reading4, ref4 = _f32c(reading4, 4), _f32c(ref4, 4)
        nrm = np.asarray(ref_normals3)
        if nrm.dtype != np.float32 or not nrm.flags.c_contiguous:
            nrm = np.ascontiguousarray(nrm, np.float32)
        stride = nrm.shape[1]
        p = params or default_params()
        n, m = reading4.shape[0], ref4.shape[0]
        t0 = colmajor(T0)
        tout = np.empty(16, np.float32)
        st = IcpStats()
        ids = np.empty(max(n, 1), np.int32) if want_ids else None
        d2 = np.empty(max(n, 1), np.float32) if want_ids else None
        hist = np.zeros((p.max_iterations, 16), np.float32) if want_hist else None
        rc = lib().ls_icp_register(self._h, ctypes.byref(p), reading4.ctypes.data, n, ref4.ctypes.data, nrm.ctypes.data,
                                   stride, m, t0.ctypes.data, tout.ctypes.data, ctypes.byref(st), _ptr(ids), _ptr(d2),
                                   _ptr(hist))
        if rc != LS_ERR_CONVERGENCE or raise_on_convergence:
            self._check(rc)
        out = dict(T=from_colmajor(tout), stats=st, rc=rc)
        if want_ids:
            out["ids"], out["d2"] = ids[:n], d2[:n]
        if want_hist:
            out["T_iter_hist"] = hist[:st.iterations].reshape(-1, 4, 4).transpose(0, 2, 1).copy()
        return out

    def nn_query(self, reading4, ref4, T0=None, params=None):
        reading4, ref4 = _f32c(reading4, 4), _f32c(ref4, 4)
        p = params or default_params()
        n = reading4.shape[0]
        t0 = colmajor(np.eye(4) if T0 is None else T0)
        ids = np.empty(max(n, 1), np.int32)
        d2 = np.empty(max(n, 1), np.float32)
        self._check(lib().ls_nn_query(self._h, ctypes.byref(p), reading4.ctypes.data, n, ref4.ctypes.data,
                                      ref4.shape[0], t0.ctypes.data, ids.ctypes.data, d2.ctypes.data))
        return ids[:n], d2[:n]

    def transform_cloud(self, T, pts4, normals3=None):
        pts4 = _f32c(pts4, 4)
        n = pts4.shape[0]
        out = np.empty_like(pts4)
        nrm = nout = None
        if normals3 is not None:
            nrm = _f32c(normals3, 3)
            nout = np.empty_like(nrm)
        t = colmajor(T)
        self._check(lib().ls_transform_cloud(self._h, t.ctypes.data, pts4.ctypes.data, _ptr(nrm), 3, n, out.ctypes.data,
                                             _ptr(nout)))
        return (out, nout) if normals3 is not None else out

    def estimate_normals(self, pts4, knn=10):
        """Surface normals of a cloud (scan frame) on the device: exact kNN -> covariance -> smallest eigenvector."""
        pts4 = _f32c(pts4, 4)
        out = np.empty((max(pts4.shape[0], 1), 3), np.float32)
        self._check(lib().ls_estimate_normals(self._h, pts4.ctypes.data, pts4.shape[0], knn, out.ctypes.data))
        return out[:pts4.shape[0]]

    def filter_cloud(self, filters, pts4, normals3=None, want_normals=None):
        """Run a per-scan input chain (PointFilter list or its YAML text) on the device: ls_filter_cloud.  Returns
        (points (m,4), normals (m,3) or None).  want_normals defaults to: the input has normals or the chain makes them."""
        arr, nf = _chain(filters)
        pts4 = _f32c(pts4, 4)
        n = pts4.shape[0]
        nrm = None if normals3 is None else _f32c(normals3, 3)
        if want_normals is None:
            want_normals = nrm is not None or any(f.type in (PF_SURFACE_NORMAL, PF_SAMPLING_SURFACE_NORMAL) for f in arr[:nf])
        out = np.empty((max(n, 1), 4), np.float32)
        nout = np.empty((max(n, 1), 3), np.float32) if want_normals else None
        m = ctypes.c_int(0)
        self._check(lib().ls_filter_cloud(self._h, ctypes.cast(arr, ctypes.c_void_p), nf, pts4.ctypes.data, _ptr(nrm), 3, n,
                                          out.ctypes.data, _ptr(nout), ctypes.byref(m)))
        return out[:m.value].copy(), (nout[:m.value].copy() if want_normals else None)

    def create_map(self, capacity_scans, max_pts_per_scan):
        return Map(self, capacity_scans, max_pts_per_scan)

    def create_local_map(self, **params):
        return LocalMap(self, **params)

    def create_occupancy_map(self, **params):
        return OccupancyMap(self, **params)


class Map:
    """Device-resident ring of the last `capacity_scans` scans (LaserTrack::laser_scans_ on the GPU)."""

    def __init__(self, ctx, capacity_scans, max_pts_per_scan):
        self.ctx = ctx
        self._h = ctypes.c_void_p()
        ctx._check(lib().ls_map_create(ctx._h, capacity_scans, max_pts_per_scan, ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().ls_map_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def push_scan(self, features4, normals3):
        f = _f32c(features4, 4)
        nrm = np.asarray(normals3)
        if nrm.dtype != np.float32 or not nrm.flags.c_contiguous:
            nrm = np.ascontiguousarray(nrm, np.float32)
        sid = ctypes.c_uint64(0)
        self.ctx._check(lib().ls_map_push_scan(self._h, f.ctypes.data, nrm.ctypes.data, nrm.shape[1], f.shape[0],
                                               ctypes.byref(sid)))
        return sid.value

    def push_scan_estimate_normals(self, features4, knn=10):
        f = _f32c(features4, 4)
        sid = ctypes.c_uint64(0)
        self.ctx._check(lib().ls_map_push_scan_estimate_normals(self._h, f.ctypes.data, f.shape[0], knn, ctypes.byref(sid)))
        return sid.value

    def push_scan_filtered(self, filters, features4, normals3=None):
        """ls_map_push_scan_filtered: a raw scan through a per-scan input chain (PointFilter list or its YAML text) into
        the next slot, all on the device.  Returns (scan id, points kept)."""
        arr, nf = _chain(filters)
        f = _f32c(features4, 4)
        nrm = None if normals3 is None else _f32c(normals3, 3)
        sid, kept = ctypes.c_uint64(0), ctypes.c_int(0)
        self.ctx._check(lib().ls_map_push_scan_filtered(self._h, ctypes.cast(arr, ctypes.c_void_p), nf, f.ctypes.data, _ptr(nrm), 3,
                                                        f.shape[0], ctypes.byref(sid), ctypes.byref(kept)))
        return sid.value, kept.value

    def push_scan_raw(self, feat_ptr, nrm_ptr, nrm_stride, n):
        """Pointer form (e.g. torch pinned tensors' data_ptr()) -- no numpy conversion on the way."""
        sid = ctypes.c_uint64(0)
        self.ctx._check(lib().ls_map_push_scan(self._h, feat_ptr, nrm_ptr, nrm_stride, n, ctypes.byref(sid)))
        return sid.value

    def push_scan_raw_async(self, feat_ptr, nrm_ptr, nrm_stride, n):
        """ls_map_push_scan_async: enqueue the upload and return; the buffers (pinned) must stay valid until `sync()`
        or until a registration that uses the scan has returned."""
        sid = ctypes.c_uint64(0)
        self.ctx._check(lib().ls_map_push_scan_async(self._h, feat_ptr, nrm_ptr, nrm_stride, n, ctypes.byref(sid)))
        return sid.value

    def sync(self):
        self.ctx._check(lib().ls_map_sync(self._h))

    def scan_size(self, scan_id):
        return int(lib().ls_map_scan_size(self._h, scan_id))

    def register(self, reading_id, part_ids, T_parts, T0, params=None, want_ids=False, want_hist=False,
                 raise_on_convergence=True):
        """Scan -> sub-map ICP on resident scans (LaserTrack::localScanToSubMap, reference laser_track.cpp:466-519)."""
        p = params or default_params()
        ids_arr = np.ascontiguousarray(part_ids, np.uint64)
        tp = np.ascontiguousarray(np.stack([colmajor(T) for T in T_parts]), np.float32)
        t0 = colmajor(T0)
        tout = np.empty(16, np.float32)
        st = IcpStats()
        n = self.scan_size(reading_id)
        ids = np.empty(max(n, 1), np.int32) if want_ids else None
        d2 = np.empty(max(n, 1), np.float32) if want_ids else None
        hist = np.zeros((p.max_iterations, 16), np.float32) if want_hist else None
        rc = lib().ls_icp_register_submap(self.ctx._h, ctypes.byref(p), self._h, reading_id, len(ids_arr),
                                          ids_arr.ctypes.data, tp.ctypes.data, t0.ctypes.data, tout.ctypes.data,
                                          ctypes.byref(st), _ptr(ids), _ptr(d2), _ptr(hist))
        if rc != LS_ERR_CONVERGENCE or raise_on_convergence:
            self.ctx._check(rc)
        out = dict(T=from_colmajor(tout), stats=st, rc=rc)
        if want_ids:
            out["ids"], out["d2"] = ids[:n], d2[:n]
        if want_hist:
            out["T_iter_hist"] = hist[:st.iterations].reshape(-1, 4, 4).transpose(0, 2, 1).copy()
        return out

    def register_sharded(self, reading_id, part_ids, T_parts, T0, params=None, raise_on_convergence=True):
        """This process's share of ONE registration sharded by queries over the GPUs of the node
        (ls_icp_register_submap_sharded): a collective -- every shard makes the same call on its own copy of the map.
        The context needs its exchange first (Context.shard_exchange_create + _connect, or dist.ShardedRegistrar)."""
        p = params or default_params()
        ids_arr = np.ascontiguousarray(part_ids, np.uint64)
        tp = np.ascontiguousarray(np.stack([colmajor(T) for T in T_parts]), np.float32)
        t0 = colmajor(T0)
        tout = np.empty(16, np.float32)
        st = IcpStats()
        rc = lib().ls_icp_register_submap_sharded(self.ctx._h, ctypes.byref(p), self._h, reading_id, len(ids_arr),
                                                  ids_arr.ctypes.data, tp.ctypes.data, t0.ctypes.data, tout.ctypes.data,
                                                  ctypes.byref(st))
        if rc != LS_ERR_CONVERGENCE or raise_on_convergence:
            self.ctx._check(rc)
        return dict(T=from_colmajor(tout), stats=st, rc=rc)

    def prepare(self, reading_id, part_ids, T_parts, T0, params=None):
        """Marshal one registration's arguments once; returns a zero-argument callable that performs the C call
        (ls_icp_register_submap) and returns (rc, T_out 4x4, stats).  For callers that pre-stage their inputs."""
        p = params or default_params()
        ids_arr = np.ascontiguousarray(part_ids, np.uint64)
        tp = np.ascontiguousarray(np.stack([colmajor(T) for T in T_parts]), np.float32)
        t0 = colmajor(T0)
        tout = np.empty(16, np.float32)
        st = IcpStats()
        fn = lib().ls_icp_register_submap
        args = (self.ctx._h, ctypes.byref(p), self._h, ctypes.c_uint64(reading_id), len(ids_arr), ids_arr.ctypes.data,
                tp.ctypes.data, t0.ctypes.data, tout.ctypes.data, ctypes.byref(st), None, None, None)
        keep = (p, ids_arr, tp, t0)

        def call(_fn=fn, _args=args, _tout=tout, _st=st, _keep=keep):
            return _fn(*_args), _tout, _st
        return call

    def prepare_batch(self, problems, params=None):
        """problems: list of (reading_id, part_ids, T_parts, T0).  Marshals once; returns a callable performing
        ls_icp_register_submap_batch and returning (rc, statuses, T_outs (B,4,4 col-major flat 16), stats array)."""
        p = params or default_params()
        B = len(problems)
        rids = np.ascontiguousarray([pr[0] for pr in problems], np.uint64)
        nparts = np.ascontiguousarray([len(pr[1]) for pr in problems], np.int32)
        pids = np.ascontiguousarray(np.concatenate([np.asarray(pr[1], np.uint64) for pr in problems]), np.uint64)
        tparts = np.ascontiguousarray(np.concatenate([np.stack([colmajor(T) for T in pr[2]]) for pr in problems]), np.float32)
        t0s = np.ascontiguousarray(np.stack([colmajor(pr[3]) for pr in problems]), np.float32)
        touts = np.empty((B, 16), np.float32)
        stats = (IcpStats * B)()
        statuses = np.zeros(B, np.int32)
        fn = lib().ls_icp_register_submap_batch
        args = (self.ctx._h, ctypes.byref(p), self._h, B, rids.ctypes.data, nparts.ctypes.data, pids.ctypes.data,
                tparts.ctypes.data, t0s.ctypes.data, touts.ctypes.data, ctypes.cast(stats, ctypes.c_void_p), statuses.ctypes.data)
        keep = (p, rids, nparts, pids, tparts, t0s)

        def call(_fn=fn, _args=args, _keep=keep):
            return _fn(*_args), statuses, touts, stats
        return call

    def prepare_begin_batch(self, problems, params=None):
        """Marshal once; returns (begin, end): `begin()` = ls_icp_register_submap_batch_begin (stage + launch, returns at once),
        `end()` = ls_icp_register_submap_batch_end -> (rc, statuses, T_outs (B,16), stats array).  For callers that pre-stage
        their inputs and interleave several contexts."""
        p = params or default_params()
        B = len(problems)
        rids = np.ascontiguousarray([pr[0] for pr in problems], np.uint64)
        nparts = np.ascontiguousarray([len(pr[1]) for pr in problems], np.int32)
        pids = np.ascontiguousarray(np.concatenate([np.asarray(pr[1], np.uint64) for pr in problems]), np.uint64)
        tparts = np.ascontiguousarray(np.concatenate([np.stack([colmajor(T) for T in pr[2]]) for pr in problems]), np.float32)
        t0s = np.ascontiguousarray(np.stack([colmajor(pr[3]) for pr in problems]), np.float32)
        touts = np.empty((B, 16), np.float32)
        stats = (IcpStats * B)()
        statuses = np.zeros(B, np.int32)
        L = lib()
        bargs = (self.ctx._h, ctypes.byref(p), self._h, B, rids.ctypes.data, nparts.ctypes.data, pids.ctypes.data,
                 tparts.ctypes.data, t0s.ctypes.data)
        eargs = (self.ctx._h, touts.ctypes.data, ctypes.cast(stats, ctypes.c_void_p), statuses.ctypes.data)
        keep = (p, rids, nparts, pids, tparts, t0s)

        def begin(_f=L.ls_icp_register_submap_batch_begin, _a=bargs, _k=keep):
            rc = _f(*_a)
            if rc != 0:
                self.ctx._check(rc)

        def end(_f=L.ls_icp_register_submap_batch_end, _a=eargs):
            return _f(*_a), statuses, touts, stats
        return begin, end

    def begin_batch(self, problems, params=None):
        """ls_icp_register_submap_batch_begin: stage and launch, return at once.  The returned callable is
        ls_icp_register_submap_batch_end: it waits and returns the same list of dicts as `register_batch`."""
        p = params or default_params()
        B = len(problems)
        rids = np.ascontiguousarray([pr[0] for pr in problems], np.uint64)
        nparts = np.ascontiguousarray([len(pr[1]) for pr in problems], np.int32)
        pids = np.ascontiguousarray(np.concatenate([np.asarray(pr[1], np.uint64) for pr in problems]), np.uint64)
        tparts = np.ascontiguousarray(np.concatenate([np.stack([colmajor(T) for T in pr[2]]) for pr in problems]), np.float32)
        t0s = np.ascontiguousarray(np.stack([colmajor(pr[3]) for pr in problems]), np.float32)
        self.ctx._check(lib().ls_icp_register_submap_batch_begin(self.ctx._h, ctypes.byref(p), self._h, B, rids.ctypes.data,
                                                                 nparts.ctypes.data, pids.ctypes.data, tparts.ctypes.data,
                                                                 t0s.ctypes.data))

        def end(_keep=(p, rids, nparts, pids, tparts, t0s)):
            touts = np.empty((B, 16), np.float32)
            stats = (IcpStats * B)()
            statuses = np.zeros(B, np.int32)
            rc = lib().ls_icp_register_submap_batch_end(self.ctx._h, touts.ctypes.data, ctypes.cast(stats, ctypes.c_void_p),
                                                        statuses.ctypes.data)
            self.ctx._check(rc if rc < 0 else 0)
            return [dict(T=from_colmajor(touts[b]), rc=int(statuses[b]), stats=stats[b]) for b in range(B)]
        return end

    def register_batch(self, problems, params=None):
        rc, statuses, touts, stats = self.prepare_batch(problems, params)()
        self.ctx._check(rc if rc < 0 else 0)
        return [dict(T=from_colmajor(touts[b]), rc=int(statuses[b]), stats=stats[b]) for b in range(len(problems))]

    def register_submaps(self, ref_ids, T_refs, reading_map, reading_ids, T_readings, T0, params=None,
                         raise_on_convergence=True):
        """Sub-map <-> sub-map ICP with both clouds assembled on the device (the loop-closure ICP of
        IncrementalEstimator::processLoopClosure, reference incremental_estimator.cpp:90-115).  `self` holds the
        reference parts, `reading_map` the reading parts (may be the same map)."""
        p = params or default_params()
        ra = np.ascontiguousarray(ref_ids, np.uint64)
        rt = np.ascontiguousarray(np.stack([colmajor(T) for T in T_refs]), np.float32)
        da = np.ascontiguousarray(reading_ids, np.uint64)
        dt = np.ascontiguousarray(np.stack([colmajor(T) for T in T_readings]), np.float32)
        t0 = colmajor(T0)
        tout = np.empty(16, np.float32)
        st = IcpStats()
        rc = lib().ls_icp_register_submaps(self.ctx._h, ctypes.byref(p), self._h, len(ra), ra.ctypes.data, rt.ctypes.data,
                                           reading_map._h, len(da), da.ctypes.data, dt.ctypes.data, t0.ctypes.data,
                                           tout.ctypes.data, ctypes.byref(st))
        if rc != LS_ERR_CONVERGENCE or raise_on_convergence:
            self.ctx._check(rc)
        return dict(T=from_colmajor(tout), stats=st, rc=rc)

    def assemble(self, part_ids, T_parts, want_normals=True):
        ids_arr = np.ascontiguousarray(part_ids, np.uint64)
        tp = np.ascontiguousarray(np.stack([colmajor(T) for T in T_parts]), np.float32)
        m = sum(self.scan_size(int(i)) for i in ids_arr)
        out = np.empty((max(m, 1), 4), np.float32)
        nout = np.empty((max(m, 1), 3), np.float32) if want_normals else None
        mo = ctypes.c_int(0)
        self.ctx._check(lib().ls_map_assemble(self.ctx._h, self._h, len(ids_arr), ids_arr.ctypes.data, tp.ctypes.data,
                                              out.ctypes.data, _ptr(nout), ctypes.byref(mo)))
        return out[:mo.value], (nout[:mo.value] if want_normals else None)


class LocalMap:
    """LaserSlamWorker's local map on the device (ls_local_map_*): local_map_, local_map_filtered_, distant_map_ and
    local_map_queue_ next to a Map ring.  Keyword arguments are the LocalMapParams fields; the defaults are
    LaserSlamWorkerParams' usual values."""

    def __init__(self, ctx, distance_to_consider_fixed=20.0, separate_distant_map=True, voxel_size_m=0.1,
                 minimum_point_number_per_voxel=0, remove_ground_from_local_map=False,
                 ground_distance_to_robot_center_m=1.0, initial_capacity_points=0):
        self.ctx = ctx
        self.params = LocalMapParams(float(distance_to_consider_fixed), int(bool(separate_distant_map)), float(voxel_size_m),
                                     int(minimum_point_number_per_voxel), int(bool(remove_ground_from_local_map)),
                                     float(ground_distance_to_robot_center_m), int(initial_capacity_points))
        self._h = ctypes.c_void_p()
        ctx._check(lib().ls_local_map_create(ctx._h, ctypes.byref(self.params), ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().ls_local_map_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add_scan(self, ring, scan_id, T_w_scan, robot_z):
        """scanCallback's map part: scan `scan_id` of `ring` moved by T_w_scan (4x4, already corrected) appended and queued,
        ground removed against robot_z.  Returns the points added."""
        t = colmajor(T_w_scan)
        n = ctypes.c_int(0)
        self.ctx._check(lib().ls_local_map_add_scan(self._h, ring._h, int(scan_id), t.ctypes.data, float(robot_z), ctypes.byref(n)))
        return n.value

    def filter(self, center):
        """getFilteredMap around `center` (the pose's position, rounded to float32 as the reference's PclPoint): returns the
        number of points of the filtered map (download(LM_FILTERED_MAP) holds them)."""
        c = np.ascontiguousarray(np.asarray(center, np.float32), np.float64)
        n = ctypes.c_int(0)
        self.ctx._check(lib().ls_local_map_filter(self._h, c.ctypes.data, ctypes.byref(n)))
        return n.value

    def get_filtered_map(self, center):
        self.filter(center)
        return self.download(LM_FILTERED_MAP)

    def size(self, which):
        n = int(lib().ls_local_map_size(self._h, which))
        if n < 0:
            raise LsError(f"ls_local_map_size: rc={n}")
        return n

    def download(self, which, cap=None):
        n = self.size(which) if cap is None else int(cap)
        out = np.empty((max(n, 1), 4), np.float32)
        got = ctypes.c_int(0)
        self.ctx._check(lib().ls_local_map_download(self._h, which, out.ctypes.data, n, ctypes.byref(got)))
        return out[:got.value].copy()

    def take_queue(self):
        """getQueuedPoints: the queued clouds in order (a list of (k,4) arrays); the queue is empty afterwards."""
        n = self.size(LM_QUEUE)
        out = np.empty((max(n, 1), 4), np.float32)
        cap_clouds = n + 1  # every queued cloud holds at least one point
        offs = np.zeros(cap_clouds + 1, np.int32)
        k = ctypes.c_int(0)
        self.ctx._check(lib().ls_local_map_take_queue(self._h, out.ctypes.data, n, offs.ctypes.data, cap_clouds, ctypes.byref(k)))
        return [out[offs[j]:offs[j + 1]].copy() for j in range(k.value)]

    def transform(self, T):
        """updateLocalMap's move: local_map_ and local_map_filtered_ by T (4x4 float32, not corrected)."""
        t = colmajor(T)
        self.ctx._check(lib().ls_local_map_transform(self._h, t.ctypes.data))

    def clear(self):
        self.ctx._check(lib().ls_local_map_clear(self._h))


class OccupancyMap:
    """laser_to_octomap's occupancy map on the device (ls_occupancy_*): scans of a Map ring inserted at their poses into
    voxels of float log-odds.  Keyword arguments are the OccupancyParams fields; the defaults are laser_to_octomap's."""

    def __init__(self, ctx, **params):
        self.ctx = ctx
        self.params = OccupancyParams()
        lib().ls_occupancy_default_params(ctypes.byref(self.params))
        for k, v in params.items():
            if not hasattr(self.params, k):
                raise TypeError(f"unknown occupancy map parameter {k!r}")
            setattr(self.params, k, v)
        self._h = ctypes.c_void_p()
        ctx._check(lib().ls_occupancy_create(ctx._h, ctypes.byref(self.params), ctypes.byref(self._h)))

    def close(self):
        if self._h:
            lib().ls_occupancy_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _sized_output(self, call, *outputs):
        """The ABI's sized outputs: call(out, cap, n) with no buffers and cap 0 counts them into n (LS_ERR_ARG with n > 0,
        or OK with n == 0); with n > 0, the call is repeated into new arrays of n rows, one per (dtype, row shape) of
        outputs.  Returns those arrays."""
        n = ctypes.c_int64(0)
        rc = call([None] * len(outputs), 0, ctypes.byref(n))
        if rc != LS_ERR_ARG or n.value == 0:
            self.ctx._check(rc)
        m = n.value
        arrays = tuple(np.empty((m,) + shape, dtype) for dtype, shape in outputs)
        if m > 0:
            self.ctx._check(call([a.ctypes.data for a in arrays], m, ctypes.byref(n)))
        return arrays

    def insert_scan(self, ring, scan_id, T_w_scan):
        """Scan `scan_id` of `ring` at pose T_w_scan (4x4, cast to float32, not corrected).  Returns OccupancyStats."""
        t = colmajor(T_w_scan)
        st = OccupancyStats()
        self.ctx._check(lib().ls_occupancy_insert_scan(self._h, ring._h, int(scan_id), t.ctypes.data, ctypes.byref(st)))
        return st

    def size(self, which=OCC_KNOWN):
        n = ctypes.c_int64(0)
        self.ctx._check(lib().ls_occupancy_size(self._h, int(which), ctypes.byref(n)))
        return n.value

    def download(self, which=OCC_KNOWN, cap=None):
        """(keys uint64, log-odds float32, centres (n,4) float32) by ascending packed key."""
        n = self.size(which) if cap is None else int(cap)
        keys = np.empty(max(n, 1), np.uint64)
        lo = np.empty(max(n, 1), np.float32)
        cen = np.empty((max(n, 1), 4), np.float32)
        got = ctypes.c_int64(0)
        self.ctx._check(lib().ls_occupancy_download(self._h, int(which), keys.ctypes.data, lo.ctypes.data, cen.ctypes.data, n,
                                                    ctypes.byref(got)))
        m = got.value
        return keys[:m].copy(), lo[:m].copy(), cen[:m].copy()

    def save_point_cloud(self, path):
        """The occupied voxels' centres as ASCII .pcd (v0.7, FIELDS x y z) or .ply, chosen by the extension (the job of
        octomap_to_point_cloud).  Returns the number of points written."""
        ext = os.path.splitext(path)[1].lower()
        if ext not in (".pcd", ".ply"):
            raise ValueError(f"unsupported point cloud extension {ext!r} (.pcd or .ply)")
        pts = self.download(OCC_OCCUPIED)[2][:, :3]
        write_point_cloud(path, pts)
        return len(pts)

    def octree(self):
        """The map as octomap's pruned tree, built on the device (ls_occupancy_build_octree): Octree(nodes, payload bytes,
        occupied leaves' centres (n,4) float32 and depths uint8 in pre-order, device ms)."""
        st = OctreeStats()
        self.ctx._check(lib().ls_occupancy_build_octree(self._h, ctypes.byref(st)))
        pay = np.empty(max(st.payload_bytes, 1), np.uint8)
        cen = np.empty((max(st.occupied_leaves, 1), 4), np.float32)
        dep = np.empty(max(st.occupied_leaves, 1), np.uint8)
        self.ctx._check(lib().ls_occupancy_download_octree(self._h, pay.ctypes.data, st.payload_bytes, cen.ctypes.data,
                                                           dep.ctypes.data, st.occupied_leaves))
        n = st.occupied_leaves
        return Octree(st.nodes, pay[:st.payload_bytes].tobytes(), cen[:n].copy(), dep[:n].copy(), st.device_ms)

    def save_octomap(self, path):
        """The map as an octomap binary file (.bt, OcTree::writeBinary), readable by octomap::OcTree(path).  Returns its
        node count."""
        st = OctreeStats()
        self.ctx._check(lib().ls_occupancy_write_octomap(self._h, os.fsencode(path), ctypes.byref(st)))
        return st.nodes

    def save_pruned_point_cloud(self, path):
        """The occupied leaves of the pruned tree as .pcd / .ply: what octomap_to_point_cloud writes from this map's .bt
        file.  Returns the number of points written."""
        ext = os.path.splitext(path)[1].lower()
        if ext not in (".pcd", ".ply"):
            raise ValueError(f"unsupported point cloud extension {ext!r} (.pcd or .ply)")
        pts = self.octree().centres[:, :3]
        write_point_cloud(path, pts)
        return len(pts)

    def read_octomap(self, path):
        """octomap's readBinary of a .bt file into this map, replacing it (ls_occupancy_read_octomap): free leaves load as
        clamp_min, occupied ones as clamp_max, and the file's resolution becomes the map's (self.params.resolution).
        Returns OctomapReadStats; on an error the map is unchanged."""
        st = OctomapReadStats()
        self.ctx._check(lib().ls_occupancy_read_octomap(self._h, os.fsencode(path), ctypes.byref(st)))
        self.params.resolution = st.resolution
        return st

    def read_octree(self, payload, nodes, resolution):
        """As read_octomap, from a payload in memory (the bytes after "data\\n", as an octomap_msgs binary message carries
        them), the node count of its size line and its resolution."""
        buf = np.frombuffer(bytes(payload), np.uint8)
        st = OctomapReadStats()
        self.ctx._check(lib().ls_occupancy_read_octree(self._h, buf.ctypes.data if len(buf) else None, len(buf), int(nodes),
                                                       float(resolution), ctypes.byref(st)))
        self.params.resolution = st.resolution
        return st

    def full_octree(self):
        """The map as octomap's full tree (every node's log-odds, pruned by value), built on the device
        (ls_occupancy_build_full_octree): FullOctree(nodes, payload bytes, device ms)."""
        st = FullOctreeStats()
        self.ctx._check(lib().ls_occupancy_build_full_octree(self._h, ctypes.byref(st)))
        pay = np.empty(max(st.payload_bytes, 1), np.uint8)
        self.ctx._check(lib().ls_occupancy_download_full_octree(self._h, pay.ctypes.data, st.payload_bytes))
        return FullOctree(st.nodes, pay[:st.payload_bytes].tobytes(), st.device_ms)

    def save_octomap_full(self, path):
        """The map as an octomap full tree file (.ot, OcTree::write), readable by octomap's AbstractOcTree::read(path).
        Unlike the .bt file it keeps every voxel's log-odds, so a map read back maps on exactly as this one would.  Returns
        its node count."""
        st = FullOctreeStats()
        self.ctx._check(lib().ls_occupancy_write_octomap_full(self._h, os.fsencode(path), ctypes.byref(st)))
        return st.nodes

    def read_octomap_full(self, path):
        """octomap's read of a .ot file into this map, replacing it (ls_occupancy_read_octomap_full): every leaf's voxels
        take its log-odds verbatim, and the file's resolution becomes the map's (self.params.resolution).  Returns
        OctomapReadStats; on an error the map is unchanged."""
        st = OctomapReadStats()
        self.ctx._check(lib().ls_occupancy_read_octomap_full(self._h, os.fsencode(path), ctypes.byref(st)))
        self.params.resolution = st.resolution
        return st

    def read_full_octree(self, payload, nodes, resolution):
        """As read_octomap_full, from a payload in memory (the bytes after "data\\n", as a full octomap message carries
        them), the node count of its size line and its resolution."""
        buf = np.frombuffer(bytes(payload), np.uint8)
        st = OctomapReadStats()
        self.ctx._check(lib().ls_occupancy_read_full_octree(self._h, buf.ctypes.data if len(buf) else None, len(buf),
                                                            int(nodes), float(resolution), ctypes.byref(st)))
        self.params.resolution = st.resolution
        return st

    # ---- queries (ls_occupancy_cell_status / _line_status / _cast_rays); self.last_query holds the last call's stats
    def cell_status(self, points):
        """getCellStatusPoint per point ((n,3), taken as float64): (status int8 CELL_*, log-odds float32, NaN when
        unknown)."""
        p = np.ascontiguousarray(np.asarray(points, np.float64).reshape(-1, 3))
        n = len(p)
        st = np.empty(max(n, 1), np.int8)
        lo = np.empty(max(n, 1), np.float32)
        self.last_query = OccupancyQueryStats()
        self.ctx._check(lib().ls_occupancy_cell_status(self._h, p.ctypes.data, n, st.ctypes.data, lo.ctypes.data,
                                                       ctypes.byref(self.last_query)))
        return st[:n].copy(), lo[:n].copy()

    def line_status(self, starts, ends, box=None, stop_at_unknown=True):
        """getLineStatus (stop_at_unknown), getVisibility or, with box = its (x, y, z) size, getLineStatusBoundingBox per
        segment ((n,3) each, taken as float64): (status int8 CELL_*, packed key uint64 that decided it, all ones when
        free)."""
        s = np.ascontiguousarray(np.asarray(starts, np.float64).reshape(-1, 3))
        e = np.ascontiguousarray(np.asarray(ends, np.float64).reshape(-1, 3))
        if len(s) != len(e):
            raise ValueError(f"{len(s)} starts for {len(e)} ends")
        b = None if box is None else np.ascontiguousarray(np.asarray(box, np.float64).reshape(3))
        n = len(s)
        st = np.empty(max(n, 1), np.int8)
        fk = np.empty(max(n, 1), np.uint64)
        self.last_query = OccupancyQueryStats()
        self.ctx._check(lib().ls_occupancy_line_status(self._h, s.ctypes.data, e.ctypes.data, n,
                                                       None if b is None else b.ctypes.data, int(bool(stop_at_unknown)),
                                                       st.ctypes.data, fk.ctypes.data, ctypes.byref(self.last_query)))
        return st[:n].copy(), fk[:n].copy()

    def cast_rays(self, origins, directions, ignore_unknown=False, max_range=-1.0):
        """octomap's castRay per ray ((n,3) each, taken as float32): (result int8 RAY_*, ends (n,3) float32: the centre
        of the voxel the result names, NaN for RAY_INVALID).  max_range <= 0: none."""
        o = np.ascontiguousarray(np.asarray(origins, np.float32).reshape(-1, 3))
        d = np.ascontiguousarray(np.asarray(directions, np.float32).reshape(-1, 3))
        if len(o) != len(d):
            raise ValueError(f"{len(o)} origins for {len(d)} directions")
        n = len(o)
        r = np.empty(max(n, 1), np.int8)
        ends = np.empty((max(n, 1), 3), np.float32)
        self.last_query = OccupancyQueryStats()
        self.ctx._check(lib().ls_occupancy_cast_rays(self._h, o.ctypes.data, d.ctypes.data, n, int(bool(ignore_unknown)),
                                                     float(max_range), r.ctypes.data, ends.ctypes.data,
                                                     ctypes.byref(self.last_query)))
        return r[:n].copy(), ends[:n].copy()

    # ---- box status and robot collision (ls_occupancy_box_status / _check_paths); self.last_query holds the stats
    def box_status(self, centres, sizes):
        """getCellStatusBoundingBox per box ((n,3) centres and sizes, or (3,) sizes for every box; taken as float64):
        status int8 CELL_* (DESIGN.md §4b''''''''''')."""
        c = np.ascontiguousarray(np.asarray(centres, np.float64).reshape(-1, 3))
        s = np.asarray(sizes, np.float64)
        s = np.ascontiguousarray(np.broadcast_to(s.reshape(-1, 3) if s.size != 3 else s.reshape(1, 3), c.shape))
        if len(s) != len(c):
            raise ValueError(f"{len(c)} centres for {len(s)} sizes")
        n = len(c)
        st = np.empty(max(n, 1), np.int8)
        self.last_query = OccupancyQueryStats()
        self.ctx._check(lib().ls_occupancy_box_status(self._h, c.ctypes.data, s.ctypes.data, n, st.ctypes.data,
                                                      ctypes.byref(self.last_query)))
        return st[:n].copy()

    def check_paths(self, positions, offsets, robot_size, unknown_as_occupied=True):
        """checkPathForCollisionsWithRobot per path: path p is positions[offsets[p]:offsets[p + 1]] ((m,3), taken as
        float64; offsets (n_paths + 1,) non-decreasing from 0), the robot a box of robot_size (3,) at each pose.  Returns
        int64 per path: the first colliding pose's index within the path, -1 when none.  A pose collides when its box is
        occupied, or, with unknown_as_occupied, when it is not free."""
        p = np.ascontiguousarray(np.asarray(positions, np.float64).reshape(-1, 3))
        o = np.ascontiguousarray(np.asarray(offsets, np.int64).reshape(-1))
        r = np.ascontiguousarray(np.asarray(robot_size, np.float64).reshape(3))
        n = max(len(o) - 1, 0)
        if n > 0 and o[-1] != len(p):
            raise ValueError(f"offsets end at {o[-1]} for {len(p)} positions")
        first = np.empty(max(n, 1), np.int64)
        self.last_query = OccupancyQueryStats()
        self.ctx._check(lib().ls_occupancy_check_paths(self._h, p.ctypes.data if len(p) else None, o.ctypes.data, n,
                                                       r.ctypes.data, int(bool(unknown_as_occupied)), first.ctypes.data,
                                                       ctypes.byref(self.last_query)))
        return first[:n].copy()

    # ---- edits (ls_occupancy_set_boxes / _clear / _box_voxels / _bounds)
    def set_boxes(self, centres, sizes, occupied):
        """volumetric_mapping's setFree / setOccupied of n boxes in order ((n,3) centres and sizes, taken as float64; occupied
        (n,) truthy for setOccupied): every voxel a box's loop reaches becomes known with clamp_min or clamp_max, the last
        box deciding.  Returns OccupancyEditStats; on an error no voxel changes."""
        c = np.ascontiguousarray(np.asarray(centres, np.float64).reshape(-1, 3))
        s = np.ascontiguousarray(np.asarray(sizes, np.float64).reshape(-1, 3))
        o = np.ascontiguousarray(np.asarray(occupied).reshape(-1).astype(bool).astype(np.int8))
        if not len(c) == len(s) == len(o):
            raise ValueError(f"{len(c)} centres, {len(s)} sizes and {len(o)} occupied flags")
        st = OccupancyEditStats()
        self.ctx._check(lib().ls_occupancy_set_boxes(self._h, c.ctypes.data, s.ctypes.data, o.ctypes.data, len(c),
                                                     ctypes.byref(st)))
        return st

    def set_free(self, centres, sizes):
        """setFree of each box ((n,3) or (3,) centres and sizes)."""
        c = np.asarray(centres, np.float64).reshape(-1, 3)
        return self.set_boxes(c, sizes, np.zeros(len(c), bool))

    def set_occupied(self, centres, sizes):
        """setOccupied of each box ((n,3) or (3,) centres and sizes)."""
        c = np.asarray(centres, np.float64).reshape(-1, 3)
        return self.set_boxes(c, sizes, np.ones(len(c), bool))

    def clear(self):
        """resetMap: no known voxel and no brick; the parameters and the device memory stay."""
        self.ctx._check(lib().ls_occupancy_clear(self._h))

    def box_voxels(self, center, size, which=OCC_OCCUPIED):
        """getOccupiedPointcloudInBoundingBox (which=OCC_OCCUPIED) or every known voxel (OCC_KNOWN) the box's loop reaches,
        in loop order with repeats: (keys uint64, log-odds float32, voxel centres (n,4) float32)."""
        c = np.ascontiguousarray(np.asarray(center, np.float64).reshape(3))
        s = np.ascontiguousarray(np.asarray(size, np.float64).reshape(3))
        return self._sized_output(
            lambda out, cap, n: lib().ls_occupancy_box_voxels(self._h, c.ctypes.data, s.ctypes.data, int(which), *out, cap, n),
            (np.uint64, ()), (np.float32, ()), (np.float32, (4,)))

    def bounds(self):
        """getMetricMin / getMetricMax over the known voxels: (min (3,) float64, max (3,) float64), zeros when empty."""
        lo, hi = np.zeros(3, np.float64), np.zeros(3, np.float64)
        self.ctx._check(lib().ls_occupancy_bounds(self._h, lo.ctypes.data, hi.ctypes.data))
        return lo, hi

    # ---- change detection (ls_occupancy_track_changes / _changes); self.last_changes holds the last call's stats
    def track_changes(self, enable=True):
        """enableChangeDetection: True takes the map as it is now as the baseline (again when tracking is on); False turns
        tracking off and frees the baseline."""
        self.ctx._check(lib().ls_occupancy_track_changes(self._h, int(bool(enable))))

    def changes(self, reset=False):
        """The voxels whose state (CELL_*) differs from the baseline's, by ascending packed key: (keys uint64, status int8
        now, previous int8 at the baseline, centres (n,4) float32).  reset=True then makes the map the new baseline
        (getChangedPoints followed by resetChangeDetection)."""
        self.last_changes = OccupancyChangeStats()
        return self._sized_output(
            lambda out, cap, n: lib().ls_occupancy_changes(self._h, *out, cap, n, int(bool(reset)),
                                                           ctypes.byref(self.last_changes)),
            (np.uint64, ()), (np.int8, ()), (np.int8, ()), (np.float32, (4,)))

    # ---- leaf boxes and marker cubes (ls_occupancy_build_leaves / _download_leaves / _marker_cubes)
    def build_leaves(self, region=None):
        """Lists the leaves of the value-pruned tree whose key cube meets region = (min (3,), max (3,)) in metres, or every
        leaf (DESIGN.md §4b'''''''''''').  Returns LeafStats; the list stays on the device for download_leaves and
        marker_cubes until the map changes."""
        st = LeafStats()
        if region is None:
            self.ctx._check(lib().ls_occupancy_build_leaves(self._h, None, None, ctypes.byref(st)))
        else:
            lo = np.ascontiguousarray(np.asarray(region[0], np.float64).reshape(3))
            hi = np.ascontiguousarray(np.asarray(region[1], np.float64).reshape(3))
            self.ctx._check(lib().ls_occupancy_build_leaves(self._h, lo.ctypes.data, hi.ctypes.data, ctypes.byref(st)))
        return st

    def download_leaves(self, which=LEAVES_ALL):
        """The last list's leaves of `which` (LEAVES_*) in octomap's leaf order: (centres (n,4) float32, depths uint8,
        states int8 CELL_*)."""
        return self._sized_output(
            lambda out, cap, n: lib().ls_occupancy_download_leaves(self._h, int(which), *out, cap, n),
            (np.float32, (4,)), (np.uint8, ()), (np.int8, ()))

    def leaf_boxes(self, which=LEAVES_ALL, region=None):
        """getAllFreeBoxes (which=LEAVES_FREE) / getAllOccupiedBoxes (LEAVES_OCCUPIED), or both in one list, optionally
        limited to a region (min (3,), max (3,)): LeafBoxes(centres (n,3) float32, edges float64 = res * 2^(16 - depth),
        depths uint8, states int8 CELL_*), in octomap's leaf order.  self.last_leaves holds the build's LeafStats."""
        self.last_leaves = self.build_leaves(region)
        cen, dep, st = self.download_leaves(which)
        edges = self.params.resolution * np.exp2(16 - dep.astype(np.float64))
        return LeafBoxes(cen[:, :3].copy(), edges, dep, st)

    def marker_cubes(self, min_z, max_z, color_factor=0.8, region=None):
        """generateMarkerArray's cube lists: MarkerCubes(occupied, free), each a list of 17 CubeList(size, points (k,3)
        float32, colors (k,4) float32) for depths 0..16; occupied cubes are coloured by height (heightMapColor), free ones
        carry no colours (an empty (0,4) array).  self.last_leaves holds the build's LeafStats."""
        self.last_leaves = self.build_leaves(region)
        occ_off, free_off = np.zeros(18, np.int64), np.zeros(18, np.int64)
        cen, rgba = self._sized_output(
            lambda out, cap, n: lib().ls_occupancy_marker_cubes(self._h, float(min_z), float(max_z), float(color_factor), *out,
                                                                occ_off.ctypes.data, free_off.ctypes.data, cap, n),
            (np.float32, (4,)), (np.float32, (4,)))
        res = self.params.resolution
        occ = [CubeList(res * 2.0 ** (16 - d), cen[occ_off[d]:occ_off[d + 1], :3].copy(),
                        rgba[occ_off[d]:occ_off[d + 1]].copy()) for d in range(17)]
        free = [CubeList(res * 2.0 ** (16 - d), cen[free_off[d]:free_off[d + 1], :3].copy(), np.zeros((0, 4), np.float32))
                for d in range(17)]
        return MarkerCubes(occ, free)

    # ---- 2D projection (ls_occupancy_build_projection / _download_projection)
    def projected_map(self, min_z=-math.inf, max_z=math.inf, min_size_x=0.0, min_size_y=0.0):
        """octomap_server's projected_map (DESIGN.md §4b'''''''''''''): the .bt tree's leaves whose z extent meets the band
        (min_z, max_z), painted into a 2D grid padded to at least min_size_x x min_size_y metres around the origin.
        Returns (grid int8 (height, width) of -1 unknown, 0 free, 100 occupied, cell (i, j) at grid[j, i]; GridInfo)."""
        info = GridInfo()
        self.ctx._check(lib().ls_occupancy_build_projection(self._h, float(min_z), float(max_z), float(min_size_x),
                                                            float(min_size_y), ctypes.byref(info)))
        grid = np.empty((info.height, info.width), np.int8)
        self.ctx._check(lib().ls_occupancy_download_projection(self._h, grid.ctypes.data if grid.size else None, grid.size))
        return grid, info

    def save_projected_map(self, stem, min_z=-math.inf, max_z=math.inf, min_size_x=0.0, min_size_y=0.0):
        """projected_map(...) saved as map_saver saves it: stem.pgm and stem.yaml (save_map).  Returns the GridInfo."""
        grid, info = self.projected_map(min_z, max_z, min_size_x, min_size_y)
        save_map(stem, grid, info.resolution, info.origin_x, info.origin_y)
        return info


def save_map(stem, grid, resolution, origin_x, origin_y):
    """map_saver's files of an occupancy grid (int8 (height, width), cell (i, j) at grid[j, i]): stem.pgm, a P5 image whose
    rows run from j = height - 1 down to 0, 0 -> 254, 100 -> 0 and anything else -> 205; and stem.yaml naming it.  The
    resolution is printed as the message's float32 holds it."""
    grid = np.asarray(grid, np.int8)
    height, width = grid.shape
    res = float(np.float32(resolution))
    pix = np.full(grid.shape, 205, np.uint8)
    pix[grid == 0] = 254
    pix[grid == 100] = 0
    image = stem + ".pgm"
    with open(image, "wb") as f:
        f.write(b"P5\n# CREATOR: map_saver.cpp %.3f m/pix\n%d %d\n255\n" % (res, width, height))
        f.write(pix[::-1].tobytes())
    with open(stem + ".yaml", "w") as f:
        f.write("image: %s\nresolution: %f\norigin: [%f, %f, %f]\nnegate: 0\noccupied_thresh: 0.65\nfree_thresh: 0.196\n\n"
                % (image, res, origin_x, origin_y, 0.0))


class DistanceMap:
    """octomap's DynamicEDTOctomap on the device (ls_distance_map_*): the Euclidean distance of every finest cell of the box
    bbx_min ... bbx_max (float triples) to its nearest obstacle, an occupied voxel (or, with treat_unknown_as_occupied, an
    unknown one), capped at max_dist.  update() recomputes it from an OccupancyMap's current state; queries read the last
    update only."""

    def __init__(self, ctx, max_dist, bbx_min, bbx_max, treat_unknown_as_occupied=False):
        self.ctx = ctx
        self.params = DistanceMapParams(float(max_dist), (ctypes.c_float * 3)(*[float(x) for x in bbx_min]),
                                        (ctypes.c_float * 3)(*[float(x) for x in bbx_max]), int(bool(treat_unknown_as_occupied)))
        self._h = ctypes.c_void_p()
        ctx._check(lib().ls_distance_map_create(ctx._h, ctypes.byref(self.params), ctypes.byref(self._h)))
        self.stats = None

    def close(self):
        if self._h:
            lib().ls_distance_map_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def update(self, occupancy_map):
        """The field of occupancy_map as it is now (ls_distance_map_update).  Returns DistanceMapStats; on an error the
        previous field stays (LS_ERR_ARG) or the handle has none (LS_ERR_NOMEM)."""
        st = DistanceMapStats()
        self.ctx._check(lib().ls_distance_map_update(self._h, occupancy_map._h, ctypes.byref(st)))
        self.stats = st
        return st

    def query(self, points):
        """getDistanceAndClosestObstacle and getSquaredDistanceInCells per point ((n,3), taken as float32): (distance
        float32 [m], squared distance in cells int32, closest obstacle's voxel centre (n,3) float32).  -1, -1 and NaN
        outside the box; NaN obstacles where none is within max_dist."""
        p = np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))
        n = len(p)
        d = np.empty(max(n, 1), np.float32)
        s = np.empty(max(n, 1), np.int32)
        o = np.empty((max(n, 1), 3), np.float32)
        self.last_query = DistanceMapQueryStats()
        self.ctx._check(lib().ls_distance_map_query(self._h, p.ctypes.data if n else None, n, d.ctypes.data, s.ctypes.data,
                                                    o.ctypes.data, ctypes.byref(self.last_query)))
        return d[:n].copy(), s[:n].copy(), o[:n].copy()

    def download(self):
        """The whole field: (squared distances (sz, sy, sx) int32, closest obstacles' packed keys (sz, sy, sx) uint64, all
        ones when none)."""
        n = ctypes.c_int64(0)
        rc = lib().ls_distance_map_download(self._h, None, None, 0, ctypes.byref(n))
        if rc != LS_ERR_ARG or n.value == 0:
            self.ctx._check(rc)
        m = n.value
        s = np.empty(max(m, 1), np.int32)
        k = np.empty(max(m, 1), np.uint64)
        self.ctx._check(lib().ls_distance_map_download(self._h, s.ctypes.data, k.ctypes.data, m, ctypes.byref(n)))
        shape = tuple(self.stats.size[::-1]) if self.stats is not None else (m,)
        return s[:m].reshape(shape), k[:m].reshape(shape)


Octree = collections.namedtuple("Octree", "nodes payload centres depths device_ms")
FullOctree = collections.namedtuple("FullOctree", "nodes payload device_ms")
LeafBoxes = collections.namedtuple("LeafBoxes", "centres edges depths states")
CubeList = collections.namedtuple("CubeList", "size points colors")
MarkerCubes = collections.namedtuple("MarkerCubes", "occupied free")

_BT_FIRST_LINE = b"# Octomap OcTree binary file"
_OT_FIRST_LINE = b"# Octomap OcTree file"


def _read_header(path, data, first_line, what):
    """(size, res, payload offset) of an octomap file's header."""
    pos = 0

    def line():
        nonlocal pos
        end = data.find(b"\n", pos)
        if end < 0:
            raise ValueError(f"{path}: header ends early")
        s, pos = data[pos:end], end + 1
        return s.rstrip(b"\r")

    if line() != first_line:
        raise ValueError(f"{path}: not an octomap {what} file (first line)")
    head = {}
    while True:
        s = line()
        if s.startswith(b"#") or not s.strip():
            continue
        if s == b"data":
            break
        key, _, value = s.partition(b" ")
        head[key.decode(errors="replace")] = value.strip().decode(errors="replace")
    if head.get("id") != "OcTree":
        raise ValueError(f"{path}: tree type {head.get('id')!r}, expected 'OcTree'")
    try:
        size, res = int(head["size"]), float(head["res"])
    except (KeyError, ValueError) as e:
        raise ValueError(f"{path}: bad or missing size / res line") from e
    if size < 0 or not res > 0:
        raise ValueError(f"{path}: bad size {size} or res {res}")
    return size, res, pos


def read_octomap(path):
    """Parse an octomap binary file (.bt) as octomap::OcTree(path) reads it, on the CPU.  Returns a dict: resolution, nodes
    (the header's size), payload, and every leaf in pre-order as first-voxel keys (n,3) int64, depths uint8 and states
    uint8 (1 free, 2 occupied).  Raises ValueError on a bad header, a truncated payload or a size that does not match."""
    data = open(path, "rb").read()
    size, res, pos = _read_header(path, data, _BT_FIRST_LINE, "binary")
    keys, depths, states = [], [], []
    start, nodes = pos, 0
    # pre-order walk (children 0 ... 7): an inner node reads its two bytes when it is reached, a leaf is listed
    stack = [(3, 0, 0, 0, 0)] if size > 0 else []  # bit pair, depth, first-voxel key
    while stack:
        bits, d, kx, ky, kz = stack.pop()
        nodes += 1
        if bits != 3:
            keys.append((kx, ky, kz))
            depths.append(d)
            states.append(2 if bits == 2 else 1)
            continue
        if d >= 16:
            raise ValueError(f"{path}: inner node at depth 16")
        if pos + 2 > len(data):
            raise ValueError(f"{path}: payload truncated")
        m = data[pos] | (data[pos + 1] << 8)
        pos += 2
        sh = 15 - d
        for i in range(7, -1, -1):
            b = (m >> (2 * i)) & 3
            if b:
                stack.append((b, d + 1, kx | ((i & 1) << sh), ky | (((i >> 1) & 1) << sh), kz | (((i >> 2) & 1) << sh)))
    if nodes != size:
        raise ValueError(f"{path}: the header's size {size} does not match the {nodes} nodes of the payload")
    return dict(resolution=res, nodes=size, payload=data[start:pos], keys=np.array(keys, np.int64).reshape(-1, 3),
                depths=np.array(depths, np.uint8), states=np.array(states, np.uint8))


def read_octomap_full(path):
    """Parse an octomap full tree file (.ot, OcTree::write) as AbstractOcTree::read reads it, on the CPU.  Returns a dict:
    resolution, nodes (the header's size), payload, and every leaf in pre-order as first-voxel keys (n,3) int64, depths
    uint8 and log-odds float32.  Raises ValueError on a bad header or tree type, a resolution that is not finite and > 0, a
    truncated payload, a node at depth 16 with children, a leaf value that is NaN or infinite, or a size that does not
    match the nodes parsed."""
    data = open(path, "rb").read()
    size, res, pos = _read_header(path, data, _OT_FIRST_LINE, "full tree")
    if not math.isfinite(res):
        raise ValueError(f"{path}: res {res} is not finite")
    keys, depths, values = [], [], []
    start, nodes = pos, 0
    unpack = struct.Struct("<fB").unpack_from
    stack = [(0, 0, 0, 0)] if size > 0 else []  # depth, first-voxel key; children pushed 7 ... 0, so read in pre-order
    while stack:
        d, kx, ky, kz = stack.pop()
        if pos + 5 > len(data):
            raise ValueError(f"{path}: payload truncated")
        v, m = unpack(data, pos)
        pos += 5
        nodes += 1
        if not m:
            if not math.isfinite(v):
                raise ValueError(f"{path}: leaf value {v} is not finite")
            keys.append((kx, ky, kz))
            depths.append(d)
            values.append(v)
            continue
        if d >= 16:
            raise ValueError(f"{path}: node at depth 16 with children")
        sh = 15 - d
        for i in range(7, -1, -1):
            if (m >> i) & 1:
                stack.append((d + 1, kx | ((i & 1) << sh), ky | (((i >> 1) & 1) << sh), kz | (((i >> 2) & 1) << sh)))
    if nodes != size:
        raise ValueError(f"{path}: the header's size {size} does not match the {nodes} nodes of the payload")
    return dict(resolution=res, nodes=size, payload=data[start:pos], keys=np.array(keys, np.int64).reshape(-1, 3),
                depths=np.array(depths, np.uint8), values=np.array(values, np.float32))


def leaf_centres(keys, depths, resolution):
    """octomap's keyToCoord(key, depth) of leaves given by their first-voxel keys (n,3): (n,3) float32."""
    k = np.asarray(keys, np.int64).reshape(-1, 3)
    s = (16 - np.asarray(depths, np.int64))[:, None]
    kc = k + np.where(s > 0, np.left_shift(1, np.maximum(s - 1, 0)), 0)
    scale = np.left_shift(1, s).astype(np.float64)
    return ((np.floor((kc.astype(np.float64) - 32768.0) / scale) + 0.5) * (float(resolution) * scale)).astype(np.float32)


def octomap_to_point_cloud(bt_path, out_path):
    """The reference tool octomap_to_point_cloud without PCL: the occupied leaves' centres of a .bt file, in its leaf
    order, written as .pcd / .ply.  Returns the number of points."""
    ext = os.path.splitext(out_path)[1].lower()
    if ext not in (".pcd", ".ply"):
        raise ValueError(f"unsupported point cloud extension {ext!r} (.pcd or .ply)")
    t = read_octomap(bt_path)
    occ = t["states"] == 2
    pts = leaf_centres(t["keys"][occ], t["depths"][occ], t["resolution"])
    write_point_cloud(out_path, pts)
    return len(pts)


def write_point_cloud(path, xyz):
    """ASCII .pcd (v0.7, FIELDS x y z) or .ply of an (n,3) float32 array, by the extension of `path`."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    ext = os.path.splitext(path)[1].lower()
    n = len(xyz)
    if ext == ".pcd":
        head = ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\n"
                f"COUNT 1 1 1\nWIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA ascii\n")
    elif ext == ".ply":
        head = f"ply\nformat ascii 1.0\nelement vertex {n}\nproperty float x\nproperty float y\nproperty float z\nend_header\n"
    else:
        raise ValueError(f"unsupported point cloud extension {ext!r} (.pcd or .ply)")
    with open(path, "w") as f:
        f.write(head)
        np.savetxt(f, xyz, fmt="%.9g")  # nine significant digits give a float32 back exactly


def check_rigid(T):
    t = colmajor(T)
    return bool(lib().ls_check_rigid(t.ctypes.data))


def correct_rigid(T):
    t = colmajor(T)
    o = np.empty(16, np.float32)
    lib().ls_correct_rigid(t.ctypes.data, o.ctypes.data)
    return from_colmajor(o)


class PoseGraph:
    """Device pose graph (gtsam::ISAM2 as IncrementalEstimator uses it).  Poses: rows [qw,qx,qy,qz,tx,ty,tz]."""

    def __init__(self, device=0):
        self._h = ctypes.c_void_p()
        rc = lib().ls_pg_create(device, ctypes.byref(self._h))
        if rc != 0:
            raise LsError(f"ls_pg_create(device={device}) failed with {rc}: no usable CUDA device (no CPU fallback)")

    def close(self):
        if self._h:
            lib().ls_pg_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc == LS_ERR_CONVERGENCE:
            raise ConvergenceError(lib().ls_pg_last_error(self._h).decode())
        if rc != 0:
            raise LsError(f"rc={rc}: {lib().ls_pg_last_error(self._h).decode()}")

    @property
    def launch_count(self):
        return int(lib().ls_pg_launch_count(self._h))

    def add_poses(self, keys, poses7, track_ids=None):
        keys = np.ascontiguousarray(keys, np.uint64)
        poses7 = np.ascontiguousarray(poses7, np.float64).reshape(-1, 7)
        tr = np.ascontiguousarray(track_ids, np.uint32) if track_ids is not None else None
        self._check(lib().ls_pg_add_poses(self._h, keys.ctypes.data, _ptr(tr), poses7.ctypes.data, len(keys)))

    def set_poses(self, keys, poses7):
        keys = np.ascontiguousarray(keys, np.uint64)
        poses7 = np.ascontiguousarray(poses7, np.float64).reshape(-1, 7)
        self._check(lib().ls_pg_set_poses(self._h, keys.ctypes.data, poses7.ctypes.data, len(keys)))

    def add_factors(self, factors):
        """factors: iterable of dicts (type, key_a, key_b, meas[7], sigma[6], robust, fix_a, fixed_a[7]).  Returns indices."""
        arr = (Factor * len(factors))()
        for i, f in enumerate(factors):
            a = arr[i]
            a.type, a.robust, a.fix_a = int(f["type"]), int(f.get("robust", 0)), int(f.get("fix_a", 0))
            a.key_a, a.key_b = int(f["key_a"]), int(f.get("key_b", 0))
            a.meas[:] = [float(x) for x in f["meas"]]
            a.sigma[:] = [float(x) for x in f["sigma"]]
            a.fixed_a[:] = [float(x) for x in f.get("fixed_a", [1, 0, 0, 0, 0, 0, 0])]
        idx = np.zeros(max(len(factors), 1), np.uint64)
        self._check(lib().ls_pg_add_factors(self._h, arr, len(factors), idx.ctypes.data))
        return idx[:len(factors)]

    def remove_factors(self, indices):
        idx = np.ascontiguousarray(indices, np.uint64)
        self._check(lib().ls_pg_remove_factors(self._h, idx.ctypes.data, len(idx)))

    def optimize(self, gn_iters=3):
        st = PgStats()
        self._check(lib().ls_pg_optimize(self._h, gn_iters, ctypes.byref(st)))
        return st

    def marginals(self, keys):
        """gtsam::Marginals::marginalCovariance per key at the current estimate: (len(keys), 6, 6), [translation; rotation]."""
        k = np.ascontiguousarray(keys, np.uint64)
        cov = np.zeros((max(len(k), 1), 6, 6), np.float64)
        self._check(lib().ls_pg_marginals(self._h, k.ctypes.data, len(k), cov.ctypes.data))
        return cov[:len(k)]

    def poses(self):
        n = ctypes.c_int(lib().ls_pg_num_poses(self._h))
        keys = np.zeros(max(n.value, 1), np.uint64)
        poses = np.zeros((max(n.value, 1), 7), np.float64)
        self._check(lib().ls_pg_get_poses(self._h, keys.ctypes.data, poses.ctypes.data, ctypes.byref(n)))
        return keys[:n.value], poses[:n.value]
