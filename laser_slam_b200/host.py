"""ctypes access to the C test hooks of the C++ host layer (laser_slam_b200/host/host_capi.cpp): drives
laser_slam::IncrementalEstimator / LaserTrack the way the ROS worker's scanCallback does
(reference laser_slam_ros/src/laser_slam_worker.cpp:124-173)."""
import ctypes
import math
import os

import numpy as np

from . import IcpStats, LsError, ConvergenceError, LS_ERR_CONVERGENCE, build as _build_all

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "libls_host.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            _build_all()
        L = ctypes.CDLL(LIB_PATH)
        vp, ci, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
        L.lsh_create.restype = vp
        L.lsh_create.argtypes = [ci, ci, ci, ci, ci, ci, ci, ci, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ci]
        L.lsh_destroy.argtypes = [vp]
        L.lsh_destroy.restype = None
        L.lsh_last_error.argtypes = [vp]
        L.lsh_last_error.restype = ctypes.c_char_p
        L.lsh_step.argtypes = [vp, ci, i64, vp, vp, vp, ci, vp, ctypes.POINTER(IcpStats)]
        L.lsh_loop_closure.argtypes = [vp, ci, i64, ci, i64, vp]
        L.lsh_step_batch.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, ci, vp, vp]
        L.lsh_begin_batch.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, ci]
        L.lsh_prefetch.argtypes = [vp, ci, vp, vp, vp, vp, vp, ci]
        L.lsh_end_batch.argtypes = [vp, ci, vp, vp]
        L.lsh_trajectory.argtypes = [vp, ci, vp, vp, ci]
        L.lsh_num_scans.argtypes = [vp, ci]
        L.lsh_build_submap.argtypes = [vp, ci, i64, ci, vp, vp, ci]
        _lib = L
    return _lib


class Estimator:
    """laser_slam::IncrementalEstimator with n_workers LaserTracks."""

    def __init__(self, n_workers=1, nscan_in_sub_map=4, use_icp_factors=True, use_odom_factors=True, robust_icp=True,
                 device=0, do_icp_step_on_loop_closures=False, loop_closures_sub_maps_radius=2, icp_yaml_path=None,
                 icp_input_filters_path=None):
        """icp_input_filters_path: a DataPointsFilters YAML list (LaserTrackParams::icp_input_filters_file) every scan
        goes through on the device before the track stores it."""
        err = ctypes.create_string_buffer(512)
        self._h = lib().lsh_create(n_workers, nscan_in_sub_map, int(use_icp_factors), int(use_odom_factors), int(robust_icp),
                                   device, int(do_icp_step_on_loop_closures), loop_closures_sub_maps_radius,
                                   icp_yaml_path.encode() if icp_yaml_path else None,
                                   icp_input_filters_path.encode() if icp_input_filters_path else None, err, 512)
        if not self._h:
            raise LsError(err.value.decode() or "lsh_create failed")

    def close(self):
        if getattr(self, "_h", None):
            lib().lsh_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc == LS_ERR_CONVERGENCE:
            raise ConvergenceError(lib().lsh_last_error(self._h).decode())
        if rc < 0:
            raise LsError(lib().lsh_last_error(self._h).decode())
        return rc

    def step(self, worker, time_ns, pose7, features4, normals3=None):
        """One scan callback; returns (icp T_a_b as 7 doubles, IcpStats).  normals3=None passes a raw scan (the input
        filters must then estimate the normals)."""
        f = np.ascontiguousarray(features4, np.float32)
        nr = None if normals3 is None else np.ascontiguousarray(normals3, np.float32)
        p = np.ascontiguousarray(pose7, np.float64)
        out = np.zeros(7, np.float64)
        st = IcpStats()
        self._check(lib().lsh_step(self._h, worker, int(time_ns), p.ctypes.data, f.ctypes.data,
                                   None if nr is None else nr.ctypes.data, f.shape[0], out.ctypes.data, ctypes.byref(st)))
        return out, st

    def step_batch(self, workers, times_ns, poses7, feat_ptrs, nrm_ptrs, ns, with_estimator=True, views=False):
        """The scan callbacks of several workers at once: one batched launch registers them all
        (IncrementalEstimator::processPosesAndLaserScans).  feat_ptrs / nrm_ptrs: host addresses of each worker's
        4xN features and 3xN normals.  views=True hands the tracks DataPoints that BORROW those arrays (no copy; they
        must stay valid while the estimator lives; pinned arrays are then uploaded asynchronously, in place).
        Returns (icp T_a_b (len,7), list of IcpStats)."""
        k = len(workers)
        w = np.ascontiguousarray(workers, np.int32)
        t = np.ascontiguousarray(times_ns, np.int64)
        p = np.ascontiguousarray(poses7, np.float64).reshape(k, 7)
        fp = (ctypes.c_void_p * k)(*[int(a) for a in feat_ptrs])
        npp = (ctypes.c_void_p * k)(*[int(a) for a in nrm_ptrs])
        nn = np.ascontiguousarray(ns, np.int32)
        out = np.zeros((k, 7), np.float64)
        st = (IcpStats * k)()
        self._check(lib().lsh_step_batch(self._h, k, w.ctypes.data, t.ctypes.data, p.ctypes.data, ctypes.cast(fp, ctypes.c_void_p),
                                         ctypes.cast(npp, ctypes.c_void_p), nn.ctypes.data, int(bool(with_estimator)) | (2 if views else 0), out.ctypes.data,
                                         ctypes.cast(st, ctypes.c_void_p)))
        return out, list(st)

    def _ptr_arrays(self, workers, times_ns, feat_ptrs, nrm_ptrs, ns):
        k = len(workers)
        return (k, np.ascontiguousarray(workers, np.int32), np.ascontiguousarray(times_ns, np.int64),
                (ctypes.c_void_p * k)(*[int(a) for a in feat_ptrs]), (ctypes.c_void_p * k)(*[int(a) for a in nrm_ptrs]),
                np.ascontiguousarray(ns, np.int32))

    def begin_batch(self, workers, times_ns, poses7, feat_ptrs, nrm_ptrs, ns, views=False):
        """First half of step_batch (IncrementalEstimator::beginPosesAndLaserScans): stage and launch, return at once."""
        k, w, t, fp, npp, nn = self._ptr_arrays(workers, times_ns, feat_ptrs, nrm_ptrs, ns)
        p = np.ascontiguousarray(poses7, np.float64).reshape(k, 7)
        self._pending_k = k
        self._check(lib().lsh_begin_batch(self._h, k, w.ctypes.data, t.ctypes.data, p.ctypes.data, ctypes.cast(fp, ctypes.c_void_p),
                                          ctypes.cast(npp, ctypes.c_void_p), nn.ctypes.data, 2 if views else 0))

    def prefetch(self, workers, times_ns, feat_ptrs, nrm_ptrs, ns, views=False):
        """Hint (IncrementalEstimator::prefetchLaserScans): upload scans a later begin_batch will be handed."""
        k, w, t, fp, npp, nn = self._ptr_arrays(workers, times_ns, feat_ptrs, nrm_ptrs, ns)
        self._check(lib().lsh_prefetch(self._h, k, w.ctypes.data, t.ctypes.data, ctypes.cast(fp, ctypes.c_void_p),
                                       ctypes.cast(npp, ctypes.c_void_p), nn.ctypes.data, 2 if views else 0))

    def end_batch(self, with_estimator=True):
        """Second half of step_batch.  Returns (icp T_a_b (len,7), list of IcpStats)."""
        k = self._pending_k
        out = np.zeros((k, 7), np.float64)
        st = (IcpStats * k)()
        self._check(lib().lsh_end_batch(self._h, int(bool(with_estimator)), out.ctypes.data, ctypes.cast(st, ctypes.c_void_p)))
        return out, list(st)

    def loop_closure(self, track_a, time_a, track_b, time_b, w_T_a_b7):
        p = np.ascontiguousarray(w_T_a_b7, np.float64)
        self._check(lib().lsh_loop_closure(self._h, track_a, int(time_a), track_b, int(time_b), p.ctypes.data))

    def _count(self, n):
        """A hook that returns a count: only a negative value is an error (1 is one node, not LS_ERR_CONVERGENCE)."""
        if n < 0:
            self._check(n)
        return n

    def trajectory(self, worker=0):
        n = self._count(lib().lsh_trajectory(self._h, worker, None, None, 0))
        times = np.zeros(max(n, 1), np.int64)
        poses = np.zeros((max(n, 1), 7), np.float64)
        self._count(lib().lsh_trajectory(self._h, worker, times.ctypes.data, poses.ctypes.data, n))
        return times[:n], poses[:n]

    def num_scans(self, worker=0):
        return self._count(lib().lsh_num_scans(self._h, worker))

    def build_submap(self, worker, time_ns, radius, cap_points):
        f = np.zeros((cap_points, 4), np.float32)
        nr = np.zeros((cap_points, 3), np.float32)
        m = self._count(lib().lsh_build_submap(self._h, worker, int(time_ns), radius, f.ctypes.data, nr.ctypes.data, cap_points))
        return f[:m], nr[:m]


class Assembler:
    """laser_slam::VelodyneAssembler (include/laser_slam/velodyne_assembler.hpp): packets in, de-skewed revolutions out."""

    def __init__(self, T_sensor_base=None, naive=False, device=0):
        L = lib()
        L.lsh_assembler_create.restype = ctypes.c_void_p
        L.lsh_assembler_create.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.lsh_assembler_destroy.argtypes = [ctypes.c_void_p]
        L.lsh_assembler_destroy.restype = None
        L.lsh_assembler_add_packet.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64,
                                               ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                               ctypes.POINTER(ctypes.c_int64)]
        t = None if T_sensor_base is None else np.ascontiguousarray(np.asarray(T_sensor_base, np.float32).T).reshape(16)
        self._h = ctypes.c_void_p(L.lsh_assembler_create(None if t is None else t.ctypes.data, int(naive), device))
        self._cap = 1 << 20
        self._out = np.empty((self._cap, 4), np.float32)

    def add_packet(self, points4, T_fixed_base, stamp_ns):
        """None, or (revolution points (m,4), stamp of its last packet)."""
        p = np.ascontiguousarray(points4, np.float32)
        t = np.ascontiguousarray(np.asarray(T_fixed_base, np.float32).T).reshape(16)   # column-major
        m, st = ctypes.c_int(0), ctypes.c_int64(0)
        rc = lib().lsh_assembler_add_packet(self._h, p.ctypes.data, len(p), t.ctypes.data, int(stamp_ns), self._out.ctypes.data,
                                            self._cap, ctypes.byref(m), ctypes.byref(st))
        if rc < 0:
            raise RuntimeError(f"lsh_assembler_add_packet failed with {rc}")
        return (self._out[:m.value].copy(), int(st.value)) if rc == 1 else None

    def close(self):
        if self._h:
            lib().lsh_assembler_destroy(self._h)
            self._h = None


LM_LOCAL, LM_LOCAL_FILTERED, LM_DISTANT, LM_FILTERED_MAP = 0, 1, 2, 3   # include/ls_b200.h LS_LM_*


class LocalMap:
    """laser_slam::LocalMap (include/laser_slam/local_map.hpp) on one worker's track of an Estimator: the worker's map
    maintenance, each call taking its pose, centre or transform from the track.  Close it before the estimator."""

    def __init__(self, estimator, worker, distance_to_consider_fixed=20.0, separate_distant_map=True, create_filtered_map=True,
                 voxel_size_m=0.1, minimum_point_number_per_voxel=0, remove_ground_from_local_map=False,
                 ground_distance_to_robot_center_m=1.0):
        L = lib()
        if not hasattr(L, "_lm_bound"):
            vp, ci, cd = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
            L.lsh_local_map_create.restype = vp
            L.lsh_local_map_create.argtypes = [vp, ci, cd, ci, ci, cd, ci, ci, cd, ctypes.c_char_p, ci]
            L.lsh_local_map_destroy.argtypes = [vp]
            L.lsh_local_map_destroy.restype = None
            L.lsh_local_map_last_error.argtypes = [vp]
            L.lsh_local_map_last_error.restype = ctypes.c_char_p
            for f in ("add_scan", "filter", "take_queue", "clear"):
                getattr(L, "lsh_local_map_" + f).argtypes = [vp]
            L.lsh_local_map_get.argtypes = [vp, ci, vp, ci]
            L.lsh_local_map_queued.argtypes = [vp, ci, vp, ci]
            L.lsh_local_map_update.argtypes = [vp, vp, ctypes.c_int64]
            L._lm_bound = True
        err = ctypes.create_string_buffer(512)
        self._h = L.lsh_local_map_create(estimator._h, worker, float(distance_to_consider_fixed), int(bool(separate_distant_map)),
                                         int(bool(create_filtered_map)), float(voxel_size_m), int(minimum_point_number_per_voxel),
                                         int(bool(remove_ground_from_local_map)), float(ground_distance_to_robot_center_m), err, 512)
        if not self._h:
            raise LsError(err.value.decode() or "lsh_local_map_create failed")

    def close(self):
        if getattr(self, "_h", None):
            lib().lsh_local_map_destroy(self._h)
            self._h = None

    def _check(self, rc):
        if rc < 0:
            raise LsError(lib().lsh_local_map_last_error(self._h).decode())
        return rc

    @staticmethod
    def _read(fn):
        n = fn(None, 0)
        out = np.zeros((max(n, 1), 4), np.float32)
        if n > 0:
            fn(out.ctypes.data, n)
        return out[:n]

    def add_scan(self):
        self._check(lib().lsh_local_map_add_scan(self._h))

    def get_filtered_map(self):
        self._check(lib().lsh_local_map_filter(self._h))
        return self.get(LM_FILTERED_MAP)

    def get(self, which):
        return self._read(lambda p, cap: self._check(lib().lsh_local_map_get(self._h, which, p, cap)))

    def get_queued_points(self):
        k = self._check(lib().lsh_local_map_take_queue(self._h))
        return [self._read(lambda p, cap, j=j: self._check(lib().lsh_local_map_queued(self._h, j, p, cap))) for j in range(k)]

    def update_local_map(self, last_pose_before_update7, time_ns):
        p = np.ascontiguousarray(last_pose_before_update7, np.float64)
        self._check(lib().lsh_local_map_update(self._h, p.ctypes.data, int(time_ns)))

    def clear_local_map(self):
        self._check(lib().lsh_local_map_clear(self._h))


class OccupancyMap:
    """laser_slam::OccupancyMap (include/laser_slam/occupancy_map.hpp) on an Estimator: laser_to_octomap's insertion of
    every track's scans.  Keyword arguments are laser_slam_b200.OccupancyParams' fields.  Close it before the estimator."""

    def __init__(self, estimator, resolution=0.075, prob_hit=0.9, prob_miss=0.4, clamp_min=0.12, clamp_max=0.97,
                 occupancy_threshold=0.7, max_range=20.0, initial_capacity=0, treat_unknown_as_occupied=True):
        L = lib()
        if not hasattr(L, "_occ_bound"):
            vp, ci, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
            L.lsh_occupancy_create.restype = vp
            L.lsh_occupancy_create.argtypes = [vp, vp, ci, ctypes.c_char_p, ci]
            L.lsh_occupancy_destroy.argtypes = [vp]
            L.lsh_occupancy_destroy.restype = None
            L.lsh_occupancy_last_error.argtypes = [vp]
            L.lsh_occupancy_last_error.restype = ctypes.c_char_p
            L.lsh_occupancy_insert_laser_tracks.argtypes = [vp]
            L.lsh_occupancy_voxels.argtypes = [vp, ci, vp, vp, i64]
            L.lsh_occupancy_voxels.restype = i64
            L.lsh_occupancy_occupied_cloud.argtypes = [vp, vp, ci]
            L.lsh_occupancy_write_binary.argtypes = [vp, ctypes.c_char_p]
            L.lsh_occupancy_read_binary.argtypes = [vp, ctypes.c_char_p]
            L.lsh_occupancy_write_full.argtypes = [vp, ctypes.c_char_p]
            L.lsh_occupancy_read_full.argtypes = [vp, ctypes.c_char_p]
            L.lsh_occupancy_write_full_data.argtypes = [vp, vp, i64, ctypes.POINTER(i64)]
            L.lsh_occupancy_write_full_data.restype = i64
            L.lsh_occupancy_read_full_data.argtypes = [vp, vp, i64, i64, ctypes.c_double]
            L.lsh_occupancy_occupied_leaf_cloud.argtypes = [vp, vp, ci]
            L.lsh_occupancy_cell_status.argtypes = [vp, vp, ci, vp, vp]
            L.lsh_occupancy_line_status.argtypes = [vp, vp, vp, ci, vp, ci, ci, vp, vp]
            L.lsh_occupancy_cast_rays.argtypes = [vp, vp, vp, ci, ci, ctypes.c_double, ci, vp, vp]
            L.lsh_occupancy_set_boxes.argtypes = [vp, vp, vp, vp, ci, ci, vp]
            L.lsh_occupancy_reset.argtypes = [vp]
            L.lsh_occupancy_box_cloud.argtypes = [vp, vp, vp, vp, ci]
            L.lsh_occupancy_bounds.argtypes = [vp, vp]
            L.lsh_occupancy_track_changes.argtypes = [vp, ci]
            L.lsh_occupancy_changed_keys.argtypes = [vp, vp, vp, vp, i64]
            L.lsh_occupancy_changed_keys.restype = i64
            L.lsh_occupancy_changed_points.argtypes = [vp, vp, vp, i64]
            L.lsh_occupancy_changed_points.restype = i64
            L.lsh_occupancy_box_status.argtypes = [vp, vp, vp, ci, ci, vp]
            L.lsh_occupancy_check_paths.argtypes = [vp, vp, vp, ci, vp, ci, vp]
            L.lsh_occupancy_boxes.argtypes = [vp, ci, vp, vp, vp, vp, i64]
            L.lsh_occupancy_boxes.restype = i64
            L.lsh_occupancy_marker_array.argtypes = [vp, ctypes.c_double, ctypes.c_double, ctypes.c_double, vp, vp, vp, vp,
                                                     i64]
            L.lsh_occupancy_marker_array.restype = i64
            L.lsh_occupancy_projected_map.argtypes = [vp, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                                      vp]
            L.lsh_occupancy_projected_map.restype = i64
            L.lsh_occupancy_projected_cells.argtypes = [vp, vp, i64]
            L.lsh_occupancy_projected_cells.restype = i64
            L.lsh_occupancy_save_projected_map.argtypes = [vp, ctypes.c_char_p, ctypes.c_double, ctypes.c_double,
                                                           ctypes.c_double, ctypes.c_double]
            L._occ_bound = True
        prm = np.array([resolution, prob_hit, prob_miss, clamp_min, clamp_max, occupancy_threshold, max_range,
                        float(bool(treat_unknown_as_occupied))], np.float64)
        err = ctypes.create_string_buffer(512)
        self._h = L.lsh_occupancy_create(estimator._h, prm.ctypes.data, int(initial_capacity), err, 512)
        if not self._h:
            raise LsError(err.value.decode() or "lsh_occupancy_create failed")

    def close(self):
        if getattr(self, "_h", None):
            lib().lsh_occupancy_destroy(self._h)
            self._h = None

    def _check(self, rc):
        if rc < 0:
            raise LsError(lib().lsh_occupancy_last_error(self._h).decode())
        return rc

    def insert_laser_tracks(self):
        return self._check(lib().lsh_occupancy_insert_laser_tracks(self._h))

    def voxels(self, which=1):
        """(keys uint64, log-odds float32) of LS_OCC_KNOWN (1) or LS_OCC_OCCUPIED (2), by ascending key."""
        n = self._check(lib().lsh_occupancy_voxels(self._h, which, None, None, 0))
        keys = np.zeros(max(n, 1), np.uint64)
        lo = np.zeros(max(n, 1), np.float32)
        self._check(lib().lsh_occupancy_voxels(self._h, which, keys.ctypes.data, lo.ctypes.data, n))
        return keys[:n], lo[:n]

    def occupied_cloud(self):
        n = self._check(lib().lsh_occupancy_occupied_cloud(self._h, None, 0))
        out = np.zeros((max(n, 1), 4), np.float32)
        self._check(lib().lsh_occupancy_occupied_cloud(self._h, out.ctypes.data, n))
        return out[:n]

    def write_binary(self, path):
        """writeBinary: the map as an octomap .bt file."""
        self._check(lib().lsh_occupancy_write_binary(self._h, os.fsencode(path)))

    def read_binary(self, path):
        """readBinary: the .bt file replaces the map.  False, with the map unchanged, when the file is refused."""
        rc = lib().lsh_occupancy_read_binary(self._h, os.fsencode(path))
        if rc == -1:  # LS_ERR_ARG
            return False
        self._check(rc)
        return True

    def write_full(self, path):
        """write: the map as an octomap .ot file (every node's log-odds)."""
        self._check(lib().lsh_occupancy_write_full(self._h, os.fsencode(path)))

    def read_full(self, path):
        """read: the .ot file replaces the map.  False, with the map unchanged, when the file is refused."""
        rc = lib().lsh_occupancy_read_full(self._h, os.fsencode(path))
        if rc == -1:  # LS_ERR_ARG
            return False
        self._check(rc)
        return True

    def write_data(self):
        """writeData: (nodes, payload bytes) of the full tree."""
        nodes = ctypes.c_int64(0)
        n = self._check(lib().lsh_occupancy_write_full_data(self._h, None, 0, ctypes.byref(nodes)))
        out = np.zeros(max(n, 1), np.uint8)
        self._check(lib().lsh_occupancy_write_full_data(self._h, out.ctypes.data, n, ctypes.byref(nodes)))
        return nodes.value, out[:n].tobytes()

    def read_data(self, payload, nodes, resolution):
        """readData: a full-tree payload replaces the map.  False, with the map unchanged, when it is refused."""
        buf = np.frombuffer(bytes(payload), np.uint8)
        rc = lib().lsh_occupancy_read_full_data(self._h, buf.ctypes.data if len(buf) else None, len(buf), int(nodes),
                                                float(resolution))
        if rc == -1:  # LS_ERR_ARG
            return False
        self._check(rc)
        return True

    def occupied_leaf_cloud(self):
        """getOccupiedLeafCloud: the pruned tree's occupied leaves, (n,4) float32."""
        n = self._check(lib().lsh_occupancy_occupied_leaf_cloud(self._h, None, 0))
        out = np.zeros((max(n, 1), 4), np.float32)
        self._check(lib().lsh_occupancy_occupied_leaf_cloud(self._h, out.ctypes.data, n))
        return out[:n]

    def cell_probability(self, points):
        """getCellProbabilityPoint per point (one query each): (status int8, probability float64, -1 when unknown)."""
        p = np.ascontiguousarray(np.asarray(points, np.float64).reshape(-1, 3))
        st = np.zeros(max(len(p), 1), np.int8)
        pr = np.zeros(max(len(p), 1), np.float64)
        self._check(lib().lsh_occupancy_cell_status(self._h, p.ctypes.data, len(p), st.ctypes.data, pr.ctypes.data))
        return st[:len(p)], pr[:len(p)]

    def line_status(self, starts, ends, box=None, stop_at_unknown=True, single=False):
        """The batched getLineStatus overload ((status, first keys)), or with single=True one getLineStatus /
        getVisibility / getLineStatusBoundingBox call per segment (status only)."""
        s = np.ascontiguousarray(np.asarray(starts, np.float64).reshape(-1, 3))
        e = np.ascontiguousarray(np.asarray(ends, np.float64).reshape(-1, 3))
        b = None if box is None else np.ascontiguousarray(np.asarray(box, np.float64).reshape(3))
        n = len(s)
        st = np.zeros(max(n, 1), np.int8)
        fk = np.zeros(max(n, 1), np.uint64)
        self._check(lib().lsh_occupancy_line_status(self._h, s.ctypes.data, e.ctypes.data, n,
                                                    None if b is None else b.ctypes.data, int(bool(stop_at_unknown)),
                                                    int(bool(single)), st.ctypes.data, fk.ctypes.data))
        return st[:n] if single else (st[:n], fk[:n])

    def cast_rays(self, origins, directions, ignore_unknown=False, max_range=-1.0, single=False, ends_in=None):
        """castRays (LS_RAY_* results, ends (n,3) float64), or with single=True one castRay per ray (1 for a hit, else 0;
        ends start as ends_in and are left alone where castRay leaves *end)."""
        o = np.ascontiguousarray(np.asarray(origins, np.float64).reshape(-1, 3))
        d = np.ascontiguousarray(np.asarray(directions, np.float64).reshape(-1, 3))
        n = len(o)
        r = np.zeros(max(n, 1), np.int32)
        ends = np.zeros((max(n, 1), 3), np.float64)
        if ends_in is not None:
            ends[:n] = ends_in
        self._check(lib().lsh_occupancy_cast_rays(self._h, o.ctypes.data, d.ctypes.data, n, int(bool(ignore_unknown)),
                                                  float(max_range), int(bool(single)), r.ctypes.data, ends.ctypes.data))
        return r[:n], ends[:n]

    def set_boxes(self, centres, sizes, occupied, single=False):
        """setBoxes ((voxels_set, new_known, known voxels)), or with single=True one setFree / setOccupied per box (None)."""
        c = np.ascontiguousarray(np.asarray(centres, np.float64).reshape(-1, 3))
        s = np.ascontiguousarray(np.asarray(sizes, np.float64).reshape(-1, 3))
        o = np.ascontiguousarray(np.asarray(occupied).reshape(-1).astype(bool).astype(np.int8))
        st = np.zeros(3, np.int64)
        self._check(lib().lsh_occupancy_set_boxes(self._h, c.ctypes.data, s.ctypes.data, o.ctypes.data, len(c),
                                                  int(bool(single)), st.ctypes.data))
        return None if single else tuple(int(x) for x in st)

    def reset_map(self):
        self._check(lib().lsh_occupancy_reset(self._h))

    def occupied_cloud_in_box(self, center, size):
        """getOccupiedPointcloudInBoundingBox: (n,4) float32 voxel centres in loop order."""
        c = np.ascontiguousarray(np.asarray(center, np.float64).reshape(3))
        s = np.ascontiguousarray(np.asarray(size, np.float64).reshape(3))
        n = self._check(lib().lsh_occupancy_box_cloud(self._h, c.ctypes.data, s.ctypes.data, None, 0))
        out = np.zeros((max(n, 1), 4), np.float32)
        self._check(lib().lsh_occupancy_box_cloud(self._h, c.ctypes.data, s.ctypes.data, out.ctypes.data, n))
        return out[:n]

    def map_bounds(self):
        """getMapBounds, getMapSize, getMapCenter: (min, max, size, centre), each (3,) float64."""
        out = np.zeros(12, np.float64)
        self._check(lib().lsh_occupancy_bounds(self._h, out.ctypes.data))
        return out[0:3], out[3:6], out[6:9], out[9:12]

    def enable_change_detection(self, enable=True):
        """enableChangeDetection; returns isChangeDetectionEnabled."""
        return bool(self._check(lib().lsh_occupancy_track_changes(self._h, int(bool(enable)))))

    def reset_change_detection(self):
        """resetChangeDetection; returns isChangeDetectionEnabled."""
        return bool(self._check(lib().lsh_occupancy_track_changes(self._h, -1)))

    def num_changes(self):
        """numChangesDetected."""
        return self._check(lib().lsh_occupancy_changed_keys(self._h, None, None, None, 0))

    def changed_keys(self):
        """getChangedKeys: (keys uint64, status int8, previous int8) by ascending key."""
        n = self.num_changes()
        k = np.zeros(max(n, 1), np.uint64)
        s = np.zeros(max(n, 1), np.int8)
        p = np.zeros(max(n, 1), np.int8)
        self._check(lib().lsh_occupancy_changed_keys(self._h, k.ctypes.data, s.ctypes.data, p.ctypes.data, n))
        return k[:n], s[:n], p[:n]

    def changed_points(self, cap):
        """getChangedPoints (then a reset): (centres (n,3) float64, occupied (n,) bool), at most cap of them."""
        pts = np.zeros((max(cap, 1), 3), np.float64)
        occ = np.zeros(max(cap, 1), np.uint8)
        n = self._check(lib().lsh_occupancy_changed_points(self._h, pts.ctypes.data, occ.ctypes.data, int(cap)))
        m = min(n, cap)
        return pts[:m], occ[:m].astype(bool)

    def boxes(self, occupied, region=None):
        """getAllOccupiedBoxes (occupied) or getAllFreeBoxes, with region = (min (3,), max (3,)) the region overload:
        (centres (n,3) float64, edges (n,) float64) in octomap's leaf order."""
        lo = hi = None
        if region is not None:
            lo = np.ascontiguousarray(np.asarray(region[0], np.float64).reshape(3))
            hi = np.ascontiguousarray(np.asarray(region[1], np.float64).reshape(3))
        args = (int(bool(occupied)), None if lo is None else lo.ctypes.data, None if hi is None else hi.ctypes.data)
        n = self._check(lib().lsh_occupancy_boxes(self._h, *args, None, None, 0))
        c = np.zeros((max(n, 1), 3), np.float64)
        e = np.zeros(max(n, 1), np.float64)
        m = self._check(lib().lsh_occupancy_boxes(self._h, *args, c.ctypes.data, e.ctypes.data, n))
        return c[:m], e[:m]

    def marker_array(self, min_z, max_z, color_factor=0.8):
        """generateMarkerArray: (occupied, free), each 17 (size, centres (k,3) float64, colours (k,4) float32) for depths
        0..16; free lists have no colours."""
        sizes, counts = np.zeros(34, np.float64), np.zeros(34, np.int64)
        n = self._check(lib().lsh_occupancy_marker_array(self._h, float(min_z), float(max_z), float(color_factor), None, None,
                                                         sizes.ctypes.data, counts.ctypes.data, 0))
        c = np.zeros((max(n, 1), 3), np.float64)
        rgba = np.zeros((max(n, 1), 4), np.float32)
        self._check(lib().lsh_occupancy_marker_array(self._h, float(min_z), float(max_z), float(color_factor), c.ctypes.data,
                                                     rgba.ctypes.data, sizes.ctypes.data, counts.ctypes.data, n))
        off = np.concatenate([[0], np.cumsum(counts)])
        lists = [(sizes[k], c[off[k]:off[k + 1]], rgba[off[k]:off[k + 1]] if k < 17 else np.zeros((0, 4), np.float32))
                 for k in range(34)]
        return lists[:17], lists[17:]

    def projected_map(self, min_z=-math.inf, max_z=math.inf, min_x_size=0.0, min_y_size=0.0):
        """getProjectedMap, called once: (grid int8 (height, width), (width, height, resolution, origin x, origin y))."""
        geo = np.zeros(5, np.float64)
        n = self._check(lib().lsh_occupancy_projected_map(self._h, float(min_z), float(max_z), float(min_x_size),
                                                          float(min_y_size), geo.ctypes.data))
        grid = np.zeros(max(n, 1), np.int8)
        lib().lsh_occupancy_projected_cells(self._h, grid.ctypes.data, n)
        w, h = int(geo[0]), int(geo[1])
        return grid[:n].reshape(h, w), (w, h, float(geo[2]), float(geo[3]), float(geo[4]))

    def save_projected_map(self, stem, min_z=-math.inf, max_z=math.inf, min_x_size=0.0, min_y_size=0.0):
        """saveProjectedMap: True when stem.pgm and stem.yaml were written."""
        return bool(self._check(lib().lsh_occupancy_save_projected_map(self._h, os.fsencode(stem), float(min_z), float(max_z),
                                                                       float(min_x_size), float(min_y_size))))

    def box_status(self, centres, sizes, single=False):
        """The batched getCellStatusBoundingBox overload, or with single=True one call per box: int8 CELL_* per box."""
        c = np.ascontiguousarray(np.asarray(centres, np.float64).reshape(-1, 3))
        s = np.ascontiguousarray(np.asarray(sizes, np.float64).reshape(-1, 3))
        st = np.zeros(max(len(c), 1), np.int8)
        self._check(lib().lsh_occupancy_box_status(self._h, c.ctypes.data, s.ctypes.data, len(c), int(bool(single)),
                                                   st.ctypes.data))
        return st[:len(c)]

    def check_paths(self, positions, offsets, robot_size, single=False):
        """setRobotSize(robot_size), then checkPathsForCollisionsWithRobot, or with single=True one
        checkPathForCollisionsWithRobot per path: int64 per path, the first colliding pose's index or -1.  The collision
        mode is the map's treat_unknown_as_occupied."""
        p = np.ascontiguousarray(np.asarray(positions, np.float64).reshape(-1, 3))
        o = np.ascontiguousarray(np.asarray(offsets, np.int64).reshape(-1))
        r = np.ascontiguousarray(np.asarray(robot_size, np.float64).reshape(3))
        n = max(len(o) - 1, 0)
        first = np.zeros(max(n, 1), np.int64)
        self._check(lib().lsh_occupancy_check_paths(self._h, p.ctypes.data, o.ctypes.data, n, r.ctypes.data,
                                                    int(bool(single)), first.ctypes.data))
        return first[:n]


class DistanceMap:
    """laser_slam::DistanceMap (include/laser_slam/distance_map.hpp) on an OccupancyMap of this module: DynamicEDTOctomap's
    calls over the device distance map.  Close it before the occupancy map."""

    def __init__(self, occupancy_map, max_dist, bbx_min, bbx_max, treat_unknown_as_occupied=False):
        L = lib()
        if not hasattr(L, "_dist_bound"):
            vp, ci = ctypes.c_void_p, ctypes.c_int
            L.lsh_distance_create.restype = vp
            L.lsh_distance_create.argtypes = [vp, ctypes.c_float, vp, ci, ctypes.c_char_p, ci]
            L.lsh_distance_destroy.argtypes = [vp]
            L.lsh_distance_destroy.restype = None
            L.lsh_distance_last_error.argtypes = [vp]
            L.lsh_distance_last_error.restype = ctypes.c_char_p
            L.lsh_distance_update.argtypes = [vp, vp]
            L.lsh_distance_query.argtypes = [vp, vp, ci, ci, vp, vp, vp]
            L._dist_bound = True
        box = np.ascontiguousarray(np.concatenate([np.asarray(bbx_min, np.float64).reshape(3),
                                                   np.asarray(bbx_max, np.float64).reshape(3)]))
        err = ctypes.create_string_buffer(512)
        self._h = L.lsh_distance_create(occupancy_map._h, float(max_dist), box.ctypes.data, int(bool(treat_unknown_as_occupied)),
                                        err, 512)
        if not self._h:
            raise LsError(err.value.decode() or "lsh_distance_create failed")

    def close(self):
        if getattr(self, "_h", None):
            lib().lsh_distance_destroy(self._h)
            self._h = None

    def _check(self, rc):
        if rc < 0:
            raise LsError(lib().lsh_distance_last_error(self._h).decode())
        return rc

    def update(self):
        """update; returns (getMaxDist, getSquaredMaxDistCells)."""
        out = np.zeros(2, np.float64)
        self._check(lib().lsh_distance_update(self._h, out.ctypes.data))
        return float(out[0]), int(out[1])

    def query(self, points, single=False):
        """The batched getDistances, or with single=True getDistance / getDistanceAndClosestObstacle /
        getSquaredDistanceInCells once per point: (distance float32, squared distance in cells int32, closest (n,3)
        float64)."""
        p = np.ascontiguousarray(np.asarray(points, np.float64).reshape(-1, 3))
        n = len(p)
        d = np.zeros(max(n, 1), np.float32)
        s = np.zeros(max(n, 1), np.int32)
        c = np.zeros((max(n, 1), 3), np.float64)
        self._check(lib().lsh_distance_query(self._h, p.ctypes.data, n, int(bool(single)), d.ctypes.data, s.ctypes.data,
                                             c.ctypes.data))
        return d[:n], s[:n], c[:n]
