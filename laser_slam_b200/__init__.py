"""laser_slam_b200 -- H100-native scan-to-local-map ICP + pose-graph hot path of ethz-asl/laser_slam.

This package is a thin ctypes front-end over the C ABI in include/ls_b200.h (libls_b200.so, built by
laser_slam_b200/csrc/Makefile for sm_90a).  The compute path is the CUDA library; there is NO CPU
fallback: loading fails loudly when the shared library is missing and ls_b200_init fails when no
CUDA device is usable.
"""
import ctypes
import os
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

    def create_map(self, capacity_scans, max_pts_per_scan):
        return Map(self, capacity_scans, max_pts_per_scan)


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
