"""ORACLE — test infrastructure only.  ctypes bindings of oracle/occupancy_oracle.cpp: laser_to_octomap's occupancy map
restated sequentially from oracle/OCCUPANCY.md.  Compiled with the flags of oracle/Makefile into its own library."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "libls_occupancy_oracle.so")
_SRC = os.path.join(_HERE, "occupancy_oracle.cpp")
_lib = None

KNOWN, OCCUPIED = 1, 2   # include/ls_b200.h LS_OCC_*
# laser_to_octomap's defaults (resolution, hit, miss, max range) and volumetric_mapping's (clamping, threshold)
DEFAULTS = dict(resolution=0.075, prob_hit=0.9, prob_miss=0.4, clamp_min=0.12, clamp_max=0.97, occupancy_threshold=0.7,
                max_range=20.0)


def build(force=False):
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < os.path.getmtime(_SRC):
        os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([cxx, "-O2", "-march=native", "-ffp-contract=off", "-fPIC", "-std=c++17", "-Wall", "-shared",
                               "-o", LIB_PATH, _SRC])
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(LIB_PATH)
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        L.occo_create.restype = vp
        L.occo_create.argtypes = [vp]
        L.occo_destroy.argtypes = [vp]
        L.occo_destroy.restype = None
        L.occo_insert.argtypes = [vp, vp, ctypes.c_int, vp, vp]
        L.occo_insert.restype = None
        L.occo_download.argtypes = [vp, ctypes.c_int, vp, vp, i64]
        L.occo_download.restype = i64
        L.occo_ray_keys.argtypes = [ctypes.c_double, vp, vp, vp, i64]
        L.occo_ray_keys.restype = i64
        L.occo_logodds.argtypes = [ctypes.c_double]
        L.occo_logodds.restype = ctypes.c_float
        _lib = L
    return _lib


def logodds(p):
    return np.float32(lib().occo_logodds(float(p)))


def ray_keys(res, origin, end):
    """The free cells of one ray (packed keys, DDA order), or None when an end key is invalid."""
    o = np.ascontiguousarray(origin, np.float32)
    e = np.ascontiguousarray(end, np.float32)
    n = lib().occo_ray_keys(float(res), o.ctypes.data, e.ctypes.data, None, 0)
    if n < 0:
        return None
    out = np.zeros(max(n, 1), np.uint64)
    lib().occo_ray_keys(float(res), o.ctypes.data, e.ctypes.data, out.ctypes.data, n)
    return out[:n]


class OccupancyMap:
    """Keyword arguments as laser_slam_b200.OccupancyMap (initial_capacity is accepted and ignored)."""

    def __init__(self, **params):
        params.pop("initial_capacity", None)
        p = dict(DEFAULTS, **params)
        self.params = p
        self._prm = np.array([p[k] for k in ("resolution", "prob_hit", "prob_miss", "clamp_min", "clamp_max",
                                             "occupancy_threshold", "max_range")], np.float64)
        self._h = lib().occo_create(self._prm.ctypes.data)

    def close(self):
        if self._h:
            lib().occo_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def insert_scan(self, pts4, T_w_scan):
        """One scan (n,4) float32 in the sensor frame at pose T_w_scan (4x4).  Returns the stats as a dict."""
        p = np.ascontiguousarray(pts4, np.float32).reshape(-1, 4)
        t = np.ascontiguousarray(np.asarray(T_w_scan, np.float32).T).ravel()
        st = np.zeros(5, np.int64)
        lib().occo_insert(self._h, p.ctypes.data, len(p), t.ctypes.data, st.ctypes.data)
        return dict(rays_cast=int(st[0]), rays_skipped=int(st[1]), free_updates=int(st[2]), occupied_updates=int(st[3]),
                    known_voxels=int(st[4]))

    def size(self, which=KNOWN):
        return int(lib().occo_download(self._h, which, None, None, 0))

    def download(self, which=KNOWN):
        """(keys uint64 ascending, log-odds float32)."""
        n = self.size(which)
        keys = np.zeros(max(n, 1), np.uint64)
        lo = np.zeros(max(n, 1), np.float32)
        lib().occo_download(self._h, which, keys.ctypes.data, lo.ctypes.data, n)
        return keys[:n], lo[:n]


def centres(keys, res):
    """Voxel centres (float32 (n,3)) of packed keys: (float)((k - 32768 + 0.5) * res)."""
    keys = np.asarray(keys, np.uint64)
    k = np.stack([(keys >> np.uint64(s)) & np.uint64(0xFFFF) for s in (0, 16, 32)], axis=1).astype(np.int64)
    return (((k - 32768).astype(np.float64) + 0.5) * float(res)).astype(np.float32)
