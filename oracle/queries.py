"""ORACLE — test infrastructure only.  ctypes bindings of oracle/query_oracle.cpp: the occupancy map's queries
(volumetric_mapping's WorldBase and octomap's castRay) restated sequentially from oracle/QUERIES.md.  The library is
compiled from query_oracle.cpp, which includes occupancy_oracle.cpp, with the flags of oracle/occupancy.py; its
OccupancyMap is the insert oracle's map with the query methods added."""
import ctypes
import os
import subprocess

import numpy as np

from oracle import occupancy

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "libls_query_oracle.so")
_SRCS = [os.path.join(_HERE, "query_oracle.cpp"), os.path.join(_HERE, "occupancy_oracle.cpp")]
_lib = None

CELL_FREE, CELL_OCCUPIED, CELL_UNKNOWN = 0, 1, 2                        # include/ls_b200.h LS_CELL_*
RAY_INVALID, RAY_HIT, RAY_UNKNOWN, RAY_MAX_RANGE, RAY_KEY_BOUND = 0, 1, 2, 3, 4   # LS_RAY_*
NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def build(force=False):
    stale = not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < max(os.path.getmtime(s) for s in _SRCS)
    if force or stale:
        os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([cxx, "-O2", "-march=native", "-ffp-contract=off", "-fPIC", "-std=c++17", "-Wall", "-shared",
                               "-o", LIB_PATH, _SRCS[0]])
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(LIB_PATH)
        vp, i64, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        L.occo_cell_status.argtypes = [vp, vp, vp, i64, vp, ci, vp, vp]
        L.occo_cell_status.restype = i64
        L.occo_line_status.argtypes = [vp, vp, vp, i64, vp, vp, ci, vp, ci, vp, vp]
        L.occo_line_status.restype = i64
        L.occo_cast_rays.argtypes = [vp, vp, vp, i64, vp, vp, ci, ci, ctypes.c_double, vp, vp]
        L.occo_cast_rays.restype = i64
        _lib = L
    return _lib


def _triples(a, dtype):
    return np.ascontiguousarray(np.asarray(a, dtype).reshape(-1, 3))


class _Queries:
    """cell_status, line_status and cast_rays over self._map() (ascending keys, log-odds) at self._prm, with the return
    values of laser_slam_b200.OccupancyMap's methods and the keys visited in self.keys_visited."""

    keys_visited = 0

    def cell_status(self, points):
        """(status int8 LS_CELL_*, log-odds float32, NaN when unknown) per double point."""
        p = _triples(points, np.float64)
        k, v = self._map()
        st = np.zeros(len(p), np.int8)
        lo = np.zeros(len(p), np.float32)
        self.keys_visited = lib().occo_cell_status(self._prm.ctypes.data, k.ctypes.data, v.ctypes.data, len(k),
                                                   p.ctypes.data, len(p), st.ctypes.data, lo.ctypes.data)
        return st, lo

    def line_status(self, starts, ends, box=None, stop_at_unknown=True):
        """(status int8 LS_CELL_*, first key uint64, all ones when free) per segment; box: the bounding box size."""
        s, e = _triples(starts, np.float64), _triples(ends, np.float64)
        b = None if box is None else np.ascontiguousarray(box, np.float64).reshape(3)
        k, v = self._map()
        st = np.zeros(len(s), np.int8)
        fk = np.zeros(len(s), np.uint64)
        self.keys_visited = lib().occo_line_status(self._prm.ctypes.data, k.ctypes.data, v.ctypes.data, len(k),
                                                   s.ctypes.data, e.ctypes.data, len(s),
                                                   None if b is None else b.ctypes.data, int(bool(stop_at_unknown)),
                                                   st.ctypes.data, fk.ctypes.data)
        return st, fk

    def cast_rays(self, origins, directions, ignore_unknown=False, max_range=-1.0):
        """(result int8 LS_RAY_*, ends (n,3) float32, NaN for an invalid ray) per float ray."""
        o, d = _triples(origins, np.float32), _triples(directions, np.float32)
        k, v = self._map()
        r = np.zeros(len(o), np.int8)
        ends = np.zeros((len(o), 3), np.float32)
        self.keys_visited = lib().occo_cast_rays(self._prm.ctypes.data, k.ctypes.data, v.ctypes.data, len(k), o.ctypes.data,
                                                 d.ctypes.data, len(o), int(bool(ignore_unknown)), float(max_range),
                                                 r.ctypes.data, ends.ctypes.data)
        return r, ends


class OccupancyMap(_Queries, occupancy.OccupancyMap):
    """The insert oracle's map with the queries."""

    _known = None

    def insert_scan(self, pts4, T_w_scan):
        self._known = None
        return super().insert_scan(pts4, T_w_scan)

    def _map(self):
        if self._known is None:
            k, v = self.download()
            self._known = (np.ascontiguousarray(k), np.ascontiguousarray(v))
        return self._known


class KnownVoxels(_Queries):
    """The queries over given known voxels (ascending packed keys and their log-odds, e.g. a device map's download);
    keyword arguments as OccupancyMap's."""

    def __init__(self, keys, log_odds, **params):
        p = dict(occupancy.DEFAULTS, **params)
        self._prm = np.array([p[k] for k in ("resolution", "prob_hit", "prob_miss", "clamp_min", "clamp_max",
                                             "occupancy_threshold", "max_range")], np.float64)
        self._known = (np.ascontiguousarray(keys, np.uint64), np.ascontiguousarray(log_odds, np.float32))

    def _map(self):
        return self._known
