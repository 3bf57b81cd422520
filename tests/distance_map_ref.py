"""Reference of the distance map (test infrastructure only).  Binds tests/ref/edt_ref.cpp: the obstacle grid of a box from
known voxels, a sequential exact separable EDT with the tie rule and the cap, and the query rule.  box() and cap() restate
how the corners are keyed and the cap; Field chains them all into what an update must give.  The rules are DESIGN.md
§4b'''''''''."""
import ctypes
import math
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "ref", "_build", "libls_edt_ref.so")
_SRC = os.path.join(_HERE, "ref", "edt_ref.cpp")
_lib = None
K0 = 32768
NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def build(force=False):
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < os.path.getmtime(_SRC):
        os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-std=c++17", "-Wall", "-shared", "-o", LIB_PATH,
                               _SRC])
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(LIB_PATH)
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        L.edt_obstacles.argtypes = [vp, vp, i64, ctypes.c_float, vp, vp, ctypes.c_int, vp]
        L.edt_obstacles.restype = None
        L.edt_transform.argtypes = [vp, vp, i64, vp, vp]
        L.edt_transform.restype = None
        L.edt_query.argtypes = [vp, vp, vp, vp, ctypes.c_double, vp, i64, vp, vp, vp]
        L.edt_query.restype = None
        _lib = L
    return _lib


def key_of(c, res):
    """The map's key of a float coordinate, None when invalid (non-finite included)."""
    c = float(np.float32(c))
    if not math.isfinite(c):
        return None
    f = math.floor(c * (1.0 / res))
    return f + K0 if -K0 <= f < K0 else None


def cap(max_dist, res):
    """(m, M, getMaxDist) of DynamicEDTOctomap's constructor."""
    m = int(float(np.float32(max_dist)) / res + 1.0)
    return m, m * m, float(np.float32(m * res))


def box(bbx_min, bbx_max, res):
    """(kmin (3,) int, size (3,) int) of the corners, or None when a corner has no valid key."""
    lo = [key_of(c, res) for c in bbx_min]
    hi = [key_of(c, res) for c in bbx_max]
    if None in lo or None in hi:
        return None
    return np.array(lo, np.int32), np.array(hi, np.int32) - np.array(lo, np.int32) + 1


def obstacles(keys, log_odds, l_occ, kmin, size, unknown_occ):
    """The obstacle grid (sz, sy, sx) uint8 of the known voxels (packed keys, float32 log-odds)."""
    k = np.ascontiguousarray(keys, np.uint64)
    v = np.ascontiguousarray(log_odds, np.float32)
    km, sz = np.ascontiguousarray(kmin, np.int32), np.ascontiguousarray(size, np.int32)
    g = np.empty(int(np.prod(sz.astype(np.int64))), np.uint8)
    lib().edt_obstacles(k.ctypes.data, v.ctypes.data, len(k), float(l_occ), km.ctypes.data, sz.ctypes.data,
                        int(bool(unknown_occ)), g.ctypes.data)
    return g.reshape(int(sz[2]), int(sz[1]), int(sz[0]))


def transform(grid, M):
    """(s (sz, sy, sx) int32, obstacle cell index (sz, sy, sx) int32, -1 when none) of an obstacle grid."""
    g = np.ascontiguousarray(grid, np.uint8)
    sz = np.array([g.shape[2], g.shape[1], g.shape[0]], np.int32)
    s = np.empty(g.shape, np.int32)
    w = np.empty(g.shape, np.int32)
    lib().edt_transform(g.ctypes.data, sz.ctypes.data, int(M), s.ctypes.data, w.ctypes.data)
    return s, w


def site_keys(site, kmin, size):
    """Obstacle cell indices as packed keys (all ones when none)."""
    w = np.asarray(site, np.int64).reshape(-1)
    x, y, z = w % size[0], (w // size[0]) % size[1], w // (int(size[0]) * int(size[1]))
    k = ((x + int(kmin[0])).astype(np.uint64) | ((y + int(kmin[1])).astype(np.uint64) << np.uint64(16)) |
         ((z + int(kmin[2])).astype(np.uint64) << np.uint64(32)))
    return np.where(w < 0, NO_KEY, k).reshape(np.shape(site))


def query(s, site, kmin, size, res, points):
    """(distance float32, sqdist int32, obstacle centres (n,3) float32) of float points."""
    p = np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))
    n = len(p)
    s, w = np.ascontiguousarray(s, np.int32), np.ascontiguousarray(site, np.int32)
    km, sz = np.ascontiguousarray(kmin, np.int32), np.ascontiguousarray(size, np.int32)
    d, q, o = np.empty(max(n, 1), np.float32), np.empty(max(n, 1), np.int32), np.empty((max(n, 1), 3), np.float32)
    lib().edt_query(s.ctypes.data, w.ctypes.data, km.ctypes.data, sz.ctypes.data, float(res), p.ctypes.data, n,
                    d.ctypes.data, q.ctypes.data, o.ctypes.data)
    return d[:n], q[:n], o[:n]


class Field:
    """What an update of a distance map gives for the known voxels: box, cap, obstacle grid and field."""

    def __init__(self, keys, log_odds, res, l_occ, max_dist, bbx_min, bbx_max, unknown_occ=False):
        self.res = res
        self.kmin, self.size = box(bbx_min, bbx_max, res)
        self.m, self.M, self.max_dist = cap(max_dist, res)
        self.grid = obstacles(keys, log_odds, l_occ, self.kmin, self.size, unknown_occ)
        self.s, self.site = transform(self.grid, self.M)
        self.cells = int(self.grid.size)
        self.obstacles = int(self.grid.sum(dtype=np.int64))

    def keys(self):
        return site_keys(self.site, self.kmin, self.size)

    def query(self, points):
        return query(self.s, self.site, self.kmin, self.size, self.res, points)
