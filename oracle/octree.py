"""ORACLE — test infrastructure only.  ctypes bindings of oracle/octree_oracle.cpp: octomap's OcTree as writeBinary
leaves it (max-likelihood states, prune, writeBinaryConst) and octomap_to_point_cloud's leaf iteration, restated from
oracle/OCTREE.md.  Input: known voxels, e.g. the occupancy oracle's map (oracle.occupancy.OccupancyMap).  Compiled with
the flags of oracle/occupancy.py into its own library."""
import ctypes
import os
import subprocess

import numpy as np

from oracle import occupancy

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "libls_octree_oracle.so")
_SRC = os.path.join(_HERE, "octree_oracle.cpp")
_lib = None

OCCUPANCY_THRESHOLD = occupancy.DEFAULTS["occupancy_threshold"]


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
        L.octo_tree_from_voxels.argtypes = [vp, vp, i64, ctypes.c_double, ctypes.c_float]
        L.octo_tree_from_voxels.restype = vp
        L.octo_tree_destroy.argtypes = [vp]
        L.octo_tree_destroy.restype = None
        for f in (L.octo_tree_counts, L.octo_tree_payload):
            f.argtypes = [vp, vp]
            f.restype = None
        L.octo_tree_leaves.argtypes = [vp, vp, vp]
        L.octo_tree_leaves.restype = None
        L.octo_tree_write.argtypes = [vp, ctypes.c_char_p]
        _lib = L
    return _lib


class Octree:
    """The pruned tree: nodes (octomap's size()), payload (the writeBinary data), occupied leaves in leaf-iterator order as
    centres (n,4) float32 and depths uint8."""

    def __init__(self, handle):
        try:
            c = np.zeros(3, np.int64)
            lib().octo_tree_counts(handle, c.ctypes.data)
            self.nodes = int(c[0])
            pay = np.zeros(max(int(c[1]), 1), np.uint8)
            lib().octo_tree_payload(handle, pay.ctypes.data)
            self.payload = pay[:int(c[1])].tobytes()
            cen = np.zeros((max(int(c[2]), 1), 4), np.float32)
            dep = np.zeros(max(int(c[2]), 1), np.uint8)
            lib().octo_tree_leaves(handle, cen.ctypes.data, dep.ctypes.data)
            self.centres, self.depths = cen[:int(c[2])], dep[:int(c[2])]
            self._h = handle
        except Exception:
            lib().octo_tree_destroy(handle)
            raise

    def write(self, path):
        """octomap's writeBinary: the .bt file."""
        if lib().octo_tree_write(self._h, os.fsencode(path)) != 0:
            raise OSError(f"cannot write {path}")

    def close(self):
        if self._h:
            lib().octo_tree_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def octree(keys, log_odds, resolution, occupancy_threshold=OCCUPANCY_THRESHOLD):
    """The pruned octree of the known voxels (packed keys, float32 log-odds) at `resolution`."""
    k = np.ascontiguousarray(keys, np.uint64)
    v = np.ascontiguousarray(log_odds, np.float32)
    return Octree(lib().octo_tree_from_voxels(k.ctypes.data, v.ctypes.data, len(k), float(resolution),
                                              float(occupancy.logodds(occupancy_threshold))))


def of_map(occupancy_map):
    """The pruned octree of an oracle.occupancy.OccupancyMap's known voxels."""
    p = occupancy_map.params
    return octree(*occupancy_map.download(), p["resolution"], p["occupancy_threshold"])
