"""Reference of the full tree (.ot) export and read (test infrastructure only).  full_octree() binds
tests/ref/octree_full_oracle.cpp, octomap's OcTree::write restated from the known voxels (value pruning,
updateInnerOccupancy, writeData).  expand() turns a file parsed by laser_slam_b200.read_octomap_full into the voxels a read
makes known, in numpy: every voxel below a leaf with the leaf's log-odds.  An insert after a read has its reference in
octomap_read_ref.seed."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "ref", "_build", "libls_octree_full_oracle.so")
_SRC = os.path.join(_HERE, "ref", "octree_full_oracle.cpp")
_lib = None


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
        L.octo_full_from_voxels.argtypes = [vp, vp, i64, ctypes.c_double]
        L.octo_full_from_voxels.restype = vp
        L.octo_full_destroy.argtypes = [vp]
        L.octo_full_destroy.restype = None
        for f in (L.octo_full_counts, L.octo_full_payload):
            f.argtypes = [vp, vp]
            f.restype = None
        L.octo_full_write.argtypes = [vp, ctypes.c_char_p]
        _lib = L
    return _lib


class FullOctree:
    """The full tree: nodes (octomap's size()), leaves and payload (the writeData bytes)."""

    def __init__(self, handle):
        try:
            c = np.zeros(3, np.int64)
            lib().octo_full_counts(handle, c.ctypes.data)
            self.nodes, self.leaves = int(c[0]), int(c[1])
            pay = np.zeros(max(int(c[2]), 1), np.uint8)
            lib().octo_full_payload(handle, pay.ctypes.data)
            self.payload = pay[:int(c[2])].tobytes()
            self._h = handle
        except Exception:
            lib().octo_full_destroy(handle)
            raise

    def write(self, path):
        """octomap's OcTree::write: the .ot file."""
        if lib().octo_full_write(self._h, os.fsencode(path)) != 0:
            raise OSError(f"cannot write {path}")

    def close(self):
        if self._h:
            lib().octo_full_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def full_octree(keys, log_odds, resolution):
    """The full tree of the known voxels (packed keys, float32 log-odds) at `resolution`."""
    k = np.ascontiguousarray(keys, np.uint64)
    v = np.ascontiguousarray(log_odds, np.float32)
    assert len(k) == len(v)
    return FullOctree(lib().octo_full_from_voxels(k.ctypes.data, v.ctypes.data, len(k), float(resolution)))


def of_map(occupancy_map):
    """The full tree of an oracle.occupancy.OccupancyMap's known voxels."""
    return full_octree(*occupancy_map.download(), occupancy_map.params["resolution"])


def expand(parsed):
    """The voxels a read of `parsed` (laser_slam_b200.read_octomap_full's dict) makes known: (packed keys uint64
    ascending, log-odds float32)."""
    keys3, depths, values = parsed["keys"], parsed["depths"], parsed["values"]
    out_k, out_v = [np.zeros(0, np.uint64)], [np.zeros(0, np.float32)]
    for d in np.unique(depths):
        sel = depths == d
        n = 1 << (16 - int(d))
        off = np.stack(np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 3)
        k = (keys3[sel][:, None, :] + off[None]).reshape(-1, 3).astype(np.uint64)
        out_k.append(k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32)))
        out_v.append(np.repeat(values[sel].astype(np.float32), n ** 3))
    k, v = np.concatenate(out_k), np.concatenate(out_v)
    order = np.argsort(k, kind="stable")
    return k[order], v[order]
