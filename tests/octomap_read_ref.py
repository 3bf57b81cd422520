"""Reference of the .bt read (test infrastructure only): octomap's readBinary restated on the CPU.  The file is parsed by
laser_slam_b200.read_octomap (the CPU parser octomap_to_point_cloud uses) and its leaves are expanded here, in numpy,
into the voxels the read makes known: every voxel below a free leaf with L_min, below an occupied leaf with L_max.
seed() fills an oracle.occupancy.OccupancyMap with given voxels, so an insert after a read has a reference."""
import ctypes
import os
import subprocess

import numpy as np

from oracle import occupancy

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "ref", "_build", "libls_occupancy_seed.so")
_SRCS = [os.path.join(_HERE, "ref", "occupancy_seed.cpp"), occupancy._SRC]
_lib = None


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
        L.occo_seed.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
        L.occo_seed.restype = None
        _lib = L
    return _lib


def clamps(clamp_min=occupancy.DEFAULTS["clamp_min"], clamp_max=occupancy.DEFAULTS["clamp_max"]):
    """(L_min, L_max): the float log-odds of the clamping probabilities, as the map computes them."""
    return occupancy.logodds(clamp_min), occupancy.logodds(clamp_max)


def expand(parsed, l_min, l_max):
    """The voxels a read of `parsed` (laser_slam_b200.read_octomap's dict) makes known: (packed keys uint64 ascending,
    log-odds float32)."""
    keys3, depths, states = parsed["keys"], parsed["depths"], parsed["states"]
    out_k, out_v = [np.zeros(0, np.uint64)], [np.zeros(0, np.float32)]
    for d in np.unique(depths):
        sel = depths == d
        n = 1 << (16 - int(d))
        off = np.stack(np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 3)
        k = (keys3[sel][:, None, :] + off[None]).reshape(-1, 3).astype(np.uint64)
        out_k.append(k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32)))
        out_v.append(np.repeat(np.where(states[sel] == 2, np.float32(l_max), np.float32(l_min)).astype(np.float32), n ** 3))
    k, v = np.concatenate(out_k), np.concatenate(out_v)
    order = np.argsort(k, kind="stable")
    return k[order], v[order]


def seed(oracle_map, keys, log_odds):
    """Replace an oracle.occupancy.OccupancyMap's known voxels by (strictly ascending packed keys, float32 log-odds)."""
    k = np.ascontiguousarray(keys, np.uint64)
    v = np.ascontiguousarray(log_odds, np.float32)
    assert len(k) == len(v) and (len(k) < 2 or (np.diff(k.astype(np.int64)) > 0).all())
    lib().occo_seed(oracle_map._h, k.ctypes.data, v.ctypes.data, len(k))
    return oracle_map
