"""ORACLE -- test infrastructure only.  numpy restatement of the per-scan input filters: the DataPointsFilters chain
LaserTrackParams::icp_input_filters_file names (reference laser_slam/src/laser_track.cpp:24-30, applied at :81 and :146).
The device path (ls_filter_cloud / ls_map_push_scan_filtered, include/ls_b200.h) is checked against it bit for bit;
the rules marked [DEFINED] are listed in oracle/INPUT_FILTERS.md.  Used by tests/test_input_filters.py and, for the CPU time
of the same chain, by bench_input_filters.py."""
import numpy as np

from . import keep_mask, knn_normals, voxel_grid


def _voxel_grid_with_normals(pts4, nrm3, leaf_size):
    """voxel_grid, plus the normals of each voxel averaged the same exact way (fixed point 2^-24, one rounding)
    [DEFINED]: not renormalised."""
    p = np.asarray(pts4, np.float32)
    leaf = np.broadcast_to(np.asarray(leaf_size, np.float32), (3,))
    inv = (np.float32(1.0) / leaf).astype(np.float32)
    ok = np.isfinite(p[:, :3]).all(1)
    q, qn = p[ok], np.asarray(nrm3, np.float32)[ok]
    if len(q) == 0:
        return np.zeros((0, 4), np.float32), np.zeros((0, 3), np.float32)
    ijk = np.floor(q[:, :3] * inv[None, :]).astype(np.int64)
    mn = ijk.min(0)
    dim = ijk.max(0) - mn + 1
    key = (ijk[:, 0] - mn[0]) + (ijk[:, 1] - mn[1]) * dim[0] + (ijk[:, 2] - mn[2]) * dim[0] * dim[1]
    order = np.argsort(key, kind="stable")
    ks = key[order]
    heads = np.flatnonzero(np.concatenate([[True], ks[1:] != ks[:-1]]))
    cnt = np.diff(np.concatenate([heads, [len(ks)]])).astype(np.float64)[:, None] * 16777216.0
    sums = np.add.reduceat(np.rint(qn[order].astype(np.float64) * 16777216.0).astype(np.int64), heads, axis=0)
    return voxel_grid(p, leaf_size), (sums.astype(np.float64) / cnt).astype(np.float32)


_FILTER_DEFAULTS = {
    # libpointmatcher's defaults, except knn / prob / ratio: the values the compat DataPointsFilters reader always used
    "RemoveNaNDataPointsFilter": {},
    "MaxDistDataPointsFilter": {"dim": -1, "maxDist": 1.0},
    "MinDistDataPointsFilter": {"dim": -1, "minDist": 1.0},
    "BoundingBoxDataPointsFilter": {"xMin": -1.0, "xMax": 1.0, "yMin": -1.0, "yMax": 1.0, "zMin": -1.0, "zMax": 1.0,
                                    "removeInside": 1},
    "RandomSamplingDataPointsFilter": {"prob": 1.0},
    "FixStepSamplingDataPointsFilter": {"startStep": 10, "stepMult": 1},
    "VoxelGridDataPointsFilter": {"vSizeX": 1.0, "vSizeY": 1.0, "vSizeZ": 1.0, "useCentroid": 1},
    "SurfaceNormalDataPointsFilter": {"knn": 10},
    "SamplingSurfaceNormalDataPointsFilter": {"knn": 10, "ratio": 1.0},
}


def apply_filters(filters, pts4, nrm3=None, num_threads=1):
    """The per-scan input filters (reference laser_slam/src/laser_track.cpp:24-30,81,146): `filters` is a list of
    (YAML filter name, {key: value}) applied in order; each sees the cloud the previous one produced, every compaction
    keeps the input order, normals (if any) travel with their points.  Returns (points (m,4), normals (m,3) or None).

      RemoveNaN            drop a point if x, y or z is NaN (+-inf is left to the distance filters)
      MaxDist / MinDist    [DEFINED] dim -1: fl(fl(fl(x*x) + fl(y*y)) + fl(z*z)) < (>) fl(d*d) in float32; dim 0/1/2:
                           |coord| < (>) d; strict
      BoundingBox          [DEFINED] inside iff min < c < max on all three axes (a point on a face is outside); keeps the
                           outside points (removeInside 1) or the inside ones (0)
      RandomSampling       keep_mask(., 0x7e11, prob) over the index in the cloud ENTERING the filter
      FixStepSampling      keep iff i % startStep == 0 (endStep != startStep / stepMult != 1 are stateful: refused)
      VoxelGrid            voxel_grid (useCentroid 1 only); normals averaged the same exact way, not renormalised [DEFINED]
      (Sampling)SurfaceNormal  knn_normals with knn clamped to [3, 16]; the Sampling variant then keep_mask(., 0x5a17, ratio)
    """
    p = np.ascontiguousarray(pts4, np.float32)
    nr = None if nrm3 is None else np.ascontiguousarray(nrm3, np.float32)
    for name, kw in filters:
        if name not in _FILTER_DEFAULTS:
            raise ValueError(f"{name} is not an input filter of this path")
        a = dict(_FILTER_DEFAULTS[name], **kw)
        keep = None
        x, y, z = p[:, 0], p[:, 1], p[:, 2]
        if name == "RemoveNaNDataPointsFilter":
            keep = ~(np.isnan(x) | np.isnan(y) | np.isnan(z))
        elif name in ("MaxDistDataPointsFilter", "MinDistDataPointsFilter"):
            d = np.float32(a["maxDist" if name.startswith("Max") else "minDist"])
            dim = int(a["dim"])
            with np.errstate(over="ignore", invalid="ignore"):
                if dim < 0:
                    v = (x * x + y * y).astype(np.float32) + (z * z).astype(np.float32)
                    lim = np.float32(d * d)
                else:
                    v = np.abs(p[:, dim])
                    lim = d
                keep = v < lim if name.startswith("Max") else v > lim
        elif name == "BoundingBoxDataPointsFilter":
            b = [np.float32(a[k]) for k in ("xMin", "xMax", "yMin", "yMax", "zMin", "zMax")]
            with np.errstate(invalid="ignore"):
                inside = (b[0] < x) & (x < b[1]) & (b[2] < y) & (y < b[3]) & (b[4] < z) & (z < b[5])
            keep = ~inside if int(a["removeInside"]) else inside
        elif name == "RandomSamplingDataPointsFilter":
            keep = keep_mask(len(p), 0x7e11, float(np.float32(a["prob"])))
        elif name == "FixStepSamplingDataPointsFilter":
            step = int(a["startStep"])
            if int(a.get("endStep", step)) != step or float(a["stepMult"]) != 1.0:
                raise ValueError("FixStepSampling with a changing step is stateful")
            keep = np.arange(len(p)) % step == 0
        elif name == "VoxelGridDataPointsFilter":
            if int(a["useCentroid"]) != 1:
                raise ValueError("VoxelGrid: only useCentroid 1")
            leaf = [a["vSizeX"], a["vSizeY"], a["vSizeZ"]]
            if nr is None:
                p = voxel_grid(p, leaf)
            else:
                p, nr = _voxel_grid_with_normals(p, nr, leaf)
            continue
        else:
            k = max(3, min(16, int(a["knn"])))
            nr = knn_normals(p, k, num_threads=num_threads) if len(p) else np.zeros((0, 3), np.float32)
            if name.startswith("Sampling"):
                keep = keep_mask(len(p), 0x5a17, float(np.float32(a["ratio"])))
        if keep is not None:
            p = np.ascontiguousarray(p[keep])
            nr = None if nr is None else np.ascontiguousarray(nr[keep])
    return p, nr


def filters_yaml(filters):
    """The YAML list (libpointmatcher DataPointsFilters file) of a `filters` list as apply_filters takes it."""
    lines = []
    for name, kw in filters:
        lines.append(f"- {name}" + (":" if kw else ""))
        lines += [f"    {k}: {v!r}" for k, v in kw.items()]
    return "\n".join(lines) + "\n"
