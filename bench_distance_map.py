"""Euclidean distance map of the resident occupancy map (ls_distance_map_*, octomap's DynamicEDTOctomap): after --scans full
synthetic HDL-64 scans (131072 points) inserted at laser_to_octomap's defaults (0.075 m voxels, 20 m range), one update of
a 20 m and a 40 m cube around the mid-trajectory pose and of the map's bounds(), with max_dist 2 m, in both modes
(occupied voxels only, and unknown cells as obstacles too).  Median ms over --repeats updates after two warm-up updates,
host clock around the synchronous call, and the median of the update's device ms; then one query of --points points in
the 40 m cube.  The reference of tests/distance_map_ref.py (tests/ref/edt_ref.cpp, one CPU thread) runs the same updates
outside the clock, and the downloaded fields are compared with it byte for byte.  The bytes the passes move follow the
model of DESIGN.md §4b''''''''' (bytes_per_cell below); GB/s is that over the device ms.  Prints one JSON line.

    python bench_distance_map.py [--scans 105] [--repeats 10] [--points 1000000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "tests"))

from bench_occupancy import gpu_info  # noqa: E402

# Bytes per cell every update must move: the grid's memset (1), the x pass (the grid read twice, the left site written and
# read, the value and site written: 2 + 4 + 4 + 8), and each of the y and z passes (the value read, the site read through
# the stack, the value and site written: 4 + 4 + 8).  Left out: the stack, whose traffic depends on the sites per column
# (at most 8 bytes written and 8 read per cell and pass), and the extraction's reads of the map, which scale with the
# known voxels.  GB/s over this count is a floor on what the kernels move.
BYTES_PER_CELL = 1 + (2 + 4 + 4 + 8) + 2 * (4 + 4 + 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=105)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--max-dist", type=float, default=2.0)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    import distance_map_ref as dr
    from oracle import occupancy as oc
    synth.build()
    dr.build()
    truth, _ = synth.trajectory(0, a.scans)
    res = 0.075
    l_occ = oc.logodds(0.7)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, 131072)
    om = ls.OccupancyMap(ctx)
    zeros = np.zeros((131072, 3), np.float32)
    for k in range(a.scans):
        om.insert_scan(ring, ring.push_scan(synth.scan(truth[k], 0, k)[0], zeros), truth[k].astype(np.float32))
    keys, vals, _ = om.download(ls.OCC_KNOWN)
    p = truth[a.scans // 2][:3, 3].astype(np.float64)
    blo, bhi = om.bounds()
    med = lambda x: round(float(np.median(x)), 3)  # noqa: E731
    result = dict(bench="distance_map", gpu=name, power_limit=limit, scans=a.scans, repeats=a.repeats, resolution=res,
                  max_dist=a.max_dist, known_voxels=len(keys), bounds=[blo.tolist(), bhi.tolist()],
                  bytes_per_cell=BYTES_PER_CELL, updates=[])
    parity = True
    boxes = {"cube_20m": (p - 10.0, p + 10.0), "cube_40m": (p - 20.0, p + 20.0), "bounds": (blo, bhi - res / 2)}
    for box, (lo, hi) in boxes.items():
        size = dr.box(lo, hi, res)[1]
        if int(np.prod(size.astype(np.int64))) > 1 << 30:  # the update refuses it
            result["updates"].append(dict(box=box, size=size.tolist(), refused="more than 2^30 cells"))
            continue
        for unknown in (False, True):
            dm = ls.DistanceMap(ctx, a.max_dist, lo, hi, unknown)
            host, dev = [], []
            for r in range(a.repeats + 2):
                t0 = time.perf_counter()
                st = dm.update(om)
                t1 = time.perf_counter()
                if r >= 2:
                    host.append((t1 - t0) * 1e3)
                    dev.append(st.device_ms)
            t0 = time.perf_counter()
            f = dr.Field(keys, vals, res, l_occ, a.max_dist, lo, hi, unknown)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            s, k = dm.download()
            same = s.tobytes() == f.s.tobytes() and k.tobytes() == f.keys().tobytes()
            parity &= same
            moved = BYTES_PER_CELL * st.cells
            result["updates"].append(dict(box=box, unknown_as_occupied=unknown, size=list(st.size), cells=st.cells,
                                          obstacles=st.obstacles, device_bytes=st.device_bytes, gpu_ms=med(host),
                                          device_ms=med(dev), gb_per_s=round(moved / (med(dev) * 1e-3) / 1e9, 1),
                                          cpu_reference_ms=round(cpu_ms, 1), parity=same))
            if box == "cube_40m" and not unknown:
                pts = np.random.default_rng(0).uniform(lo, hi, (a.points, 3)).astype(np.float32)
                qh, qd = [], []
                for r in range(a.repeats + 2):
                    t0 = time.perf_counter()
                    got = dm.query(pts)
                    t1 = time.perf_counter()
                    if r >= 2:
                        qh.append((t1 - t0) * 1e3)
                        qd.append(dm.last_query.device_ms)
                want = f.query(pts)
                qsame = all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(got, want))
                parity &= qsame
                result["query"] = dict(points=a.points, gpu_ms=med(qh), device_ms=med(qd), parity=qsame)
            dm.close()
            del f, s, k
    result["parity"] = bool(parity)
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if not parity:
        sys.exit("the distance map differs from the reference")


if __name__ == "__main__":
    main()
