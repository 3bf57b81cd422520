"""The 2D projection of the resident occupancy map (ls_occupancy_build_projection / _download_projection): octomap_server's
projected_map.  --scans full synthetic HDL-64 scans (131072 points) inserted at laser_to_octomap's defaults (0.075 m voxels,
20 m range), then four workloads, each a synchronous Python call of projected_map (build and download) timed on the host
clock, median of --repeats after 2 warm-ups: the whole map and a 0.3 ... 2.0 m band, each with the .bt build cached and with
it not cached (before each of those calls, setOccupied rewrites one voxel 5 m above the map, which invalidates the cached
builds; it is set once before any timing, so every call projects the same map).  The device ms of each call (the .bt build it needed included) is reported beside them, and the
restatement (tests/projected_map_ref.py) is timed once per workload on one CPU thread, projecting the .bt payload's leaves
(walked before its clock), and checked against the device grid.  Prints one JSON line with the GPU's name and power limit.

    python bench_occupancy_projection.py [--scans 105] [--repeats 10]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=105)
    ap.add_argument("--repeats", type=int, default=10)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    import projected_map_ref as pr
    synth.build()
    truth, _ = synth.trajectory(0, a.scans)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, 131072)
    om = ls.OccupancyMap(ctx)
    zeros = np.zeros((131072, 3), np.float32)
    for k in range(a.scans):
        om.insert_scan(ring, ring.push_scan(synth.scan(truth[k], 0, k)[0], zeros), truth[k].astype(np.float32))
    t = om.octree()
    res = om.params.resolution
    band = dict(min_z=0.3, max_z=2.0)
    lo, hi = om.bounds()
    above = [float((lo[0] + hi[0]) / 2), float((lo[1] + hi[1]) / 2), float(hi[2] + 5.0)]
    om.set_occupied([above], [[res / 2, res / 2, res / 2]])
    t = om.octree()

    def stale():
        om.set_occupied([above], [[res / 2, res / 2, res / 2]])

    workloads = {"whole_map_cached": (dict(), None), "band_0.3_2.0_cached": (band, None),
                 "whole_map_not_cached": (dict(), stale), "band_0.3_2.0_not_cached": (band, stale)}
    out = {}
    for wname, (kw, before) in workloads.items():
        host, dev = [], []
        for r in range(a.repeats + 2):
            if before:
                before()
            t0 = time.perf_counter()
            grid, info = om.projected_map(**kw)
            t1 = time.perf_counter()
            if r >= 2:
                host.append(t1 - t0)
                dev.append(info.device_ms)
        out[wname] = dict(host_ms=round(float(np.median(host)) * 1e3, 3), device_ms=round(float(np.median(dev)), 3),
                          width=info.width, height=info.height, free_cells=info.free_cells,
                          occupied_cells=info.occupied_cells)
    leaves = pr.bt_leaves(t.payload)
    parity = True
    ref_s = {}
    for wname, kw in (("whole_map", dict()), ("band_0.3_2.0", band)):
        t0 = time.perf_counter()
        want = pr.project(leaves, res, **kw)[0]
        ref_s[wname] = round(time.perf_counter() - t0, 3)
        parity = parity and bool(np.array_equal(om.projected_map(**kw)[0], want))
    result = dict(bench="occupancy_projection", gpu=name, power_limit=limit, scans=a.scans, resolution=res,
                  known_voxels=om.size(ls.OCC_KNOWN), bt_nodes=t.nodes, bt_leaves=len(leaves[1]), workloads=out,
                  reference_s=ref_s, parity=parity)
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if not parity:
        sys.exit("the projection differs from the restatement")


if __name__ == "__main__":
    main()
