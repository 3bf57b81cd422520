"""Leaf boxes and marker cubes of the resident occupancy map (ls_occupancy_build_leaves / _download_leaves /
_marker_cubes): --scans full synthetic HDL-64 scans (131072 points) inserted at laser_to_octomap's defaults (0.075 m
voxels, 20 m range), then three workloads, each a synchronous Python call timed on the host clock (median of --repeats
after 2 warm-ups): leaf_boxes of every leaf of the whole map, leaf_boxes of a 20 m box around the last pose, and
marker_cubes over the whole map.  The .ot build is cached, so the timed calls measure the listing and its copies; the .ot
build's own device time (its second build, after its buffers exist) is reported beside them.  The reference walk of the
.ot payload (tests/leaf_boxes_ref.py) is timed once on one CPU thread, and the whole-map listing is checked against it
outside the clock.  Prints one JSON line with the GPU's name and power limit.

    python bench_occupancy_leaves.py [--scans 105] [--repeats 10]
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
    import leaf_boxes_ref as lr
    from oracle import occupancy as oc
    synth.build()
    truth, _ = synth.trajectory(0, a.scans)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, 131072)
    om = ls.OccupancyMap(ctx)
    zeros = np.zeros((131072, 3), np.float32)
    for k in range(a.scans):
        om.insert_scan(ring, ring.push_scan(synth.scan(truth[k], 0, k)[0], zeros), truth[k].astype(np.float32))
    om.full_octree()  # the first build allocates the tree's buffers; the second is timed
    ft = om.full_octree()
    last = np.asarray(truth[-1])[:3, 3].astype(np.float64)
    region = (last - 10.0, last + 10.0)
    workloads = {"leaf_boxes_whole_map": lambda: om.leaf_boxes(ls.LEAVES_ALL),
                 "leaf_boxes_20m_box": lambda: om.leaf_boxes(ls.LEAVES_ALL, region),
                 "marker_cubes": lambda: om.marker_cubes(-1.0, 3.0, 0.8)}
    out = {}
    for wname, call in workloads.items():
        host, dev = [], []
        for r in range(a.repeats + 2):
            t0 = time.perf_counter()
            got = call()
            t1 = time.perf_counter()
            if r >= 2:
                host.append(t1 - t0)
                dev.append(om.last_leaves.device_ms)
        st = om.last_leaves
        out[wname] = dict(host_ms=round(float(np.median(host)) * 1e3, 3), device_ms=round(float(np.median(dev)), 3),
                          free_leaves=st.free_leaves, occupied_leaves=st.occupied_leaves)
    boxes = om.leaf_boxes(ls.LEAVES_ALL)
    t0 = time.perf_counter()
    keys, depths, values = lr.walk(ft.payload)
    ref_s = time.perf_counter() - t0
    l_occ = oc.logodds(0.7)
    states = np.where(values >= np.float32(l_occ), lr.CELL_OCCUPIED, lr.CELL_FREE)
    centres = ls.leaf_centres(keys, depths, om.params.resolution)
    parity = bool(np.array_equal(boxes.depths, depths) and np.array_equal(boxes.states, states) and
                  np.array_equal(boxes.centres.view(np.uint32), centres.view(np.uint32)))
    result = dict(bench="occupancy_leaves", gpu=name, power_limit=limit, scans=a.scans, resolution=om.params.resolution,
                  known_voxels=om.size(ls.OCC_KNOWN), ot_nodes=ft.nodes, ot_build_device_ms=round(ft.device_ms, 3),
                  leaves=len(depths), workloads=out, reference_walk_s=round(ref_s, 3), parity=parity)
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if not parity:
        sys.exit("the leaf list differs from the reference walk")


if __name__ == "__main__":
    main()
