"""Octree export of the resident occupancy map (ls_occupancy_build_octree / _write_octomap): after --scans full synthetic
HDL-64 scans (131072 points) inserted at laser_to_octomap's defaults (0.075 m voxels, 20 m range), the median ms of
OccupancyMap.octree() (build on the device, then download of the payload and the occupied leaves) and of save_octomap()
(download and .bt file write of the current tree), host clock around the synchronous calls, plus the build's device ms.
The oracle's CPU time for the same export is octomap's structure restated (pointer tree, prune, writeBinary, leaf
iteration) built from the device map's known voxels; parity (the .bt files byte for byte, the leaves bit for bit) is
checked outside the clock.  Prints one JSON line.

    python bench_octomap.py [--scans 105] [--repeats 20] [--resolution 0.075] [--max-range 20]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_occupancy import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=105)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--resolution", type=float, default=0.075)
    ap.add_argument("--max-range", type=float, default=20.0)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    from oracle import octree as oc
    synth.build()
    oc.build()
    truth, _ = synth.trajectory(0, a.scans)
    params = dict(resolution=a.resolution, max_range=a.max_range)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, 131072)
    om = ls.OccupancyMap(ctx, **params)
    zeros = np.zeros((131072, 3), np.float32)
    for k in range(a.scans):
        om.insert_scan(ring, ring.push_scan(synth.scan(truth[k], 0, k)[0], zeros), truth[k].astype(np.float32))
    with tempfile.TemporaryDirectory() as tmp:
        bt = os.path.join(tmp, "map.bt")
        t_exp, t_dev, t_write = [], [], []
        for r in range(a.repeats + 2):  # two warm-up rounds
            t0 = time.perf_counter()
            tree = om.octree()
            t1 = time.perf_counter()
            om.save_octomap(bt)
            t2 = time.perf_counter()
            if r >= 2:
                t_exp.append(t1 - t0)
                t_dev.append(tree.device_ms * 1e-3)
                t_write.append(t2 - t1)
        keys, lo, _ = om.download(ls.OCC_KNOWN)
        t0 = time.perf_counter()
        ot = oc.octree(keys, lo, a.resolution)
        t_oracle = time.perf_counter() - t0
        obt = os.path.join(tmp, "oracle.bt")
        ot.write(obt)
        parity = (open(bt, "rb").read() == open(obt, "rb").read() and tree.payload == ot.payload and
                  np.array_equal(tree.centres.view(np.uint32), ot.centres.view(np.uint32)) and
                  np.array_equal(tree.depths, ot.depths))
    ms = lambda v: round(float(np.median(v)) * 1e3, 3)  # noqa: E731
    result = dict(bench="octomap", gpu=name, power_limit=limit, scans=a.scans, repeats=a.repeats, params=params,
                  known_voxels=len(keys), occupied_voxels=om.size(ls.OCC_OCCUPIED), nodes=tree.nodes,
                  payload_bytes=len(tree.payload), occupied_leaves=len(tree.depths), gpu_ms_export=ms(t_exp),
                  gpu_device_ms_export=ms(t_dev), gpu_ms_write_bt=ms(t_write), oracle_cpu_ms_export=round(t_oracle * 1e3, 1),
                  parity=parity)
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if not parity:
        sys.exit("octree export differs from the oracle")


if __name__ == "__main__":
    main()
