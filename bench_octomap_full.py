"""The occupancy map as octomap's full tree (.ot): after --scans full synthetic HDL-64 scans (131072 points) inserted at
laser_to_octomap's defaults (0.075 m voxels, 20 m range), the full tree is built (ls_occupancy_build_full_octree),
downloaded (_download_full_octree), saved (save_octomap_full, with the build current: download and file write) and read
back into a second map (read_octomap_full: file read, header parse, upload, device parse and expansion).  Median ms per
step, host clock around the synchronous call, plus the device ms the build and the read report.  The oracle's CPU time is
tests/octomap_full_ref.py's full_octree of the same voxels.  Parity (the device payload against the oracle's, the loaded
map's known keys and log-odds bit for bit, and the written-back file byte for byte) is checked outside the clock.  Prints
one JSON line.

    python bench_octomap_full.py [--scans 105] [--repeats 10] [--resolution 0.075] [--max-range 20]
"""
import argparse
import ctypes
import json
import os
import sys
import tempfile
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
    ap.add_argument("--resolution", type=float, default=0.075)
    ap.add_argument("--max-range", type=float, default=20.0)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    import octomap_full_ref as fr
    synth.build()
    truth, _ = synth.trajectory(0, a.scans)
    params = dict(resolution=a.resolution, max_range=a.max_range)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, 131072)
    om = ls.OccupancyMap(ctx, **params)
    zeros = np.zeros((131072, 3), np.float32)
    for k in range(a.scans):
        om.insert_scan(ring, ring.push_scan(synth.scan(truth[k], 0, k)[0], zeros), truth[k].astype(np.float32))
    L = ls.lib()
    st = ls.FullOctreeStats()
    loaded = ls.OccupancyMap(ctx, **params)
    t = {k: [] for k in ("build", "build_dev", "download", "save", "read", "read_dev")}
    with tempfile.TemporaryDirectory() as tmp:
        ot, back = os.path.join(tmp, "map.ot"), os.path.join(tmp, "back.ot")
        for r in range(a.repeats + 2):  # two warm-up rounds
            t0 = time.perf_counter()
            ctx._check(L.ls_occupancy_build_full_octree(om._h, ctypes.byref(st)))
            t1 = time.perf_counter()
            pay = np.empty(st.payload_bytes, np.uint8)
            t2 = time.perf_counter()
            ctx._check(L.ls_occupancy_download_full_octree(om._h, pay.ctypes.data, st.payload_bytes))
            t3 = time.perf_counter()
            om.save_octomap_full(ot)
            t4 = time.perf_counter()
            rst = loaded.read_octomap_full(ot)
            t5 = time.perf_counter()
            if r >= 2:
                t["build"].append(t1 - t0)
                t["build_dev"].append(st.device_ms * 1e-3)
                t["download"].append(t3 - t2)
                t["save"].append(t4 - t3)
                t["read"].append(t5 - t4)
                t["read_dev"].append(rst.device_ms * 1e-3)
        keys, lo, _ = om.download(ls.OCC_KNOWN)
        t0 = time.perf_counter()
        oracle = fr.full_octree(keys, lo, a.resolution)
        t_oracle = time.perf_counter() - t0
        k, v, _ = loaded.download(ls.OCC_KNOWN)
        loaded.save_octomap_full(back)
        parity = (pay.tobytes() == oracle.payload and st.nodes == oracle.nodes and np.array_equal(k, keys) and
                  np.array_equal(v.view(np.uint32), lo.view(np.uint32)) and open(ot, "rb").read() == open(back, "rb").read())
    ms = lambda x: round(float(np.median(x)) * 1e3, 3)  # noqa: E731
    result = dict(bench="octomap_full", gpu=name, power_limit=limit, scans=a.scans, repeats=a.repeats, params=params,
                  nodes=st.nodes, leaves=st.leaves, payload_bytes=st.payload_bytes, known_voxels=rst.known_voxels,
                  bricks=rst.bricks, gpu_ms_build=ms(t["build"]), gpu_device_ms_build=ms(t["build_dev"]),
                  gpu_ms_download=ms(t["download"]), gpu_ms_save=ms(t["save"]), gpu_ms_read=ms(t["read"]),
                  gpu_device_ms_read=ms(t["read_dev"]), oracle_cpu_ms_build=round(t_oracle * 1e3, 1), parity=parity)
    loaded.close()
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if not parity:
        sys.exit("full octree differs from the oracle")


if __name__ == "__main__":
    main()
