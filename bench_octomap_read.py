"""Reading a .bt file into the resident occupancy map (ls_occupancy_read_octomap): after --scans full synthetic HDL-64
scans (131072 points) inserted at laser_to_octomap's defaults (0.075 m voxels, 20 m range), the map is saved and read
back into a second map.  Median ms of the read, host clock around the synchronous call (file read, header parse, upload,
device parse and expansion), plus its device ms.  The oracle's CPU time for the same read is the CPU parser
(laser_slam_b200.read_octomap) and the numpy expansion of tests/octomap_read_ref.py.  Parity (the loaded map's known keys
and log-odds against the oracle, and the written-back file byte for byte) is checked outside the clock.  Prints one JSON
line.

    python bench_octomap_read.py [--scans 105] [--repeats 10] [--resolution 0.075] [--max-range 20]
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
    import octomap_read_ref as rr
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
    loaded = ls.OccupancyMap(ctx, **params)
    with tempfile.TemporaryDirectory() as tmp:
        bt, back = os.path.join(tmp, "map.bt"), os.path.join(tmp, "back.bt")
        nodes = om.save_octomap(bt)
        t_read, t_dev = [], []
        for r in range(a.repeats + 2):  # two warm-up rounds
            t0 = time.perf_counter()
            st = loaded.read_octomap(bt)
            t1 = time.perf_counter()
            if r >= 2:
                t_read.append(t1 - t0)
                t_dev.append(st.device_ms * 1e-3)
        t0 = time.perf_counter()
        parsed = ls.read_octomap(bt)
        keys, lo = rr.expand(parsed, *rr.clamps())
        t_oracle = time.perf_counter() - t0
        k, v, _ = loaded.download(ls.OCC_KNOWN)
        loaded.save_octomap(back)
        parity = (np.array_equal(k, keys) and np.array_equal(v.view(np.uint32), lo.view(np.uint32)) and
                  open(bt, "rb").read() == open(back, "rb").read())
        payload_bytes = len(parsed["payload"])
    ms = lambda x: round(float(np.median(x)) * 1e3, 3)  # noqa: E731
    result = dict(bench="octomap_read", gpu=name, power_limit=limit, scans=a.scans, repeats=a.repeats, params=params,
                  nodes=nodes, payload_bytes=payload_bytes, inner_nodes=st.inner_nodes, known_voxels=st.known_voxels,
                  bricks=st.bricks, gpu_ms_read=ms(t_read), gpu_device_ms_read=ms(t_dev),
                  oracle_cpu_ms_read=round(t_oracle * 1e3, 1), parity=parity)
    loaded.close()
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if not parity:
        sys.exit("octomap read differs from the oracle")


if __name__ == "__main__":
    main()
