"""Resident occupancy map (ls_occupancy_*, laser_to_octomap's insertion loop): ms per insert_scan of full synthetic HDL-64
scans (131072 points) at laser_to_octomap's defaults (0.075 m voxels, 20 m range), after warm-up.  Host clock around the
synchronous call; voxel updates per second from the call's counters; map size and device memory at the end.  The oracle's
ms per scan on one CPU thread over the first --oracle-scans scans is the reference figure, and the device map after those
scans is checked against the oracle's bit for bit, outside the clock.  Prints one JSON line.

    python bench_occupancy.py [--scans 100] [--warmup 5] [--oracle-scans 10] [--resolution 0.075] [--max-range 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, limit = [x.strip() for x in out[0].split(",")]
        return name, limit
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "not measured"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--oracle-scans", type=int, default=10)
    ap.add_argument("--resolution", type=float, default=0.075)
    ap.add_argument("--max-range", type=float, default=20.0)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    from oracle import occupancy as oc
    synth.build()
    oc.build()
    total = a.warmup + a.scans
    truth, _ = synth.trajectory(0, total)
    params = dict(resolution=a.resolution, max_range=a.max_range)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, 131072)
    om = ls.OccupancyMap(ctx, **params)
    o = oc.OccupancyMap(**params)
    zeros = np.zeros((131072, 3), np.float32)
    t_ins, t_dev, updates, t_oracle = [], [], [], []
    parity = None
    for k in range(total):
        scan = synth.scan(truth[k], 0, k)[0]
        T = truth[k].astype(np.float32)
        sid = ring.push_scan(scan, zeros)
        ring.sync()
        t0 = time.perf_counter()
        st = om.insert_scan(ring, sid, T)
        t1 = time.perf_counter()
        if k >= a.warmup:
            t_ins.append(t1 - t0)
            t_dev.append(st.device_ms * 1e-3)
            updates.append(st.free_updates + st.occupied_updates)
        if k < a.oracle_scans:
            t0 = time.perf_counter()
            o.insert_scan(scan, T)
            t_oracle.append(time.perf_counter() - t0)
            if k == a.oracle_scans - 1:  # outside the clock
                same = lambda x, y: np.array_equal(x[0], y[0]) and np.array_equal(x[1].view(np.uint32), y[1].view(np.uint32))
                parity = (same(om.download(ls.OCC_KNOWN)[:2], o.download(oc.KNOWN)) and
                          same(om.download(ls.OCC_OCCUPIED)[:2], o.download(oc.OCCUPIED)))
                o.close()
    known, occupied = om.size(ls.OCC_KNOWN), om.size(ls.OCC_OCCUPIED)
    ms = lambda v: round(float(np.median(v)) * 1e3, 3) if v else None
    result = dict(bench="occupancy", gpu=name, power_limit=limit, scans=a.scans, warmup=a.warmup, params=params,
                  points_per_scan=131072, gpu_ms_insert_scan=ms(t_ins), gpu_device_ms_insert_scan=ms(t_dev),
                  voxel_updates_per_scan=int(np.median(updates)) if updates else None,
                  voxel_updates_per_s=round(float(np.sum(updates) / np.sum(t_ins)), 1) if t_ins else None,
                  known_voxels=known, occupied_voxels=occupied, bricks=st.bricks, device_mb=round(st.device_bytes / 2**20, 1),
                  oracle_scans=len(t_oracle), oracle_cpu_ms_insert_scan=ms(t_oracle), parity=parity)
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if parity is False:
        sys.exit("occupancy map differs from the oracle")


if __name__ == "__main__":
    main()
