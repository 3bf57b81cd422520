"""Per-scan input filters: ms per scan of ls_map_push_scan_filtered (raw cloud -> filtered cloud with normals in a ring
slot) for the chain RemoveNaN -> MinDist 1 -> MaxDist 60 -> BoundingBox (ego box) -> RandomSampling 0.5 -> VoxelGrid 0.1
-> SurfaceNormal 10, on full synthetic scans with injected NaN and far points, against the oracle's CPU time for the same
chain.  Host clock around synchronous calls, after warm-up.  Prints one JSON line.

    python bench_input_filters.py [--scans 50] [--warmup 5] [--sizes 131072,262144] [--oracle-threads 1]
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

CHAIN = [("RemoveNaNDataPointsFilter", {}),
         ("MinDistDataPointsFilter", {"minDist": 1.0}),
         ("MaxDistDataPointsFilter", {"dim": -1, "maxDist": 60.0}),
         ("BoundingBoxDataPointsFilter", {"xMin": -3.0, "xMax": 3.0, "yMin": -2.0, "yMax": 2.0, "zMin": -3.0, "zMax": 3.0}),
         ("RandomSamplingDataPointsFilter", {"prob": 0.5}),
         ("VoxelGridDataPointsFilter", {"vSizeX": 0.1, "vSizeY": 0.1, "vSizeZ": 0.1}),
         ("SurfaceNormalDataPointsFilter", {"knn": 10})]


def raw_scan(synth, truth, k, n):
    """n points: full 131072-point scans concatenated (the second one from the next pose), NaN and far points injected."""
    parts, j = [], 0
    while sum(len(p) for p in parts) < n:
        parts.append(synth.scan(truth[k + j], 0, k + j)[0])
        j += 1
    p = np.ascontiguousarray(np.concatenate(parts)[:n])
    p[::97, 0] = np.nan
    p[7::89, :3] *= 40.0
    return p


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
    ap.add_argument("--scans", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sizes", default="131072,262144")
    ap.add_argument("--oracle-threads", type=int, default=1)
    ap.add_argument("--oracle-reps", type=int, default=2)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    import oracle
    from oracle import input_filters
    synth.build()
    oracle.build()
    yaml = input_filters.filters_yaml(CHAIN)
    chain = ls.point_filters_from_yaml(yaml)
    truth, _ = synth.trajectory(0, 8)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    res = dict(bench="input_filters", gpu=name, power_limit=limit, scans=a.scans, warmup=a.warmup, chain=[c[0] for c in CHAIN],
               sizes={})
    for n in [int(s) for s in a.sizes.split(",")]:
        clouds = [raw_scan(synth, truth, k, n) for k in range(4)]
        mp = ctx.create_map(8, n)
        for i in range(a.warmup):
            mp.push_scan_filtered(chain, clouds[i % 4])
        launches, kept = [], []
        t0 = time.perf_counter()
        for i in range(a.scans):
            l0 = ctx.launch_count
            _, m = mp.push_scan_filtered(chain, clouds[i % 4])
            launches.append(ctx.launch_count - l0)
            kept.append(m)
        dt = (time.perf_counter() - t0) / a.scans
        mp.close()
        t_or = []
        for r in range(a.oracle_reps):
            t1 = time.perf_counter()
            want = input_filters.apply_filters(CHAIN, clouds[r % 4], num_threads=a.oracle_threads)
            t_or.append(time.perf_counter() - t1)
        res["sizes"][str(n)] = dict(gpu_ms_per_scan=round(dt * 1e3, 3), launches_per_scan=sorted(set(launches)),
                                    points_kept=int(np.median(kept)), oracle_cpu_ms=round(min(t_or) * 1e3, 1),
                                    oracle_threads=a.oracle_threads, oracle_points=int(len(want[0])))
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
