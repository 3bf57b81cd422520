"""Resident local map (ls_local_map_*, LaserSlamWorker's map maintenance): ms per add_scan and per filter on a synthetic
HDL-64 sequence pushed through the ring, add_scan every step and filter (getFilteredMap) every k-th step, against the
oracle's CPU time for the same steps.  Host clock around synchronous calls, after warm-up.  The last step's maps are
checked against the oracle bit for bit, outside the clock.  Prints one JSON line.

    python bench_local_map.py [--steps 60] [--warmup 10] [--every 5] [--voxel 0.1] [--min-points 3] [--radius 20]
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
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--every", type=int, default=5)
    ap.add_argument("--voxel", type=float, default=0.1)
    ap.add_argument("--min-points", type=int, default=3)
    ap.add_argument("--radius", type=float, default=20.0)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    import oracle
    from oracle import local_map as olm
    synth.build()
    oracle.build()
    total = a.warmup + a.steps
    truth, _ = synth.trajectory(0, total)
    scans = [synth.scan(truth[k], 0, k)[0] for k in range(total)]
    poses = [ls.correct_rigid(truth[k].astype(np.float32)) for k in range(total)]
    zeros = np.zeros((len(scans[0]), 3), np.float32)
    params = dict(distance_to_consider_fixed=a.radius, separate_distant_map=True, voxel_size_m=a.voxel,
                  minimum_point_number_per_voxel=a.min_points, remove_ground_from_local_map=True,
                  ground_distance_to_robot_center_m=1.5)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, len(scans[0]))
    lm = ls.LocalMap(ctx, **params)
    o = olm.LocalMap(**params)
    t_add, t_filter, t_or_add, t_or_filter = [], [], [], []
    sizes = {}
    for k in range(total):
        sid = ring.push_scan(scans[k], zeros)
        ring.sync()
        z = float(truth[k][2, 3])
        t0 = time.perf_counter()
        lm.add_scan(ring, sid, poses[k], z)
        t1 = time.perf_counter()
        o.add_scan(scans[k], poses[k], z)
        t2 = time.perf_counter()
        if k >= a.warmup:
            t_add.append(t1 - t0)
            t_or_add.append(t2 - t1)
        if k % a.every == a.every - 1:
            c = truth[k][:3, 3]
            t0 = time.perf_counter()
            n = lm.filter(c)
            t1 = time.perf_counter()
            want = o.get_filtered_map(c)
            t2 = time.perf_counter()
            if k >= a.warmup:
                t_filter.append(t1 - t0)
                t_or_filter.append(t2 - t1)
            # outside the clock: drain the queues as a SegMatch reader would, and record the sizes reached
            lm.take_queue()
            o.get_queued_points()
            sizes = dict(local=lm.size(ls.LM_LOCAL), local_filtered=lm.size(ls.LM_LOCAL_FILTERED),
                         distant=lm.size(ls.LM_DISTANT), filtered_map=n)
            last_want = want
    same = lambda x, y: x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32))
    parity = (same(lm.download(ls.LM_LOCAL), o.local_map) and same(lm.download(ls.LM_LOCAL_FILTERED), o.local_map_filtered)
              and same(lm.download(ls.LM_DISTANT), o.distant_map) and same(lm.download(ls.LM_FILTERED_MAP), last_want))
    lm.close()
    ring.close()
    ctx.close()
    ms = lambda v: round(float(np.median(v)) * 1e3, 3) if v else None
    print(json.dumps(dict(bench="local_map", gpu=name, power_limit=limit, steps=a.steps, warmup=a.warmup, filter_every=a.every,
                          params=params, points_per_scan=len(scans[0]), gpu_ms_add_scan=ms(t_add), gpu_ms_filter=ms(t_filter),
                          oracle_cpu_ms_add_scan=ms(t_or_add), oracle_cpu_ms_filter=ms(t_or_filter), sizes_reached=sizes,
                          parity=bool(parity))))
    if not parity:
        sys.exit("local map differs from the oracle")


if __name__ == "__main__":
    main()
