"""Queries of the resident occupancy map (ls_occupancy_cell_status / _line_status / _cast_rays): after --scans full synthetic
HDL-64 scans (131072 points) of sequence 0 inserted at laser_to_octomap's defaults (0.075 m voxels, 20 m range), as
bench_octomap.py builds it, the median ms of each synchronous query call (host clock, after two warm-up calls):
  cells   1 M points uniform over the map's bounding box
  lines   100 k segments of 1-10 m from near the scan poses (getLineStatus)
  boxes   1 k segments of 1-10 m with a 0.6 x 0.6 x 0.3 m box (getLineStatusBoundingBox)
  rays    131072 rays, the directions of the HDL-64 scan at pose --ray-pose, from that pose, max range 20, ignore_unknown
          0 and 1 (castRay)
with queries/s and keys visited/s.  The oracle (one CPU thread, over the device map's known voxels) is timed on the first
--oracle-subset queries of each kind; parity on that subset (status, first keys, log-odds and ends bit for bit) is
checked outside the clock.  Prints one JSON line.

    python bench_occupancy_queries.py [--scans 105] [--repeats 10] [--oracle-subset 10000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_occupancy import gpu_info  # noqa: E402


def _same(a, b):
    x, y = np.asarray(a[1]), np.asarray(b[1])
    if x.dtype == np.float32:
        x, y = x.view(np.uint32), y.view(np.uint32)
    return bool(np.array_equal(a[0], b[0]) and np.array_equal(x, y))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=105)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--oracle-subset", type=int, default=10000)
    ap.add_argument("--ray-pose", type=int, default=50)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    from oracle import occupancy, queries
    synth.build()
    queries.build()
    truth, _ = synth.trajectory(0, a.scans)
    params = dict(resolution=0.075, max_range=20.0)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, 131072)
    om = ls.OccupancyMap(ctx, **params)
    zeros = np.zeros((131072, 3), np.float32)
    for k in range(a.scans):
        om.insert_scan(ring, ring.push_scan(synth.scan(truth[k], 0, k)[0], zeros), truth[k].astype(np.float32))
    keys, lo, _ = om.download(ls.OCC_KNOWN)
    cen = occupancy.centres(keys, params["resolution"]).astype(np.float64)
    rng = np.random.default_rng(0)
    pts = rng.uniform(cen.min(axis=0), cen.max(axis=0), (1_000_000, 3))
    poses = np.array([truth[k][:3, 3] for k in range(a.scans)])

    def segments(n):
        s = poses[rng.integers(0, a.scans, n)] + rng.uniform(-3.0, 3.0, (n, 3)) * [1, 1, 0.3]
        d = rng.normal(size=(n, 3))
        d /= np.linalg.norm(d, axis=1)[:, None]
        return s, s + d * rng.uniform(1.0, 10.0, (n, 1))

    s_l, e_l = segments(100_000)
    s_b, e_b = segments(1000)
    box = (0.6, 0.6, 0.3)
    k = min(a.ray_pose, a.scans - 1)
    T = truth[k]
    dirs = (synth.scan(T, 0, k)[0][:, :3].astype(np.float64) @ T[:3, :3].T).astype(np.float32)
    origins = np.repeat(T[:3, 3][None].astype(np.float32), len(dirs), axis=0)
    kinds = {
        "cells": (lambda: om.cell_status(pts), lambda o, m: o.cell_status(pts[:m])),
        "lines": (lambda: om.line_status(s_l, e_l), lambda o, m: o.line_status(s_l[:m], e_l[:m])),
        "boxes": (lambda: om.line_status(s_b, e_b, box=box), lambda o, m: o.line_status(s_b[:m], e_b[:m], box=box)),
        "rays_ignore0": (lambda: om.cast_rays(origins, dirs, False, 20.0),
                         lambda o, m: o.cast_rays(origins[:m], dirs[:m], False, 20.0)),
        "rays_ignore1": (lambda: om.cast_rays(origins, dirs, True, 20.0),
                         lambda o, m: o.cast_rays(origins[:m], dirs[:m], True, 20.0)),
    }
    n_of = dict(cells=len(pts), lines=len(s_l), boxes=len(s_b), rays_ignore0=len(dirs), rays_ignore1=len(dirs))
    oracle = queries.KnownVoxels(keys, lo, **params)
    out, parity = {}, True
    for kind, (dev_call, oracle_call) in kinds.items():
        times, dev_ms = [], []
        for r in range(a.repeats + 2):
            t0 = time.perf_counter()
            got = dev_call()
            t1 = time.perf_counter()
            if r >= 2:
                times.append(t1 - t0)
                dev_ms.append(om.last_query.device_ms)
        visited = om.last_query.keys_visited
        m = min(a.oracle_subset, n_of[kind])
        t0 = time.perf_counter()
        want = oracle_call(oracle, m)
        t_oracle = time.perf_counter() - t0
        ok = _same((got[0][:m], got[1][:m]), want)
        if kind != "boxes":  # the device's box pass may read lines past the failing one before they stop
            ok = ok and (m < n_of[kind] or visited == oracle.keys_visited)
        parity = parity and ok
        ms = float(np.median(times)) * 1e3
        out[kind] = dict(queries=n_of[kind], gpu_ms=round(ms, 3), gpu_device_ms=round(float(np.median(dev_ms)), 3),
                         queries_per_s=round(n_of[kind] / ms * 1e3), keys_visited=int(visited),
                         keys_visited_per_s=round(visited / ms * 1e3), oracle_subset=m,
                         oracle_cpu_ms=round(t_oracle * 1e3, 1), parity=ok)
    result = dict(bench="occupancy_queries", gpu=name, power_limit=limit, scans=a.scans, repeats=a.repeats, params=params,
                  known_voxels=len(keys), box=box, ray_pose=k, **out, parity=parity)
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    print(f"parity: {str(parity).lower()}")
    if not parity:
        sys.exit("queries differ from the oracle")


if __name__ == "__main__":
    main()
