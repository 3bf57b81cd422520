"""Box status and robot collision on the resident occupancy map (ls_occupancy_box_status / _check_paths): --scans full
synthetic HDL-64 scans (131072 points) inserted at laser_to_octomap's defaults (0.075 m voxels, 20 m range), then
10^6 boxes of 1 x 1 x 0.5 m and of 0.5 x 0.5 x 0.3 m centred within 10 m (3 m in z) of the trajectory's poses, and 10^4
paths of 100 waypoints 0.1 m apart from the poses in random directions, with a 1 x 1 x 0.5 m robot, in both
unknown_as_occupied modes.  Reports per workload the median host-clock ms of --repeats calls after 2 warm-ups (each call
is synchronous), the median device_ms, boxes per second and voxel states read per second of host time.  The CPU
restatement (tests/occupancy_collision_ref.py, the grid form) is timed on a subset, and parity against it is checked
outside the clock on --parity boxes and paths of each workload.  Prints one JSON line with the GPU's name and power limit.

    python bench_occupancy_collision.py [--scans 105] [--repeats 10] [--parity 20000]
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
    ap.add_argument("--boxes", type=int, default=1000000)
    ap.add_argument("--paths", type=int, default=10000)
    ap.add_argument("--parity", type=int, default=20000)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    import occupancy_collision_ref as cr
    from oracle import occupancy as oc
    synth.build()
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
    rng = np.random.default_rng(0)
    poses = np.asarray(truth)[:, :3, 3].astype(np.float64)

    def around(n):
        return poses[rng.integers(0, len(poses), n)] + rng.uniform(-1.0, 1.0, (n, 3)) * (10.0, 10.0, 3.0)

    robot = np.array([1.0, 1.0, 0.5])
    starts = around(a.paths)
    d = rng.normal(size=(a.paths, 3)) * (1.0, 1.0, 0.1)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pos = (starts[:, None, :] + 0.1 * np.arange(100)[None, :, None] * d[:, None, :]).reshape(-1, 3)
    offsets = np.arange(a.paths + 1, dtype=np.int64) * 100
    workloads = {"boxes_1x1x0.5": (around(a.boxes), np.array([1.0, 1.0, 0.5])),
                 "boxes_0.5x0.5x0.3": (around(a.boxes), np.array([0.5, 0.5, 0.3]))}
    out = {}
    parity = True
    sub = a.parity
    for wname, (c, size) in workloads.items():
        calls = lambda: om.box_status(c, size)  # noqa: E731
        out[wname] = timed(calls, om, a.repeats, len(c))
        got = om.box_status(c[:sub], size)
        lo, shape = cr.BoxGrid.covering(c[:sub], size, res)
        grid = cr.BoxGrid(keys, vals, l_occ, lo, shape)
        t0 = time.perf_counter()
        want = grid.statuses(c[:sub], size, res)
        out[wname]["cpu_restatement_us_per_box"] = round((time.perf_counter() - t0) / sub * 1e6, 2)
        out[wname]["status_counts"] = [int((want == s).sum()) for s in range(3)]
        parity &= bool(np.array_equal(got, want))
    n_sub = max(sub // 100, 1)
    lo, shape = cr.BoxGrid.covering(pos[:n_sub * 100], robot, res)
    grid = cr.BoxGrid(keys, vals, l_occ, lo, shape)
    st = grid.statuses(pos[:n_sub * 100], robot, res)
    for unknown_occ in (True, False):
        wname = f"paths_unknown_as_occupied_{int(unknown_occ)}"
        calls = lambda: om.check_paths(pos, offsets, robot, unknown_occ)  # noqa: E731
        out[wname] = timed(calls, om, a.repeats, len(pos))
        first = om.check_paths(pos, offsets, robot, unknown_occ)
        out[wname]["paths_colliding"] = int((first >= 0).sum())
        want = cr.first_collisions(st, offsets[:n_sub + 1], unknown_occ)
        parity &= bool(np.array_equal(first[:n_sub], want))
    result = dict(bench="occupancy_collision", gpu=name, power_limit=limit, scans=a.scans, resolution=res,
                  known_voxels=len(keys), workloads=out, parity=bool(parity))
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if not parity:
        sys.exit("box status or path checks differ from the restatement")


def timed(call, om, repeats, boxes):
    host, dev, visited = [], [], []
    for r in range(repeats + 2):
        t0 = time.perf_counter()
        call()
        t1 = time.perf_counter()
        if r >= 2:
            host.append(t1 - t0)
            dev.append(om.last_query.device_ms)
            visited.append(om.last_query.keys_visited)
    ms = float(np.median(host)) * 1e3
    return dict(host_ms=round(ms, 3), device_ms=round(float(np.median(dev)), 3), boxes=boxes,
                boxes_per_s=round(boxes / (ms / 1e3)), voxels_read_per_s=round(float(np.median(visited)) / (ms / 1e3)),
                keys_visited=int(np.median(visited)))


if __name__ == "__main__":
    main()
