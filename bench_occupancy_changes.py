"""Change detection of the resident occupancy map (ls_occupancy_track_changes / _changes): --scans full synthetic HDL-64
scans (131072 points) inserted at laser_to_octomap's defaults (0.075 m voxels, 20 m range) into two maps, one tracking
changes and one not, alternating which inserts first.  After every scan the tracking map is asked for its changes with a
reset (volumetric_mapping's getChangedPoints).  Reports the median ms of the changes call, the changed voxels per scan,
the insert with and without tracking, a baseline capture of the final map and one full download(LS_OCC_KNOWN) of it for
comparison.  Host clock around each synchronous call.  Parity is checked outside the clock: at three scans the changes
equal the diff of two downloads (tests/occupancy_changes_ref.py), and at the end both maps hold the same voxels.  Prints
one JSON line.

    python bench_occupancy_changes.py [--scans 105] [--repeats 10]
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
    import occupancy_changes_ref as cr
    from oracle import occupancy as oc
    synth.build()
    truth, _ = synth.trajectory(0, a.scans)
    res = 0.075
    l_occ = oc.logodds(0.7)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, 131072)
    plain, tracked = ls.OccupancyMap(ctx), ls.OccupancyMap(ctx)
    tracked.track_changes()
    zeros = np.zeros((131072, 3), np.float32)
    checks = {0, a.scans // 2, a.scans - 1}
    t_plain, t_tracked, t_changes, changed = [], [], [], []
    parity = True
    for k in range(a.scans):
        sid = ring.push_scan(synth.scan(truth[k], 0, k)[0], zeros)
        T = truth[k].astype(np.float32)
        base = tracked.download(ls.OCC_KNOWN)[:2] if k in checks else None
        for m in ((plain, tracked) if k % 2 == 0 else (tracked, plain)):
            t0 = time.perf_counter()
            m.insert_scan(ring, sid, T)
            (t_plain if m is plain else t_tracked).append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        got = tracked.changes(reset=True)
        t_changes.append(time.perf_counter() - t0)
        changed.append(len(got[0]))
        if base is not None:
            want = cr.diff_arrays(*base, *tracked.download(ls.OCC_KNOWN)[:2], l_occ)
            want += (cr.centres(want[0], want[1], res, res),)
            parity &= all(np.array_equal(np.asarray(g).view(np.uint8), np.asarray(w).view(np.uint8)) for g, w in zip(got, want))
    stats = tracked.last_changes
    kp, vp, _ = plain.download(ls.OCC_KNOWN)
    kt, vt, _ = tracked.download(ls.OCC_KNOWN)
    parity &= np.array_equal(kp, kt) and np.array_equal(vp.view(np.uint32), vt.view(np.uint32))
    t_capture, t_download = [], []
    for r in range(a.repeats + 2):
        t0 = time.perf_counter()
        tracked.track_changes()
        t1 = time.perf_counter()
        plain.download(ls.OCC_KNOWN)
        t2 = time.perf_counter()
        if r >= 2:
            t_capture.append(t1 - t0)
            t_download.append(t2 - t1)
    parity &= all(len(x) == 0 for x in tracked.changes())
    ms = lambda x: round(float(np.median(x)) * 1e3, 3)  # noqa: E731
    result = dict(bench="occupancy_changes", gpu=name, power_limit=limit, scans=a.scans, resolution=res,
                  known_voxels=len(kp), baseline_bricks=stats.baseline_bricks, change_device_bytes=stats.device_bytes,
                  gpu_ms_changes_reset=ms(t_changes), changed_voxels_median=int(np.median(changed)),
                  changed_voxels_max=int(np.max(changed)), gpu_ms_insert_untracked=ms(t_plain),
                  gpu_ms_insert_tracked=ms(t_tracked), gpu_ms_baseline_capture=ms(t_capture),
                  gpu_ms_download_known=ms(t_download), parity=bool(parity))
    plain.close()
    tracked.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if not parity:
        sys.exit("change detection differs from the diff of two downloads")


if __name__ == "__main__":
    main()
