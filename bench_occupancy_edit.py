"""Edits of the resident occupancy map (ls_occupancy_set_boxes / _box_voxels / _bounds / _clear): after --scans full
synthetic HDL-64 scans (131072 points) inserted at laser_to_octomap's defaults (0.075 m voxels, 20 m range), setFree of
1 m, 5 m and 20 m cubes at a pose mid-trajectory, the occupied voxels of a 20 m cube, the bounds and a reset.  Every timed
call starts from the same map (read back from its .ot file outside the clock).  Median ms over --repeats calls after two
warm-up calls, host clock around the synchronous call.  Parity against the restatement of tests/occupancy_edits_ref.py
(its per-axis loop, vectorised over the box in numpy) is checked outside the clock.  Prints one JSON line.

    python bench_occupancy_edit.py [--scans 105] [--repeats 10]
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


def box_keys(er, center, size, res):
    """The restatement's loop keys of a box (x outer, z inner), as a uint64 array."""
    ax = [np.array(er.axis_keys(center[a], size[a], res), np.uint64) for a in range(3)]
    x, y, z = np.meshgrid(*ax, indexing="ij")
    return (x | (y << np.uint64(16)) | (z << np.uint64(32))).reshape(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=105)
    ap.add_argument("--repeats", type=int, default=10)
    a = ap.parse_args()
    import laser_slam_b200 as ls
    from laser_slam_b200 import synth
    import occupancy_edits_ref as er
    import octomap_read_ref as rr
    from oracle import occupancy as oc
    synth.build()
    truth, _ = synth.trajectory(0, a.scans)
    res = 0.075
    l_min, _ = rr.clamps()
    l_occ = oc.logodds(0.7)
    ctx = ls.Context(0)
    name, limit = gpu_info()
    ring = ctx.create_map(8, 131072)
    om = ls.OccupancyMap(ctx)
    zeros = np.zeros((131072, 3), np.float32)
    for k in range(a.scans):
        om.insert_scan(ring, ring.push_scan(synth.scan(truth[k], 0, k)[0], zeros), truth[k].astype(np.float32))
    k0, v0, _ = om.download(ls.OCC_KNOWN)
    p = truth[a.scans // 2][:3, 3].astype(np.float64)
    ms = lambda x: round(float(np.median(x)) * 1e3, 3)  # noqa: E731
    result = dict(bench="occupancy_edit", gpu=name, power_limit=limit, scans=a.scans, repeats=a.repeats, resolution=res,
                  known_voxels=len(k0), bricks=None)
    parity = True
    with tempfile.TemporaryDirectory() as tmp:
        ot = os.path.join(tmp, "map.ot")
        om.save_octomap_full(ot)

        def timed(call, reload=True):
            t = []
            for r in range(a.repeats + 2):
                if reload:
                    om.read_octomap_full(ot)
                t0 = time.perf_counter()
                out = call()
                t1 = time.perf_counter()
                if r >= 2:
                    t.append(t1 - t0)
            return out, ms(t)

        for side in (1.0, 5.0, 20.0):
            st, result[f"gpu_ms_set_free_{side:g}m"] = timed(lambda: om.set_free(p, (side,) * 3))
            bk = np.unique(box_keys(er, p, (side,) * 3, res))
            keep = ~np.isin(k0, bk)
            wk = np.concatenate([k0[keep], bk])
            wv = np.concatenate([v0[keep], np.full(len(bk), l_min, np.float32)])
            order = np.argsort(wk)
            k, v, _ = om.download(ls.OCC_KNOWN)
            parity &= np.array_equal(k, wk[order]) and np.array_equal(v.view(np.uint32), wv[order].view(np.uint32))
            result[f"voxels_set_{side:g}m"] = st.voxels_set
        om.read_octomap_full(ot)
        result["bricks"] = om.set_boxes(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros(0)).bricks
        (ck, cv, _), result["gpu_ms_crop_20m"] = timed(lambda: om.box_voxels(p, (20.0,) * 3), reload=False)
        bk = box_keys(er, p, (20.0,) * 3, res)
        idx = np.clip(np.searchsorted(k0, bk), 0, len(k0) - 1)
        hit = (k0[idx] == bk) & (v0[idx] >= l_occ)
        parity &= np.array_equal(ck, bk[hit]) and np.array_equal(cv.view(np.uint32), v0[idx][hit].view(np.uint32))
        result["crop_points_20m"] = len(ck)
        (lo, hi), result["gpu_ms_bounds"] = timed(om.bounds, reload=False)
        wlo, whi = er.Edits(res, l_min, 0, l_occ).bounds(dict.fromkeys([int(k0.min())] + [int(x) for x in _extremes(k0)]))
        parity &= np.array_equal(lo, wlo) and np.array_equal(hi, whi)
        _, result["gpu_ms_clear"] = timed(om.clear)
        parity &= om.size(ls.OCC_KNOWN) == 0
    result["parity"] = bool(parity)
    om.close()
    ring.close()
    ctx.close()
    print(json.dumps(result))
    if not parity:
        sys.exit("occupancy edits differ from the restatement")


def _extremes(keys):
    """Keys holding the smallest and largest key of each axis (the bounds depend on nothing else)."""
    out = []
    for a in range(3):
        ka = (keys >> np.uint64(16 * a)) & np.uint64(0xFFFF)
        out += [keys[np.argmin(ka)], keys[np.argmax(ka)]]
    return out


if __name__ == "__main__":
    main()
