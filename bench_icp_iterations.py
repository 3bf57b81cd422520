#!/usr/bin/env python
"""bench_icp_iterations.py -- where the time of bench.py's config-2 launch goes, iteration by iteration.

Stages bench.py's config-2 batch (the same synthetic pools, the same tracks, the same per-step arguments) and runs it with
max_iterations = k for several k, the differential checker off: a k-iteration run is then exactly the first k iterations
of the 30-iteration run, so differences of the median icp_ms between two k are the cost of the iterations in between.
Prints one JSON line (device name and power limit included: the numbers mean nothing without them).
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# bench.py configs[1]: scan size, scans per map, pool of scans per track
N_SCAN, K_MAP, POOL, SENSOR = 131072, 4, 24, 0
KS = (1, 2, 3, 4, 6, 10, 20, 30)


def walk(step):
    period = 2 * (POOL - 1)
    j = step % period
    return j if j < POOL else period - j


def make_pool(seq):
    from laser_slam_b200 import synth
    truth, odom = synth.trajectory(seq, POOL, y_start=-20.0)
    return truth, odom, [synth.scan(truth[k], seq, k, sensor=SENSOR) for k in range(POOL)]


def stage_track(truth, odom, n_steps):
    """bench.py's stage_track: sub-map scans, their transforms and the initial guess of each step."""
    h = [walk(s) for s in range(K_MAP + 1)]
    out = []
    for s in range(n_steps):
        idx = walk(s + K_MAP + 1)
        h.append(idx)
        ref = h[-2]
        ks = h[-2:-2 - K_MAP:-1]
        Ts = [np.eye(4, dtype=np.float32) if k == ref else (np.linalg.inv(truth[ref]) @ truth[k]).astype(np.float32) for k in ks]
        T0 = (np.linalg.inv(truth[ref]) @ odom[idx]).astype(np.float32) if abs(idx - ref) == 1 else np.eye(4, dtype=np.float32)
        out.append((idx, ks, Ts, T0))
    return out


def device_info():
    import torch
    name = torch.cuda.get_device_name(0)
    power = None
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        power = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:
        import subprocess
        try:
            out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                 capture_output=True, text=True, timeout=10).stdout.strip()
            power = float(out.splitlines()[0])
        except Exception:
            pass
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=8, help="timed launches per iteration count")
    ap.add_argument("--warmup", type=int, default=3, help="untimed launches per iteration count")
    ap.add_argument("--tracks", type=int, default=0, help="registrations per launch (default: as bench.py, 4 CTAs each)")
    args = ap.parse_args()

    import torch
    import laser_slam_b200 as ls
    from concurrent.futures import ThreadPoolExecutor
    from laser_slam_b200 import synth
    torch.cuda.set_device(0)
    ctx = ls.Context(0)
    B = args.tracks or min(160, ctx.set_icp_cta_budget(0) // 4)
    synth.build()
    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
        tracks = list(ex.map(make_pool, range(B)))
    n_steps = args.warmup + args.launches
    staged = [stage_track(tr[0], tr[1], n_steps) for tr in tracks]
    feats = [[torch.from_numpy(s[0]).pin_memory() for s in tr[2]] for tr in tracks]
    nrms = [[torch.from_numpy(s[1]).pin_memory() for s in tr[2]] for tr in tracks]
    mp = ctx.create_map(B * POOL + 2, N_SCAN)
    sid = [[mp.push_scan_raw(feats[t][k].data_ptr(), nrms[t][k].data_ptr(), 3, N_SCAN) for k in range(POOL)] for t in range(B)]

    rows = {}
    for k in KS:
        prm = ls.default_params(max_iterations=k, use_differential=0)
        icp, build, dev = [], [], []
        for s in range(n_steps):   # every k runs the same steps
            probs = [(sid[t][staged[t][s][0]], [sid[t][j] for j in staged[t][s][1]], staged[t][s][2], staged[t][s][3])
                     for t in range(B)]
            begin, end = mp.prepare_begin_batch(probs, prm)
            begin()
            rc, statuses, _, stats = end()
            if rc != 0 or statuses.any():
                raise RuntimeError(f"registration failed rc={rc} {list(statuses)}")
            if s >= args.warmup:
                icp.append(stats[0].icp_ms)
                build.append(stats[0].build_ms)
                dev.append(max(st.device_ms for st in stats))
        rows[k] = {"icp_ms": float(np.median(icp)), "build_ms": float(np.median(build)), "device_ms": float(np.median(dev)),
                   "icp_ms_min": float(np.min(icp)), "icp_ms_max": float(np.max(icp))}
    mp.close()
    ctx.close()

    bands, prev = [], None
    for k in KS:
        if prev is not None:
            d = rows[k]["icp_ms"] - rows[prev]["icp_ms"]
            bands.append({"iterations": f"{prev}..{k - 1}", "ms": d, "ms_per_iteration": d / (k - prev)})
        else:
            bands.append({"iterations": f"0..{k - 1}", "ms": rows[k]["icp_ms"], "ms_per_iteration": rows[k]["icp_ms"] / k})
        prev = k
    name, power = device_info()
    print(json.dumps({"device": name, "power_limit_w": power, "registrations_per_launch": B, "launches_per_k": args.launches,
                      "per_k": {str(k): v for k, v in rows.items()}, "bands": bands}))


if __name__ == "__main__":
    main()
