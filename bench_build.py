#!/usr/bin/env python
"""bench_build.py -- where the device time of bench.py's config-2 step goes outside the ICP kernel.

Stages bench.py's config-2 batch (the pools, walk and per-step arguments of bench_icp_iterations.py) and runs it at the
benchmark's 30 iterations.  Two runs of the same steps:
  - with torch.profiler (CUDA activities), whose trace is written under --out; from it, per kernel name, the device time
    of the map build and the reading sort, the icp_kernel time, the memset and copy times, and the idle gap between one
    step's last device operation and the next step's first;
  - without the profiler: the wall time per step (begin + end, as bench.py's resident arm with one group).
Prints one JSON line (device name and power limit included: the numbers mean nothing without them).
"""
import argparse
import collections
import json
import os
import re
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_icp_iterations import N_SCAN, POOL, device_info, make_pool, stage_track  # noqa: E402

ITERS = 30


def kernel_name(full):
    """'void ls::count0_kernel(ls::BuildJob const*)' -> 'count0_kernel'"""
    m = re.search(r"(\w+)\s*(<[^(]*>)?\s*\(", full)
    return m.group(1) if m else full


def split_trace(path):
    """Device operations of the trace, in start order: (kind, name, start_us, dur_us)."""
    with open(path) as f:
        tr = json.load(f)
    ops = []
    for e in tr.get("traceEvents", []):
        cat = e.get("cat", "")
        if e.get("ph") != "X" or cat not in ("kernel", "gpu_memcpy", "gpu_memset"):
            continue
        name = kernel_name(e["name"]) if cat == "kernel" else e["name"]
        ops.append((cat, name, float(e["ts"]), float(e["dur"])))
    ops.sort(key=lambda o: o[2])
    return ops


def per_step(ops):
    """Cut the device operations into steps.  A step begins with the upload of its build jobs (a host-to-device copy)
    and ends with what the launch queues after icp_kernel (result gathering, device-to-host copies)."""
    steps, cur, after_icp = [], [], False
    for o in ops:
        if after_icp and o[0] == "gpu_memcpy" and "HtoD" in o[1]:
            steps.append(cur)
            cur, after_icp = [], False
        cur.append(o)
        if o[0] == "kernel" and o[1] == "icp_kernel":
            after_icp = True
    if cur and after_icp:
        steps.append(cur)
    return steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per run")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps before each run")
    ap.add_argument("--tracks", type=int, default=0, help="registrations per launch (default: as bench.py, 4 CTAs each)")
    ap.add_argument("--out", default=None, help="directory of the profiler trace (default: a new temporary directory)")
    args = ap.parse_args()
    if args.out is None:
        args.out = tempfile.mkdtemp(prefix="bench_build_")

    import torch
    import laser_slam_b200 as ls
    from concurrent.futures import ThreadPoolExecutor
    from laser_slam_b200 import synth
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.set_device(0)
    ctx = ls.Context(0)
    B = args.tracks or min(160, ctx.set_icp_cta_budget(0) // 4)
    synth.build()
    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
        tracks = list(ex.map(make_pool, range(B)))
    n_steps = 2 * (args.warmup + args.steps)
    staged = [stage_track(tr[0], tr[1], n_steps) for tr in tracks]
    feats = [[torch.from_numpy(s[0]).pin_memory() for s in tr[2]] for tr in tracks]
    nrms = [[torch.from_numpy(s[1]).pin_memory() for s in tr[2]] for tr in tracks]
    mp = ctx.create_map(B * POOL + 2, N_SCAN)
    sid = [[mp.push_scan_raw(feats[t][k].data_ptr(), nrms[t][k].data_ptr(), 3, N_SCAN) for k in range(POOL)] for t in range(B)]
    prm = ls.default_params(max_iterations=ITERS, use_differential=0)
    prepared = [mp.prepare_begin_batch([(sid[t][staged[t][s][0]], [sid[t][j] for j in staged[t][s][1]], staged[t][s][2],
                                         staged[t][s][3]) for t in range(B)], prm) for s in range(n_steps)]
    build_ms, device_ms = [], []

    def run(s0, n, record):
        for s in range(s0, s0 + n):
            begin, end = prepared[s]
            begin()
            rc, statuses, _, stats = end()
            if rc != 0 or statuses.any():
                raise RuntimeError(f"registration failed rc={rc} {list(statuses)}")
            if record:
                build_ms.append(stats[0].build_ms)
                device_ms.append(max(st.device_ms for st in stats))

    # profiler off: wall time per step
    run(0, args.warmup, False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(args.warmup, args.steps, True)
    torch.cuda.synchronize()
    wall_ms = (time.perf_counter() - t0) * 1e3 / args.steps

    # profiler on: device operations of the same kind of steps
    s1 = args.warmup + args.steps
    run(s1, args.warmup, False)
    torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "trace.json")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(s1 + args.warmup, args.steps, False)
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    mp.close()
    ctx.close()

    steps = per_step(split_trace(trace))
    if len(steps) != args.steps:
        raise RuntimeError(f"trace holds {len(steps)} steps, expected {args.steps}")
    kern = collections.defaultdict(float)
    icp = memset = h2d = d2h = other_copy = 0.0
    n_copies = 0
    for st in steps:
        for kind, name, _, dur in st:
            if kind == "kernel":
                if name == "icp_kernel":
                    icp += dur
                else:
                    kern[name] += dur
            elif kind == "gpu_memset":
                memset += dur
            else:
                n_copies += 1
                if "HtoD" in name:
                    h2d += dur
                elif "DtoH" in name:
                    d2h += dur
                else:
                    other_copy += dur
    gaps = [steps[k + 1][0][2] - max(o[2] + o[3] for o in steps[k]) for k in range(len(steps) - 1)]
    span = [max(o[2] + o[3] for o in st) - st[0][2] for st in steps]
    per = len(steps) * 1e3   # us summed over the steps -> ms per step
    name, power = device_info()
    print(json.dumps({
        "device": name, "power_limit_w": power, "registrations_per_launch": B, "steps": args.steps,
        "build_kernels_ms": {k: v / per for k, v in sorted(kern.items(), key=lambda kv: -kv[1])},
        "build_and_sort_ms": sum(kern.values()) / per,
        "icp_kernel_ms": icp / per,
        "memset_ms": memset / per,
        "copy_ms": {"htod": h2d / per, "dtoh": d2h / per, "other": other_copy / per,
                    "copies_per_step": n_copies / len(steps)},
        "device_span_ms": float(np.median(span)) / 1e3,
        "gap_ms": {"median": float(np.median(gaps)) / 1e3, "min": float(np.min(gaps)) / 1e3,
                   "max": float(np.max(gaps)) / 1e3} if gaps else None,
        "wall_ms_per_step": wall_ms,
        "stats_build_ms": float(np.median(build_ms)),
        "stats_device_ms": float(np.median(device_ms)),
        "trace": trace,
    }))


if __name__ == "__main__":
    main()
