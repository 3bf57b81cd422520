"""CPU rehearsal of phase A's list builds on config-2-shaped data: the search and the list collection in one walk
(nn_search_collect) against a second walk of their own after the search (the previous kernel).

For each registration (bench.py config 2's synthetic scans, staged as bench_icp_iterations.py stages them: a
131072-point scan against a 524288-point sub-map) the oracle runs the 30 iterations; its T_iter history is then replayed
through tests/sim/fused_sim.cpp's sim_vlists_paths once per path, with the kernel's cap policy.  Per iteration it prints
the queries answered from their list, the list builds and the refused ones (more than LS_VK points), and the dependent
round trips (ls_sim_steps) per searched query.  Both paths must give every query the same match as the plain search.

    python tools/fused_rehearsal.py [--registrations 2] [--iters 30]
"""
import argparse
import ctypes
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SIM_SRC = os.path.join(ROOT, "tests", "sim", "fused_sim.cpp")
SIM_LIB = os.path.join(ROOT, "tests", "sim", "libfused_sim.so")


def sim_lib():
    deps = [SIM_SRC, os.path.join(ROOT, "tests", "sim", "grid_sim.cpp")] + [os.path.join(ROOT, "laser_slam_b200", "csrc", f) for f in ("ls_grid.cuh", "ls_math.cuh")]
    if not os.path.exists(SIM_LIB) or os.path.getmtime(SIM_LIB) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared",
                               "-I/usr/local/cuda/include", "-o", SIM_LIB, SIM_SRC])
    L = ctypes.CDLL(SIM_LIB)
    vp = ctypes.c_void_p
    L.sim_vlists_paths.restype = ctypes.c_int
    L.sim_vlists_paths.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, vp,
                                   ctypes.c_int, vp, ctypes.c_int, vp, vp, vp, vp, vp, vp]
    return L


def replay(L, rd, refc, Ts, caps, fused):
    K, n = len(Ts), len(rd)
    Tcm = np.ascontiguousarray(np.stack([np.asarray(T, np.float32).T.ravel() for T in Ts]))
    caps = np.ascontiguousarray(caps, np.float32)
    hits, builds, refused = (np.zeros(K, np.int32) for _ in range(3))
    steps = np.zeros(K, np.int64)
    ids, d2 = np.empty(n, np.int32), np.empty(n, np.float32)
    bad = L.sim_vlists_paths(rd.ctypes.data, n, refc.ctypes.data, len(refc), 1.0, 1 << 22, 32, Tcm.ctypes.data, K,
                             caps.ctypes.data, int(fused), hits.ctypes.data, builds.ctypes.data, refused.ctypes.data,
                             steps.ctypes.data, ids.ctypes.data, d2.ctypes.data)
    return dict(bad=bad, hits=hits, builds=builds, refused=refused, steps=steps, ids=ids)


def caps_of(rd, refc, Ts, trim_ratio):
    """The kernel's cap policy (ls_kernels.cuh): 0.04 m^2 first, then the previous trimmed limit times 0.5 (after the
    first iteration) or 2, times 4 while the trimmed quantile would fall among the unmatched queries (the redo rounds)."""
    from scipy.spatial import cKDTree
    tree = cKDTree(refc.astype(np.float64))
    caps, cap = [], 0.04
    k = max(int(np.ceil(trim_ratio * len(rd))) - 1, 0)
    for t, T in enumerate(Ts):
        q = rd.astype(np.float64) @ np.asarray(T, np.float64)[:3, :3].T + np.asarray(T, np.float64)[:3, 3]
        d2 = tree.query(q)[0] ** 2
        while np.count_nonzero(d2 <= cap) <= k and cap < np.inf:
            cap = cap * 4 if cap < 64 else np.inf
        caps.append(cap)
        limit = np.partition(d2, k)[k]
        cap = max(limit * (0.5 if t == 0 else 2.0), 1e-12)
    return caps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--registrations", type=int, default=2, help="registrations of the first track, replayed one by one")
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()

    import bench_icp_iterations as bi
    import oracle
    from laser_slam_b200 import synth
    synth.build()
    L = sim_lib()
    truth, odom, scans = bi.make_pool(0)
    rows = {0: [], 1: []}
    for s, (idx, ks, Ts_map, T0) in enumerate(bi.stage_track(truth, odom, args.registrations)):
        parts = [oracle.transform_cloud(T, *scans[k]) for k, T in zip(ks, Ts_map)]
        refp, refn = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
        reading = scans[idx][0]
        prm = oracle.default_params(max_iterations=args.iters, use_differential=0, num_threads=os.cpu_count() or 1)
        r = oracle.icp(reading, refp, refn, T0, prm, want_hist=True)
        mu = oracle.mean(refp)
        refc = np.ascontiguousarray(refp[:, :3] - mu, np.float32)
        Tpre = np.asarray(T0, np.float32).copy()
        Tpre[:3, 3] -= mu
        rd = np.ascontiguousarray(oracle.transform_points(Tpre, reading)[:, :3], np.float32)
        Ts = [np.eye(4, dtype=np.float32)] + [np.asarray(T, np.float32) for T in r["T_iter_hist"][:-1]]
        caps = caps_of(rd, refc, Ts, prm.trim_ratio)
        with ThreadPoolExecutor(2) as ex:
            res = list(ex.map(lambda f: replay(L, rd, refc, Ts, caps, f), (0, 1)))
        for f in (0, 1):
            assert res[f]["bad"] == 0, f"path {f}: {res[f]['bad']} answers differ from the plain search"
            found = res[f]["ids"] >= 0  # the capped search: nothing found beyond the cap
            assert np.array_equal(res[f]["ids"][found], r["ids_hist"][-1][found]), "last iteration differs from the oracle"
            rows[f].append(res[f])
        print(f"registration {s}: {len(rd)} queries, {len(refc)} map points, {len(Ts)} iterations, both paths exact",
              flush=True)

    def tot(f, key):
        return sum(x[key].astype(np.int64) for x in rows[f])
    n = len(rd) * len(rows[0])
    print(f"\nsummed over {len(rows[0])} registrations ({n} queries per iteration); steps = dependent round trips of the "
          "searches and list builds, per searched query")
    print(f"{'it':>3} | {'two walks: hits':>15} {'builds':>7} {'refused':>7} {'steps/srch':>10} | "
          f"{'one walk: hits':>14} {'builds':>7} {'refused':>7} {'steps/srch':>10} | {'steps':>6}")
    for t in range(len(Ts)):
        cells = []
        for f in (0, 1):
            h, b, rf, st = tot(f, "hits")[t], tot(f, "builds")[t], tot(f, "refused")[t], tot(f, "steps")[t]
            cells.append(f"{h:>{15 if f == 0 else 14}} {b:>7} {rf:>7} {st / max(n - h, 1):>10.1f}")
        ratio = tot(1, "steps")[t] / max(tot(0, "steps")[t], 1)
        print(f"{t:>3} | {cells[0]} | {cells[1]} | {ratio:>6.3f}")
    for lo, hi in ((1, 4), (4, len(Ts)), (0, len(Ts))):
        s0, s1 = tot(0, "steps")[lo:hi].sum(), tot(1, "steps")[lo:hi].sum()
        h0, h1 = tot(0, "hits")[lo:hi].sum() / (n * (hi - lo)), tot(1, "hits")[lo:hi].sum() / (n * (hi - lo))
        print(f"iterations {lo}..{hi - 1}: steps {s0} -> {s1} ({s1 / max(s0, 1):.3f}x), hit rate {100 * h0:.2f} % -> "
              f"{100 * h1:.2f} %")


if __name__ == "__main__":
    main()
