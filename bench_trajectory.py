"""bench.py --config 3: BASELINE.json configs[2], the batched trajectory.

World-size independent synthetic sequences, sequence r on GPU r (one LaserTrack per GPU, the reference's
n_laser_slam_workers tracks, reference laser_slam/src/incremental_estimator.cpp:22-26), each `--steps` CONSECUTIVE scans
long (no recycled pool): scan k is registered against the rolling map of the previous 4 scans with 30 ICP iterations
(LaserTrack::localScanToSubMap, reference laser_slam/src/laser_track.cpp:466-519), its upload overlapping the previous
registration.  After every registration the rank posts ONE 32-byte record {delta[6], status, key} into a single
ncclAllGather over NVLink (ls_comm_*); the records of all ranks come back one step later and EVERY rank feeds them into its
replica of the shared pose graph (ls_pg_*: one node + one Cauchy ICP factor per track per step, priors at the start),
which is re-estimated (3 Gauss-Newton iterations = one IncrementalEstimator::estimate) every --pg-every steps and at the
end.  value = all ranks' registrations / wall time of the slowest rank; per-rank times are reported (imbalance)."""
import json
import os
import time

import numpy as np


def main(args):
    import torch
    import torch.distributed as dist
    import laser_slam_b200 as ls
    from laser_slam_b200 import dist as lsd, synth
    import bench
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    wl = bench.select_workload(2)
    N, K, ITERS = bench.N_SCAN, bench.K_MAP, bench.ITERS
    warm = 1 + max(args.warmup, K)                 # scan 0 + the warm-up registrations; the first K of them fill the first map
    n_scans = warm + args.steps                    # the rest are timed
    pg_every = int(os.environ.get("LS_PG_EVERY", "10"))
    seq = int(os.environ.get("LS_BENCH_SEQ_BASE", "0")) + rank
    from concurrent.futures import ThreadPoolExecutor
    truth, odom = synth.trajectory(seq, n_scans, y_start=-100.0)
    with ThreadPoolExecutor(max_workers=max(1, min(16, bench.usable_threads() // max(1, min(world, 8))))) as ex_:
        scans = list(ex_.map(lambda k: synth.scan(truth[k], seq, k), range(n_scans)))
    feats = [torch.from_numpy(s[0]).pin_memory() for s in scans]
    nrms = [torch.from_numpy(s[1]).pin_memory() for s in scans]
    ctx = ls.Context(local)
    prm = ls.default_params(max_iterations=ITERS, use_differential=0)
    ring = ctx.create_map(K + 6, N)
    graph_dev = ls.PoseGraph(local)
    graph = lsd.ReplicatedGraph(world, sink=graph_dev)
    exchange = lsd.Exchange(rank, world, device=local)
    sid = {}

    def problem(k):
        ref = k - 1
        ks = [ref - j for j in range(K) if ref - j >= 0]
        Ts = [np.eye(4, dtype=np.float32) if j == ref else (np.linalg.inv(truth[ref]) @ truth[j]).astype(np.float32) for j in ks]
        T0 = (np.linalg.inv(truth[ref]) @ odom[k]).astype(np.float32) if k >= 1 else np.eye(4, dtype=np.float32)
        T0 = (np.linalg.inv(odom[ref]) @ odom[k]).astype(np.float32)      # the odometry increment, as the trajectory gives it
        return (sid[k], [sid[j] for j in ks], Ts, T0)

    def upload(k):
        if k < n_scans:
            sid[k] = ring.push_scan_raw_async(feats[k].data_ptr(), nrms[k].data_ptr(), 3, N)

    pg_ms, icp_ms, dev_ms = [], [], []

    def feed(records, step):
        if records is None:
            return
        graph.feed(records)
        if graph.count[0] % pg_every == 0:
            st = graph_dev.optimize(3)
            pg_ms.append(st.device_ms)

    def step(k, record):
        end = ring.begin_batch([problem(k)], prm)     # stage + launch scan k, returns at once
        upload(k + 1)                                 # the next scan goes up while this one is registered
        feed(exchange.collect(), k)                   # last step's records from every rank -> the replicated graph
        out = end()[0]
        exchange.post(lsd.pose_record(out["T"], status=out["rc"], key=k))
        if record:
            icp_ms.append(out["stats"].icp_ms)
            dev_ms.append(out["stats"].device_ms)
        return out

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    upload(0)
    ring.sync()
    exchange.post(lsd.pose_record(np.eye(4), status=0, key=0))   # every track's first node (prior)
    upload(1)
    for k in range(1, warm):
        step(k, False)
    sampler = bench.ClockSampler(local)
    sampler.start()
    l0 = ctx.launch_count + graph_dev.launch_count
    barrier()
    t0 = time.perf_counter()
    last = None
    for k in range(warm, n_scans):
        last = step(k, True)
    feed(exchange.collect(), n_scans)
    st_final = graph_dev.optimize(3)
    torch.cuda.synchronize()
    t_rank = time.perf_counter() - t0
    barrier()
    t_all = time.perf_counter() - t0
    launches = ctx.launch_count + graph_dev.launch_count - l0
    clocks = sampler.summary()
    timed = n_scans - warm
    t_max, = lsd.max_over_ranks([t_all], device=local)
    per_rank = [t_rank]
    digest = graph.digest()
    if world > 1:
        tt = torch.tensor([t_rank], dtype=torch.float64, device="cuda")
        gl = [torch.zeros_like(tt) for _ in range(world)]
        dist.all_gather(gl, tt)
        per_rank = [float(x.item()) for x in gl]
        dg = [None] * world
        dist.all_gather_object(dg, digest)
        same_graph = all(d == dg[0] for d in dg)
    else:
        same_graph = True
    truth_rel = np.linalg.inv(truth[n_scans - 2]) @ truth[n_scans - 1]
    pose_err = float(np.abs(last["T"][:3, 3] - truth_rel[:3, 3]).max())
    exchange.close()
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    peak, peak_src = bench.load_peaks()
    t_icp = float(np.mean(icp_ms)) * 1e-3
    out = {
        "metric": "trajectory registrations/s (one synthetic sequence per GPU, 131072-pt scan vs 524288-pt rolling map, 30 iterations)",
        "value": world * timed / t_max, "unit": "registrations/s", "n_gpus": args.gpus, "steps": timed, "warmup": warm - 1,
        "ms_per_step": 1e3 * t_max / timed, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
        "data": "synthetic",
        "config": {"workload": f"configs[2]: batched trajectory, {world} independent synthetic sequences of {timed} consecutive scans "
                               f"(+{warm} to fill the first map), 1 per GPU, rolling map of {K} scans, {ITERS} ICP iterations, "
                               "NCCL pose-record allgather feeding a replicated shared pose graph",
                   "sequences": world, "scans_per_sequence": timed,
                   "per_rank_wall_s": per_rank, "imbalance_max_over_min": max(per_rank) / min(per_rank),
                   "collective": "one 32 B/rank ncclAllGather of {delta[6], status, key} per step, split-phase (posted after "
                                 "registration k, collected during registration k+1)",
                   "estimator": {"replicas": world, "identical_across_ranks": bool(same_graph), "poses": len(graph.keys),
                                 "factors": len(graph.factors), "optimize_every_steps": pg_every,
                                 "optimize_ms_mean": float(np.mean(pg_ms)) if pg_ms else None,
                                 "final_optimize_ms": st_final.device_ms, "final_cost": st_final.cost_last},
                   "l2": f"inputs larger than L2: every step registers a new scan ({timed} distinct scans per rank, "
                         f"{timed * N * 32 / 1e6:.0f} MB) against a sub-map rebuilt from the last {K}",
                   "final_pose_err_vs_truth_m": pose_err},
        "e2e": {"value": world * timed / t_max, "unit": "registrations/s",
                "h2d_bytes_per_step": int(N * 28 + 16 * 4 * (K + 1) + 8 * (K + 1)), "d2h_bytes_per_step": 216 + 212,
                "note": "this workload IS the end-to-end path: every step uploads its scan from pinned host memory "
                        "(ls_map_push_scan_async), registers through the C ABI and reads the 4x4 result back"},
        "gpu_launches": int(launches), "clocks": clocks,
        "roofline": {"bound": "hbm", "kernel": "ls::icp_kernel (one registration per launch)",
                     "achieved": bench.ALG_BYTES_ICP / t_icp / 1e9, "peak": peak, "unit": "GB/s",
                     "frac": bench.ALG_BYTES_ICP / t_icp / 1e9 / peak, "traffic": None, "peak_source": peak_src,
                     "kernel_ms": t_icp * 1e3, "device_ms_per_registration": float(np.mean(dev_ms))},
    }
    print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()
