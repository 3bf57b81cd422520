"""The batched registration (ls_icp_register_submap_batch) against the oracle at the schedules only a batch reaches:
few CTAs per problem (CTA budgets, the 160-problem launch), problems leaving the loop in different iterations
(differential checker), re-search rounds under the dynamic schedule (up to the uncapped search), ragged and empty
problems in one launch, and many queries tied at the trimmed limit.

Every problem is compared bit for bit with `oracle.icp` on the host-assembled sub-map and with its own single call
(`Map.register`, static schedule).  The tests not marked `gpu` are the preconditions: they show, from the oracle alone,
that each case really reaches the branch it is meant for, so a change of the synthetic data cannot quietly turn a case
into one that exercises nothing."""
import os
import struct
import sys

import numpy as np
import pytest

from oracle import input_filters as fo

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

N_SCANS = 14          # scans of the pool (sequence 0); problems use scans 2..13 as readings
THREADS = min(16, os.cpu_count() or 1)
DEFAULT = {}                                                      # icp_default.yaml: 40 iterations, differential, 0.75
FIXED = dict(max_iterations=12, use_differential=0)
NOTHING = [("MaxDistDataPointsFilter", {"maxDist": 0.001}), ("SurfaceNormalDataPointsFilter", {})]


# ---- problems ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pool(synth_mod):
    """Full (131072-point) and sub-sampled (8192-point) scans of one synthetic sequence, with truth and odometry."""
    truth, odom = synth_mod.trajectory(0, N_SCANS, y_start=-20.0)
    full = [synth_mod.scan(truth[k], 0, k) for k in range(N_SCANS)]
    return dict(truth=truth, odom=odom, full=full, sub=[synth_mod.subsample(*s, 16) for s in full])


def _pert(dx, dyaw_deg, dy=0.0):
    c, s = np.cos(np.deg2rad(dyaw_deg)), np.sin(np.deg2rad(dyaw_deg))
    P = np.eye(4)
    P[:2, :2] = [[c, -s], [s, c]]
    P[:3, 3] = [dx, dy, 0.0]
    return P


_submaps = {}


def problem(oracle_mod, pool, r, K, dx=0.0, dyaw=0.0, reading=None, name=None):
    """LaserTrack::localScanToSubMap's registration of scan r: the sub-map is scans r-1 .. r-K in the frame of scan r-1,
    T0 the odometry guess times a perturbation (dx metres along x, dyaw degrees about z).  `reading` replaces the
    sub-sampled scan r as the reading: ("full",) the whole scan, ("head", k) its first k points, ("outliers", f, d) a
    fraction f of its points moved d metres off the map, ("empty",) a scan the input chain filtered to nothing."""
    truth, odom = pool["truth"], pool["odom"]
    ref = r - 1
    ks = [ref - j for j in range(K)]
    Ts = [np.eye(4, dtype=np.float32) if k == ref else (np.linalg.inv(truth[ref]) @ truth[k]).astype(np.float32) for k in ks]
    T0 = (np.linalg.inv(truth[ref]) @ odom[r] @ _pert(dx, dyaw)).astype(np.float32)
    if (r, K) not in _submaps:
        parts = [pool["sub"][k] if k == ref else oracle_mod.transform_cloud(T, *pool["sub"][k]) for k, T in zip(ks, Ts)]
        _submaps[(r, K)] = (np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))
    reading = reading or ("sub",)
    pts, nrm = pool["sub"][r]
    if reading[0] == "full":
        pts, nrm = pool["full"][r]
    elif reading[0] == "head":
        pts, nrm = pts[:reading[1]].copy(), nrm[:reading[1]].copy()
    elif reading[0] == "outliers":
        pts = pts.copy()
        moved = np.random.default_rng(r).random(len(pts)) < reading[1]
        pts[moved, 2] += np.float32(reading[2])
    elif reading[0] == "empty":
        pts, nrm = np.zeros((0, 4), np.float32), np.zeros((0, 3), np.float32)
    refp, refn = _submaps[(r, K)]
    return dict(name=name or f"r{r} K{K} dx{dx} yaw{dyaw} {reading}", r=r, ks=ks, Ts=Ts, T0=T0, reading=reading,
                pts=pts, nrm=nrm, refp=refp, refn=refn, empty_submap=False)


def track_problems(oracle_mod, pool, count, perts=((0.0, 0.0),)):
    """`count` distinct scan -> sub-map problems cycling over readings 4..13, sub-maps of 2..4 scans and `perts`."""
    out = []
    for j in range(count):
        r, K = 4 + j % 10, 2 + (j // 10) % 3
        dx, dyaw = perts[j % len(perts)]
        out.append(problem(oracle_mod, pool, r, K, dx, dyaw))
    return out


def oracle_result(oracle_mod, pr, kw, want_hist=False):
    if pr["empty_submap"]:
        return dict(rc=1, T=pr["T0"], stats=None)
    po = oracle_mod.default_params(num_threads=THREADS, **kw)
    return oracle_mod.icp(pr["pts"], pr["refp"], pr["refn"], pr["T0"], po, want_hist=want_hist)


def cap_rounds(oracle_mod, pr, r, ratio=0.75):
    """Replay of the kernel's trim-aware search cap (DESIGN §4) on the oracle's iterates: per iteration, the number of
    extra search rounds and whether the last one was uncapped.  The cap starts at 0.04 m^2, is half the first limit in
    the second iteration and twice the previous limit afterwards; a round whose trimmed quantile has no match inside the
    cap is followed by one with a 4x larger cap, and by an uncapped one once the cap has reached 64 m^2."""
    mu = oracle_mod.mean(pr["refp"])
    refc = (pr["refp"][:, :3] - mu).astype(np.float32)
    Tpre = pr["T0"].copy()
    Tpre[:3, 3] -= mu
    rd = oracle_mod.transform_points(Tpre, pr["pts"])
    cap, out = np.float32(0.04), []
    hist = r["T_iter_hist"]
    n = len(pr["pts"])
    rank = min(int(np.float32(n) * np.float32(ratio)), n - 1)     # the limit is the rank-th smallest d2 (from 0)
    for it in range(len(hist)):
        q = rd if it == 0 else oracle_mod.transform_points(hist[it - 1], rd)
        _, d2 = oracle_mod.nn_kdtree(q[:, :3].copy(), refc, THREADS)
        rounds = 0
        while (d2 <= cap).sum() <= rank:                          # the quantile falls among the unmatched queries
            assert np.isfinite(cap), "uncapped and still no quantile: empty map"
            cap = np.float32(cap * 4) if cap < 64 else np.float32(np.inf)
            rounds += 1
        out.append((rounds, not np.isfinite(cap)))
        limit = np.float32(oracle_mod.trim_limit(d2, ratio)[0])
        cap = max(np.float32(limit * np.float32(0.5 if it == 0 else 2.0)), np.float32(1e-12))
    return out


def lattice_problem(dxyz=(0.25, 0.125, 0.0625), pad=4):
    """A 41 x 41 lattice (0.5 m) on the plane z = 0 with normals +z, and a reading on the same lattice, offset by exactly
    representable steps and reaching `pad` lattice steps past two edges: the squared distances take a handful of
    values, the 0.75 quantile falls inside a long run of equal keys, ties between two map points are everywhere
    (x offset of half a step) and the point-to-plane system has rank 3."""
    g = np.arange(41, dtype=np.float32) * np.float32(0.5)
    X, Y = np.meshgrid(g, g, indexing="ij")
    ref = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size, np.float32), np.ones(X.size, np.float32)], 1).astype(np.float32)
    nrm = np.tile(np.array([0, 0, 1], np.float32), (len(ref), 1))
    h = np.arange(-pad, 41, dtype=np.float32) * np.float32(0.5)
    X, Y = np.meshgrid(h, h, indexing="ij")
    rd = np.stack([X.ravel() + np.float32(dxyz[0]), Y.ravel() + np.float32(dxyz[1]),
                   np.full(X.size, np.float32(dxyz[2])), np.ones(X.size, np.float32)], 1).astype(np.float32)
    return dict(name="lattice", reading=("lattice",), pts=rd, nrm=np.tile(np.array([0, 0, 1], np.float32), (len(rd), 1)),
                refp=ref, refn=nrm, ks=None, Ts=[np.eye(4, dtype=np.float32)], T0=np.eye(4, dtype=np.float32),
                empty_submap=False)


def convergence_problems(oracle_mod, pool):
    perts = [(0.0, 0.0), (0.05, 0.25), (0.15, 0.5), (0.3, 1.0), (0.5, 1.5), (0.8, 2.0), (1.0, 2.5), (1.2, 3.0),
             (1.5, 3.5), (1.8, 4.5), (2.0, 5.0), (-1.0, -3.0)]
    # a 33-point reading (one arc of the first ring) never settles and runs into the counter
    return track_problems(oracle_mod, pool, 12, perts) + [
        problem(oracle_mod, pool, 5, 2, reading=("head", 33)),
        problem(oracle_mod, pool, 8, 4, reading=("outliers", 0.4, 40.0), name="40 % of the reading 40 m off")]


def research_problems(oracle_mod, pool):
    return [problem(oracle_mod, pool, 6, 3), problem(oracle_mod, pool, 7, 2, dx=2.0, name="2 m offset"),
            problem(oracle_mod, pool, 8, 4, reading=("outliers", 0.4, 40.0), name="40 % of the reading 40 m off"),
            problem(oracle_mod, pool, 9, 3, dx=0.5, dyaw=1.0)]


# ---- preconditions (CPU, oracle only) --------------------------------------------------------------------------------
def test_precondition_early_convergence_gives_distinct_iteration_counts(oracle_mod, synth_mod, pool):
    """Case C stops its problems in different iterations, some by the differential checker and some by the counter, for
    every smooth_length it runs."""
    for smooth in (4, 1, 15):
        rs = [oracle_result(oracle_mod, pr, dict(smooth_length=smooth)) for pr in convergence_problems(oracle_mod, pool)]
        its = {r["stats"].iterations for r in rs if r["rc"] == 0}
        assert len(its) >= 3, (smooth, its)
        assert any(r["stats"].converged for r in rs), smooth
        assert any(r["stats"].max_iter_reached for r in rs), smooth


def test_precondition_research_reaches_later_iterations_and_the_uncapped_search(oracle_mod, synth_mod, pool):
    """Case D: some problem needs a re-search after iteration 0, and some problem's search ends uncapped; the same with
    trim_ratio 1.0."""
    for ratio in (0.75, 1.0):
        reps = [cap_rounds(oracle_mod, pr, oracle_result(oracle_mod, pr, dict(FIXED, trim_ratio=ratio), want_hist=True), ratio)
                for pr in research_problems(oracle_mod, pool)]
        assert any(rounds > 0 for rep in reps for rounds, _ in rep[1:]), ratio
        assert any(unc for rep in reps for _, unc in rep), ratio
    two_m = cap_rounds(oracle_mod, research_problems(oracle_mod, pool)[1],
                       oracle_result(oracle_mod, research_problems(oracle_mod, pool)[1], FIXED, want_hist=True))
    assert two_m[0][0] >= 2


def test_precondition_lattice_ties_at_the_limit(oracle_mod):
    """Case F: many queries sit exactly at the trimmed limit, so the kept count exceeds the quantile's rank."""
    pr = lattice_problem()
    r = oracle_result(oracle_mod, pr, DEFAULT, want_hist=True)
    assert r["rc"] == 0
    d2 = r["d2_last"]
    limit = np.float32(r["stats"].last_limit)
    assert (d2 == limit).sum() > 1
    assert r["stats"].last_kept == (d2 <= limit).sum() > int(np.float32(len(d2)) * np.float32(0.75)) + 1
    assert len(np.unique(d2)) <= 32


# ---- the device ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bctx():
    """A context of this file's own, so CTA budgets and 160 workspaces never reach the session's context."""
    import laser_slam_b200 as ls
    ctx = ls.Context(0)
    yield ctx
    ctx.close()


class Ring:
    """One scan ring for the whole file: the pool is pushed once, other readings get a slot of their own."""

    def __init__(self, ctx, pool):
        self.mp = ctx.create_map(40, 131072)
        self.sub = [self.mp.push_scan(*s) for s in pool["sub"]]
        self.extra = {}
        self.empty = self.mp.push_scan_filtered(fo.filters_yaml(NOTHING), pool["full"][0][0])
        assert self.empty[1] == 0 and self.mp.scan_size(self.empty[0]) == 0
        self.empty = self.empty[0]

    def stage(self, pr):
        """(reading id, part ids, T_parts, T0) of a problem."""
        key = (pr["reading"], pr["r"]) if "r" in pr else pr["name"]
        if pr["reading"] == ("sub",):
            rid = self.sub[pr["r"]]
        elif pr["reading"] == ("empty",):
            rid = self.empty
        else:
            if key not in self.extra:
                self.extra[key] = self.mp.push_scan(pr["pts"], pr["nrm"])
            rid = self.extra[key]
        if pr["empty_submap"]:
            return (rid, [self.empty], [np.eye(4, dtype=np.float32)], pr["T0"])
        if pr["ks"] is None:
            if ("map", pr["name"]) not in self.extra:
                self.extra[("map", pr["name"])] = self.mp.push_scan(pr["refp"], pr["refn"])
            return (rid, [self.extra[("map", pr["name"])]], pr["Ts"], pr["T0"])
        return (rid, [self.sub[k] for k in pr["ks"]], pr["Ts"], pr["T0"])


@pytest.fixture(scope="module")
def ring(bctx, pool):
    rg = Ring(bctx, pool)
    yield rg
    rg.mp.close()


def _f32bits(x):
    return struct.pack("<f", x)


def _stats_tuple(st):
    return (st.iterations, st.converged, st.max_iter_reached, st.last_kept, _f32bits(st.last_limit))


def check_batch(oracle_mod, ring, probs, kw, hist=0, begin_end=False):
    """One launch of `probs`; every problem equals the oracle and its own single call, bit for bit.  Problem `hist`
    (or none if None) is also compared iteration by iteration and in its final correspondences."""
    import laser_slam_b200 as ls
    pg = ls.default_params(**kw)
    staged = [ring.stage(pr) for pr in probs]
    if begin_end:
        got = ring.mp.begin_batch(staged, pg)()
    else:
        got = ring.mp.register_batch(staged, pg)
    assert len(got) == len(probs)
    for b, (pr, st) in enumerate(zip(probs, staged)):
        r = oracle_result(oracle_mod, pr, kw)
        g = got[b]
        what = f"problem {b}: {pr['name']}"
        assert g["rc"] == r["rc"], what
        assert np.array_equal(g["T"], r["T"]), what + ": final transform differs from the oracle"
        one = ring.mp.register(*st, pg, raise_on_convergence=False)
        assert one["rc"] == g["rc"] and np.array_equal(one["T"], g["T"]), what + ": batch differs from its single call"
        assert _stats_tuple(one["stats"]) == _stats_tuple(g["stats"]), what
        if r["rc"] == 0:
            assert _stats_tuple(g["stats"]) == _stats_tuple(r["stats"]), what
        else:
            assert np.array_equal(g["T"], pr["T0"]), what
        if len(pr["pts"]) == 0 or pr["empty_submap"]:
            assert g["rc"] == ls.LS_ERR_CONVERGENCE and _stats_tuple(g["stats"]) == _stats_tuple(ls.IcpStats()), what
    if hist is not None:
        pr = probs[hist]
        r = oracle_result(oracle_mod, pr, kw, want_hist=True)
        h = ring.mp.register(*staged[hist], pg, want_ids=True, want_hist=True)
        assert r["rc"] == 0 and h["rc"] == 0
        assert np.array_equal(h["T_iter_hist"], r["T_iter_hist"])
        assert np.array_equal(h["ids"], r["ids_hist"][-1]) and np.array_equal(h["d2"], r["d2_last"])
    return got


@pytest.mark.gpu
def test_a_cta_budgets_from_one_cta_per_problem_to_the_full_device(bctx, ring, oracle_mod, pool):
    probs = track_problems(oracle_mod, pool, 8, [(0.0, 0.0), (0.3, 1.0), (-0.2, -0.5), (0.6, 2.0)])
    B = len(probs)
    full = bctx.set_icp_cta_budget(0)
    try:
        # 1, 2 (17 does not divide by 8), 3 CTAs per problem, fewer CTAs than problems (still one each), the device
        for budget in (B, 2 * B + 1, 3 * B, B - 3, full):
            assert bctx.set_icp_cta_budget(budget) == budget
            check_batch(oracle_mod, ring, probs, FIXED, hist=None)
            check_batch(oracle_mod, ring, probs, DEFAULT, hist=None)
        for budget in (1, 2, 3):                       # one problem alone: static schedule on 1, 2, 3 CTAs
            bctx.set_icp_cta_budget(budget)
            check_batch(oracle_mod, ring, probs[1:2], DEFAULT, hist=0)
    finally:
        bctx.set_icp_cta_budget(0)
    assert bctx.set_icp_cta_budget(0) == full


@pytest.mark.gpu
def test_b_the_largest_batch(bctx, ring, oracle_mod, pool):
    import torch
    import laser_slam_b200 as ls
    probs = track_problems(oracle_mod, pool, 140, [(0.0, 0.0), (0.4, 1.0), (1.0, 3.0), (-0.3, -2.0), (2.0, 5.0)])
    probs += research_problems(oracle_mod, pool)
    probs += [problem(oracle_mod, pool, 5, 2, reading=("head", k)) for k in (1, 31, 32, 33, 4097)]
    probs += [problem(oracle_mod, pool, 12, 3, reading=("empty",), name="empty reading")]
    probs += track_problems(oracle_mod, pool, 160 - len(probs), [(0.7, -1.5)])
    assert len(probs) == 160
    free0, total = torch.cuda.mem_get_info()
    check_batch(oracle_mod, ring, probs, dict(max_iterations=30), hist=3)
    free1, _ = torch.cuda.mem_get_info()
    print(f"\n160-problem launch: {(total - free1) / 2**20:.0f} MiB of {total / 2**20:.0f} MiB in use on the device "
          f"({(free0 - free1) / 2**20:.0f} MiB more than before it)")
    staged = [ring.stage(pr) for pr in probs] + [ring.stage(probs[0])]
    with pytest.raises(ls.LsError, match="batch <= 160"):
        ring.mp.register_batch(staged, ls.default_params())


@pytest.mark.gpu
@pytest.mark.parametrize("smooth", [4, 1, 15])
def test_c_problems_leaving_the_loop_in_different_iterations(bctx, ring, oracle_mod, pool, smooth):
    check_batch(oracle_mod, ring, convergence_problems(oracle_mod, pool), dict(smooth_length=smooth), hist=2)


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [0.75, 1.0])
def test_d_research_rounds_under_the_dynamic_schedule(bctx, ring, oracle_mod, pool, ratio):
    probs = research_problems(oracle_mod, pool) + track_problems(oracle_mod, pool, 6, [(0.2, 0.5)])
    check_batch(oracle_mod, ring, probs, dict(FIXED, trim_ratio=ratio), hist=2)
    check_batch(oracle_mod, ring, probs, dict(trim_ratio=ratio), hist=1)


@pytest.mark.gpu
def test_e_empty_and_ragged_problems_in_one_launch(bctx, ring, oracle_mod, pool):
    empty_sub = problem(oracle_mod, pool, 10, 2, name="empty sub-map")
    empty_sub["empty_submap"] = True
    probs = [problem(oracle_mod, pool, 4, 3),
             problem(oracle_mod, pool, 12, 3, reading=("empty",), name="empty reading"),
             *[problem(oracle_mod, pool, 5 + j % 3, 2, reading=("head", k)) for j, k in enumerate((1, 31, 32, 33, 4097))],
             empty_sub,
             problem(oracle_mod, pool, 13, 4, reading=("full",), name="full scan"),
             problem(oracle_mod, pool, 9, 2, dx=0.3)]
    for kw in (DEFAULT, FIXED):
        check_batch(oracle_mod, ring, probs, kw, hist=0)
        check_batch(oracle_mod, ring, probs, kw, hist=None, begin_end=True)
    # a batch of empty problems only launches nothing and keeps every initial guess
    check_batch(oracle_mod, ring, [probs[1], empty_sub, probs[1]], DEFAULT, hist=None)
    check_batch(oracle_mod, ring, [empty_sub], DEFAULT, hist=None, begin_end=True)
    # the context is free afterwards
    check_batch(oracle_mod, ring, probs[:1], FIXED, hist=0)


@pytest.mark.gpu
def test_f_ties_at_the_trimmed_limit(bctx, ring, oracle_mod, pool):
    lat = [lattice_problem(), lattice_problem((0.25, 0.25, -0.125), pad=6)]
    lat[1]["name"] = "lattice 2"
    for kw in (DEFAULT, FIXED):
        check_batch(oracle_mod, ring, lat[:1], kw, hist=0)                      # alone: static schedule
        check_batch(oracle_mod, ring, lat + track_problems(oracle_mod, pool, 3), kw, hist=1)


@pytest.mark.gpu
def test_g_estimator_keeps_the_guess_of_a_track_whose_scan_is_filtered_to_nothing(oracle_mod, synth_mod, tmp_path):
    """host.Estimator with two workers and an input-filter file: in the last step worker 1's raw scan lies entirely
    inside the MinDist radius (a blocked sensor).  That worker keeps its odometry guess, worker 0 registers as usual
    (both in one batched launch), and each track equals the per-scan oracle flow."""
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    from test_host_layer import oracle_flow
    o = oracle_mod
    n_scans, K, W = 5, 3, 2
    chain = [("RemoveNaNDataPointsFilter", {}), ("MinDistDataPointsFilter", {"minDist": 1.0}),
             ("MaxDistDataPointsFilter", {"maxDist": 60.0}), ("SurfaceNormalDataPointsFilter", {"knn": 10})]
    path = tmp_path / "input_filters.yaml"
    path.write_text(fo.filters_yaml(chain))
    raw, filt, odom7 = [], [], []
    for w in range(W):
        truth, odom = synth_mod.trajectory(w + 1, n_scans)
        raw.append([synth_mod.subsample(*synth_mod.scan(truth[k], w + 1, k), 16)[0].copy() for k in range(n_scans)])
        odom7.append(pg.se3_from_matrix(odom))
    blocked = raw[1][-1].copy()
    blocked[:, :3] *= np.float32(0.5) / np.linalg.norm(blocked[:, :3], axis=1, keepdims=True).astype(np.float32)
    raw[1][-1] = blocked
    for w in range(W):
        filt.append([fo.apply_filters(chain, p) for p in raw[w]])
    assert len(filt[1][-1][0]) == 0 and all(len(f[0]) > 1000 for f in filt[0] + filt[1][:-1])
    po = o.default_params(trim_ratio=0.85, min_diff_rot=0.001, min_diff_trans=0.001, smooth_length=3)
    est = host.Estimator(n_workers=W, nscan_in_sub_map=K, icp_input_filters_path=str(path),
                         icp_yaml_path=None)
    got = [[], []]
    for k in range(n_scans):
        feats = [np.ascontiguousarray(raw[w][k]) for w in range(W)]
        icp, st = est.step_batch(list(range(W)), [k * 100_000_000] * W, [odom7[w][k] for w in range(W)],
                                 [f.ctypes.data for f in feats], [0] * W, [len(f) for f in feats])
        for w in range(W):
            got[w].append(icp[w])
    for w in range(W):
        ref_traj, ref_icp = oracle_flow(o, filt[w], odom7[w], K, po)
        g = np.stack(got[w])
        assert np.abs(g[:, 4:] - ref_icp[:, 4:]).max() < 1e-6, w
        _, traj = est.trajectory(w)
        assert np.abs(traj[:, 4:] - ref_traj[:, 4:]).max() < 1e-6, w
    rel = pg.se3_compose(pg.se3_inverse(odom7[1][-2]), odom7[1][-1])        # the odometry guess of the blocked step
    assert np.abs(np.stack(got[1])[-1][4:] - rel[4:]).max() < 1e-5
    assert est.num_scans(1) == n_scans
    est.close()
