"""The map build and the reading sort (count0 / count1 / scatter, q_count / q_scatter in ls_kernels.cuh) at the point
layouts their warp-aggregated counters depend on: lanes of one warp that share a counter form one group, take one atomic
and split its slots by rank.  So the cases are the layouts that make those groups large, ragged or trivial: every point in
one fine cell (duplicates included), runs of 32 consecutive points in one level-0 cell (aligned to a warp and straddling
two), cells holding exactly leaf_split and leaf_split + 1 points, one point per cell, a ragged batch of many problems, and
a reading whose points share a few cells.

Every case compares the registration bit for bit with `oracle.icp` (transform, per-iteration transforms, correspondences)
and the grid statistics with a CPU count made with the same float32 cell expressions (test_grid_shapes.device_grid)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_grid_shapes import cell_counts, device_grid, homog, leaf_blocks, sim  # noqa: E402,F401

F32 = np.float32
SPLIT = 32          # the device's default leaf_split
PARAMS = dict(max_iterations=8, use_differential=0)


def normals(n, seed):
    v = np.random.default_rng(seed).normal(size=(n, 3))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(F32)


def near(pts3, seed, sigma=0.02, count=None):
    """A reading: points of the map (or `count` of them) moved by a little noise."""
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, len(pts3), count) if count else np.arange(len(pts3))
    return homog((pts3[idx] + rng.normal(0, sigma, (len(idx), 3))).astype(F32))


def one_fine_cell():
    """300 points inside one 12.5 cm fine cell, a third of them duplicates; the level-0 cell holds them all (> split)."""
    rng = np.random.default_rng(1)
    p = rng.uniform(0.02, 0.10, (200, 3))
    return np.concatenate([p, p[:100]]).astype(F32)


def runs_of_32(head):
    """64 runs of 32 consecutive points, each run inside its own level-0 cell (exactly split points: leaves).  `head`
    points come first in a cell of their own, among them the origin, which pins the lattice to whole metres: with a head
    of 32 the runs are aligned to warps, with 16 every warp straddles two runs."""
    rng = np.random.default_rng(2 + head)
    runs = [np.array([2 + 2 * (c % 8), 2 * ((c // 8) % 4), 2 * (c // 32)], np.float64) + rng.uniform(0.1, 0.9, (32, 3))
            for c in range(64)]
    first = np.concatenate([np.zeros((1, 3)), rng.uniform(0.1, 0.9, (head - 1, 3))])
    return np.concatenate([first] + runs).astype(F32)


def lattice():
    """One point per level-0 cell: the centres of a 16 x 12 x 4 lattice of 1 m cells, and the origin (alone in its cell,
    it pins the lattice to whole metres)."""
    r = [np.arange(1, k + 1, dtype=np.float64) for k in (16, 12, 4)]
    g = np.stack(np.meshgrid(*r, indexing="ij"), -1).reshape(-1, 3) + 0.5
    return np.concatenate([np.zeros((1, 3)), g]).astype(F32)


def blocks():
    pts, counts = leaf_blocks(SPLIT)
    assert {SPLIT, SPLIT + 1} <= set(counts.tolist())
    return pts


def check_grid(sim, oracle_mod, ref3, stats):
    g = device_grid(sim, oracle_mod, ref3)
    assert stats.grid_overflow == 0
    assert stats.grid_cells == g["n_cells0"]
    assert stats.grid_tables == int((cell_counts(g) > g["split"]).sum())


def check_single(gpu_ctx, oracle_mod, sim, reading4, ref3, T0=None):
    import laser_slam_b200 as ls
    T0 = np.eye(4, dtype=F32) if T0 is None else T0
    ref4, nrm = homog(ref3), normals(len(ref3), len(ref3))
    g = gpu_ctx.icp_register(reading4, ref4, nrm, T0, ls.default_params(**PARAMS), want_ids=True, want_hist=True,
                             raise_on_convergence=False)
    r = oracle_mod.icp(reading4, ref4, nrm, T0, oracle_mod.default_params(**PARAMS), want_hist=True)
    assert (g["rc"] == 0) == (r["rc"] == 0)
    assert np.array_equal(g["T"], r["T"])
    assert np.array_equal(g["T_iter_hist"], r["T_iter_hist"])
    if r["rc"] == 0:
        assert np.array_equal(g["ids"], r["ids_hist"][-1])
    check_grid(sim, oracle_mod, ref3, g["stats"])
    return g


# ---- CPU: each layout reaches what it is meant to -----------------------------------------------------------------
def test_precondition_layouts(sim, oracle_mod):
    g = device_grid(sim, oracle_mod, one_fine_cell())
    c = cell_counts(g)
    assert (c > 0).sum() == 1 and c.max() == 300
    fine = np.floor((g["centred"] - g["centred"].min(0)) * (F32(8.0) / g["H0"])).astype(np.int64)
    assert len(np.unique(fine, axis=0)) == 1
    for head in (32, 16):
        g = device_grid(sim, oracle_mod, runs_of_32(head))
        c = cell_counts(g)
        assert sorted(c[c > 0].tolist()) == sorted([head] + [SPLIT] * 64)
    g = device_grid(sim, oracle_mod, lattice())
    assert cell_counts(g).max() == 1
    g = device_grid(sim, oracle_mod, blocks())
    c = cell_counts(g)
    assert {SPLIT, SPLIT + 1} <= set(c.tolist()) and (c > SPLIT).sum() > 0


# ---- the device ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_fine_cell(gpu_ctx, oracle_mod, sim):
    ref = one_fine_cell()
    check_single(gpu_ctx, oracle_mod, sim, near(ref, 10, sigma=0.01, count=200), ref)


@pytest.mark.gpu
@pytest.mark.parametrize("head", [32, 16])
def test_runs_of_32_in_one_cell(gpu_ctx, oracle_mod, sim, head):
    ref = runs_of_32(head)
    check_single(gpu_ctx, oracle_mod, sim, near(ref, 11 + head), ref)


@pytest.mark.gpu
def test_split_and_split_plus_one(gpu_ctx, oracle_mod, sim):
    ref = blocks()
    check_single(gpu_ctx, oracle_mod, sim, near(ref, 12), ref)


@pytest.mark.gpu
def test_one_point_per_cell(gpu_ctx, oracle_mod, sim):
    ref = lattice()
    check_single(gpu_ctx, oracle_mod, sim, near(ref, 13, sigma=0.05), ref)


@pytest.mark.gpu
def test_reading_in_a_few_cells(gpu_ctx, oracle_mod, sim, synth_mod):
    truth, _ = synth_mod.trajectory(0, 2)
    ref, _ = synth_mod.subsample(*synth_mod.scan(truth[0], 0, 0), 8)
    ref3 = ref[:, :3].copy()
    # 3000 reading points from three level-0 cells of the map, many per warp in each
    g = device_grid(sim, oracle_mod, ref3)
    c = cell_counts(g)
    t = np.clip(np.floor((g["centred"] - g["lo"]) * (F32(1.0) / g["H0"])), 0, g["dim"] - 1).astype(np.int64)
    key = (t[:, 2] * g["dim"][1] + t[:, 1]) * g["dim"][0] + t[:, 0]
    busy = np.argsort(c)[-3:]
    src = ref3[np.isin(key, busy)]
    rng = np.random.default_rng(14)
    reading = homog((src[rng.integers(0, len(src), 3000)] + rng.normal(0, 0.01, (3000, 3))).astype(F32))
    check_single(gpu_ctx, oracle_mod, sim, reading, ref3)


@pytest.mark.gpu
def test_ragged_batch(gpu_ctx, oracle_mod, sim, synth_mod):
    """24 problems in one launch: sub-maps of 1..3 scans cut to different lengths, readings of 37 .. 8192 points."""
    import laser_slam_b200 as ls
    truth, odom = synth_mod.trajectory(0, 6, y_start=-20.0)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 0, k), 16) for k in range(6)]
    mp = gpu_ctx.create_map(128, 8192)
    try:
        problems, expect = [], []
        for b in range(24):
            r = 1 + b % 5
            K = 1 + b % 3
            cut = [8192, 5000, 1234, 333][b % 4]
            ks = [max(0, r - 1 - j) for j in range(K)]
            parts = [(scans[k][0][:cut].copy(), scans[k][1][:cut].copy()) for k in ks]
            Ts = [(np.linalg.inv(truth[ks[0]]) @ truth[k]).astype(F32) for k in ks]
            n = [8192, 37, 4000, 777, 2048, 100][b % 6]
            rd = (scans[r][0][:n].copy(), scans[r][1][:n].copy())
            T0 = (np.linalg.inv(truth[ks[0]]) @ odom[r]).astype(F32)
            problems.append((mp.push_scan(*rd), [mp.push_scan(*p) for p in parts], Ts, T0))
            tp = [oracle_mod.transform_cloud(T, *p) for T, p in zip(Ts, parts)]
            refp, refn = np.concatenate([p[0] for p in tp]), np.concatenate([p[1] for p in tp])
            expect.append((oracle_mod.icp(rd[0], refp, refn, T0, oracle_mod.default_params(**PARAMS)), refp[:, :3]))
        got = mp.register_batch(problems, ls.default_params(**PARAMS))
        for b, (g, (r, refp)) in enumerate(zip(got, expect)):
            assert (g["rc"] == 0) == (r["rc"] == 0), b
            assert np.array_equal(g["T"], r["T"]), b
            assert g["stats"].iterations == r["stats"].iterations, b
            check_grid(sim, oracle_mod, refp, g["stats"])
    finally:
        mp.close()
