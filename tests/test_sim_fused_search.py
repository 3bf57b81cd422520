"""The search and the candidate-list build in one walk (ls_grid.cuh nn_search_collect), on the CPU where the same header
compiles (tests/sim/fused_sim.cpp): its match equals nn_search's on every query, and every list it builds holds exactly
the map points within its radius -- checked by brute force -- or is refused at more than LS_VK of them."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, "sim", "fused_sim.cpp")
SIM_LIB = os.path.join(HERE, "sim", "libfused_sim.so")


@pytest.fixture(scope="module")
def lib():
    deps = [SIM_SRC, os.path.join(HERE, "sim", "grid_sim.cpp")] + [os.path.join(HERE, "..", "laser_slam_b200", "csrc", f) for f in ("ls_grid.cuh", "ls_math.cuh")]
    if not os.path.exists(SIM_LIB) or os.path.getmtime(SIM_LIB) < max(os.path.getmtime(d) for d in deps):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared",
                               "-I/usr/local/cuda/include", "-o", SIM_LIB, SIM_SRC])
    L = ctypes.CDLL(SIM_LIB)
    vp = ctypes.c_void_p
    L.sim_search_collect.restype = ctypes.c_int
    L.sim_search_collect.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int] + [vp] * 12
    L.sim_vlists_paths.restype = ctypes.c_int
    L.sim_vlists_paths.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, vp,
                                   ctypes.c_int, vp, ctypes.c_int, vp, vp, vp, vp, vp, vp]
    return L


def _d2(q, p):
    """fl(fl(fl(dx*dx) + fl(dy*dy)) + fl(dz*dz)) in float32, as the query computes it."""
    d = (p[None, :, :] - q[:, None, :]).astype(np.float32)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _check(L, q, ref, warm, caps, motion, cell=1.0, split=32):
    q = np.ascontiguousarray(q, np.float32)
    ref = np.ascontiguousarray(ref, np.float32)
    n, m = len(q), len(ref)
    warm = np.ascontiguousarray(warm, np.int32)
    caps = np.ascontiguousarray(np.broadcast_to(np.float32(caps), (n,)), np.float32)
    motion = np.ascontiguousarray(np.broadcast_to(np.float32(motion), (n,)), np.float32)
    ids, ref_ids, pos, ref_pos = (np.empty(n, np.int32) for _ in range(4))
    d2, ref_d2, rv = (np.empty(n, np.float32) for _ in range(3))
    vq = np.empty((n, 4), np.float32)
    K = 15
    vpts = np.empty((K, n, 4), np.float32)  # room for any LS_VK
    K = L.sim_search_collect(q.ctypes.data, n, ref.ctypes.data, m, cell, 1 << 22, split, warm.ctypes.data, caps.ctypes.data,
                             motion.ctypes.data, ids.ctypes.data, d2.ctypes.data, pos.ctypes.data, ref_ids.ctypes.data,
                             ref_d2.ctypes.data, ref_pos.ctypes.data, vq.ctypes.data, vpts.ctypes.data, rv.ctypes.data)
    # the search half: exactly nn_search, ties and caps included
    assert np.array_equal(ids, ref_ids) and np.array_equal(pos, ref_pos) and np.array_equal(d2, ref_d2)
    # the list half
    bits = vq[:, 3].view(np.uint32)
    built = rv > 0
    assert (bits[~built] == 0).all()                          # no list wanted: the header is left as it was (zero here)
    assert np.array_equal(vq[built, :3], q[built])            # q0
    full = built & (bits == 0)                                # refused: more than LS_VK points
    listed = built & (bits != 0)
    vp = vpts[:K].transpose(1, 0, 2)                          # n x K x 4, .w = original index
    n_full = n_listed = 0
    for s in range(0, n, 512):
        sl = slice(s, min(n, s + 512))
        dd = _d2(q[sl], ref)
        r2 = (rv[sl] * rv[sl]).astype(np.float32)
        inside = dd <= r2[:, None]
        for j in np.flatnonzero(built[sl]):
            i = s + j
            want = np.flatnonzero(inside[j])
            if full[i]:
                assert len(want) > K, (i, len(want))
                n_full += 1
                continue
            cnt = int(bits[i] & 15)
            # the stored radius is Rv rounded down, then the count bits
            assert bits[i] & ~np.uint32(15) == np.float32(rv[i] * np.float32(0.9999999)).view(np.uint32) & ~np.uint32(15)
            got = vp[i, :cnt, 3].view(np.int32)
            assert cnt == len(want) and np.array_equal(np.sort(got), want), (i, cnt, len(want))
            assert np.array_equal(vp[i, :cnt, :3], ref[got])
            n_listed += 1
    return int(built.sum()), n_listed, n_full


def _lidar(small_pair, oracle_mod):
    mu = oracle_mod.mean(small_pair["ref"])
    refc = (small_pair["ref"][:, :3] - mu).astype(np.float32)
    q = (oracle_mod.transform_points(small_pair["T0"], small_pair["reading"])[:, :3] - mu).astype(np.float32)
    return q, refc


@pytest.mark.parametrize("cap", [np.inf, 0.04, 0.0025])
def test_fused_walk_on_lidar_with_warm_matches(lib, oracle_mod, small_pair, cap):
    """Warm start = the true match of a nearby position (the steady state), and motions that pass or fail the gate."""
    q, refc = _lidar(small_pair, oracle_mod)
    rng = np.random.default_rng(1)
    ib, _ = oracle_mod.nn_brute(q, refc)
    q2 = (q + rng.normal(scale=0.01, size=q.shape)).astype(np.float32)
    motion = rng.choice([0.0, 0.001, 0.01, 0.05, 1.0], size=len(q)).astype(np.float32)
    built, listed, full = _check(lib, q2, refc, ib, cap, motion)
    assert built > len(q) // 4 and listed > 0


def test_fused_walk_random_and_missing_warm_starts(lib, oracle_mod, small_pair):
    """Any map point as the warm start (often far beyond the cap: the 'not found' radius), or none (the seed)."""
    q, refc = _lidar(small_pair, oracle_mod)
    q = q[:3000]
    rng = np.random.default_rng(2)
    for warm in (rng.integers(0, len(refc), len(q)), np.full(len(q), -1)):
        for cap in (np.inf, 0.04):
            built, listed, full = _check(lib, q, refc, warm, cap, 0.002)
            assert listed > 0


def test_fused_walk_ties_on_a_lattice(lib):
    """Integer lattice with duplicates: exact ties inside the search and on the list radius."""
    rng = np.random.default_rng(3)
    g = np.stack(np.meshgrid(np.arange(10), np.arange(10), np.arange(5), indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    ref = np.concatenate([g, g[rng.permutation(len(g))[:200]]]).astype(np.float32)
    q = np.concatenate([g + 0.5, g, g + np.float32(0.25), rng.uniform(-2, 11, (400, 3))]).astype(np.float32)
    for cell, split in [(1.0, 16), (2.0, 32), (0.5, 16)]:
        for warm in (rng.integers(0, len(ref), len(q)), np.full(len(q), -1)):
            for cap, motion in ((np.inf, 0.0), (1.0, 0.01), (0.3, 0.0), (2.0, 0.3)):
                _check(lib, q, ref, warm, cap, motion, cell=cell, split=split)


def test_both_list_paths_reproduce_the_search_over_an_icp_run(lib, oracle_mod, small_pair):
    """Every query of every iteration of a real ICP run, with lists built in the search's walk and in a walk of their
    own: both answer exactly as the plain search, and the lists certify the converged iterations."""
    o = oracle_mod
    r = o.icp(small_pair["reading"], small_pair["ref"], small_pair["ref_normals"], small_pair["T0"],
              o.default_params(max_iterations=20, use_differential=0), want_hist=True)
    mu = o.mean(small_pair["ref"])
    refc = np.ascontiguousarray(small_pair["ref"][:, :3] - mu, np.float32)
    Tpre = small_pair["T0"].copy()
    Tpre[:3, 3] -= mu
    rd = np.ascontiguousarray(o.transform_points(Tpre, small_pair["reading"])[:, :3], np.float32)
    Ts = [np.eye(4, dtype=np.float32)] + [np.asarray(T, np.float32) for T in r["T_iter_hist"][:-1]]
    K, n = len(Ts), len(rd)
    Tcm = np.ascontiguousarray(np.stack([T.T.ravel() for T in Ts]))
    for caps in ([0.25] + [0.02] * (K - 1), [np.inf] * K):
        caps = np.ascontiguousarray(caps, np.float32)
        out = {}
        for fused in (0, 1):
            hits, builds, refused = (np.zeros(K, np.int32) for _ in range(3))
            steps = np.zeros(K, np.int64)
            ids, d2 = np.empty(n, np.int32), np.empty(n, np.float32)
            bad = lib.sim_vlists_paths(rd.ctypes.data, n, refc.ctypes.data, len(refc), 1.0, 1 << 22, 32, Tcm.ctypes.data, K,
                                       caps.ctypes.data, fused, hits.ctypes.data, builds.ctypes.data, refused.ctypes.data,
                                       steps.ctypes.data, ids.ctypes.data, d2.ctypes.data)
            assert bad == 0
            assert hits[0] == 0 and hits[-1] > 0.9 * n, hits
            out[fused] = (ids, steps)
        assert np.array_equal(out[0][0], out[1][0])
        assert out[1][1][1:].sum() < out[0][1][1:].sum()   # one walk instead of two: fewer dependent round trips
