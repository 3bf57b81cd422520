"""Pose-graph solver (laser_slam_b200/csrc/ls_pg.cu) at the graph shapes its structure depends on.

The device solver orders the poses track by track, labels every factor "chain" (between consecutive poses of one track)
or "border" (everything else), solves the chain part by block cyclic reduction over log2 P levels, adds the border
through the Woodbury identity with a dense Cholesky factor in 16-wide panels, damps the first pose of every chain
segment that has no prior, and reuses all of it for the marginals in chunks of 64 poses.  Each of those steps depends on
the graph's shape, so the graphs below are built to hit the edges: every parity of P at every reduction level, track
boundaries and single-pose tracks, reversed / duplicate / skip factors, border counts on both sides of a panel boundary,
marginal queries across the chunk boundary, chain gaps and more poses than one launch grid holds.

References (the oracle's conventions, oracle/posegraph_oracle.py):
  * dense_step: the dense Hessian of pg.hessian (with the damping), the gradient of pg.linearize, numpy.linalg.solve --
    nothing in it depends on cyclic reduction or on Woodbury; for graphs up to about a thousand poses;
  * sparse_step: every factor linearised in one vectorised batch, COO assembly, scipy.sparse.linalg.spsolve; for the
    large graphs, where the oracle's per-factor loop would take minutes.
Both are checked against pg.gauss_newton_step on the CPU.  The device is compared with them after one Gauss-Newton step
from the same values, translations directly and rotations as Log(R_ref^T R_dev), relative to the largest step component.
"""
import re

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import posegraph_oracle as pg

SIG = np.array([0.005] * 3 + [0.0015] * 3)          # odometry / ICP / loop closure (laser_slam's defaults)
PRIOR_SIG = np.array([1e-3] * 3 + [1e-4] * 3)       # tight priors, but no tighter than 1e-4
LOOSE_PRIOR_SIG = np.array([0.05] * 3 + [0.01] * 3)  # GPS-like priors along the large graphs
FIXED_SIG = np.array([0.01] * 3 + [0.003] * 3)
IDENTITY7 = np.array([1.0, 0, 0, 0, 0, 0, 0])

# Bounds on |device - reference| / max|reference step| (+ 1e-12 absolute).  Both sides solve the same float64 normal
# equations; they differ only in the order of the sums (cyclic reduction + Woodbury vs LAPACK / SuperLU), so the
# difference is rounding amplified by the conditioning: a 1e-4 rad prior at one end of a chain of P poses gives
# cond(H) ~ P^2 x 1e3, and a damped segment makes H_c itself nearly singular (the damping is far weaker than any
# factor), which the Woodbury correction then has to cancel.  Largest ratios measured on an H100 SXM 80 GB: 6.2e-9 for
# the damped track of test_anchors_damping_and_key_range (the dense and the sparse reference agree there to 8e-13, so
# this is the device's own rounding; it is deterministic), 1.3e-9 for the 5100-pose reuse graph, 3.2e-10 for the
# 1025-pose chain, 6.4e-11 after three steps, 1.3e-11 for the marginals.  A single 131071-pose chain with one such
# prior reached 6e-6 (cond(H) ~ 1e13, on both sides' rounding alone), so the large graphs carry a prior every 256
# poses.  A wrong coupling, a missed border row or a different damping moves the step by 1e-3 or more.
TOL_STEP = 1e-8          # one step vs the dense or sparse reference
TOL_ITER = 1e-9          # three steps vs pg.optimize (the later steps are smaller; bound relative to the first)
TOL_MARG = 1e-9          # marginal blocks vs numpy.linalg.inv, relative to the largest entry of each block


# ---------------------------------------------------------------- vectorised SE3 on [qw qx qy qz tx ty tz] rows
def quat_mul(p, q):
    pw, px, py, pz = np.moveaxis(p, -1, 0)
    qw, qx, qy, qz = np.moveaxis(q, -1, 0)
    return np.stack([pw * qw - px * qx - py * qy - pz * qz, pw * qx + px * qw + py * qz - pz * qy,
                     pw * qy - px * qz + py * qw + pz * qx, pw * qz + px * qy - py * qx + pz * qw], -1)


def quat_exp(w):
    th = np.linalg.norm(w, axis=-1, keepdims=True)
    small = th < 1e-8
    sc = np.where(small, 0.5 - th * th / 48.0, np.sin(0.5 * th) / np.where(small, 1.0, th))
    return np.concatenate([np.cos(0.5 * th), sc * w], -1)


def se3_mul(A, B):
    q = quat_mul(A[..., :4], B[..., :4])
    t = A[..., 4:] + (pg.quat_to_R(A[..., :4]) @ B[..., 4:, None])[..., 0]
    return np.concatenate([q / np.linalg.norm(q, axis=-1, keepdims=True), t], -1)


def se3_between(A, B):
    """A^-1 B."""
    qa_inv = A[..., :4] * np.array([1.0, -1.0, -1.0, -1.0])
    q = quat_mul(qa_inv, B[..., :4])
    t = (np.swapaxes(pg.quat_to_R(A[..., :4]), -1, -2) @ (B[..., 4:] - A[..., 4:])[..., None])[..., 0]
    return np.concatenate([q / np.linalg.norm(q, axis=-1, keepdims=True), t], -1)


def se3_noise(rng, n, st, sr):
    return np.concatenate([quat_exp(rng.normal(scale=sr, size=(n, 3))), rng.normal(scale=st, size=(n, 3))], -1)


def retract(poses, d):
    """t += dt, R <- R Exp(dr), as pg.retract, without its per-pose loop."""
    q = poses[:, :4] / np.linalg.norm(poses[:, :4], axis=-1, keepdims=True)
    q = quat_mul(q, quat_exp(d[:, 3:]))
    return np.concatenate([q / np.linalg.norm(q, axis=-1, keepdims=True), poses[:, 4:] + d[:, :3]], -1)


def rot_err(A, B):
    return np.abs(pg.so3_log(np.swapaxes(pg.quat_to_R(A[:, :4]), -1, -2) @ pg.quat_to_R(B[:, :4]))).max()


# ---------------------------------------------------------------- graph generator
class Graph:
    """keys / tracks / truth / init in insertion order, factor dicts (pg.make_factor), and what the solver is expected
    to make of them: the number of border factors, the keys it damps and whether it must refuse the graph."""

    def __init__(self, keys, tracks, truth, init, factors):
        self.keys, self.tracks, self.truth, self.init, self.factors = keys, tracks, truth, init, factors
        self.n_border, self.damp, self.free = classify(keys, tracks, factors)

    def subgraph(self, keep_keys, factor_mask=None):
        keep = np.isin(self.keys, np.asarray(list(keep_keys), np.uint64))
        ks = set(int(k) for k in self.keys[keep])
        fac = [f for i, f in enumerate(self.factors) if (factor_mask is None or factor_mask[i])
               and int(f["key_b" if f["type"] == pg.BETWEEN else "key_a"]) in ks
               and (f["type"] == pg.PRIOR or f["fix_a"] or int(f["key_a"]) in ks)]
        return Graph(self.keys[keep], self.tracks[keep], self.truth[keep], self.init[keep], fac)


def classify(keys, tracks, factors):
    """The solver's labelling restated: a between factor from pose k to pose k + 1 of the same track (in insertion
    order) is chain, every other between factor is border; a chain segment is a maximal run of poses joined by chain
    factors; a segment with a prior or a fixed-node factor is anchored, one without but touched by a border factor gets
    its first pose damped, one with neither leaves the gauge free."""
    pos, count = {}, {}
    for k, t in zip(keys.tolist(), tracks.tolist()):
        pos[k] = (t, count.get(t, 0))
        count[t] = count.get(t, 0) + 1
    joined, anchored, linked, n_border = set(), set(), set(), 0
    for f in factors:
        if f["type"] == pg.PRIOR:
            anchored.add(int(f["key_a"]))
        elif f["fix_a"]:
            anchored.add(int(f["key_b"]))
        else:
            (ta, ka), (tb, kb) = pos[int(f["key_a"])], pos[int(f["key_b"])]
            if ta == tb and kb == ka + 1:
                joined.add(int(f["key_b"]))
            else:
                n_border += 1
                linked.update((int(f["key_a"]), int(f["key_b"])))
    by_track = {}
    for k in keys.tolist():
        by_track.setdefault(pos[k][0], []).append(k)
    damp, free = [], []
    for ks in by_track.values():
        segs = []
        for k in ks:
            if k in joined:
                segs[-1].append(k)
            else:
                segs.append([k])
        for s in segs:
            if not anchored.intersection(s):
                (damp if linked.intersection(s) else free).append(s[0])
    return n_border, damp, free


def make_graph(lengths, ids=None, priors=None, fixed=(), extra=(), gaps=(), robust_icp=True, meas_noise=True,
               init_noise=(0.05, 0.01), seed=0, counter0=1000, prior_sigma=PRIOR_SIG):
    """lengths[t] poses in track t, track id ids[t] (default t), inserted round-robin across the tracks (time order is
    kept inside a track) with laser_slam's keys (track_id << 48 | global counter, LaserTrack::extendTrajectory).
      priors : (t, k, robust) -- default: one prior on the first pose of every track
      fixed  : (t, k)         -- a between factor from a fixed pose outside the graph (fix_a) to pose k of track t
      extra  : ((ta, ka), (tb, kb), robust) -- between factors besides the odometry (loop closures, skips, reversed...)
      gaps   : (t, k)         -- no odometry between poses k - 1 and k of track t
    Odometry: one factor between consecutive poses and, with robust_icp, a second (Cauchy) one on every third edge."""
    rng = np.random.default_rng(seed)
    T = len(lengths)
    ids = list(range(T)) if ids is None else list(ids)
    priors = [(t, 0, 0) for t in range(T)] if priors is None else list(priors)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    P = int(off[-1])
    # smooth trajectories (closed form, so this stays vectorised at 200000 poses): a heading that turns slowly, a small
    # roll / pitch wobble, 0.5 m between poses; each track starts at its own random pose
    truth = np.zeros((P, 7))
    for t in range(T):
        k = np.arange(lengths[t], dtype=np.float64)
        yaw = 0.02 * k
        wob = np.stack([0.05 * np.sin(0.07 * k), 0.04 * np.cos(0.05 * k), np.zeros_like(k)], -1)
        q = quat_mul(quat_exp(np.stack([np.zeros_like(k), np.zeros_like(k), yaw], -1)), quat_exp(wob))
        x = np.stack([25.0 * np.sin(yaw), 25.0 * (1.0 - np.cos(yaw)), 0.3 * np.sin(0.03 * k)], -1)
        start = np.concatenate([quat_exp(rng.normal(scale=0.3, size=(1, 3))), rng.normal(scale=20.0, size=(1, 3))], -1)
        truth[off[t]:off[t + 1]] = se3_mul(np.broadcast_to(start, (lengths[t], 7)), np.concatenate([q, x], -1))
    counter = counter0 + np.arange(P, dtype=np.uint64)
    track_of = np.repeat(np.arange(T), lengths)
    keys = np.array([((int(ids[t]) << 48) & 0xFFFFFFFFFFFFFFFF) | int(c) for t, c in zip(track_of, counter)], np.uint64)

    def idx(t, k):
        k = k if k >= 0 else lengths[t] + k
        assert 0 <= k < lengths[t]
        return int(off[t] + k)

    def noisy(m, st=0.004, sr=0.001):
        return se3_mul(m, se3_noise(rng, len(m), st, sr)) if meas_noise else m

    factors = []
    for (t, k, rob) in priors:
        i = idx(t, k)
        factors.append(pg.make_factor(pg.PRIOR, keys[i], keys[i], noisy(truth[i:i + 1])[0], prior_sigma, robust=rob))
    gapset = set((t, k if k >= 0 else lengths[t] + k) for t, k in gaps)
    ia, ib, rob = [], [], []
    for t in range(T):
        for k in range(1, lengths[t]):
            if (t, k) in gapset:
                continue
            ia.append(off[t] + k - 1); ib.append(off[t] + k); rob.append(0)
            if robust_icp and k % 3 == 0:
                ia.append(off[t] + k - 1); ib.append(off[t] + k); rob.append(1)
    for (a, b, r) in extra:
        ia.append(idx(*a)); ib.append(idx(*b)); rob.append(r)
    ia, ib = np.asarray(ia, np.int64), np.asarray(ib, np.int64)
    if len(ia):
        meas = noisy(se3_between(truth[ia], truth[ib]))
        sig = np.broadcast_to(SIG, (len(ia), 6))
        factors += [dict(type=pg.BETWEEN, key_a=int(keys[a]), key_b=int(keys[b]), meas=m, sigma=s, robust=int(r), fix_a=0,
                         fixed_a=IDENTITY7) for a, b, m, s, r in zip(ia, ib, meas, sig, rob)]
    for (t, k) in fixed:
        i = idx(t, k)
        anchor = se3_mul(truth[i:i + 1], se3_noise(rng, 1, 1.0, 0.1))
        m = noisy(se3_between(anchor, truth[i:i + 1]))[0]
        factors.append(pg.make_factor(pg.BETWEEN, keys[idx(t, 0)], keys[i], m, FIXED_SIG, fix_a=1, fixed_a7=anchor[0]))
    init = se3_mul(truth, se3_noise(rng, P, *init_noise))
    # insertion order: round-robin across the tracks, time order inside each
    rank = np.concatenate([np.arange(n) for n in lengths])
    order = np.lexsort((track_of, rank))
    return Graph(keys[order], np.asarray(ids, np.uint32)[track_of[order]], truth[order], init[order], factors)


def random_links(rng, lengths, n, first=None):
    """n border factors between random poses (pose a from index first[t] on), robust or not at random."""
    out = []
    while len(out) < n:
        ta, tb = int(rng.integers(len(lengths))), int(rng.integers(len(lengths)))
        ka = int(rng.integers(0 if first is None else first[ta], lengths[ta]))
        kb = int(rng.integers(lengths[tb]))
        if (ta, ka) != (tb, kb) and not (ta == tb and kb == ka + 1):
            out.append(((ta, ka), (tb, kb), int(rng.integers(2))))
    return out


# ---------------------------------------------------------------- references
def gradient(factors, keys, poses):
    r, Ja, Jb, ia, ib, _ = pg.linearize(factors, keys, poses)
    g = np.zeros((len(keys), 6))
    np.add.at(g, ib, np.einsum("fmi,fm->fi", Jb, r))
    m = ia >= 0
    np.add.at(g, ia[m], np.einsum("fmi,fm->fi", Ja[m], r[m]))
    return g.ravel()


def dense_step(G, poses, damp=None):
    """One Gauss-Newton step with dense linear algebra: H from pg.hessian (with the gauge damping), numpy.linalg.solve."""
    damp = G.damp if damp is None else damp
    H = pg.hessian(G.factors, G.keys, poses, damp)
    d = np.linalg.solve(H, -gradient(G.factors, G.keys, poses)).reshape(-1, 6)
    return retract(poses, d), np.abs(d).max()


class FactorArrays:
    def __init__(self, factors, keys):
        index = {int(k): i for i, k in enumerate(keys)}
        F = len(factors)
        self.prior = np.array([f["type"] == pg.PRIOR for f in factors], bool)
        self.fix_a = np.array([bool(f["fix_a"]) and f["type"] == pg.BETWEEN for f in factors], bool)
        self.robust = np.array([bool(f["robust"]) for f in factors], bool)
        self.ib = np.array([index[int(f["key_a" if f["type"] == pg.PRIOR else "key_b"])] for f in factors], np.int64)
        self.ia = np.array([-1 if (f["type"] == pg.PRIOR or f["fix_a"]) else index[int(f["key_a"])] for f in factors],
                           np.int64)
        self.meas = np.stack([f["meas"] for f in factors]).reshape(F, 7)
        self.sigma = np.stack([f["sigma"] for f in factors]).reshape(F, 6)
        self.fixed = np.stack([f["fixed_a"] for f in factors]).reshape(F, 7)


def linearize_batch(fa, poses):
    """pg.linearize for all factors at once (a prior is a between factor from the identity)."""
    T = lambda M: np.swapaxes(M, -1, -2)
    A = poses[np.maximum(fa.ia, 0)].copy()
    A[fa.fix_a] = fa.fixed[fa.fix_a]
    A[fa.prior] = IDENTITY7
    B = poses[fa.ib]
    Rm, Ra, Rb = pg.quat_to_R(fa.meas[:, :4]), pg.quat_to_R(A[:, :4]), pg.quat_to_R(B[:, :4])
    RmT, RaT = T(Rm), T(Ra)
    v = (RaT @ (B[:, 4:] - A[:, 4:])[..., None])[..., 0]
    rt = (RmT @ (v - fa.meas[:, 4:])[..., None])[..., 0]
    rR = pg.so3_log(RmT @ RaT @ Rb)
    Ji = pg.jr_inv(rR)
    F = len(fa.ib)
    Ja, Jb = np.zeros((F, 6, 6)), np.zeros((F, 6, 6))
    Ja[:, :3, :3] = -RmT @ RaT
    Ja[:, :3, 3:] = RmT @ pg.skew(v)
    Ja[:, 3:, 3:] = -Ji @ T(Rb) @ Ra
    Jb[:, :3, :3] = RmT @ RaT
    Jb[:, 3:, 3:] = Ji
    Ja[fa.ia < 0] = 0.0
    r = np.concatenate([rt, rR], -1) / fa.sigma
    Ja, Jb = Ja / fa.sigma[:, :, None], Jb / fa.sigma[:, :, None]
    sw = np.where(fa.robust, np.sqrt(1.0 / (1.0 + (r * r).sum(-1))), 1.0)
    return r * sw[:, None], Ja * sw[:, None, None], Jb * sw[:, None, None]


def sparse_step(G, poses, fa=None):
    """One Gauss-Newton step, vectorised linearisation + COO assembly + scipy.sparse.linalg.spsolve."""
    fa = FactorArrays(G.factors, G.keys) if fa is None else fa
    P = len(G.keys)
    r, Ja, Jb = linearize_batch(fa, poses)
    g = np.zeros((P, 6))
    np.add.at(g, fa.ib, np.einsum("fmi,fm->fi", Jb, r))
    m = fa.ia >= 0
    np.add.at(g, fa.ia[m], np.einsum("fmi,fm->fi", Ja[m], r[m]))
    blk = np.arange(6)
    rows, cols, vals = [], [], []

    def add(i, j, Ji, Jj):
        rows.append(np.broadcast_to((6 * i)[:, None, None] + blk[None, :, None], (len(i), 6, 6)).ravel())
        cols.append(np.broadcast_to((6 * j)[:, None, None] + blk[None, None, :], (len(i), 6, 6)).ravel())
        vals.append(np.einsum("fmi,fmj->fij", Ji, Jj).ravel())

    add(fa.ib, fa.ib, Jb, Jb)
    add(fa.ia[m], fa.ia[m], Ja[m], Ja[m])
    add(fa.ia[m], fa.ib[m], Ja[m], Jb[m])
    add(fa.ib[m], fa.ia[m], Jb[m], Ja[m])
    index = {int(k): i for i, k in enumerate(G.keys)}
    for k in G.damp:
        i = 6 * index[int(k)] + blk
        rows.append(i); cols.append(i); vals.append(np.array([1.0] * 3 + [4.0] * 3))
    H = sp.csc_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * P, 6 * P))
    d = spla.spsolve(H, -g.ravel()).reshape(P, 6)
    return retract(poses, d), np.abs(d).max()


# ---------------------------------------------------------------- device helpers
def device_graph(G, poses=None):
    import laser_slam_b200 as ls
    g = ls.PoseGraph(0)
    g.add_poses(G.keys, G.init if poses is None else poses, G.tracks)
    idx = g.add_factors(G.factors)
    return g, idx


def assert_close(dev, ref, scale, tol, what):
    """|t_dev - t_ref| and |Log(R_ref^T R_dev)| within tol * scale + 1e-12 (scale: the largest reference step)."""
    et, er = np.abs(dev[:, 4:] - ref[:, 4:]).max(), rot_err(ref, dev)
    print(f"[{what}] step {scale:.3e}  rel err t {et / scale:.2e}  r {er / scale:.2e}")
    assert et <= tol * scale + 1e-12, f"{what}: translation differs by {et:.3e} (step {scale:.3e})"
    assert er <= tol * scale + 1e-12, f"{what}: rotation differs by {er:.3e} (step {scale:.3e})"


def check_one_step(G, ref=dense_step, iters3=False, what=""):
    """optimize(1) on the device vs the reference step; with iters3 also optimize(3) vs pg.optimize."""
    g, _ = device_graph(G)
    try:
        st = g.optimize(1)
        assert st.n_border == G.n_border and st.n_poses == len(G.keys) and st.n_factors == len(G.factors)
        k2, est = g.poses()
        assert np.array_equal(k2, G.keys)
        want, scale = ref(G, G.init)
        assert scale > 1e-3                       # a real step, not a fixed point
        assert_close(est, want, scale, TOL_STEP, what or "one step")
        if iters3:
            g.set_poses(G.keys, G.init)
            st = g.optimize(3)
            want3, _ = pg.optimize(G.factors, G.keys, G.init, iters=3, damp_keys=G.damp)
            assert_close(g.poses()[1], want3, scale, TOL_ITER, (what or "") + " x3")
    finally:
        g.close()


# ---------------------------------------------------------------- CPU: the references themselves
def small_mixed_graph():
    """Three tracks (one damped, one anchored by a fixed-node factor only), robust factors, reversed / skip / cross-track
    border factors, duplicate chain factors."""
    return make_graph([6, 5, 4], ids=[9, 3, 0xFFFFFFFF], priors=[(0, 0, 0), (0, 3, 1)], fixed=[(1, 2)],
                      extra=[((0, 4), (0, 3), 1), ((0, 1), (0, 4), 0), ((0, 5), (2, 0), 0), ((2, 3), (1, 0), 1),
                             ((2, 1), (2, 2), 0)], seed=3)


def test_references_match_the_oracle_step():
    G = small_mixed_graph()
    assert G.n_border == 4 and len(G.damp) == 1 and not G.free
    assert int(G.damp[0]) >> 48 == 0xFFFF                      # track 0xFFFFFFFF: its key is >= 2^63
    want, dmax, _ = pg.gauss_newton_step(G.factors, G.keys, G.init, G.damp)
    for ref in (dense_step, sparse_step):
        got, scale = ref(G, G.init)
        assert abs(scale - dmax) <= 1e-10 * dmax
        assert np.abs(got[:, 4:] - want[:, 4:]).max() < 1e-10 and rot_err(got, want) < 1e-10


def test_references_match_the_oracle_on_a_damped_chain_with_loop_closures():
    G = make_graph([30, 20], priors=[(0, 0, 1)], extra=[((0, 5), (1, 3), 1), ((1, 19), (0, 29), 0), ((0, 2), (0, 20), 1)],
                   seed=4)
    assert G.n_border == 3 and len(G.damp) == 1
    want, _, _ = pg.gauss_newton_step(G.factors, G.keys, G.init, G.damp)
    for ref in (dense_step, sparse_step):
        got, _ = ref(G, G.init)
        assert np.abs(got[:, 4:] - want[:, 4:]).max() < 1e-10 and rot_err(got, want) < 1e-10
    r0, Ja0, Jb0, _, _, _ = pg.linearize(G.factors, G.keys, G.init)
    r1, Ja1, Jb1 = linearize_batch(FactorArrays(G.factors, G.keys), G.init)
    assert np.abs(r0 - r1).max() < 1e-12 and np.abs(Ja0 - Ja1).max() < 1e-9 and np.abs(Jb0 - Jb1).max() < 1e-9


def test_classification_model():
    """The generator's own expectations, checked by hand on the shapes the GPU tests use."""
    G = make_graph([4, 4], gaps=[(0, 2)], extra=[((0, 1), (0, 3), 0)], robust_icp=False)
    assert G.n_border == 1 and [int(k) & 0xFFFFFFFFFFFF for k in G.damp] == [1000 + 2] and not G.free
    G = make_graph([4], gaps=[(0, 2)], robust_icp=False)
    assert G.n_border == 0 and not G.damp and [int(k) & 0xFFFFFFFFFFFF for k in G.free] == [1002]
    G = make_graph([3, 3], extra=[((0, 2), (1, 0), 0), ((1, 1), (1, 0), 0), ((1, 0), (1, 1), 0)], robust_icp=False)
    assert G.n_border == 2 and not G.damp
    G = make_graph([3, 2], ids=[7, 1], priors=[(0, 0, 0)], fixed=[(1, 1)], robust_icp=False)
    assert G.n_border == 0 and not G.damp and not G.free
    assert list(G.tracks) == [7, 1, 7, 1, 7]                 # round-robin insertion, time order inside a track


# ---------------------------------------------------------------- GPU: cyclic-reduction shapes
CR_SIZES = [1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025]


@pytest.mark.gpu
@pytest.mark.parametrize("P", CR_SIZES)
def test_cr_single_track(P):
    """One track of P poses: every parity of P at every reduction level; one loop closure from the first to the last
    pose (from P = 3 on) so the last node also carries a border column."""
    extra = [((0, 0), (0, P - 1), 1)] if P >= 3 else []
    G = make_graph([P], extra=extra, seed=P)
    assert G.n_border == len(extra)
    check_one_step(G, iters3=P in (5, 33, 129), what=f"P={P}")


# ---------------------------------------------------------------- GPU: track boundaries
@pytest.mark.gpu
@pytest.mark.parametrize("lengths", [[1, 1, 1], [1, 2, 3, 4, 5], [7, 1, 8], [15, 1, 16], [31, 1, 32], [63, 1, 64],
                                     [127, 1, 128], [2, 1, 1, 2, 1, 3, 1, 1]],
                         ids=lambda v: "-".join(map(str, v)))
def test_track_boundaries(lengths):
    """Tracks of every length around the reduction strides, single-pose tracks with a prior, interleaved insertion of
    unsorted track ids; every other track linked to the next by a loop closure."""
    T = len(lengths)
    ids = [(0x9E3779B1 * (t + 1)) & 0xFFFFFFFF for t in range(T)]       # unsorted, some >= 2^31
    extra = [((t, lengths[t] // 2), (t + 1, -1), 1) for t in range(0, T - 1, 2)]
    G = make_graph(lengths, ids=ids, extra=extra, seed=sum(lengths))
    assert G.n_border == len(extra) and not G.damp
    check_one_step(G, iters3=lengths == [7, 1, 8], what=str(lengths))


@pytest.mark.gpu
def test_anchors_damping_and_key_range():
    """Track ids 5, 0xFFFFFFFF, 2, 17 inserted interleaved (keys >= 2^48, the 0xFFFFFFFF track's >= 2^63):
      5          prior on its first pose, a single-pose track (17) with a prior
      0xFFFFFFFF anchored only by a fixed-node factor: must not be damped
      2          no prior, linked to track 5 by a loop closure: its first pose is damped"""
    G = make_graph([40, 33, 25, 1], ids=[5, 0xFFFFFFFF, 2, 17], priors=[(0, 0, 0), (3, 0, 0)], fixed=[(1, 10)],
                   extra=[((0, 20), (2, 7), 0), ((0, 30), (2, 20), 1), ((2, 24), (3, 0), 0)], seed=11)
    assert G.n_border == 3 and len(G.damp) == 1 and int(G.damp[0]) >> 48 == 2
    assert G.keys.max() >= 1 << 63 and (G.keys >= 1 << 48).all()
    check_one_step(G, iters3=True, what="anchors")
    # the damping is that of the oracle: the same graph without it is a different step
    want_undamped, scale = dense_step(G, G.init, damp=[])
    damped, _ = dense_step(G, G.init)
    assert np.abs(want_undamped[:, 4:] - damped[:, 4:]).max() > 1e3 * (TOL_STEP * scale + 1e-12)


# ---------------------------------------------------------------- GPU: factor classification
@pytest.mark.gpu
def test_factor_classification():
    """Reversed consecutive factor (k+1 -> k: border), duplicate chain factors (chain), skip factors (border), last pose of
    one track to the first of the next in sorted order (adjacent positions, different tracks: border), border factors
    on position 0 and position P-1, a prior on a middle pose, two priors in one track, a robust prior."""
    L = [20, 17, 23]
    extra = [((0, 6), (0, 5), 1),                # reversed consecutive
             ((1, 3), (1, 4), 0), ((1, 3), (1, 4), 1),   # duplicate chain factors
             ((0, 2), (0, 4), 0), ((2, 0), (2, 9), 1),   # skips
             ((0, -1), (1, 0), 0),               # last of track 0 -> first of track 1: adjacent after sorting
             ((1, -1), (2, 0), 1),               # same for tracks 1 -> 2
             ((0, 0), (2, -1), 0),               # position 0 <-> position P-1
             ((2, -1), (0, 0), 1)]
    G = make_graph(L, ids=[1, 2, 3], priors=[(0, 0, 0), (1, 8, 1), (2, 0, 0), (2, 11, 0)], extra=extra, seed=21)
    assert G.n_border == 7 and not G.damp
    check_one_step(G, iters3=True, what="classification")


# ---------------------------------------------------------------- GPU: border sizes (16-wide panels of 6 E rows)
@pytest.mark.gpu
@pytest.mark.parametrize("E", [0, 1, 2, 3, 8, 11, 16, 43])
def test_border_sizes(E):
    """6 E rows padded to 16: 0 (no border solve), 6 / 12 (one padded panel), 18 (two panels, one trailing update),
    48 / 96 (exact multiples of 16), 66 and 258 (padded, several panels and trailing updates)."""
    L = [70, 60]
    extra = random_links(np.random.default_rng(100 + E), L, E)
    G = make_graph(L, extra=extra, seed=200 + E)
    assert G.n_border == E
    check_one_step(G, iters3=E in (3, 43), what=f"E={E}")


# ---------------------------------------------------------------- GPU: marginals
def marginal_graph():
    """Tracks with and without border factors: 0 prior + loop closures (one ends on its last pose), 1 anchored by a
    fixed-node factor only, 2 no prior (damped), 3 prior and no border factor."""
    return make_graph([40, 50, 45, 30], ids=[4, 1, 9, 6], priors=[(0, 0, 0), (3, 0, 0)], fixed=[(1, 0)],
                      extra=[((0, 3), (0, -1), 1), ((2, 10), (0, -1), 0), ((1, 20), (2, 5), 1), ((2, -1), (0, 12), 0),
                             ((1, -1), (1, 30), 0)], seed=31)


@pytest.mark.gpu
@pytest.mark.parametrize("nq", [1, 63, 64, 65, 129])
def test_marginals(nq):
    """nq keys (across the 64-key chunks) spread over all four tracks, before any optimize, vs numpy.linalg.inv of the
    dense Hessian at the same values; the last query repeats an earlier key."""
    G = marginal_graph()
    assert G.n_border == 5 and len(G.damp) == 1
    rng = np.random.default_rng(nq)
    q = G.keys[rng.permutation(len(G.keys))[:nq]]
    if nq > 1:
        q[-1] = q[0]
    g, _ = device_graph(G)
    try:
        got = g.marginals(q)
        assert np.array_equal(g.poses()[1], G.init)          # marginals do not move the estimate
    finally:
        g.close()
    C = np.linalg.inv(pg.hessian(G.factors, G.keys, G.init, G.damp))
    index = {int(k): i for i, k in enumerate(G.keys)}
    want = np.stack([C[6 * index[int(k)]:6 * index[int(k)] + 6, 6 * index[int(k)]:6 * index[int(k)] + 6] for k in q])
    rel = np.abs(got - want).max(axis=(1, 2)) / np.abs(want).max(axis=(1, 2))
    print(f"[marginals nq={nq}] rel err {rel.max():.2e}")
    assert rel.max() <= TOL_MARG
    if nq > 1:
        assert np.array_equal(got[-1], got[0])


@pytest.mark.gpu
def test_marginals_every_pose_of_each_track_after_optimize():
    """All poses of the graph after two iterations (three chunks, the last partial), every track's last pose included."""
    G = marginal_graph()
    g, _ = device_graph(G)
    try:
        g.optimize(2)
        est = g.poses()[1]
        got = g.marginals(G.keys)
    finally:
        g.close()
    C = np.linalg.inv(pg.hessian(G.factors, G.keys, est, G.damp))
    want = np.stack([C[6 * i:6 * i + 6, 6 * i:6 * i + 6] for i in range(len(G.keys))])
    rel = np.abs(got - want).max(axis=(1, 2)) / np.abs(want).max(axis=(1, 2))
    print(f"[marginals all] rel err {rel.max():.2e}")
    assert rel.max() <= TOL_MARG


# ---------------------------------------------------------------- GPU: one graph object across calls
@pytest.mark.gpu
def test_graph_reuse_across_calls():
    """Optimise, remove border factors, then grow P past the buffers' earlier capacity (P + P/4 + 64): every call against
    a fresh reference, so a stale device buffer would show; two identical calls give bit-identical poses."""
    L0, L1 = [1500, 1200, 900], [2000, 1700, 1400]
    rng = np.random.default_rng(41)
    extra = random_links(rng, L0, 14) + random_links(rng, L1, 9, first=L0)   # the last 9 need the grown tracks
    full = make_graph(L1, ids=[12, 7, 30], extra=extra, seed=42)
    rank = {}
    keep = []
    for k, t in zip(full.keys.tolist(), full.tracks.tolist()):
        rank[t] = rank.get(t, -1) + 1
        if rank[t] < L0[[12, 7, 30].index(t)]:
            keep.append(k)
    G0 = full.subgraph(keep)
    assert G0.n_border == 14 and len(G0.keys) == sum(L0) and sum(L1) > 1.25 * sum(L0) + 64
    import laser_slam_b200 as ls
    g = ls.PoseGraph(0)
    try:
        g.add_poses(G0.keys, G0.init, G0.tracks)
        idx = g.add_factors(G0.factors)
        st = g.optimize(1)
        want, scale = sparse_step(G0, G0.init)
        assert st.n_border == G0.n_border
        assert_close(g.poses()[1], want, scale, TOL_STEP, "reuse: first")
        # remove five of the loop closures
        border = [i for i, f in enumerate(G0.factors) if f["type"] == pg.BETWEEN and not f["fix_a"]][-14:]
        gone = set(border[::3])
        g.remove_factors(idx[sorted(gone)])
        G1 = Graph(G0.keys, G0.tracks, G0.truth, G0.init, [f for i, f in enumerate(G0.factors) if i not in gone])
        assert G1.n_border == 14 - len(gone)
        g.set_poses(G0.keys, G0.init)
        st = g.optimize(1)
        want, scale = sparse_step(G1, G1.init)
        assert st.n_border == G1.n_border
        assert_close(g.poses()[1], want, scale, TOL_STEP, "reuse: removed")
        # grow to the full graph (the removed loop closures stay removed)
        have = set(int(k) for k in G0.keys)
        new = np.array([k not in have for k in full.keys.tolist()])
        g.add_poses(full.keys[new], full.init[new], full.tracks[new])
        old_ids = {id(f) for f in G0.factors}
        g.add_factors([f for f in full.factors if id(f) not in old_ids])
        gone_ids = {id(G0.factors[i]) for i in gone}
        G2 = Graph(full.keys, full.tracks, full.truth, full.init, [f for f in full.factors if id(f) not in gone_ids])
        assert G2.n_border == 23 - len(gone)
        # the device keeps insertion order: the original poses first, then the new ones
        order = np.concatenate([np.flatnonzero(~new), np.flatnonzero(new)])
        G2 = Graph(G2.keys[order], G2.tracks[order], G2.truth[order], G2.init[order], G2.factors)
        g.set_poses(G2.keys, G2.init)
        st = g.optimize(1)
        want, scale = sparse_step(G2, G2.init)
        assert st.n_border == G2.n_border and st.n_poses == len(G2.keys)
        k2, est = g.poses()
        assert np.array_equal(k2, G2.keys)
        assert_close(est, want, scale, TOL_STEP, "reuse: grown")
        g.set_poses(G2.keys, G2.init)
        g.optimize(1)
        assert np.array_equal(g.poses()[1], est)
    finally:
        g.close()


# ---------------------------------------------------------------- GPU: refusals and chain gaps
@pytest.mark.gpu
def test_pose_without_factors_is_refused():
    import laser_slam_b200 as ls
    G = make_graph([12, 9], extra=[((0, 3), (1, 4), 1)], seed=51)
    g, _ = device_graph(G)
    try:
        lone = np.uint64((1 << 48) | 999999)
        g.add_poses([lone], G.init[:1], [int(G.tracks[0])])
        before = g.poses()
        with pytest.raises(ls.LsError, match=str(int(lone))):
            g.optimize(1)
        after = g.poses()
        assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    finally:
        g.close()


@pytest.mark.gpu
def test_chain_gap_bridged_by_a_skip_factor():
    """Removing the odometry between poses 14 and 15 leaves a skip factor 13 -> 16 bridging the gap: poses 15.. are a
    chain segment of their own, without prior but linked, so its first pose is damped -- the solution of the oracle
    with the damping at the segment head."""
    G = make_graph([40], extra=[((0, 13), (0, 16), 0)], robust_icp=False, seed=61)
    g, idx = device_graph(G)
    try:
        odo = [i for i, f in enumerate(G.factors) if f["type"] == pg.BETWEEN and
               (int(f["key_b"]) & 0xFFFFFFFFFFFF) == 1000 + 15 and (int(f["key_a"]) & 0xFFFFFFFFFFFF) == 1000 + 14]
        assert len(odo) == 1
        g.remove_factors(idx[odo])
        H = Graph(G.keys, G.tracks, G.truth, G.init, [f for i, f in enumerate(G.factors) if i != odo[0]])
        assert H.n_border == 1 and [int(k) & 0xFFFFFFFFFFFF for k in H.damp] == [1015]
        st = g.optimize(1)
        want, scale = dense_step(H, H.init)
        assert st.n_border == 1
        assert_close(g.poses()[1], want, scale, TOL_STEP, "gap")
        g.set_poses(H.keys, H.init)
        g.optimize(3)
        want3, _ = pg.optimize(H.factors, H.keys, H.init, iters=3, damp_keys=H.damp)
        assert_close(g.poses()[1], want3, scale, TOL_ITER, "gap x3")
    finally:
        g.close()


@pytest.mark.gpu
def test_pose_linked_only_by_border_factors():
    """A pose in the middle of a track whose only factors are loop closures: a one-pose segment, damped."""
    G = make_graph([20, 15], gaps=[(0, 8), (0, 9)], extra=[((1, 3), (0, 8), 0), ((0, 8), (0, 12), 1)], seed=71)
    assert G.n_border == 2 and len(G.damp) == 2               # pose 8 and the segment 9.. of track 0
    check_one_step(G, iters3=True, what="border-only pose")


@pytest.mark.gpu
def test_unlinked_segment_is_refused_naming_its_first_pose():
    import laser_slam_b200 as ls
    G = make_graph([20], gaps=[(0, 11)], seed=81)
    assert len(G.free) == 1
    g, _ = device_graph(G)
    try:
        with pytest.raises(ls.LsError, match=re.escape(str(int(G.free[0])))):
            g.optimize(1)
        assert np.array_equal(g.poses()[1], G.init)
    finally:
        g.close()


@pytest.mark.gpu
def test_border_limit_is_refused_before_allocation():
    """10921 border factors would need a 65536-row dense border system (gridDim.y is at most 65535 rows, 10920
    factors): refused with the limit in the message, before any device buffer is sized for it."""
    import laser_slam_b200 as ls
    P = 10922
    G = make_graph([P], extra=[((0, k), (0, k + 2), 0) for k in range(P - 2)] + [((0, 0), (0, 3), 0)], robust_icp=False,
                   meas_noise=False, seed=91)
    assert G.n_border == 10921
    g, _ = device_graph(G)
    try:
        with pytest.raises(ls.LsError, match="10920"):
            g.optimize(1)
    finally:
        g.close()


# ---------------------------------------------------------------- GPU: more poses than one launch grid row holds
@pytest.mark.gpu
@pytest.mark.parametrize("lengths,n_lc", [([131071], 0), ([90000, 70001, 39999], 10)], ids=["P131071", "P200000"])
def test_large_graphs(lengths, n_lc):
    """P = 131071 (level 0 has 65536 eliminated nodes: one more than gridDim.y allows) and three tracks of 200000 poses
    with about ten loop closures: one step vs the sparse reference; then, from truth plus small independent noise and
    noise-free measurements, five iterations return to truth."""
    T = len(lengths)
    extra = random_links(np.random.default_rng(sum(lengths)), lengths, n_lc)
    priors = [(t, k, 0) for t in range(T) for k in range(0, lengths[t], 256)]     # GPS-like: keeps cond(H) ~ 1e6
    kw = dict(ids=[3, 1, 2][:T], priors=priors, prior_sigma=LOOSE_PRIOR_SIG, extra=extra, robust_icp=False)
    G = make_graph(lengths, seed=len(lengths), **kw)
    assert G.n_border == n_lc
    check_one_step(G, ref=sparse_step, what=f"P={sum(lengths)}")
    C = make_graph(lengths, meas_noise=False, init_noise=(0.01, 0.002), seed=len(lengths), **kw)
    g, _ = device_graph(C)
    try:
        g.optimize(5)
        est = g.poses()[1]
    finally:
        g.close()
    assert np.abs(est[:, 4:] - C.truth[:, 4:]).max() < 1e-8 and rot_err(est, C.truth) < 1e-8
