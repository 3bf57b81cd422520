"""A handle's results must not depend on the calls made on it before.  Each GPU test creates its own context, ring or
occupancy map and runs a scripted sequence of calls on it: sizes exactly at a group's capacity, one past it, smaller
again and larger, parameters that regrow or shrink what the kernels use, and refused or empty calls in between.  After
every call the result is compared bit for bit with the plain reference of that operation (the oracle, or a dict of
log-odds for the occupancy map) and with the same call on a newly created handle.

The capacity boundaries are derived from the growth rules of the library, restated below with the function that owns
each rule; the CPU tests check that the sequences cross them where they say they do."""
import numpy as np
import pytest

import laser_slam_b200 as ls
from oracle import input_filters as fo
from oracle import occupancy as oc
from oracle import octree as ot_oracle
from test_grid_shapes import THREADS, gpu_nn_check, homog, pool_block
from test_input_filters import CHAIN

F32 = np.float32
K0 = 32768


# ---- growth rules (retarget these when the library's rules change) ---------------------------------------------------
def grow(cap, n):
    """Workspace reading and sub-map groups (ensure_capacity), context staging (ensure_staging) and the filter chain's
    ChainBuffers (lsf::reserve): nothing when n fits, else n + n/8 + 1024."""
    return cap if n <= cap else n + n // 8 + 1024


def table_pool(m_cap):
    """Fine tables of a sub-map group of m_cap points (ensure_capacity): cap/17 + 1024, at most 1.5 GB of tables."""
    return min(m_cap // 17 + 1024, (1536 * 1024 * 1024) // (512 * 12))


def stage_need(n, stride):
    """Device normals staging of one ring push (ls_map_push_scan_async): (n-1)*stride + 3 floats, reserved with 1024
    to spare, per staging slot (16 slots, used round-robin)."""
    return (n - 1) * stride + 3


def host_stage_need(n, stride):
    """Pinned host staging of one ring push (ls_map_push_scan): the 4n feature floats and the normals, reserved with
    1024 to spare, per staging slot."""
    return 4 * n + stage_need(n, stride)


STAGE_SPARE, STAGE_RING = 1024, 16


def grow_stage(cap, n, stride, need=stage_need):
    return cap if need(n, stride) <= cap else need(n, stride) + STAGE_SPARE


# Ring rounds (points, normals stride), 16 pushes each so that every staging slot sees them: the device rule exactly at
# its capacity and one past it, then the host rule exactly at its capacity and one past it, then smaller and larger.
RING_ROUNDS = [(936, 3), (548, 7), (767, 5), (842, 5), (758, 6), (936, 3), (2000, 3)]


def nrm_raw_need(m, stride):
    """The context's normals upload of a host reference (upload_normals, strides up to 8): (m-1)*stride + 3 floats,
    reserved with 4096 to spare."""
    return (m - 1) * stride + 3


def grow_nrm_raw(cap, m, stride):
    return cap if nrm_raw_need(m, stride) <= cap else nrm_raw_need(m, stride) + 4096


# Reference sizes and normals strides of the upload sequence: at its capacity, one past it, smaller, larger.
NRM_RAW_STEPS = [(3001, 3), (1638, 8), (1872, 7), (1000, 3), (4000, 5)]


def pg_grow(cap, n):
    """The pose graph's per-factor and per-pose groups (pg_run in ls_pg.cu): nothing when n fits, else n + n/4 + 64."""
    return cap if n <= cap else n + n // 4 + 64


POOL_BYTES_PER_BRICK = 512 * 4 + 48 * 4 + 8 + 4 + 4   # lso::device_bytes: log-odds, three mark words, key, touched, list
TABLE_BYTES_PER_SLOT = 8 + 4                          # lso::device_bytes: key and value per hash slot
MAX_PROBE = 64                                        # kMaxProbe of ls_occupancy.cu (insert and find_brick)


def first_table(initial_bricks):
    """lso::init: 1024 slots, doubled until the table is at least twice the initial pool."""
    cap = 1024
    while cap < 2 * initial_bricks:
        cap *= 2
    return cap


def pool_after(initial_bricks, n_bricks):
    """The occupancy pool after bricks arrive one per insert: doubled on each pool overflow (insert's retry loop)."""
    cap = initial_bricks
    while cap < n_bricks:
        cap *= 2
    return cap


# ---- the occupancy hash, restated ------------------------------------------------------------------------------------
M64 = (1 << 64) - 1


def hash64_int(k):
    """hash64 of ls_occupancy.cu on Python integers (MurmurHash3's 64-bit finaliser, truncated to 32 bits)."""
    k ^= k >> 33
    k = (k * 0xff51afd7ed558ccd) & M64
    k ^= k >> 33
    k = (k * 0xc4ceb9fe1a85ec53) & M64
    k ^= k >> 33
    return k & 0xffffffff


def hash64(k):
    k = np.asarray(k, np.uint64).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xff51afd7ed558ccd)
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xc4ceb9fe1a85ec53)
        k ^= k >> np.uint64(33)
    return (k & np.uint64(0xffffffff)).astype(np.uint32)


def brick_key(b):
    b = np.asarray(b, np.uint64)
    return b[..., 0] | (b[..., 1] << np.uint64(13)) | (b[..., 2] << np.uint64(26))


def colliding_bricks(count=130, bits=12, radius=48):
    """`count` bricks near the origin whose hashes share their low `bits` bits with the origin brick's, nearest first
    (Chebyshev distance, then brick key): a linear-probed table of up to 2^bits slots puts them all in one run."""
    r = np.arange(-radius, radius + 1)
    b = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3) + K0 // 8
    h = hash64(brick_key(b)) & np.uint32((1 << bits) - 1)
    target = hash64(brick_key(np.array([K0 // 8] * 3))) & np.uint32((1 << bits) - 1)
    b = b[h == target]
    order = np.lexsort((brick_key(b), np.abs(b - K0 // 8).max(1)))
    assert len(b) >= count
    return b[order[:count]]


def _pack(k):
    return int(k[0]) | (int(k[1]) << 16) | (int(k[2]) << 32)


RES = 0.1


def brick_voxel(b):
    """A voxel inside brick b (its (3,3,3) voxel) and that voxel's centre."""
    k = np.asarray(b, np.int64) * 8 + 3
    return k, ((k - K0).astype(np.float64) + 0.5) * RES


def one_voxel_scan(b):
    """Brick b as a scan: one point 0.017 m from an origin inside the same voxel, so the ray marks no free cell."""
    k, c = brick_voxel(b)
    T = np.eye(4, dtype=F32)
    T[:3, 3] = c.astype(F32)
    return np.array([[0.01, 0.01, 0.01, 1]], F32), T, _pack(k)


# ---- CPU: the restatements and the sequences' assumptions --------------------------------------------------------------
FMIX64_1 = 0xb456bcfc34c2cb2c   # MurmurHash3's fmix64(1), the published value


def test_hash64_restatement():
    keys = [0, 1, 2, 4096 | (4096 << 13) | (4096 << 26), (1 << 39) - 1, M64, 0x123456789abcdef]
    assert hash64_int(0) == 0 and int(hash64(np.array([0], np.uint64))[0]) == 0
    assert hash64_int(1) == FMIX64_1 & 0xffffffff == int(hash64(np.array([1], np.uint64))[0])
    assert [int(x) for x in hash64(np.array(keys, np.uint64))] == [hash64_int(k) for k in keys]
    rng = np.random.default_rng(5)
    ks = rng.integers(0, 1 << 39, 2000, dtype=np.uint64)
    assert [int(x) for x in hash64(ks)] == [hash64_int(int(k)) for k in ks]
    assert hash64_int(1) != hash64_int(2) and hash64_int(1) < (1 << 32)


def test_colliding_bricks_are_realisable():
    b = colliding_bricks()
    assert len(b) == 130 and len({tuple(x) for x in b}) == 130
    h = hash64(brick_key(b))
    assert len(set((h & 0xfff).tolist())) == 1                     # one run in every table of up to 4096 slots
    assert ((b >= 0) & (b < 8192)).all()                           # 13-bit brick coordinates
    for x in b[:10].tolist() + b[-10:].tolist():
        pts, T, key = one_voxel_scan(x)
        p = pts[0, :3].astype(F32) + T[:3, 3]
        kp = np.floor(p.astype(np.float64) * (1.0 / RES)).astype(np.int64) + K0
        ko = np.floor(T[:3, 3].astype(np.float64) * (1.0 / RES)).astype(np.int64) + K0
        assert _pack(kp) == _pack(ko) == key and np.array_equal(kp >> 3, x)
    # 64 of them fill a run of 1024, 2048 and 4096 slots: the 65th forces the table to at least 8192
    assert MAX_PROBE + 1 <= len(b) and first_table(256) == first_table(16) == first_table(17) == 1024


def test_sequence_boundaries():
    # the ICP sequences: s = 3000, exactly c(s), c(s) + 1, s/3, then one past each later capacity
    assert grow(0, 3000) == 4399 and grow(4399, 4399) == 4399 and grow(4399, 4400) == 5974
    assert grow(5974, 1000) == 5974 and grow(5974, 5974) == 5974 and grow(5974, 5975) == 7745 and 7746 <= 8192
    assert table_pool(grow(0, len(pool_block()))) == 262144
    # ring staging rounds: device rule at / one past its capacity, then host rule at / one past its capacity
    dev = host = 0
    hits = []
    for n, s in RING_ROUNDS:
        hits.append((stage_need(n, s) - dev, host_stage_need(n, s) - host))
        dev, host = grow_stage(dev, n, s), grow_stage(host, n, s, host_stage_need)
    assert [h for h, _ in hits[1:3]] == [0, 1] and [h for _, h in hits[1:3]] < [0, 0]
    assert [h for _, h in hits[3:5]] == [0, 1] and [h for h, _ in hits[3:5]] < [0, 0]
    assert hits[5][0] < 0 and hits[5][1] < 0 and hits[6][0] > 0 and hits[6][1] > 0
    # the context's normals upload: exactly at its capacity, one past it, smaller, larger
    cap, rel = 0, []
    for m, s in NRM_RAW_STEPS:
        rel.append(nrm_raw_need(m, s) - cap)
        cap = grow_nrm_raw(cap, m, s)
    assert rel[1:3] == [0, 1] and rel[3] < 0 and rel[4] > 0
    # the pose graph's groups
    assert pg_grow(0, 200) == 314 and pg_grow(314, 314) == 314 and pg_grow(314, 315) == 457
    assert grow(0, 2000) == 3274 and grow(3274, 3274) == 3274 and grow(3274, 3275) > 3274
    assert pool_after(16, 65) == 128 and pool_after(16, 64) == 64 and pool_after(17, 65) == 68


# ---- GPU helpers -----------------------------------------------------------------------------------------------------
def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


ICP_GRID = ("cell_size", "leaf_split", "max_cells")


def _oracle_icp(o, rd, ref, nrm, T0, kw):
    po = o.default_params(num_threads=THREADS, **{k: v for k, v in kw.items() if k not in ICP_GRID})
    return o.icp(rd, ref, np.ascontiguousarray(nrm[:, :3]), T0, po, want_hist=True)


def _register(ctx, rd, ref, nrm, T0, kw):
    return ctx.icp_register(rd, ref, nrm, T0, ls.default_params(**kw), want_ids=True, want_hist=True,
                            raise_on_convergence=False)


STAT_FIELDS = ("iterations", "converged", "max_iter_reached", "last_kept", "last_limit", "grid_cells", "grid_tables",
               "grid_overflow")


def _same_icp(a, b):
    for k in ("T", "ids", "d2", "T_iter_hist"):
        assert _same(a[k], b[k]), k
    assert a["rc"] == b["rc"]
    for f in STAT_FIELDS:
        assert getattr(a["stats"], f) == getattr(b["stats"], f), f


def _check_icp(ctx, o, rd, ref, nrm, T0, kw, what):
    g = _register(ctx, rd, ref, nrm, T0, kw)
    r = _oracle_icp(o, rd, ref, nrm, T0, kw)
    assert g["rc"] == r["rc"] == 0, what
    assert np.array_equal(g["T_iter_hist"], r["T_iter_hist"]), what
    assert np.array_equal(g["ids"], r["ids_hist"][-1]) and np.array_equal(g["d2"], r["d2_last"]), what
    assert np.array_equal(g["T"], r["T"]), what
    assert g["stats"].last_kept == r["stats"].last_kept, what
    fresh = ls.Context(0)
    try:
        _same_icp(g, _register(fresh, rd, ref, nrm, T0, kw))
    finally:
        fresh.close()
    return g


def _with_stride(nrm, stride):
    """Normals as the first three floats of `stride`-float rows (a descriptor block); the rest is garbage."""
    if stride == 3:
        return np.ascontiguousarray(nrm, F32)
    pad = np.full((len(nrm), stride - 3), np.nan, F32)
    return np.ascontiguousarray(np.concatenate([nrm, pad], 1))


# ---- 1. ICP workspace and context staging ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_icp_workspace_sequence(oracle_mod, small_pair):
    """ls_icp_register / ls_nn_query / ls_estimate_normals on one context: the reading and sub-map groups and the
    staging at s, exactly c(s), c(s)+1, s/3 and past the next capacity; max_cells regrowing the cell group and shrinking
    again, cell_size 1.0 -> 0.3 -> 1.0, leaf_split 64 <-> 16, T_hist growing; a refused call, an empty reading and a map
    that exhausts the fine-table pool in between."""
    o = oracle_mod
    rng = np.random.default_rng(11)
    pr, pm = rng.permutation(len(small_pair["reading"])), rng.permutation(len(small_pair["ref"]))
    RD = np.ascontiguousarray(small_pair["reading"][pr])
    REF = np.ascontiguousarray(small_pair["ref"][pm])
    NRM = np.ascontiguousarray(small_pair["ref_normals"][pm])
    T0 = small_pair["T0"]
    ctx = ls.Context(0)
    cap = 0                                                        # reading, sub-map and staging capacity (all grow alike)

    def icp(n, kw, stride=3):
        nonlocal cap
        g = _check_icp(ctx, o, RD[:n], REF[:n], _with_stride(NRM[:n], stride), T0, kw, f"n=m={n} {kw} stride {stride}")
        cap = grow(cap, n)
        return g

    try:
        icp(3000, dict(max_iterations=4, use_differential=0, max_cells=256))
        assert cap == 4399
        icp(cap, dict(max_iterations=6, use_differential=0, max_cells=256, leaf_split=64), stride=8)      # exactly at c(s)
        with pytest.raises(ls.LsError, match="rc=-1"):                                                   # refused
            ctx.icp_register(RD[:cap + 1], REF[:cap + 1], NRM[:cap + 1], T0, ls.default_params(trim_ratio=0.0))
        icp(cap + 1, dict(max_iterations=6, use_differential=0, max_cells=5000, cell_size=0.3))          # c(s)+1, cells regrow
        assert cap == 5974
        e = ctx.icp_register(RD[:0], REF[:cap], NRM[:cap], T0, ls.default_params(), raise_on_convergence=False)
        assert e["rc"] == ls.LS_ERR_CONVERGENCE and np.array_equal(e["T"], T0)                            # empty reading
        icp(1000, dict(max_iterations=8, use_differential=0, cell_size=1.0, leaf_split=16))              # s/3
        # ls_nn_query exactly at the capacity, then normals one past it
        gpu_nn_check(ctx, o, RD[:cap, :3], REF[:1500, :3])
        cap = grow(cap, cap)
        pts = REF[:cap + 1]
        nr = ctx.estimate_normals(pts, 10)
        assert np.array_equal(nr, o.knn_normals(pts, 10, num_threads=THREADS))
        cap = grow(cap, cap + 1)
        assert cap == 7745
        icp(cap + 1, dict(max_iterations=12, max_cells=64))                                              # larger again
        icp(3000, dict(max_iterations=10, use_differential=0, cell_size=0.3, leaf_split=64))
        # more cells over leaf_split than fine tables (test_grid_shapes' pool_block), then small problems again
        p3 = pool_block()
        ref4 = homog(p3)
        nrm = rng.normal(size=(len(p3), 3))
        nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(F32)
        rd = homog(p3[rng.choice(len(p3), 20000, replace=False)])
        Tp = np.eye(4, dtype=F32)
        Tp[:3, 3] = [0.05, -0.03, 0.02]
        g = _check_icp(ctx, o, rd, ref4, nrm, Tp, dict(max_iterations=3, use_differential=0, leaf_split=16), "pool block")
        assert g["stats"].grid_overflow == 1 and g["stats"].grid_tables > table_pool(grow(0, len(p3)))
        del p3, ref4, nrm, rd
        icp(1000, dict(max_iterations=8, use_differential=0, leaf_split=16, max_cells=256))
        icp(5000, dict(max_iterations=8, use_differential=0, cell_size=0.3, leaf_split=16), stride=8)
        gpu_nn_check(ctx, o, RD[:4000, :3], REF[:2000, :3], leaf_split=64)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_icp_normals_upload_sequence(oracle_mod, small_pair):
    """ls_icp_register with the reference normals in descriptor rows of 3 to 8 floats: the context's normals upload
    (need + 4096) exactly at its capacity, one past it, smaller and larger (NRM_RAW_STEPS)."""
    o = oracle_mod
    rng = np.random.default_rng(14)
    pm = rng.permutation(len(small_pair["ref"]))
    REF = np.ascontiguousarray(small_pair["ref"][pm])
    NRM = np.ascontiguousarray(small_pair["ref_normals"][pm])
    rd, T0 = small_pair["reading"][:2000], small_pair["T0"]
    ctx = ls.Context(0)
    try:
        for m, stride in NRM_RAW_STEPS:
            _check_icp(ctx, o, rd, REF[:m], _with_stride(NRM[:m], stride), T0, dict(max_iterations=5, use_differential=0),
                       f"m={m} stride {stride}")
    finally:
        ctx.close()


def _submap(o, parts, Ts):
    pts, nrm = [], []
    for (p, n), T in zip(parts, Ts):
        if np.array_equal(T, np.eye(4, dtype=F32)):
            pts.append(p), nrm.append(n)
        else:
            q, m = o.transform_cloud(T, p, n)
            pts.append(q), nrm.append(m)
    return np.concatenate(pts), np.concatenate(nrm)


@pytest.mark.gpu
def test_icp_submap_sequence(oracle_mod, scans, traj):
    """ls_icp_register_submap and _batch on resident scans: sub-maps of s, exactly c(s) and c(s)+1 points, then a batch
    with an empty reading and a smaller and a larger problem, then single registrations again on the grown workspaces."""
    o = oracle_mod
    truth, odom = traj
    rng = np.random.default_rng(12)
    sub = []
    for k in range(5):
        p, n = scans[k]
        keep = rng.permutation(len(p))[:8192]
        sub.append((np.ascontiguousarray(p[keep]), np.ascontiguousarray(n[keep])))
    ref_k, rd_k = 1, 2
    Ts = [np.eye(4, dtype=F32), (np.linalg.inv(truth[ref_k]) @ truth[0]).astype(F32)]
    T0 = (np.linalg.inv(truth[ref_k]) @ odom[rd_k]).astype(F32)
    kw = dict(max_iterations=6, use_differential=0)

    def problem(ring, n, m):
        """Reading: the first n points of scan 2; sub-map: m points split over scans 1 and 0 (scan 1 is the frame)."""
        a = m // 2
        parts = [(sub[ref_k][0][:a], sub[ref_k][1][:a]), (sub[0][0][:m - a], sub[0][1][:m - a])]
        rid = ring.push_scan(sub[rd_k][0][:n], sub[rd_k][1][:n])
        pids = [ring.push_scan(*parts[0]), ring.push_scan(*parts[1])]
        return dict(rid=rid, pids=pids, n=n, m=m, parts=parts)

    def oracle(pr):
        ref, nrm = _submap(o, pr["parts"], Ts)
        assert len(ref) == pr["m"]
        return _oracle_icp(o, sub[rd_k][0][:pr["n"]], ref, nrm, T0, kw)

    def single(ring, n, m):
        pr = problem(ring, n, m)
        g = ring.register(pr["rid"], pr["pids"], Ts, T0, ls.default_params(**kw), want_ids=True, want_hist=True)
        r = oracle(pr)
        assert g["rc"] == r["rc"] == 0 and np.array_equal(g["T_iter_hist"], r["T_iter_hist"])
        assert np.array_equal(g["ids"], r["ids_hist"][-1]) and np.array_equal(g["T"], r["T"]), (n, m)
        fctx = ls.Context(0)
        fring = fctx.create_map(8, 8192)
        try:
            fp = problem(fring, n, m)
            _same_icp(g, fring.register(fp["rid"], fp["pids"], Ts, T0, ls.default_params(**kw), want_ids=True,
                                        want_hist=True))
        finally:
            fring.close(), fctx.close()

    ctx = ls.Context(0)
    ring = ctx.create_map(32, 8192)
    try:
        s = 3000
        cap = grow(0, s)
        single(ring, s, s)
        single(ring, cap, cap)                 # exactly at c(s)
        single(ring, cap + 1, cap + 1)         # one past it
        cap = grow(cap, cap + 1)
        # a batch: a smaller problem, an empty reading, a larger one (workspaces 1 and 2 start empty)
        sizes = [(s // 3, s // 3), (0, 2000), (cap + 1, cap + 1)]
        prs = [problem(ring, n, m) for n, m in sizes]
        res = ring.register_batch([(p["rid"], p["pids"], Ts, T0) for p in prs], ls.default_params(**kw))
        # the same batch on a fresh context, and every problem alone on a fresh context (the batch returns no
        # correspondences or iterates, so those are compared through the single call)
        fctx = ls.Context(0)
        fring = fctx.create_map(16, 8192)
        try:
            fprs = [problem(fring, n, m) for n, m in sizes]
            fres = fring.register_batch([(p["rid"], p["pids"], Ts, T0) for p in fprs], ls.default_params(**kw))
            for pr, g, f in zip(prs, res, fres):
                assert g["rc"] == f["rc"] and _same(g["T"], f["T"]), (pr["n"], pr["m"])
                for name in STAT_FIELDS:
                    assert getattr(g["stats"], name) == getattr(f["stats"], name), name
                if pr["n"] == 0:
                    assert g["rc"] == ls.LS_ERR_CONVERGENCE and np.array_equal(g["T"], T0)
                    continue
                r = oracle(pr)
                assert g["rc"] == r["rc"] == 0 and np.array_equal(g["T"], r["T"]), (pr["n"], pr["m"])
                assert g["stats"].iterations == r["stats"].iterations
                assert g["stats"].last_kept == r["stats"].last_kept
                sp = problem(fring, pr["n"], pr["m"])
                one = fring.register(sp["rid"], sp["pids"], Ts, T0, ls.default_params(**kw), want_ids=True, want_hist=True)
                assert _same(one["T"], g["T"]) and np.array_equal(one["T_iter_hist"], r["T_iter_hist"])
                assert np.array_equal(one["ids"], r["ids_hist"][-1])
                for name in STAT_FIELDS:
                    assert getattr(one["stats"], name) == getattr(g["stats"], name), name
        finally:
            fring.close(), fctx.close()
        cap = grow(cap, cap + 1)
        single(ring, s // 3, s // 3)           # smaller again, on the grown workspace 0
        single(ring, s, 2 * s)
    finally:
        ring.close()
        ctx.close()


# ---- 2. scan ring and its staging ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ring_staging_sequence(oracle_mod, scans):
    """Pushes exactly at and one past both staging rules (device normals and pinned host copy, need + 1024 per staging
    slot) with normals strides 3, 5, 6, 7, then smaller and larger; pushes
    that estimate normals across the workspace boundary, and filtered pushes across the ChainBuffers boundary
    interleaved with ls_filter_cloud on the same context.  Every round is assembled and compared with the oracle's
    transform of the pushed clouds and with a fresh ring fed the same scans."""
    o = oracle_mod
    rng = np.random.default_rng(13)
    P, N = scans[3]
    ctx = ls.Context(0)
    ring = ctx.create_map(64, 8192)
    yaml = fo.filters_yaml(CHAIN)

    def check(ids, clouds):
        Ts = []
        for j in range(len(ids)):
            c, s = np.cos(0.1 * j), np.sin(0.1 * j)
            T = np.eye(4, dtype=F32)
            T[:2, :2] = [[c, -s], [s, c]]
            T[:3, 3] = [0.5 * j, -0.25 * j, 0.125]
            Ts.append(T if j else np.eye(4, dtype=F32))
        got = ring.assemble(ids, Ts)
        want = _submap(o, clouds, Ts)
        assert _same(got[0], want[0]) and _same(got[1], want[1])
        fring = ctx.create_map(16, 8192)
        try:
            fids = [fring.push_scan(p, n) for p, n in clouds]
            fgot = fring.assemble(fids, Ts)
            assert _same(got[0], fgot[0]) and _same(got[1], fgot[1])
        finally:
            fring.close()

    def push_round(n, stride):
        ids, clouds = [], []
        for j in range(STAGE_RING):
            sel = rng.choice(len(P), n, replace=False)
            p, nr = np.ascontiguousarray(P[sel]), np.ascontiguousarray(N[sel])
            ids.append(ring.push_scan(p, _with_stride(nr, stride)))
            clouds.append((p, nr))
        check(ids, clouds)

    try:
        for n, stride in RING_ROUNDS:  # see test_sequence_boundaries for which rule each round meets
            push_round(n, stride)
        # normals estimated on the device: the workspace at s, exactly c(s), c(s)+1, smaller
        cap = 0
        ids, clouds = [], []
        for n in (2000, 3274, 3275, 700):
            sel = rng.choice(len(P), n, replace=False)
            p = np.ascontiguousarray(P[sel])
            ids.append(ring.push_scan_estimate_normals(p, knn=10))
            clouds.append((p, o.knn_normals(p, 10, num_threads=THREADS)))
            cap = grow(cap, n)
        check(ids, clouds)
        # filtered pushes across the chain buffers, with ls_filter_cloud on the same context in between
        raw = P.copy()
        raw[::97, 0] = np.nan
        raw[7::89, :3] *= 40.0
        ids, clouds = [], []
        for n, direct in ((2000, 1500), (3274, 3275), (3275, 800), (900, 6000)):
            sid, kept = ring.push_scan_filtered(yaml, raw[:n])
            want = fo.apply_filters(CHAIN, raw[:n], num_threads=THREADS)
            assert kept == len(want[0]) and ring.scan_size(sid) == kept
            ids.append(sid)
            clouds.append(want)
            got = ctx.filter_cloud(yaml, raw[:direct])
            want_d = fo.apply_filters(CHAIN, raw[:direct], num_threads=THREADS)
            assert _same(got[0], want_d[0]) and _same(got[1], want_d[1])
        check(ids, clouds)
    finally:
        ring.close()
        ctx.close()


# ---- 3. occupancy map: the probe bound --------------------------------------------------------------------------------
OCC_PARAMS = dict(resolution=RES, max_range=12.0)


def _occ_state(m):
    k, v, _ = m.download(ls.OCC_KNOWN)
    ko, vo, _ = m.download(ls.OCC_OCCUPIED)
    return k, v, ko, vo


@pytest.mark.gpu
@pytest.mark.parametrize("initial_capacity", [256, 16, 17])
def test_occupancy_probe_bound_overflow(oracle_mod, scans, traj, initial_capacity, tmp_path):
    """130 bricks whose hashes share their low 12 bits, inserted one per scan: the 65th overflows the probe bound of the
    1024-slot table, and the insert's retry rebuilds the table until it holds them (at least 8192 slots, read back
    from device_bytes).  At 16 initial bricks the same insert also overflows the pool.  After every insert the known and
    occupied voxels equal the oracle, a dict of log-odds, and a map created with room for everything; cell_status on
    every colliding brick reads through the 64-probe lookup.  Then a full scan, refused calls and another full scan."""
    truth, _ = traj
    bricks = colliding_bricks()
    voxels = [one_voxel_scan(b) for b in bricks]
    qpts = np.stack([brick_voxel(b)[1] for b in bricks])
    L_hit, L_max, L_occ = oc.logodds(0.9), oc.logodds(0.97), oc.logodds(0.7)
    ctx = ls.Context(0)
    ring = ctx.create_map(4, 131072)
    dev = ls.OccupancyMap(ctx, initial_capacity=initial_capacity, **OCC_PARAMS)
    roomy = ls.OccupancyMap(ctx, **OCC_PARAMS)                 # 32768 bricks, 65536 slots: never overflows here
    o = oc.OccupancyMap(**OCC_PARAMS)
    lo = {}
    try:
        st0, _ = dev.cell_status(qpts)                        # sizes the query staging before device_bytes is read
        assert (st0 == ls.CELL_UNKNOWN).all()
        schedule = list(range(len(voxels))) + [0]             # the first voxel again at the end: clamped at L_max
        K = None
        tabs = []
        for t, j in enumerate(schedule):
            pts, T, key = voxels[j]
            sid = ring.push_scan(pts, np.zeros((1, 3), F32))
            st = dev.insert_scan(ring, sid, T)
            roomy.insert_scan(ring, sid, T)
            o.insert_scan(pts, T)
            lo[key] = min(F32(lo.get(key, F32(0)) + L_hit), L_max)
            n_b = len(set(schedule[:t + 1]))
            assert st.bricks == n_b
            pool = pool_after(initial_capacity, n_b) * POOL_BYTES_PER_BRICK
            if t == 1:
                K = st.device_bytes - pool - first_table(initial_capacity) * TABLE_BYTES_PER_SLOT
            if t >= 1:
                tab, rem = divmod(st.device_bytes - pool - K, TABLE_BYTES_PER_SLOT)
                assert rem == 0 and tab & (tab - 1) == 0, (t, st.device_bytes)
                tabs.append(tab)
                if t < MAX_PROBE:
                    assert tab == 1024, t
                elif t == MAX_PROBE:
                    assert tab >= 8192, "the 65th colliding brick did not rebuild the table"
            # the known and occupied voxels: the oracle, the dict, the roomy map
            k, v, ko, vo = _occ_state(dev)
            ok, ov = o.download(oc.KNOWN)
            assert np.array_equal(k, ok) and _same(v, ov), t
            want_k = np.array(sorted(lo), np.uint64)
            assert np.array_equal(k, want_k) and _same(v, np.array([lo[int(x)] for x in want_k], F32)), t
            ook, oov = o.download(oc.OCCUPIED)
            assert np.array_equal(ko, ook) and _same(vo, oov) and (vo >= L_occ).all(), t
            rk, rv, rko, rvo = _occ_state(roomy)
            assert np.array_equal(k, rk) and _same(v, rv) and np.array_equal(ko, rko) and _same(vo, rvo), t
            # every colliding brick through the read-only lookup: inserted ones occupied, the rest unknown
            cs, cl = dev.cell_status(qpts)
            want_s = np.array([ls.CELL_OCCUPIED if voxels[i][2] in lo else ls.CELL_UNKNOWN for i in range(len(voxels))])
            assert np.array_equal(cs, want_s), t
            inside = want_s == ls.CELL_OCCUPIED
            assert _same(cl[inside], np.array([lo[voxels[i][2]] for i in np.flatnonzero(inside)], F32))
            assert np.isnan(cl[~inside]).all()
        assert max(tabs) >= 8192
        # a full scan, refused calls, another full scan: equal to a fresh map fed the accepted scans only
        nrm = np.zeros((131072, 3), F32)
        for k in (0, 1):
            sid = ring.push_scan(scans[k][0], nrm)
            dev.insert_scan(ring, sid, truth[k])
            roomy.insert_scan(ring, sid, truth[k])
            o.insert_scan(scans[k][0], truth[k])
            if k == 0:
                with pytest.raises(ls.LsError, match=f"rc={ls.LS_ERR_STATE}"):
                    dev.insert_scan(ring, sid + 100, truth[k])          # never pushed
                with pytest.raises(ls.LsError, match=f"rc={ls.LS_ERR_ARG}"):
                    dev.size(7)
        k, v, ko, vo = _occ_state(dev)
        ok, ov = o.download(oc.KNOWN)
        assert np.array_equal(k, ok) and _same(v, ov) and len(k) > 10000
        rk, rv, rko, rvo = _occ_state(roomy)
        assert np.array_equal(k, rk) and _same(v, rv) and np.array_equal(ko, rko) and _same(vo, rvo)
        cs, cl = dev.cell_status(qpts)
        rs, rl = roomy.cell_status(qpts)
        assert np.array_equal(cs, rs) and _same(cl, rl)
        ot = ot_oracle.of_map(o)
        dev.save_octomap(str(tmp_path / "d.bt"))
        ot.write(str(tmp_path / "o.bt"))
        assert (tmp_path / "d.bt").read_bytes() == (tmp_path / "o.bt").read_bytes()
        ot.close()
    finally:
        dev.close()
        roomy.close()
        ring.close()
        ctx.close()


# ---- 4. local map ----------------------------------------------------------------------------------------------------
def local_map_capacity(cap, initial, need):
    """grow_cloud (ls_api.cu): nothing when need fits, else the larger of the capacity and the initial one, doubled
    until it holds need."""
    if need <= cap:
        return cap
    c = max(cap, initial)
    while c < need:
        c *= 2
    return c


def test_local_map_capacities():
    assert local_map_capacity(0, 4096, 4096) == 4096 and local_map_capacity(4096, 4096, 4097) == 8192
    assert local_map_capacity(8192, 4096, 30000) == 32768


@pytest.mark.gpu
def test_local_map_sequence(scans, traj):
    """add_scan / filter / transform / take_queue / clear on a local map created with room for 4096 points: the clouds
    exactly at that capacity, one past it, far past it after a clear, refused calls in between.  Every cloud equals
    oracle.local_map and a local map created with the default room that gets the same calls."""
    from oracle import local_map as olm
    truth, _ = traj
    params = dict(distance_to_consider_fixed=20.0, separate_distant_map=True, voxel_size_m=0.1,
                  minimum_point_number_per_voxel=0, remove_ground_from_local_map=False, ground_distance_to_robot_center_m=1.5)
    ctx = ls.Context(0)
    ring = ctx.create_map(2, 131072)
    dev = ls.LocalMap(ctx, initial_capacity_points=4096, **params)
    roomy = ls.LocalMap(ctx, **params)
    o = olm.LocalMap(**params)
    poses = [ls.correct_rigid(truth[k].astype(F32)) for k in range(len(scans))]
    clouds = (ls.LM_LOCAL, ls.LM_LOCAL_FILTERED, ls.LM_DISTANT)

    def check(filtered=None, queue=False):
        for w, want in zip(clouds, (o.local_map, o.local_map_filtered, o.distant_map)):
            got = dev.download(w)
            assert _same(got, want) and _same(got, roomy.download(w)), w
        if filtered is not None:
            got = dev.download(ls.LM_FILTERED_MAP)
            assert _same(got, filtered) and _same(got, roomy.download(ls.LM_FILTERED_MAP))
        if queue:
            q, rq, oq = dev.take_queue(), roomy.take_queue(), o.get_queued_points()
            assert len(q) == len(oq) == len(rq) and all(_same(a, b) and _same(a, c) for a, b, c in zip(q, oq, rq))

    def add(k, n):
        s = np.ascontiguousarray(scans[k][0][:n])
        sid = ring.push_scan(s, np.zeros((len(s), 3), F32))
        z = float(truth[k][2, 3])
        got = dev.add_scan(ring, sid, poses[k], z)
        assert got == roomy.add_scan(ring, sid, poses[k], z) == o.add_scan(s, poses[k], z)
        check()
        return sid

    def filt(k):
        want = o.get_filtered_map(truth[k][:3, 3])
        assert dev.filter(truth[k][:3, 3]) == roomy.filter(truth[k][:3, 3]) == len(want)
        check(filtered=want)

    try:
        add(0, 4096)
        assert dev.size(ls.LM_LOCAL) == 4096                    # exactly the initial capacity
        first = add(1, 1)                                       # one past it
        scratch = grow(0, max(dev.size(ls.LM_LOCAL), 4096))     # reserve_scratch: ChainBuffers for max(n, initial)
        filt(1)
        ring.push_scan(scans[3][0][:10], np.zeros((10, 3), F32))
        ring.push_scan(scans[3][0][:10], np.zeros((10, 3), F32))     # evicts `first`
        with pytest.raises(ls.LsError, match=f"rc={ls.LS_ERR_STATE}"):
            dev.add_scan(ring, first, poses[1], 0.0)
        with pytest.raises(ls.LsError, match="rc=-1"):
            dev.size(9)
        # the filter's scratch exactly at its capacity, then one past it
        for extra in (0, 1):
            dev.clear(), roomy.clear(), o.clear_local_map()
            add(2, scratch + extra)
            assert dev.size(ls.LM_LOCAL) == scratch + extra
            filt(2)
        assert grow(scratch, scratch + 1) > scratch
        # a filter refused part-way: the crop has run when the voxel grid finds more than 9e18 cells (a point 3e5 m
        # out on every axis at 0.1 m); nothing changes, and the next filter after a clear equals the oracle again
        far = np.concatenate([scans[3][0][:1000], np.array([[3e5, 3e5, 3e5, 1]], F32)])
        sid = ring.push_scan(far, np.zeros((len(far), 3), F32))
        z = float(truth[3][2, 3])
        assert dev.add_scan(ring, sid, poses[3], z) == roomy.add_scan(ring, sid, poses[3], z) == o.add_scan(far, poses[3], z)
        check()
        before = dev.download(ls.LM_FILTERED_MAP)
        for m in (dev, roomy):
            with pytest.raises(ls.LsError, match="rc=-1"):
                m.filter(truth[3][:3, 3])
        check()
        assert _same(dev.download(ls.LM_FILTERED_MAP), before)
        T = np.eye(4, dtype=F32)
        T[:3, 3] = [0.05, -0.03, 0.01]
        dev.transform(T), roomy.transform(T), o.update_local_map(T)
        check(queue=True)
        dev.clear(), roomy.clear(), o.clear_local_map()
        check()
        add(4, 20000)                                           # several doublings at once
        filt(4)
        add(5, len(scans[5][0]))
        filt(5)
        add(0, 500)                                             # smaller again
        filt(0)
        check(queue=True)
    finally:
        dev.close()
        roomy.close()
        ring.close()
        ctx.close()


# ---- 5. pose graph ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_pose_graph_sequence():
    """Poses and factors of a two-track graph with loop closures added in steps on one graph: the per-factor group
    exactly at its capacity (padded with loose priors) and one past it, the per-pose group exactly at its capacity and
    one past it, then loop closures, duplicate odometry and the padding removed, then both groups grown again.  After
    every step one Gauss-Newton step from the same values equals the dense reference (test_posegraph_shapes' tolerance),
    and the poses are bit-equal to a fresh graph fed the same poses and only the surviving factors, in the same order."""
    from test_posegraph_shapes import LOOSE_PRIOR_SIG, TOL_STEP, Graph, assert_close, dense_step, make_graph, pg, random_links
    rng = np.random.default_rng(51)
    L = [260, 260]
    full = make_graph(L, ids=[5, 9], extra=random_links(rng, L, 24), seed=52)
    g = ls.PoseGraph(0)
    n_poses, added, log = 0, set(), []           # log: [factor, device index, active] in the order the graph got them

    def sync(P, F=None):
        nonlocal n_poses
        g.add_poses(full.keys[n_poses:P], full.init[n_poses:P], full.tracks[n_poses:P])
        n_poses = P
        have = set(int(k) for k in full.keys[:P])
        new = [f for f in full.factors if id(f) not in added and int(f["key_a"]) in have and int(f["key_b"]) in have]
        if F is not None:
            active = sum(1 for e in log if e[2]) + len(new)
            assert active <= F
            new += [pg.make_factor(pg.PRIOR, full.keys[j % P], full.keys[j % P], full.truth[j % P], LOOSE_PRIOR_SIG)
                    for j in range(F - active)]
        if new:
            for f, i in zip(new, g.add_factors(new)):
                added.add(id(f))
                log.append([f, int(i), True])
        return sum(1 for e in log if e[2])

    def step(what):
        keys, init, tracks = full.keys[:n_poses], full.init[:n_poses], full.tracks[:n_poses]
        act = [e[0] for e in log if e[2]]
        G = Graph(keys, tracks, full.truth[:n_poses], init, act)
        g.set_poses(keys, init)
        st = g.optimize(1)
        k2, est = g.poses()
        assert np.array_equal(k2, keys) and st.n_poses == n_poses and st.n_factors == len(act) and st.n_border == G.n_border
        want, scale = dense_step(G, init)
        assert_close(est, want, scale, TOL_STEP, what)
        fresh = ls.PoseGraph(0)
        try:
            fresh.add_poses(keys, init, tracks)
            fresh.add_factors(act)
            fst = fresh.optimize(1)
            assert np.array_equal(fresh.poses()[1], est), what
            assert (fst.n_factors, fst.n_border, fst.iterations) == (st.n_factors, st.n_border, st.iterations)
            # the reported cost is a float64 atomicAdd over the factors: its last bits follow the order of the atomics
            assert np.isclose(fst.cost_first, st.cost_first, rtol=1e-12, atol=0) and \
                np.isclose(fst.cost_last, st.cost_last, rtol=1e-12, atol=0)
        finally:
            fresh.close()

    try:
        F0 = sync(200)
        cap_f, cap_p = pg_grow(0, F0), pg_grow(0, 200)
        step("first")
        sync(200, cap_f)
        step("factors exactly at capacity")
        F = sync(200, cap_f + 1)
        step("factors one past capacity")
        cap_f = pg_grow(cap_f, F)
        F = sync(cap_p)
        step("poses exactly at capacity")
        cap_f = pg_grow(cap_f, F)
        F = sync(cap_p + 1)
        step("poses one past capacity")
        cap_f, cap_p = pg_grow(cap_f, F), pg_grow(cap_p, cap_p + 1)
        # remove a third of the loop closures, every other duplicate (robust) odometry factor and the padding priors
        pos = {int(k): i for i, k in enumerate(full.keys)}
        track = {int(k): int(t) for k, t in zip(full.keys, full.tracks)}
        border = [e for e in log if e[0]["type"] == pg.BETWEEN and not (
            track[int(e[0]["key_a"])] == track[int(e[0]["key_b"])] and pos[int(e[0]["key_b"])] == pos[int(e[0]["key_a"])] + 2)]
        in_border = {id(e) for e in border}
        robust_odo = [e for e in log if e[0]["type"] == pg.BETWEEN and e[0]["robust"] and id(e) not in in_border]
        padding = [e for e in log if e[0]["type"] == pg.PRIOR and e[0]["sigma"][0] == LOOSE_PRIOR_SIG[0]]
        gone = border[::3] + robust_odo[::2] + padding
        assert border and robust_odo and padding
        g.remove_factors([e[1] for e in gone])
        for e in gone:
            e[2] = False
        step("after removal")
        F = sync(520)                                  # larger: both groups regrow, the removed factors stay removed
        assert n_poses > cap_p and F > cap_f
        step("larger")
    finally:
        g.close()
