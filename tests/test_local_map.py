"""LaserSlamWorker's local map (ls_local_map_*; reference laser_slam_ros/src/laser_slam_worker.cpp): the oracle's rules
against an independent per-point restatement on the CPU, the device map against the oracle bit for bit on the GPU."""
import ctypes

import numpy as np
import pytest

import oracle
from oracle import local_map as olm

F32 = np.float32


# ---- an independent per-point restatement: plain loops, a dict of voxels --------------------------------------------
def _naive_xform(T, p):
    T = np.asarray(T, F32)
    if np.array_equal(T, np.eye(4, dtype=F32)):
        return [F32(v) for v in p[:3]]
    out = []
    for r in range(3):
        s = F32(F32(T[r, 0] * p[0]) + F32(T[r, 1] * p[1]))
        s = F32(s + F32(T[r, 2] * p[2]))
        out.append(F32(s + T[r, 3]))
    return out


def _naive_inside(p, c, r, h, outside=False):
    dx, dy = float(p[0]) - c[0], float(p[1]) - c[1]
    d2 = dx * dx + dy * dy
    dz = abs(float(p[2]) - c[2])
    if outside:
        return d2 >= r * r or dz >= h / 2.0
    return d2 <= r * r and dz <= h / 2.0


def _naive_voxel(points, leaf, min_points):
    inv = F32(1.0) / F32(leaf)
    cells = {}
    for p in points:
        if not all(np.isfinite(p[:3])):
            continue
        key = tuple(int(np.floor(F32(p[a]) * inv)) for a in (2, 1, 0))  # (k, j, i): the linear index order, x fastest
        s = cells.setdefault(key, [0, 0, 0, 0])
        for a in range(3):
            s[a] += round(float(p[a]) * 16777216.0)
        s[3] += 1
    out = []
    for key in sorted(cells):
        s = cells[key]
        if min_points > 1 and s[3] < min_points:
            continue
        out.append([F32(s[a] / (s[3] * 16777216.0)) for a in range(3)] + [F32(1.0)])
    return out


class NaiveLocalMap:
    def __init__(self, r, separate, leaf, min_points, ground, ground_dist):
        self.r, self.separate, self.leaf, self.min_points, self.ground, self.gd = r, separate, leaf, min_points, ground, ground_dist
        self.local, self.filtered, self.distant, self.queue = [], [], [], []

    def add_scan(self, scan, T, robot_z):
        cloud = []
        for p in scan:
            q = _naive_xform(T, p) + [p[3]]
            if not self.ground or float(q[2]) > robot_z - self.gd:
                cloud.append(q)
        if cloud:
            self.local += cloud
            self.queue.append(cloud)

    def get_filtered_map(self, center):
        c = [float(F32(v)) for v in center]
        snapshot = self.local
        self.local = [p for p in snapshot if _naive_inside(p, c, self.r, 40.0)]
        if not self.separate:
            return list(snapshot)
        v = _naive_voxel(snapshot, self.leaf, self.min_points)
        self.filtered = [p for p in v if _naive_inside(p, c, self.r, 40.0)]
        self.distant = self.distant + [p for p in v if _naive_inside(p, c, self.r, 40.0, outside=True)]
        return self.filtered + self.distant

    def update_local_map(self, T):
        T = np.asarray(T, F32)
        move = lambda p: [F32(F32(F32(F32(T[r, 0] * p[0]) + F32(T[r, 1] * p[1])) + F32(T[r, 2] * p[2])) + T[r, 3])
                          for r in range(3)] + [p[3]]
        self.local = [move(p) for p in self.local]
        self.filtered = [move(p) for p in self.filtered]


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, F32).reshape(-1, 4)).view(np.uint32)


def _same(a, b):
    a, b = _bits(a), _bits(b)
    return a.shape == b.shape and np.array_equal(a, b)


def _rigid(yaw, t):
    c, s = np.cos(yaw), np.sin(yaw)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:3, 3] = t
    return T.astype(F32)


def _cpu_scans(rng, k, n=2000):
    """Small clouds around the origin: a ground plane at z ~ -1.5, scattered points, some exactly on voxel boundaries."""
    out = []
    for _ in range(k):
        p = np.ones((n, 4), F32)
        p[:, :3] = rng.uniform(-25, 25, (n, 3)).astype(F32)
        p[: n // 3, 2] = rng.normal(-1.5, 0.05, n // 3).astype(F32)
        p[n // 3: n // 3 + 300, :3] = np.round(p[n // 3: n // 3 + 300, :3] * 4) / 4   # on 0.25 m boundaries, many share voxels
        out.append(p)
    return out


@pytest.mark.parametrize("separate, ground, min_points, leaf", [(True, False, 0, 0.25), (True, True, 3, 0.25),
                                                                (False, True, 0, 0.5), (True, False, 2, 1.0)])
def test_oracle_matches_per_point_restatement(separate, ground, min_points, leaf):
    rng = np.random.default_rng(7)
    scans = _cpu_scans(rng, 6)
    kw = dict(distance_to_consider_fixed=12.0, separate_distant_map=separate, voxel_size_m=leaf,
              minimum_point_number_per_voxel=min_points, remove_ground_from_local_map=ground, ground_distance_to_robot_center_m=1.0)
    o = olm.LocalMap(**kw)
    nv = NaiveLocalMap(12.0, separate, leaf, min_points, ground, 1.0)
    for k, s in enumerate(scans):
        T = np.eye(4, dtype=F32) if k == 0 else _rigid(0.1 * k, [1.5 * k, 0.3 * k, 0.01 * k])
        robot_z = 0.01 * k
        o.add_scan(s, T, robot_z)
        nv.add_scan(s, T, robot_z)
        if k % 2 == 1:
            center = T[:3, 3].astype(np.float64) + 0.1
            assert _same(o.get_filtered_map(center), nv.get_filtered_map(center))
            for a, b in ((o.local_map, nv.local), (o.local_map_filtered, nv.filtered), (o.distant_map, nv.distant)):
                assert _same(a, b)
            q, nq = o.get_queued_points(), nv.queue
            nv.queue = []
            assert len(q) == len(nq) and all(_same(a, b) for a, b in zip(q, nq))
        if k == 3:
            T2 = _rigid(-0.05, [0.2, -0.1, 0.0])
            o.update_local_map(T2)
            nv.update_local_map(T2)
            assert _same(o.local_map, nv.local) and _same(o.local_map_filtered, nv.filtered)


def test_min_points_zero_is_todays_voxel_grid():
    """min_points 0 and 1 give oracle.voxel_grid's bits; a minimum keeps exactly the voxels the per-point restatement
    counts at least that many points in."""
    rng = np.random.default_rng(3)
    p = np.ones((5000, 4), F32)
    p[:, :3] = rng.normal(0, 5, (5000, 3)).astype(F32)
    p[17, 0] = np.nan
    for leaf in (0.1, 0.25, 1.0):
        ref = oracle.voxel_grid(p, leaf)
        for m in (0, 1):
            assert _same(olm.voxel_grid(p, leaf, min_points=m), ref)
            assert _same(_naive_voxel(p, leaf, m), ref)
        for m in (2, 3, 7):
            got = olm.voxel_grid(p, leaf, min_points=m)
            assert _same(got, _naive_voxel(p, leaf, m)) and len(got) < len(ref)


def test_minimum_above_every_count_empties_the_voxels():
    p = np.ones((100, 4), F32)
    p[:, :3] = np.arange(300, dtype=F32).reshape(100, 3) * F32(0.01)
    counts = len(p)  # no voxel can hold more than every point
    assert len(olm.voxel_grid(p, 0.1, min_points=counts + 1)) == 0
    o = olm.LocalMap(distance_to_consider_fixed=5.0, minimum_point_number_per_voxel=counts + 1)
    o.add_scan(p, np.eye(4, dtype=F32), 0.0)
    assert len(o.get_filtered_map([0, 0, 0])) == 0 and len(o.local_map_filtered) == 0 and len(o.distant_map) == 0


def test_centroid_on_the_boundary_lands_in_both_maps():
    p = np.array([[10.0, 0, 0, 1], [0, 0, 0, 1]], F32)        # leaf 0.5: each point is its own voxel's centroid
    o = olm.LocalMap(distance_to_consider_fixed=10.0, voxel_size_m=0.5)
    o.add_scan(p, np.eye(4, dtype=F32), 0.0)
    out = o.get_filtered_map([0, 0, 0])
    assert any((o.local_map_filtered[:, 0] == 10.0)) and any((o.distant_map[:, 0] == 10.0))
    assert len(o.local_map_filtered) == 2 and len(o.distant_map) == 1 and len(out) == 3


def test_non_separating_filter_returns_the_uncropped_snapshot():
    p = np.array([[1, 0, 0, 1], [50, 0, 0, 1], [1, 0, 30, 1]], F32)
    o = olm.LocalMap(distance_to_consider_fixed=10.0, separate_distant_map=False)
    o.add_scan(p, np.eye(4, dtype=F32), 0.0)
    out = o.get_filtered_map([0, 0, 0])
    assert _same(out, p) and _same(o.local_map, p[:1]) and len(o.local_map_filtered) == 0


def test_update_and_clear_leave_distant_map_and_queue():
    rng = np.random.default_rng(1)
    s = _cpu_scans(rng, 2)
    o = olm.LocalMap(distance_to_consider_fixed=8.0)
    o.add_scan(s[0], np.eye(4, dtype=F32), 0.0)
    o.get_filtered_map([0, 0, 0])
    o.add_scan(s[1], _rigid(0.2, [1, 2, 0]), 0.0)
    dist, queue = o.distant_map.copy(), [q.copy() for q in o.queue]
    assert len(dist) > 0 and len(queue) == 2
    local_before = o.local_map.copy()
    o.update_local_map(_rigid(0.3, [5, 0, 0]))
    assert _same(o.distant_map, dist) and all(_same(a, b) for a, b in zip(o.queue, queue))
    assert not _same(o.local_map, local_before)
    o.clear_local_map()
    assert len(o.local_map) == 0 and len(o.local_map_filtered) == 0
    assert _same(o.distant_map, dist) and len(o.get_queued_points()) == 2 and o.get_queued_points() == []


def test_all_ground_cloud_is_not_queued():
    p = np.ones((50, 4), F32)
    p[:, 2] = -2.0
    o = olm.LocalMap(remove_ground_from_local_map=True, ground_distance_to_robot_center_m=1.0)
    assert o.add_scan(p, np.eye(4, dtype=F32), 0.0) == 0
    assert len(o.local_map) == 0 and o.queue == []
    p[0, 2] = -0.999
    assert o.add_scan(p, np.eye(4, dtype=F32), 0.0) == 1 and len(o.queue) == 1


# ---- GPU ------------------------------------------------------------------------------------------------------------
N_STEPS = 40


@pytest.fixture(scope="module")
def seq(synth_mod):
    import laser_slam_b200 as ls
    truth, _ = synth_mod.trajectory(0, N_STEPS)
    scans = [synth_mod.scan(truth[k], 0, k)[0] for k in range(N_STEPS)]
    poses = [ls.correct_rigid(truth[k].astype(F32)) for k in range(N_STEPS)]
    return truth, scans, poses


def _lm_params(**kw):
    base = dict(distance_to_consider_fixed=20.0, separate_distant_map=True, voxel_size_m=0.1, minimum_point_number_per_voxel=0,
                remove_ground_from_local_map=False, ground_distance_to_robot_center_m=1.5)
    base.update(kw)
    return base


def _check_all(ls, dev, o, filtered=None, want_filtered=None):
    assert _same(dev.download(ls.LM_LOCAL), o.local_map)
    assert _same(dev.download(ls.LM_LOCAL_FILTERED), o.local_map_filtered)
    assert _same(dev.download(ls.LM_DISTANT), o.distant_map)
    if want_filtered is not None:
        assert _same(dev.download(ls.LM_FILTERED_MAP), want_filtered)
    q, oq = dev.take_queue(), o.get_queued_points()
    assert len(q) == len(oq) and all(_same(a, b) for a, b in zip(q, oq))


def _run_sequence(ls, ctx, seq, params, stray_at=None, initial_capacity=0, begin_batch=None):
    truth, scans, poses = seq
    ring = ctx.create_map(8, 131072)
    dev = ls.LocalMap(ctx, initial_capacity_points=initial_capacity, **params)
    o = olm.LocalMap(**params)
    T_mid = _rigid(0.004, [0.05, -0.03, 0.01])
    n_filters, stray_space = 0, 0
    for k in range(N_STEPS):
        s = scans[k]
        if stray_at == k:
            s = s.copy()
            s[100, :3] = [4000.0, 3000.0, 200.0]
        sid = ring.push_scan(s, np.zeros((len(s), 3), F32))
        robot_z = float(truth[k][2, 3])
        assert dev.add_scan(ring, sid, poses[k], robot_z) == o.add_scan(s, poses[k], robot_z)
        if k == N_STEPS // 2:
            dev.transform(T_mid)
            o.update_local_map(T_mid)
            assert len(o.local_map) > 0 and (len(o.local_map_filtered) > 0) == params["separate_distant_map"]
            assert _same(dev.download(ls.LM_LOCAL), o.local_map)                    # both moved ...
            assert _same(dev.download(ls.LM_LOCAL_FILTERED), o.local_map_filtered)
            assert _same(dev.download(ls.LM_DISTANT), o.distant_map)                # ... the distant map is not
        if k % 5 == 4:
            center = truth[k][:3, 3]
            snap = o.local_map[np.isfinite(o.local_map[:, :3]).all(1)]
            if len(snap):  # the snapshot's voxel index space (cells), as the voxel grid sizes it
                ijk = np.floor(snap[:, :3] * (F32(1) / F32(params["voxel_size_m"]))).astype(np.int64)
                stray_space = max(stray_space, int(np.prod(ijk.max(0) - ijk.min(0) + 1)))
            want = o.get_filtered_map(center)
            assert dev.filter(center) == len(want)
            _check_all(ls, dev, o, want_filtered=want)
            n_filters += 1
    assert n_filters == N_STEPS // 5
    dev.close()
    ring.close()
    return stray_space


PARAM_SETS = [
    dict(separate_distant_map=True, remove_ground_from_local_map=False, minimum_point_number_per_voxel=0, voxel_size_m=0.1),
    dict(separate_distant_map=True, remove_ground_from_local_map=True, minimum_point_number_per_voxel=3, voxel_size_m=0.25),
    dict(separate_distant_map=False, remove_ground_from_local_map=True, minimum_point_number_per_voxel=0, voxel_size_m=0.1),
    dict(separate_distant_map=True, remove_ground_from_local_map=False, minimum_point_number_per_voxel=3, voxel_size_m=0.1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(PARAM_SETS)))
def test_sequence_matches_oracle(gpu_ctx, seq, i):
    import laser_slam_b200 as ls
    stray_at = 12 if i == 3 else None
    space = _run_sequence(ls, gpu_ctx, seq, _lm_params(**PARAM_SETS[i]), stray_at=stray_at)
    if stray_at is not None:
        assert space > 2 ** 31   # pcl::VoxelGrid would have returned this snapshot unfiltered
    else:
        assert space < 2 ** 31   # the synthetic scene alone stays below that


@pytest.mark.gpu
def test_growth_from_a_small_capacity(gpu_ctx, seq):
    import laser_slam_b200 as ls
    _run_sequence(ls, gpu_ctx, seq, _lm_params(minimum_point_number_per_voxel=2), initial_capacity=1000)


@pytest.mark.gpu
def test_append_equals_the_assembled_world_cloud_and_nan_handling(gpu_ctx, seq):
    import laser_slam_b200 as ls
    truth, scans, poses = seq
    ring = gpu_ctx.create_map(4, 131072)
    s = scans[3].copy()
    s[::997, 0] = np.nan
    s[5::1009, 2] = np.nan
    n_nan = int(np.isnan(s[:, :3]).any(1).sum())
    sid = ring.push_scan(s, np.zeros((len(s), 3), F32))
    world, _ = ring.assemble([sid], [poses[3]], want_normals=False)
    for ground in (False, True):
        dev = ls.LocalMap(gpu_ctx, **_lm_params(remove_ground_from_local_map=ground))
        robot_z = float(truth[3][2, 3])
        n = dev.add_scan(ring, sid, poses[3], robot_z)
        want = world if not ground else world[world[:, 2].astype(np.float64) > robot_z - 1.5]
        got = dev.download(ls.LM_LOCAL)
        assert n == len(want) and _same(got, want)
        if not ground:
            assert int(np.isnan(got[:, :3]).any(1).sum()) == n_nan     # carried by the append
        dev.filter(truth[3][:3, 3])
        o = olm.LocalMap(**_lm_params(remove_ground_from_local_map=ground))
        o.add_scan(s, poses[3], robot_z)
        want_f = o.get_filtered_map(truth[3][:3, 3])
        assert not np.isnan(dev.download(ls.LM_LOCAL)).any()             # dropped by the crop ...
        assert not np.isnan(dev.download(ls.LM_FILTERED_MAP)).any()      # ... and by the voxel grid
        assert _same(dev.download(ls.LM_FILTERED_MAP), want_f) and _same(dev.download(ls.LM_LOCAL), o.local_map)
        dev.close()
    ring.close()


@pytest.mark.gpu
def test_calls_between_batch_begin_and_end(seq):
    import laser_slam_b200 as ls
    truth, scans, poses = seq
    ctx = ls.Context(0)
    ring = ctx.create_map(16, 131072)
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(6)]
    problems = [(ids[k + 1], [ids[k]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[k]) @ poses[k + 1]) for k in range(3)]
    p = ls.default_params(max_iterations=5)
    alone = ring.register_batch(problems, p)
    dev = ls.LocalMap(ctx, **_lm_params())
    o = olm.LocalMap(**_lm_params())
    end = ring.begin_batch(problems, p)
    for k in range(6):
        assert dev.add_scan(ring, ids[k], poses[k], float(truth[k][2, 3])) == o.add_scan(scans[k], poses[k], float(truth[k][2, 3]))
    want = o.get_filtered_map(truth[5][:3, 3])
    assert dev.filter(truth[5][:3, 3]) == len(want)
    res = end()
    for a, b in zip(res, alone):
        assert a["rc"] == b["rc"] and np.array_equal(a["T"], b["T"])
    _check_all(ls, dev, o, want_filtered=want)
    dev.close()
    ring.close()
    ctx.close()


@pytest.mark.gpu
def test_errors_leave_the_map_unchanged(gpu_ctx, seq):
    import laser_slam_b200 as ls
    truth, scans, poses = seq
    for bad in (dict(voxel_size_m=-0.1), dict(voxel_size_m=0.0), dict(distance_to_consider_fixed=-1.0),
                dict(minimum_point_number_per_voxel=-1), dict(distance_to_consider_fixed=float("nan"))):
        with pytest.raises(ls.LsError, match="rc=-1"):
            ls.LocalMap(gpu_ctx, **_lm_params(**bad))
    ring = gpu_ctx.create_map(2, 131072)
    nrm = np.zeros((131072, 3), F32)
    first = ring.push_scan(scans[0], nrm)
    dev = ls.LocalMap(gpu_ctx, **_lm_params())
    dev.add_scan(ring, first, poses[0], 0.0)
    dev.filter(truth[0][:3, 3])
    dev.add_scan(ring, first, poses[0], 0.0)
    before = {w: dev.download(w) for w in (ls.LM_LOCAL, ls.LM_LOCAL_FILTERED, ls.LM_DISTANT, ls.LM_FILTERED_MAP, ls.LM_QUEUE)}
    ring.push_scan(scans[1], nrm)
    ring.push_scan(scans[2], nrm)                       # evicts `first`
    n = ctypes.c_int(-7)
    t = ls.colmajor(poses[0])
    assert ls.lib().ls_local_map_add_scan(dev._h, ring._h, first, t.ctypes.data, 0.0, ctypes.byref(n)) == ls.LS_ERR_STATE
    small = np.empty((10, 4), F32)
    assert ls.lib().ls_local_map_download(dev._h, ls.LM_LOCAL, small.ctypes.data, 10, ctypes.byref(n)) == ls.LS_ERR_ARG
    offs = np.zeros(2, np.int32)
    assert ls.lib().ls_local_map_take_queue(dev._h, small.ctypes.data, 10, offs.ctypes.data, 1, ctypes.byref(n)) == ls.LS_ERR_ARG
    assert ls.lib().ls_local_map_size(dev._h, 9) == ls.LS_ERR_ARG
    for w, a in before.items():
        assert _same(dev.download(w), a)
    dev.close()
    ring.close()


# ---- host layer: laser_slam::LocalMap on the tracks of an IncrementalEstimator ---------------------------------------
def _rot(q):
    """compat RotationQuaternion::getRotationMatrix (row-major, the quaternion as stored), in the same double order."""
    w, x, y, z = (float(v) for v in q)
    return [1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
            2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
            2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]


def _rotate(q, v):
    R = _rot(q)
    return [R[0] * v[0] + R[1] * v[1] + R[2] * v[2], R[3] * v[0] + R[4] * v[1] + R[5] * v[2],
            R[6] * v[0] + R[7] * v[1] + R[8] * v[2]]


def _se3_inverse(p):
    qi = [float(p[0]), -float(p[1]), -float(p[2]), -float(p[3])]
    t = _rotate(qi, [float(v) for v in p[4:7]])
    return qi + [-t[0], -t[1], -t[2]]


def _se3_compose(a, b):
    t = _rotate(a[:4], [float(v) for v in b[4:7]])
    a0, a1, a2, a3 = (float(v) for v in a[:4])
    b0, b1, b2, b3 = (float(v) for v in b[:4])
    r = [a0 * b0 - a1 * b1 - a2 * b2 - a3 * b3, a0 * b1 + a1 * b0 + a2 * b3 - a3 * b2,
         a0 * b2 - a1 * b3 + a2 * b0 + a3 * b1, a0 * b3 + a1 * b2 - a2 * b1 + a3 * b0]
    n = float(np.sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]))
    return [v / n for v in r] + [t[0] + float(a[4]), t[1] + float(a[5]), t[2] + float(a[6])]


def _float_matrix(p):
    """SE3::getTransformationMatrix().cast<float>() of a pose (qw,qx,qy,qz,tx,ty,tz)."""
    R = _rot(p[:4])
    T = np.eye(4, dtype=F32)
    for r in range(3):
        for c in range(3):
            T[r, c] = F32(R[3 * r + c])
        T[r, 3] = F32(p[4 + r])
    return T


@pytest.mark.gpu
def test_host_layer_local_map_per_worker_with_loop_closure(synth_mod):
    """Two workers in batch mode (IncrementalEstimator::processPosesAndLaserScans), one laser_slam::LocalMap per worker
    reading its track's scans from the estimator's shared ring; a loop closure between the tracks, then updateLocalMap.
    Every map equals oracle.local_map fed with the tracks' scans and the poses lsh_trajectory reports."""
    import laser_slam_b200 as ls
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    n_scans = 8
    truth, odom = synth_mod.trajectory(3, 2 * n_scans + 2)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 3, k), 8) for k in range(2 * n_scans)]
    odom7 = pg.se3_from_matrix(odom)
    off = pg.se3_from_matrix(np.array([[1, 0, 0, 50.0], [0, 1, 0, 20.0], [0, 0, 1, 0], [0, 0, 0, 1.0]]))
    params = dict(distance_to_consider_fixed=15.0, separate_distant_map=True, voxel_size_m=0.25, minimum_point_number_per_voxel=2,
                  remove_ground_from_local_map=True, ground_distance_to_robot_center_m=1.5)
    est = host.Estimator(n_workers=2, nscan_in_sub_map=3)
    lms = [host.LocalMap(est, w, **params) for w in range(2)]
    ors = [olm.LocalMap(**params) for _ in range(2)]

    def compare(w):
        assert _same(lms[w].get(host.LM_LOCAL), ors[w].local_map)
        assert _same(lms[w].get(host.LM_LOCAL_FILTERED), ors[w].local_map_filtered)
        assert _same(lms[w].get(host.LM_DISTANT), ors[w].distant_map)

    def step(k):
        data = [scans[k], scans[n_scans + k]]
        feats = [np.ascontiguousarray(d[0]) for d in data]
        nrms = [np.ascontiguousarray(d[1]) for d in data]
        est.step_batch([0, 1], [k * 10**8] * 2, [odom7[k], pg.se3_compose(off, odom7[n_scans + k])], [f.ctypes.data for f in feats],
                       [n.ctypes.data for n in nrms], [len(f) for f in feats])
        for w in range(2):
            lms[w].add_scan()
            times, traj = est.trajectory(w)
            assert times[-1] == k * 10**8
            T = _float_matrix(traj[-1])
            if not ls.check_rigid(T):                      # correctTransformationMatrix
                T = ls.correct_rigid(T)
            ors[w].add_scan(feats[w], T, float(traj[-1][6]))
            if k % 3 == 2:
                got = lms[w].get_filtered_map()
                want = ors[w].get_filtered_map(traj[-1][4:7])
                assert len(want) > 0 and _same(got, want)
                q, oq = lms[w].get_queued_points(), ors[w].get_queued_points()
                assert len(q) == len(oq) == 3 and all(_same(a, b) for a, b in zip(q, oq))
                compare(w)

    for k in range(5):
        step(k)
    before = [est.trajectory(w) for w in range(2)]
    rel_true = pg.se3_from_matrix(np.linalg.inv(truth[4]) @ truth[n_scans])
    w_T = pg.se3_compose(pg.se3_compose(before[0][1][4], rel_true), pg.se3_inverse(before[1][1][0]))
    est.loop_closure(0, 4 * 10**8, 1, 0, w_T)
    moved = 0.0
    for w in range(2):
        t_last, p_last = before[w][0][-1], before[w][1][-1]
        lms[w].update_local_map(p_last, t_last)
        times, traj = est.trajectory(w)
        new_last = traj[list(times).index(t_last)]
        moved = max(moved, float(np.abs(new_last[4:] - p_last[4:]).max()))
        ors[w].update_local_map(_float_matrix(_se3_compose(new_last, _se3_inverse(p_last))))
        assert len(ors[w].local_map) > 0 and len(ors[w].local_map_filtered) > 0
        compare(w)
    assert moved > 1.0                                     # the loop closure moved a track: the transform is not the identity
    for k in range(5, n_scans):
        step(k)
    for w in range(2):
        lms[w].clear_local_map()
        assert len(lms[w].get(host.LM_LOCAL)) == 0 and len(lms[w].get(host.LM_LOCAL_FILTERED)) == 0
        assert _same(lms[w].get(host.LM_DISTANT), ors[w].distant_map)
        lms[w].close()
    est.close()
