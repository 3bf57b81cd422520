"""Occupancy map (laser_to_octomap's insertion loop): the oracle against an independent restatement and known answers on
the CPU; the device map (ls_occupancy_*), the Python wrapper and laser_slam::OccupancyMap bit for bit against the oracle
on the GPU.  The rules are oracle/OCCUPANCY.md."""
import ctypes
import math

import numpy as np
import pytest

from oracle import occupancy as oc

F32 = np.float32
K0 = 32768


def _key(c, res):
    s = math.floor(float(F32(c)) * (1.0 / res))
    return s + K0 if -K0 <= s < K0 else None


def _key3(p, res):
    k = [_key(c, res) for c in p]
    return None if None in k else tuple(k)


def _pack(k):
    return k[0] | (k[1] << 16) | (k[2] << 32)


def _rel(*k):
    return _pack((K0 + k[0], K0 + k[1], K0 + k[2]))


# ---- independent restatement: float64 segment-cube intersection, a dict of voxels, the scan rules ----------------------
def segment_cells(o, e, res, margin=None):
    """The voxels the segment o -> e passes through before the end voxel, in order (float64 geometry).  With a margin,
    None when a boundary crossing comes within `margin` of another boundary (an edge or corner tie) or an end lies
    within it of a boundary."""
    o = [float(v) for v in o]
    e = [float(v) for v in e]
    ko, ke = _key3(o, res), _key3(e, res)
    if ko is None or ke is None:
        return []
    if ko == ke:
        return []
    d = [e[i] - o[i] for i in range(3)]
    ts = []
    for a in range(3):
        if d[a] == 0.0:
            continue
        lo, hi = sorted((o[a], e[a]))
        for j in range(math.floor(lo / res) + 1, math.floor(hi / res) + 1):
            ts.append(((j * res) - o[a]) / d[a])
    ts = sorted(t for t in ts if 0.0 < t < 1.0)
    if margin is not None:
        for p in (o, e):
            if any(abs(c / res - round(c / res)) * res < margin for c in p):
                return None
        for t in ts:
            q = [o[i] + t * d[i] for i in range(3)]
            if sum(abs(c / res - round(c / res)) * res < margin for c in q) > 1:
                return None
        if any(b - a < margin for a, b in zip(ts, ts[1:])):
            return None
    cells, bounds = [], [0.0] + ts + [1.0]
    for a, b in zip(bounds, bounds[1:]):
        m = 0.5 * (a + b)
        k = tuple(math.floor((o[i] + m * d[i]) / res) + K0 for i in range(3))
        if k == ke:
            break
        if not cells or cells[-1] != k:
            cells.append(k)
    return cells


class Restated:
    def __init__(self, resolution, max_range, **_):
        self.res, self.max_range = resolution, max_range
        self.l = {p: oc.logodds(v) for p, v in (("hit", 0.9), ("miss", 0.4), ("min", 0.12), ("max", 0.97))}
        self.vox = {}

    def insert(self, pts, origin):
        occ, free = set(), set()
        o = np.asarray(origin, F32)
        for p in np.asarray(pts, F32)[:, :3]:
            if not np.isfinite(p).all():
                continue
            k = _key3(p, self.res)
            if k is not None and k in occ:
                continue
            d = (p - o).astype(F32)
            if self.max_range < 0 or math.sqrt(float(np.sum(d.astype(np.float64) ** 2))) <= self.max_range:
                free.update(segment_cells(o, p, self.res))
                if k is not None:
                    occ.add(k)
            else:
                free.update(segment_cells(o, cut_end(o, p, self.max_range), self.res))
        for k in occ | free:
            v = F32(self.vox.get(k, F32(0)) + (self.l["hit"] if k in occ else self.l["miss"]))
            self.vox[k] = min(max(v, self.l["min"]), self.l["max"])

    def download(self):
        ks = sorted(self.vox, key=lambda k: (k[2], k[1], k[0]))
        return np.array([_pack(k) for k in ks], np.uint64), np.array([self.vox[k] for k in ks], F32)


def cut_end(o, p, max_range):
    """o + dir * max_range in float32, dir = (p - o) / (float)|p - o| (the rules' order)."""
    d = (np.asarray(p, F32) - np.asarray(o, F32)).astype(F32)
    n2 = F32(F32(d[0] * d[0]) + F32(d[1] * d[1])) + F32(d[2] * d[2])
    fl = F32(math.sqrt(float(F32(n2))))
    return (np.asarray(o, F32) + (d / fl).astype(F32) * F32(max_range)).astype(F32)


def _translate(t):
    T = np.eye(4, dtype=F32)
    T[:3, 3] = t
    return T


def _bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def _same_map(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(_bits(a[1]), _bits(b[1]))


# ---- CPU: DDA and scan rules ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("res", [0.1, 0.075])
def test_dda_equals_segment_voxel_intersection(res):
    rng = np.random.default_rng(7)
    checked = 0
    while checked < 300:
        o = rng.uniform(-2.0, 2.0, 3).astype(F32)
        e = (o + rng.uniform(-1.5, 1.5, 3)).astype(F32)
        want = segment_cells(o, e, res, margin=1e-6)
        if want is None:
            continue
        got = oc.ray_keys(res, o, e)
        assert [int(k) for k in got] == [_pack(k) for k in want], (o, e)
        checked += 1


def _tie_free_cloud(rng, n, res, origin, max_range):
    pts = []
    while len(pts) < n:
        p = (origin + rng.uniform(-3.0, 3.0, 3)).astype(F32)
        d = (p - origin).astype(np.float64)
        r = float(np.sqrt(np.sum(d * d)))
        if max_range >= 0 and abs(r - max_range) < 1e-3:
            continue
        e = p if max_range < 0 or r <= max_range else cut_end(origin, p, max_range)
        if segment_cells(origin, e, res, margin=1e-6) is None:
            continue
        pts.append([p[0], p[1], p[2], 1.0])
    return np.array(pts, F32)


@pytest.mark.parametrize("res", [0.1, 0.075])
def test_oracle_matches_restatement(res):
    rng = np.random.default_rng(11)
    origin = np.array([0.013, -0.021, 0.037], F32)
    T = _translate(origin)
    for max_range in (2.0, -1.0):
        o, r = oc.OccupancyMap(resolution=res, max_range=max_range), Restated(res, max_range)
        for s in range(3):
            cloud = _tie_free_cloud(rng, 150, res, origin, max_range)
            cloud = np.concatenate([cloud, cloud[:10]])   # repeated endpoints
            o.insert_scan(cloud - np.array([*origin, 0], F32), T)
            r.insert(cloud, origin)
            assert _same_map(o.download(), r.download())
        assert o.size() > 1000 and o.size(oc.OCCUPIED) > 0


# Known-answer cases: (params, [(cloud, T)], check(oracle map, list of stats))
L_HIT, L_MISS = oc.logodds(0.9), oc.logodds(0.4)


def _x_run(a, b):
    return [_rel(i, 0, 0) for i in range(a, b)]


def _vox(m):
    k, v = m.download()
    return dict(zip((int(x) for x in k), v))


CASES = {}


def case(name, params, scans):
    def deco(check):
        CASES[name] = (params, scans, check)
        return check
    return deco


@case("one_voxel", dict(resolution=0.1, max_range=-1.0), [(np.array([[0.03, 0.04, 0.02, 1]], F32), np.eye(4, dtype=F32))])
def _one_voxel(m, st):
    assert _vox(m) == {_rel(0, 0, 0): L_HIT}


@case("axis_parallel", dict(resolution=0.1, max_range=-1.0),
      [(np.array([[0.55, 0.05, 0.05, 1], [0.05, -0.35, 0.05, 1], [0.05, 0.05, 0.25, 1]], F32), np.eye(4, dtype=F32))])
def _axis_parallel(m, st):
    want = {k: L_MISS for k in _x_run(0, 5) + [_rel(0, -i, 0) for i in range(0, 4)] + [_rel(0, 0, i) for i in range(0, 2)]}
    want.update({_rel(5, 0, 0): L_HIT, _rel(0, -4, 0): L_HIT, _rel(0, 0, 2): L_HIT})
    assert _vox(m) == want


@case("edge_tie", dict(resolution=0.1, max_range=-1.0), [(np.array([[0.2, 0.2, 0.0, 1]], F32), _translate([0.05, 0.05, 0.05]))])
def _edge_tie(m, st):   # equal tMax in x and y: the later axis (y) steps first
    want = {k: L_MISS for k in (_rel(0, 0, 0), _rel(0, 1, 0), _rel(1, 1, 0), _rel(1, 2, 0))}
    want[_rel(2, 2, 0)] = L_HIT
    assert _vox(m) == want


@case("corner_tie", dict(resolution=0.1, max_range=-1.0), [(np.array([[0.2, 0.2, 0.2, 1]], F32), _translate([0.05, 0.05, 0.05]))])
def _corner_tie(m, st):  # three-way ties: z, then y, then x
    want = {k: L_MISS for k in (_rel(0, 0, 0), _rel(0, 0, 1), _rel(0, 1, 1), _rel(1, 1, 1), _rel(1, 1, 2), _rel(1, 2, 2))}
    want[_rel(2, 2, 2)] = L_HIT
    assert _vox(m) == want


@case("at_max_range", dict(resolution=0.1, max_range=2.0), [(np.array([[2.0, 0.0, 0.0, 1]], F32), np.eye(4, dtype=F32))])
def _at_max_range(m, st):
    # voxel 19 is not listed: the (float) half step puts its far boundary at 2.0000000007, past the 2.0 m length
    want = {k: L_MISS for k in _x_run(0, 19)}
    want[_rel(20, 0, 0)] = L_HIT
    assert _vox(m) == want


@case("beyond_max_range", dict(resolution=0.1, max_range=1.999), [(np.array([[2.0, 0.0, 0.0, 1]], F32), np.eye(4, dtype=F32))])
def _beyond_max_range(m, st):  # cut at 1.999: free cells up to the cut end's voxel, no occupied voxel
    assert _vox(m) == {k: L_MISS for k in _x_run(0, 19)}
    assert st[0]["rays_cast"] == 1 and st[0]["occupied_updates"] == 0


@case("past_key_space", dict(resolution=0.1, max_range=-1.0), [(np.array([[5000.0, 0.0, 0.0, 1]], F32), np.eye(4, dtype=F32))])
def _past_key_space(m, st):
    assert _vox(m) == {} and st[0]["rays_cast"] == 1


_NEG_T = _translate([-0.01, -0.02, -0.03])


@case("negative", dict(resolution=0.1, max_range=-1.0), [(np.array([[-0.54, -0.23, -0.02, 1]], F32), _NEG_T)])
def _negative(m, st):
    p = np.array([-0.54, -0.23, -0.02], F32) + _NEG_T[:3, 3]
    want = {_pack(k): L_MISS for k in segment_cells(_NEG_T[:3, 3], p, 0.1)}
    want[_rel(-6, -3, -1)] = L_HIT
    assert _vox(m) == want and len(want) > 5


# from (0.05, 0.05) to (0.99, 0.31) and to (0.91, 0.39): one endpoint voxel, rays through different voxels
_A, _B = [0.94, 0.26, 0.0, 1], [0.86, 0.34, 0.0, 1]


@case("duplicate_a_first", dict(resolution=0.1, max_range=-1.0), [(np.array([_A, _B], F32), _translate([0.05, 0.05, 0.05]))])
def _dup_a(m, st):
    r = Restated(0.1, -1.0)
    r.insert(np.array([_A, _B], F32) + np.array([0.05, 0.05, 0.05, 0], F32), [0.05, 0.05, 0.05])
    assert _same_map(m.download(), r.download())
    assert _rel(1, 1, 0) not in _vox(m) and st[0]["rays_skipped"] == 1


@case("duplicate_b_first", dict(resolution=0.1, max_range=-1.0), [(np.array([_B, _A], F32), _translate([0.05, 0.05, 0.05]))])
def _dup_b(m, st):
    assert _vox(m)[_rel(1, 1, 0)] == L_MISS and _rel(2, 0, 0) not in _vox(m) and st[0]["rays_skipped"] == 1


@case("free_and_occupied", dict(resolution=0.1, max_range=-1.0),
      [(np.array([[0.55, 0.05, 0.05, 1], [1.05, 0.05, 0.05, 1]], F32), np.eye(4, dtype=F32))])
def _free_and_occupied(m, st):
    want = {k: L_MISS for k in _x_run(0, 10)}
    want[_rel(5, 0, 0)] = L_HIT
    want[_rel(10, 0, 0)] = L_HIT
    assert _vox(m) == want and st[0]["free_updates"] == 9 and st[0]["occupied_updates"] == 2


@case("clamping", dict(resolution=0.1, max_range=-1.0), [(np.array([[0.35, 0.05, 0.05, 1]], F32), np.eye(4, dtype=F32))] * 30)
def _clamping(m, st):
    v_hit, v_miss = F32(0), F32(0)
    for _ in range(30):
        v_hit = min(F32(v_hit + L_HIT), oc.logodds(0.97))
        v_miss = max(F32(v_miss + L_MISS), oc.logodds(0.12))
    assert v_hit == oc.logodds(0.97) and v_miss == oc.logodds(0.12)
    assert _vox(m) == {**{k: v_miss for k in _x_run(0, 3)}, _rel(3, 0, 0): v_hit}


_NAN_CLOUD = np.array([[0.55, 0.05, 0.05, 1], [np.nan, 0.1, 0.1, 1], [0.05, 0.05, np.nan, 1], [0.05, 0.45, 0.05, 1]], F32)


@case("nan", dict(resolution=0.1, max_range=-1.0), [(_NAN_CLOUD, _translate([0.01, 0.02, 0.03]))])
def _nan(m, st):
    clean = oc.OccupancyMap(resolution=0.1, max_range=-1.0)
    clean.insert_scan(_NAN_CLOUD[[0, 3]], _translate([0.01, 0.02, 0.03]))
    assert _same_map(m.download(), clean.download())
    assert st[0]["rays_skipped"] == 2 and st[0]["rays_cast"] == 2


@pytest.mark.parametrize("name", sorted(CASES))
def test_known_answers(name):
    params, scans, check = CASES[name]
    m = oc.OccupancyMap(**params)
    st = [m.insert_scan(c, T) for c, T in scans]
    check(m, st)


def test_occupied_is_known_and_above_the_threshold():
    m = oc.OccupancyMap(resolution=0.1, max_range=-1.0)
    for _ in range(3):
        m.insert_scan(np.array([[0.35, 0.05, 0.05, 1]], F32), np.eye(4, dtype=F32))
    k, v = m.download(oc.OCCUPIED)
    assert list(k) == [_rel(3, 0, 0)] and v[0] >= oc.logodds(0.7)


@pytest.mark.parametrize("ext", [".pcd", ".ply"])
def test_point_cloud_files_parse_back(tmp_path, ext):
    import laser_slam_b200 as ls
    rng = np.random.default_rng(3)
    keys = np.sort(rng.integers(K0 - 3000, K0 + 3000, (500, 3)).astype(np.uint64) @ np.array([1, 1 << 16, 1 << 32], np.uint64))
    xyz = oc.centres(keys, 0.075)
    path = str(tmp_path / ("map" + ext))
    ls.write_point_cloud(path, xyz)
    lines = open(path).read().splitlines()
    end = lines.index("DATA ascii") if ext == ".pcd" else lines.index("end_header")
    if ext == ".pcd":
        assert "FIELDS x y z" in lines and "VERSION 0.7" in lines and f"POINTS {len(xyz)}" in lines
    else:
        assert lines[0] == "ply" and f"element vertex {len(xyz)}" in lines
    back = np.array([[F32(t) for t in ln.split()] for ln in lines[end + 1:]], F32)
    assert np.array_equal(_bits(back), _bits(xyz))
    with pytest.raises(ValueError):
        ls.write_point_cloud(str(tmp_path / "map.bt"), xyz)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _dev_map(ls, dev):
    k, v, _ = dev.download(ls.OCC_KNOWN)
    return k, v


def _stats_dict(st):
    return dict(rays_cast=st.rays_cast, rays_skipped=st.rays_skipped, free_updates=st.free_updates,
                occupied_updates=st.occupied_updates, known_voxels=st.known_voxels)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_known_answers_on_the_device(gpu_ctx, name):
    import laser_slam_b200 as ls
    params, scans, check = CASES[name]
    ring = gpu_ctx.create_map(2, 1024)
    dev = ls.OccupancyMap(gpu_ctx, **params)
    o = oc.OccupancyMap(**params)
    for c, T in scans:
        sid = ring.push_scan(c, np.zeros((len(c), 3), F32))
        assert _stats_dict(dev.insert_scan(ring, sid, T)) == o.insert_scan(c, T)
    assert _same_map(_dev_map(ls, dev), o.download())
    k, v, cen = dev.download(ls.OCC_OCCUPIED)
    assert _same_map((k, v), o.download(oc.OCCUPIED))
    assert np.array_equal(_bits(cen[:, :3]), _bits(oc.centres(k, params["resolution"]))) and (cen[:, 3] == 1).all()
    dev.close()
    ring.close()


N_FULL = 12


@pytest.fixture(scope="module")
def full_scans(synth_mod):
    truth, _ = synth_mod.trajectory(0, N_FULL)
    return [synth_mod.scan(truth[k], 0, k)[0] for k in range(N_FULL)], [truth[k].astype(F32) for k in range(N_FULL)]


def _run_full(ls, ctx, full_scans, params, initial_capacity=0, check_at=(1, 6, 12)):
    scans, poses = full_scans
    ring = ctx.create_map(4, 131072)
    dev = ls.OccupancyMap(ctx, initial_capacity=initial_capacity, **params)
    o = oc.OccupancyMap(**params)
    nrm = np.zeros((131072, 3), F32)
    bricks = []
    for k in range(N_FULL):
        sid = ring.push_scan(scans[k], nrm)
        st = dev.insert_scan(ring, sid, poses[k])
        assert _stats_dict(st) == o.insert_scan(scans[k], poses[k])
        bricks.append(st.bricks)
        if k + 1 in check_at:
            assert _same_map(_dev_map(ls, dev), o.download())
            assert _same_map(dev.download(ls.OCC_OCCUPIED)[:2], o.download(oc.OCCUPIED))
    out = (_dev_map(ls, dev), bricks)
    dev.close()
    ring.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("params", [dict(), dict(resolution=0.1, max_range=-1.0)], ids=["defaults", "res0.1_unlimited"])
def test_full_scans_match_the_oracle(gpu_ctx, full_scans, params):
    import laser_slam_b200 as ls
    (keys, _), _ = _run_full(ls, gpu_ctx, full_scans, params)
    assert len(keys) > 1_000_000


@pytest.mark.gpu
def test_growth_from_a_tiny_capacity(gpu_ctx, full_scans):
    import laser_slam_b200 as ls
    params = dict(resolution=0.1, max_range=12.0)
    scans = (full_scans[0][:4], full_scans[1][:4])
    global N_FULL
    n_saved, N_FULL = N_FULL, 4
    try:
        small, bricks = _run_full(ls, gpu_ctx, scans, params, initial_capacity=16, check_at=(4,))
        big, _ = _run_full(ls, gpu_ctx, scans, params, check_at=())
    finally:
        N_FULL = n_saved
    assert bricks[0] > 16 and bricks[-1] > bricks[0]      # it grew, and kept growing across scans
    assert _same_map(small, big)


@pytest.mark.gpu
def test_errors_leave_the_map_unchanged(gpu_ctx, full_scans):
    import laser_slam_b200 as ls
    scans, poses = full_scans
    for bad in (dict(resolution=0.0), dict(resolution=-0.1), dict(prob_hit=1.0), dict(clamp_min=0.99),
                dict(max_range=float("nan"))):
        with pytest.raises(ls.LsError, match="rc=-1"):
            ls.OccupancyMap(gpu_ctx, **bad)
    ring = gpu_ctx.create_map(2, 131072)
    nrm = np.zeros((131072, 3), F32)
    first = ring.push_scan(scans[0], nrm)
    dev = ls.OccupancyMap(gpu_ctx)
    dev.insert_scan(ring, first, poses[0])
    before = (dev.download(ls.OCC_KNOWN), dev.download(ls.OCC_OCCUPIED))
    ring.push_scan(scans[1], nrm)
    ring.push_scan(scans[2], nrm)                        # evicts `first`
    st = ls.OccupancyStats()
    t = ls.colmajor(poses[0])
    assert ls.lib().ls_occupancy_insert_scan(dev._h, ring._h, first, t.ctypes.data, ctypes.byref(st)) == ls.LS_ERR_STATE
    n = ctypes.c_int64(-7)
    small = np.empty(10, np.uint64)
    assert ls.lib().ls_occupancy_download(dev._h, ls.OCC_KNOWN, small.ctypes.data, None, None, 10, ctypes.byref(n)) == ls.LS_ERR_ARG
    assert n.value == -7
    assert ls.lib().ls_occupancy_size(dev._h, 3, ctypes.byref(n)) == ls.LS_ERR_ARG
    after = (dev.download(ls.OCC_KNOWN), dev.download(ls.OCC_OCCUPIED))
    for a, b in zip(before, after):
        assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_insert_between_batch_begin_and_end(full_scans):
    import laser_slam_b200 as ls
    scans, poses = full_scans
    ctx = ls.Context(0)
    ring = ctx.create_map(16, 131072)
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(4)]
    problems = [(ids[k + 1], [ids[k]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[k]) @ poses[k + 1]) for k in range(3)]
    p = ls.default_params(max_iterations=5)
    alone = ring.register_batch(problems, p)
    dev = ls.OccupancyMap(ctx)
    o = oc.OccupancyMap()
    end = ring.begin_batch(problems, p)
    for k in range(2):
        dev.insert_scan(ring, ids[k], poses[k])
        o.insert_scan(scans[k], poses[k])
    res = end()
    for a, b in zip(res, alone):
        assert a["rc"] == b["rc"] and np.array_equal(a["T"], b["T"])
    assert _same_map(_dev_map(ls, dev), o.download())
    dev.close()
    ring.close()
    ctx.close()


@pytest.mark.gpu
def test_save_point_cloud_writes_the_occupied_centres(gpu_ctx, full_scans, tmp_path):
    import laser_slam_b200 as ls
    scans, poses = full_scans
    ring = gpu_ctx.create_map(2, 131072)
    dev = ls.OccupancyMap(gpu_ctx)
    dev.insert_scan(ring, ring.push_scan(scans[0], np.zeros((131072, 3), F32)), poses[0])
    want = dev.download(ls.OCC_OCCUPIED)[2][:, :3]
    for ext in (".pcd", ".ply"):
        path = str(tmp_path / ("map" + ext))
        assert dev.save_point_cloud(path) == len(want) > 0
        lines = open(path).read().splitlines()
        start = lines.index("DATA ascii" if ext == ".pcd" else "end_header") + 1
        assert np.array_equal(_bits(np.loadtxt(lines[start:], dtype=F32)), _bits(want))
    with pytest.raises(ValueError):
        dev.save_point_cloud(str(tmp_path / "map.bt"))
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_host_layer_insert_laser_tracks(synth_mod):
    """laser_slam::OccupancyMap::insertLaserTracks on an estimator with two workers, each with a time-0 scan: equals the
    oracle fed every scan by time (ties by track), the second time-0 scan dropped, at the poses lsh_trajectory reports."""
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    from test_local_map import _float_matrix
    n = 5
    truth, odom = synth_mod.trajectory(3, 2 * n + 2)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 3, k), 8) for k in range(2 * n)]
    odom7 = pg.se3_from_matrix(odom)
    off = pg.se3_from_matrix(np.array([[1, 0, 0, 3.0], [0, 1, 0, 2.0], [0, 0, 1, 0], [0, 0, 0, 1.0]]))
    est = host.Estimator(n_workers=2, nscan_in_sub_map=3)
    times = [[k * 10**8 for k in range(n)], [k * 10**8 + 5 * 10**7 * (k > 0) for k in range(n)]]
    for k in range(n):
        data = [scans[k], scans[n + k]]
        feats = [np.ascontiguousarray(d[0]) for d in data]
        nrms = [np.ascontiguousarray(d[1]) for d in data]
        est.step_batch([0, 1], [times[0][k], times[1][k]], [odom7[k], pg.se3_compose(off, odom7[n + k])],
                       [f.ctypes.data for f in feats], [x.ctypes.data for x in nrms], [len(f) for f in feats])
    params = dict(resolution=0.1, max_range=15.0)
    occ = host.OccupancyMap(est, **params)
    assert occ.insert_laser_tracks() == 2 * n - 1
    o = oc.OccupancyMap(**params)
    entries = []
    for w in range(2):
        ts, traj = est.trajectory(w)
        assert list(ts) == times[w]
        entries += [(int(ts[k]), w, k, _float_matrix(traj[k])) for k in range(n)]
    entries.sort(key=lambda e: e[:3])
    zero = False
    for t, w, k, T in entries:
        if t == 0:
            if zero:
                continue
            zero = True
        o.insert_scan(scans[w * n + k][0], T)
    assert _same_map(occ.voxels(1), o.download())
    k_occ, v_occ = occ.voxels(2)
    assert _same_map((k_occ, v_occ), o.download(oc.OCCUPIED)) and len(k_occ) > 0
    cloud = occ.occupied_cloud()
    assert np.array_equal(_bits(cloud[:, :3]), _bits(oc.centres(k_occ, 0.1)))
    occ.close()
    est.close()
