"""Euclidean distance map of the occupancy map (ls_distance_map_*): octomap's DynamicEDTOctomap over a box.  CPU: the
reference (tests/distance_map_ref.py) against an all-pairs brute force on random small grids, cases built to reach each
rule, scipy's EDT on the 12-scan map, and the query rule.  GPU: the device against the reference bit for bit, then the
snapshot rule, a read at a foreign resolution, repeatability, refusals, batches and laser_slam::DistanceMap.  The rules are
DESIGN.md §4b'''''''''."""
import ctypes
import math

import numpy as np
import pytest

import distance_map_ref as dr
import laser_slam_b200 as ls
from oracle import occupancy as oc
from test_occupancy import F32, K0, full_scans  # noqa: F401  (full_scans: fixture)

L_OCC = oc.logodds(0.7)


def _bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def _key(x, y, z):
    return (x + K0) | ((y + K0) << 16) | ((z + K0) << 32)


# ---- CPU: the reference against brute force -------------------------------------------------------------------------
def brute(grid, M):
    """Every cell against every obstacle: the least s, then the smallest cell index (= packed key), capped at M."""
    sz, sy, sx = grid.shape
    z, y, x = np.meshgrid(np.arange(sz), np.arange(sy), np.arange(sx), indexing="ij")
    cells = np.stack([x.ravel(), y.ravel(), z.ravel()], 1).astype(np.int64)
    obs = np.flatnonzero(grid.ravel())
    if len(obs) == 0:
        return np.full(grid.shape, M, np.int32), np.full(grid.shape, -1, np.int32)
    d = ((cells[:, None, :] - cells[obs][None, :, :]) ** 2).sum(-1)
    j = np.argmin(d, axis=1)  # the first least: obstacles are in ascending index
    s = d[np.arange(len(cells)), j]
    keep = s <= M
    return (np.where(keep, s, M).astype(np.int32).reshape(grid.shape),
            np.where(keep, obs[j], -1).astype(np.int32).reshape(grid.shape))


def test_reference_equals_brute_force_on_random_grids():
    rng = np.random.default_rng(11)
    ties = 0
    for i in range(200):
        shape = tuple(int(v) for v in rng.choice([1, 2, 3, 5, 8, 11], 3))
        density = [0.0, 0.02, 0.1, 0.3, 0.7, 1.0][i % 6]
        grid = (rng.random(shape) < density).astype(np.uint8)
        s0, _ = brute(grid, 1 << 30)
        present = np.unique(s0[s0 > 0])
        # maxdist: small, large, and exactly a squared distance the grid holds (cells at s == M and M + 1)
        M = [1, 4, 9, 1 << 30][i % 4] if len(present) == 0 or i % 3 else int(rng.choice(present))
        s, w = dr.transform(grid, M)
        ws, ww = brute(grid, M)
        assert np.array_equal(s, ws) and np.array_equal(w, ww), (i, shape, density, M)
        ties += int((s0 == M).any())
    assert ties > 10


def _tied(grid, cell):
    """The obstacles at the least s of a cell (x, y, z), by index."""
    sz, sy, sx = grid.shape
    obs = np.flatnonzero(grid.ravel())
    c = np.array([(o % sx, (o // sx) % sy, o // (sx * sy)) for o in obs])
    d = ((c - np.array(cell)) ** 2).sum(1)
    return obs[d == d.min()], int(d.min())


def _index(shape, x, y, z):
    return (z * shape[1] + y) * shape[2] + x


CASES = {}  # name: (shape (sz, sy, sx), obstacle cells (x, y, z), M, the cell to look at, its (s, obstacle cell))


def case(name, shape, obstacles, M, cell, want):
    CASES[name] = (shape, obstacles, M, cell, want)


case("left_right", (1, 1, 9), [(1, 0, 0), (7, 0, 0)], 100, (4, 0, 0), (9, (1, 0, 0)))
case("above_below", (9, 1, 1), [(0, 0, 1), (0, 0, 7)], 100, (0, 0, 4), (9, (0, 0, 1)))
case("front_back", (1, 9, 1), [(0, 2, 0), (0, 6, 0)], 100, (0, 4, 0), (4, (0, 2, 0)))
case("z_beats_x", (5, 1, 5), [(4, 0, 2), (2, 0, 0)], 100, (2, 0, 2), (4, (2, 0, 0)))
case("y_beats_x", (1, 5, 5), [(4, 2, 0), (2, 0, 0)], 100, (2, 2, 0), (4, (2, 0, 0)))
case("diagonal_ties", (5, 5, 5), [(4, 4, 2), (2, 4, 4), (4, 2, 4), (0, 4, 2)], 100, (2, 2, 2), (8, (0, 4, 2)))
case("at_M", (1, 3, 6), [(0, 0, 0)], 4, (2, 0, 0), (4, (0, 0, 0)))
case("at_M_plus_1", (1, 3, 6), [(0, 0, 0)], 4, (2, 1, 0), (4, None))
case("one_obstacle_is_its_own", (3, 3, 3), [(1, 1, 1)], 1, (1, 1, 1), (0, (1, 1, 1)))
case("far_beats_capped", (1, 1, 40), [(0, 0, 0), (39, 0, 0)], 400, (25, 0, 0), (196, (39, 0, 0)))


def _grid(shape, obstacles):
    g = np.zeros(shape, np.uint8)
    for x, y, z in obstacles:
        g[z, y, x] = 1
    return g


@pytest.mark.parametrize("name", sorted(CASES))
def test_constructed_cases(name):
    shape, obstacles, M, cell, (s_want, o_want) = CASES[name]
    g = _grid(shape, obstacles)
    tied, s_min = _tied(g, cell)
    if name in ("left_right", "above_below", "front_back", "z_beats_x", "y_beats_x", "diagonal_ties"):
        assert len(tied) >= 2  # precondition: the cell has equidistant obstacles
    if name == "at_M":
        assert s_min == M
    if name == "at_M_plus_1":
        assert s_min == M + 1
    s, w = dr.transform(g, M)
    x, y, z = cell
    assert s[z, y, x] == s_want
    assert w[z, y, x] == (-1 if o_want is None else _index(shape, *o_want))
    ws, ww = brute(g, M)
    assert np.array_equal(s, ws) and np.array_equal(w, ww)


def test_obstacle_one_key_outside_the_box():
    kmin, size = np.array([K0 + 10, K0 - 5, K0], np.int32), np.array([6, 4, 3], np.int32)
    keys = np.array([_key(9, -5, 0), _key(16, -5, 0), _key(10, -6, 0), _key(10, -5, 3), _key(15, -2, 2)], np.uint64)
    lo = np.full(len(keys), 2.0, np.float32)
    g = dr.obstacles(keys, lo, L_OCC, kmin, size, False)
    assert g.sum() == 1 and g[2, 3, 5] == 1  # only the last is inside
    g0 = dr.obstacles(keys[:4], lo[:4], L_OCC, kmin, size, False)
    assert g0.sum() == 0  # precondition: each of the four is one key outside on one axis
    s, w = dr.transform(g0, 16)
    assert (s == 16).all() and (w == -1).all()


def test_obstacle_rule():
    kmin, size = np.array([K0, K0, K0], np.int32), np.array([3, 1, 1], np.int32)
    keys = np.array([_key(0, 0, 0), _key(1, 0, 0)], np.uint64)
    lo = np.array([L_OCC, np.nextafter(F32(L_OCC), F32(-1))], np.float32)  # exactly L_occ is occupied, one ulp below free
    assert dr.obstacles(keys, lo, L_OCC, kmin, size, False).ravel().tolist() == [1, 0, 0]
    assert dr.obstacles(keys, lo, L_OCC, kmin, size, True).ravel().tolist() == [1, 0, 1]  # cell 2 is unknown


def test_unknown_as_occupied_on_an_empty_map():
    kmin, size = np.array([K0 - 2, K0, K0 + 1], np.int32), np.array([4, 3, 2], np.int32)
    g = dr.obstacles(np.zeros(0, np.uint64), np.zeros(0, np.float32), L_OCC, kmin, size, True)
    assert g.all()
    s, w = dr.transform(g, 1)
    assert (s == 0).all() and np.array_equal(w.ravel(), np.arange(24))


def test_box_and_cap_rules():
    kmin, size = dr.box((-0.75, -0.01, 0.0), (-0.05, 0.0, 0.25), 0.25)  # negative corners; both ends included
    assert kmin.tolist() == [K0 - 3, K0 - 1, K0] and size.tolist() == [3, 2, 2]
    kmin, size = dr.box((-0.3, 0, 0), (-0.3, 0, 0), 0.1)  # (float)-0.3 * 10 is below -3: the key is floor's, -4
    assert kmin.tolist() == [K0 - 4, K0, K0] and size.tolist() == [1, 1, 1]
    kmin, size = dr.box((32766.5, -32768.0, 0.0), (32767.9, -32767.5, 0.0), 1.0)  # the key-space edges
    assert kmin.tolist() == [65534, 0, K0] and size.tolist() == [2, 1, 1]
    assert dr.box((0, 0, 0), (32768.0, 0, 0), 1.0) is None and dr.box((-32768.5, 0, 0), (0, 0, 0), 1.0) is None
    assert dr.box((np.nan, 0, 0), (0, 0, 0), 1.0) is None
    assert dr.cap(1.0, 0.075) == (14, 196, float(F32(14 * 0.075)))
    assert dr.cap(0.15, 0.075)[0] == int(float(F32(0.15)) / 0.075 + 1.0)


def test_query_rule_at_the_faces():
    res = 0.25
    kmin, size = np.array([K0 - 4, K0 + 2, K0], np.int32), np.array([5, 3, 2], np.int32)
    g = np.zeros((2, 3, 5), np.uint8)
    g[1, 2, 4] = 1
    s, w = dr.transform(g, 25)
    lo = (kmin - K0) * res  # the lower faces, exact at res 0.25
    hi = (kmin + size - K0) * res  # one key past the upper faces
    inside = [lo, hi - 1e-3, np.nextafter(hi.astype(F32), F32(-np.inf))]
    outside = [np.nextafter(lo.astype(F32), F32(-np.inf)), hi]
    pts = []
    for a in range(3):
        for p, want in [(q, True) for q in inside] + [(q, False) for q in outside]:
            x = (lo + hi) / 2
            x[a] = p[a]
            pts.append((x, want))
    for bad in (np.nan, np.inf, -np.inf):
        pts.append((np.array([bad, lo[1], lo[2]]), False))
        pts.append((np.array([lo[0], lo[1], bad]), False))
    d, q, o = dr.query(s, w, kmin, size, res, np.array([p for p, _ in pts]))
    for i, (p, want) in enumerate(pts):
        if not want:
            assert d[i] == -1.0 and q[i] == -1 and np.isnan(o[i]).all(), p
            continue
        c = [math.floor(float(F32(p[a])) * (1 / res)) + K0 - kmin[a] for a in range(3)]
        assert q[i] == s[c[2], c[1], c[0]]
        assert _bits(d[i]) == _bits(F32(float(F32(math.sqrt(q[i]))) * res))
        assert np.array_equal(_bits(o[i]), _bits(np.array([(k - K0 + 0.5) * res for k in (kmin[0] + 4, kmin[1] + 2,
                                                                                            kmin[2] + 1)], F32)))
    g[:] = 0
    s, w = dr.transform(g, 25)
    d, q, o = dr.query(s, w, kmin, size, res, [(lo + hi) / 2])
    assert q[0] == 25 and d[0] == F32(5 * res) and np.isnan(o[0]).all()  # no obstacle: the cap, NaN obstacle


# ---- CPU: the reference against scipy on the 12-scan map ------------------------------------------------------------
@pytest.fixture(scope="module")
def oracle_voxels(full_scans):
    scans, poses = full_scans
    o = oc.OccupancyMap(**oc.DEFAULTS)
    for k in range(len(scans)):
        o.insert_scan(scans[k], poses[k])
    k, v = o.download()
    o.close()
    return k, v


def test_reference_equals_scipy_on_the_twelve_scan_map(full_scans, oracle_voxels):
    from scipy import ndimage
    p = full_scans[1][6][:3, 3].astype(np.float64)
    f = dr.Field(*oracle_voxels, 0.075, L_OCC, 3.0, p - 7.5, p + 7.5)
    assert f.obstacles > 1000 and f.cells > 10 ** 6
    d, idx = ndimage.distance_transform_edt(f.grid == 0, return_indices=True)
    s = np.rint(d * d).astype(np.int64)
    assert np.array_equal(f.s, np.minimum(s, f.M).astype(np.int32))
    assert (s > f.M).any() and (s < f.M).any()  # both sides of the cap
    keep = f.site >= 0
    w = f.site[keep].astype(np.int64)
    sx, sy = int(f.size[0]), int(f.size[1])
    zz, yy, xx = np.nonzero(keep)
    dist = (w % sx - xx) ** 2 + ((w // sx) % sy - yy) ** 2 + (w // (sx * sy) - zz) ** 2
    assert np.array_equal(dist, f.s[keep]) and f.grid.ravel()[w].all()


# ---- GPU ----------------------------------------------------------------------------------------------------------
@pytest.fixture
def keep():
    """keep(h) returns h and closes it when the test ends, in reverse order, even when the test fails."""
    opened = []

    def add(h):
        opened.append(h)
        return h

    yield add
    for h in reversed(opened):
        h.close()


def _same_field(dm, f, st):
    assert (list(st.min_key), list(st.size)) == (f.kmin.tolist(), f.size.tolist())
    assert (st.cells, st.obstacles, st.max_sqdist_cells) == (f.cells, f.obstacles, f.M)
    assert F32(st.max_dist) == F32(f.max_dist)
    s, k = dm.download()
    assert s.shape == f.s.shape and np.array_equal(s, f.s) and np.array_equal(k, f.keys())


def _same_queries(dm, f, pts):
    got, want = dm.query(pts), f.query(pts)
    assert np.array_equal(got[1], want[1])
    assert np.array_equal(_bits(got[0]), _bits(want[0])) and np.array_equal(_bits(got[2]), _bits(want[2]))
    return got


def _centres(keys, res):
    return np.stack([((keys >> np.uint64(16 * a)) & np.uint64(0xFFFF)).astype(np.float64) for a in range(3)], 1)


def _query_points(f, keys, res, rng):
    """Every known voxel's centre, random points in and around the box, points outside, NaN."""
    lo = (f.kmin - K0) * res
    hi = (f.kmin + f.size - K0) * res
    cen = ((_centres(keys, res) - K0 + 0.5) * res).astype(F32)
    rnd = rng.uniform(lo - 1.0, hi + 1.0, (50_000, 3)).astype(F32)
    out = np.array([lo - 0.5, hi + 0.5, [lo[0], lo[1], hi[2] + 0.01], [np.nan, 0, 0], [0, np.inf, 0]], F32)
    return np.concatenate([cen, rnd, out])


def _case_map(ctx, name, keep_, res=0.1):
    """The case's obstacles as occupied voxels (one-voxel setOccupied boxes) and a free voxel beside each, in a map at res;
    the distance map's box is the case's grid at keys K0 + 3 ...."""
    shape, obstacles, M, cell, _ = CASES[name]
    om = keep_(ls.OccupancyMap(ctx, resolution=res))
    base = np.array([3, -2, 5])
    for x, y, z in obstacles:
        om.set_occupied(((np.array([x, y, z]) + base) + 0.5) * res, (res, res, res))
    om.set_free(((base - 1) + 0.5) * res, (res, res, res))
    lo = base * res + res / 2
    hi = (base + np.array(shape[::-1]) - 1) * res + res / 2
    m = int(math.isqrt(M))
    return om, lo, hi, (m - 0.5) * res  # maxdist: m cells


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_constructed_cases_on_the_device(gpu_ctx, name, keep):
    om, lo, hi, maxdist = _case_map(gpu_ctx, name, keep)
    k, v, _ = om.download(ls.OCC_KNOWN)
    for unknown in (False, True):
        dm = keep(ls.DistanceMap(gpu_ctx, maxdist, lo, hi, unknown))
        f = dr.Field(k, v, 0.1, L_OCC, maxdist, lo, hi, unknown)
        if not unknown:
            assert f.obstacles == len(CASES[name][1]) and f.M == CASES[name][2]  # the map holds the case
        _same_field(dm, f, dm.update(om))
        _same_queries(dm, f, _query_points(f, k, 0.1, np.random.default_rng(1)))
        dm.close()
    om.close()


@pytest.fixture(scope="module")
def twelve(full_scans, gpu_ctx):
    scans, poses = full_scans
    ring = gpu_ctx.create_map(2, 131072)
    om = ls.OccupancyMap(gpu_ctx)
    nrm = np.zeros((131072, 3), F32)
    for k in range(len(scans)):
        om.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
    yield om, ring, poses
    om.close()
    ring.close()


@pytest.mark.gpu
@pytest.mark.parametrize("unknown", [False, True], ids=["occupied", "unknown_as_occupied"])
def test_twelve_scan_map(gpu_ctx, twelve, unknown, keep):
    om, _, poses = twelve
    k, v, _ = om.download(ls.OCC_KNOWN)
    p = poses[6][:3, 3].astype(np.float64)
    blo, bhi = om.bounds()
    rng = np.random.default_rng(3)
    for lo, hi in ((p - 10.0, p + 10.0), (blo, bhi - 0.01)):
        for maxdist in (1.0, 10.0):
            dm = keep(ls.DistanceMap(gpu_ctx, maxdist, lo, hi, unknown))
            st = dm.update(om)
            f = dr.Field(k, v, 0.075, L_OCC, maxdist, lo, hi, unknown)
            assert f.obstacles > 1000 and (f.s < f.M).any() and (unknown or maxdist > 1.0 or (f.s == f.M).any())
            _same_field(dm, f, st)
            _same_queries(dm, f, _query_points(f, k, 0.075, rng))
            assert dm.last_query.outside > 0
            dm.close()


@pytest.mark.gpu
def test_snapshot_rule(gpu_ctx, full_scans, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    om = keep(ls.OccupancyMap(gpu_ctx, resolution=0.1))
    nrm = np.zeros((131072, 3), F32)
    om.insert_scan(ring, ring.push_scan(scans[0], nrm), poses[0])
    p = poses[0][:3, 3]
    dm = keep(ls.DistanceMap(gpu_ctx, 2.0, p - 8.0, p + 8.0))
    with pytest.raises(ls.LsError, match="rc=-4"):
        dm.query([p])
    with pytest.raises(ls.LsError, match="rc=-4"):
        dm.download()
    dm.update(om)
    before = dm.download()
    pts = p + np.random.default_rng(2).uniform(-9.0, 9.0, (20_000, 3))
    q0 = dm.query(pts)
    om.insert_scan(ring, ring.push_scan(scans[3], nrm), poses[3])
    om.set_occupied(p, (1.0, 1.0, 1.0))
    after = dm.download()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    q1 = dm.query(pts)
    assert all(np.array_equal(_bits(a) if a.dtype == F32 else a, _bits(b) if b.dtype == F32 else b) for a, b in zip(q0, q1))
    st = dm.update(om)
    fresh = keep(ls.DistanceMap(gpu_ctx, 2.0, p - 8.0, p + 8.0))
    fresh.update(om)
    assert all(np.array_equal(a, b) for a, b in zip(dm.download(), fresh.download()))
    k, v, _ = om.download(ls.OCC_KNOWN)
    _same_field(dm, dr.Field(k, v, 0.1, L_OCC, 2.0, p - 8.0, p + 8.0), st)
    assert not np.array_equal(before[0], dm.download()[0])
    dm.close(), fresh.close(), om.close(), ring.close()


@pytest.mark.gpu
def test_update_after_a_read_at_a_foreign_resolution(gpu_ctx, twelve, tmp_path, keep):
    om, _, poses = twelve
    path = str(tmp_path / "map.ot")
    om.save_octomap_full(path)
    other = keep(ls.OccupancyMap(gpu_ctx, resolution=0.2))
    p = poses[4][:3, 3]
    dm = keep(ls.DistanceMap(gpu_ctx, 3.0, p - 6.0, p + 6.0, True))
    st0 = dm.update(other)
    assert st0.resolution == 0.2 and st0.obstacles == st0.cells  # an empty map, unknown as occupied
    other.read_octomap_full(path)
    st = dm.update(other)
    assert st.resolution == 0.075
    k, v, _ = other.download(ls.OCC_KNOWN)
    f = dr.Field(k, v, 0.075, L_OCC, 3.0, p - 6.0, p + 6.0, True)
    _same_field(dm, f, st)
    _same_queries(dm, f, _query_points(f, k[::5], 0.075, np.random.default_rng(4)))
    dm.close(), other.close()


@pytest.mark.gpu
def test_two_updates_give_identical_bytes(gpu_ctx, twelve, keep):
    om, _, poses = twelve
    p = poses[9][:3, 3]
    for unknown in (False, True):
        dm = keep(ls.DistanceMap(gpu_ctx, 2.0, p - 12.0, p + 12.0, unknown))
        dm.update(om)
        a = dm.download()
        dm.update(om)
        b = dm.download()
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
        dm.close()


def _occ_snapshot(om):
    k, v, _ = om.download(ls.OCC_KNOWN)
    return k, _bits(v)


@pytest.mark.gpu
def test_refusals(gpu_ctx, twelve, keep):
    om, _, poses = twelve
    occ0 = _occ_snapshot(om)
    p = poses[2][:3, 3]
    L = ls.lib()
    for maxdist, lo, hi in ((0.0, p - 1, p + 1), (-1.0, p - 1, p + 1), (np.nan, p - 1, p + 1), (np.inf, p - 1, p + 1),
                            (1.0, p + 1, p - 1), (1.0, (np.nan, 0, 0), p), (1.0, p, (0, np.inf, 0))):
        with pytest.raises(ls.LsError, match="rc=-1"):
            ls.DistanceMap(gpu_ctx, maxdist, lo, hi)
    dm = keep(ls.DistanceMap(gpu_ctx, 1.0, p - 5.0, p + 5.0))
    dm.update(om)
    field = dm.download()
    pts = p + np.random.default_rng(6).uniform(-6.0, 6.0, (5000, 3))
    q = dm.query(pts)
    refused = [keep(ls.DistanceMap(gpu_ctx, 0.075 * 46340.5, p - 1, p + 1)),            # m > 46340
               keep(ls.DistanceMap(gpu_ctx, 1.0, (-2500.0, 0, 0), (2500.0, 0, 0))),     # corner keys invalid
               keep(ls.DistanceMap(gpu_ctx, 1.0, (0, 0, 0), (80.0, 80.0, 80.0)))]       # 1067^3 cells > 2^30
    for r in refused:
        with pytest.raises(ls.LsError, match="rc=-1"):
            r.update(om)
        with pytest.raises(ls.LsError, match="rc=-4"):
            r.query(pts[:3])
    ok = keep(ls.DistanceMap(gpu_ctx, 0.075 * 46339.5, p - 1, p + 1))  # m = 46340 is accepted
    assert ok.update(om).max_sqdist_cells == 46340 * 46340
    # a refused update keeps the previous field: the box's corner has no key at 0.001 m (40 m is key 40000 + 32768)
    small = keep(ls.OccupancyMap(gpu_ctx, resolution=0.001))
    far = keep(ls.DistanceMap(gpu_ctx, 1.0, (40.0, 0.0, 0.0), (41.0, 1.0, 1.0)))
    far.update(om)
    far_field = far.download()
    with pytest.raises(ls.LsError, match="rc=-1"):
        far.update(small)
    assert all(np.array_equal(a, b) for a, b in zip(far_field, far.download()))
    h = dm._h
    s3 = np.zeros(3, F32)
    out = np.zeros(3, np.float32)
    assert L.ls_distance_map_query(h, None, 1, out.ctypes.data, None, None, None) == ls.LS_ERR_ARG
    assert L.ls_distance_map_query(h, s3.ctypes.data, -1, out.ctypes.data, None, None, None) == ls.LS_ERR_ARG
    assert L.ls_distance_map_query(h, None, 0, None, None, None, None) == 0
    assert L.ls_distance_map_update(h, None, None) == ls.LS_ERR_ARG
    n = ctypes.c_int64(0)
    assert L.ls_distance_map_download(h, None, None, 0, ctypes.byref(n)) == ls.LS_ERR_ARG and n.value == field[0].size
    assert L.ls_distance_map_download(h, None, None, 0, None) == ls.LS_ERR_ARG
    assert all(np.array_equal(a, b) for a, b in zip(field, dm.download()))
    q2 = dm.query(pts)
    assert all(np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)) for a, b in zip(q, q2))
    occ1 = _occ_snapshot(om)
    assert np.array_equal(occ0[0], occ1[0]) and np.array_equal(occ0[1], occ1[1])
    for h_ in [dm, ok, far, small] + refused:
        h_.close()


@pytest.mark.gpu
def test_calls_between_batch_begin_and_end(full_scans, keep):
    scans, poses = full_scans
    ctx = keep(ls.Context(0))
    ring = keep(ctx.create_map(4, 131072))
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(2)]
    om = keep(ls.OccupancyMap(ctx, resolution=0.1))
    om.insert_scan(ring, ids[0], poses[0])
    p = poses[0][:3, 3]
    dm = keep(ls.DistanceMap(ctx, 2.0, p - 6.0, p + 6.0))
    pts = p + np.random.default_rng(8).uniform(-7.0, 7.0, (10_000, 3))
    end = ring.begin_batch([(ids[1], [ids[0]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[0]) @ poses[1])])
    try:  # the batch always ends, so a failed comparison cannot leave it open
        st = dm.update(om)
        field = dm.download()
        got = dm.query(pts)
    finally:
        end()
    k, v, _ = om.download(ls.OCC_KNOWN)
    f = dr.Field(k, v, 0.1, L_OCC, 2.0, p - 6.0, p + 6.0)
    assert (st.cells, st.obstacles) == (f.cells, f.obstacles)
    assert np.array_equal(field[0], f.s) and np.array_equal(field[1], f.keys())
    want = f.query(pts)
    assert np.array_equal(got[1], want[1]) and np.array_equal(_bits(got[0]), _bits(want[0]))
    assert np.array_equal(_bits(got[2]), _bits(want[2]))
    dm.close(), om.close(), ring.close(), ctx.close()


@pytest.mark.gpu
def test_host_layer_equals_the_abi(gpu_ctx, synth_mod, keep):
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    n = 3
    truth, odom = synth_mod.trajectory(3, n + 2)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 3, k), 8) for k in range(n)]
    odom7 = pg.se3_from_matrix(odom)
    est = keep(host.Estimator(n_workers=1, nscan_in_sub_map=3))
    for k in range(n):
        f, x = np.ascontiguousarray(scans[k][0]), np.ascontiguousarray(scans[k][1])
        est.step_batch([0], [k * 10**8], [odom7[k]], [f.ctypes.data], [x.ctypes.data], [len(f)])
    hm = keep(host.OccupancyMap(est, resolution=0.1, max_range=15.0))
    hm.insert_laser_tracks()
    k, v = hm.voxels(1)
    p = truth[1][:3, 3]
    lo, hi = p - 5.0, p + 5.0
    pts = np.concatenate([p + np.random.default_rng(9).uniform(-6.0, 6.0, (3000, 3)), [[np.nan, 0, 0]]])
    for unknown in (False, True):
        hd = keep(host.DistanceMap(hm, 1.5, lo, hi, unknown))
        with pytest.raises(ls.LsError):
            hd.query(pts[:2])  # before the first update
        max_dist, max_sq = hd.update()
        f = dr.Field(k, v, 0.1, L_OCC, 1.5, lo, hi, unknown)
        assert (F32(max_dist), max_sq) == (F32(f.max_dist), f.M)
        want = f.query(pts)
        for single in (False, True):
            d, s, c = hd.query(pts, single=single)
            assert np.array_equal(s, want[1]) and np.array_equal(_bits(d), _bits(want[0]))
            assert np.array_equal(_bits(c.astype(F32)), _bits(want[2]))
        hd.close()
    with pytest.raises(ls.LsError):
        host.DistanceMap(hm, 0.0, lo, hi)
    hm.close()
    est.close()
