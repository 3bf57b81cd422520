"""Box status and robot collision on the resident occupancy map (ls_occupancy_box_status / _check_paths; DESIGN.md
§4b''''''''''').  CPU: the literal restatement (tests/occupancy_collision_ref.py) equals the grid restatement and itself in
reverse and random order; answers derived by hand; cases found by search, each with a precondition that it reaches its
branch.  GPU: every result bit for bit against the restatement, on the hand and searched cases, on the 12-scan map, after
edits, a .ot read and clear; the calls change nothing; refusals; calls inside a batch; the C++ layer against the ABI."""
import numpy as np
import pytest

import laser_slam_b200 as ls
import occupancy_collision_ref as cr
import occupancy_edits_ref as er
from oracle import occupancy as oc
from test_occupancy import full_scans  # noqa: F401  (fixture)

F32 = np.float32
K0 = cr.K0
L_OCC = oc.logodds(0.7)
L_MIN, L_MAX = F32(oc.logodds(0.12)), F32(oc.logodds(0.97))
FREE, OCC, UNK = cr.CELL_FREE, cr.CELL_OCCUPIED, cr.CELL_UNKNOWN


def _vox(edits, res):
    """The map {packed key: log-odds} that setFree / setOccupied of the edit boxes (centre, size, occupied) make."""
    vox = {}
    if edits:
        er.Edits(res, L_MIN, L_MAX, L_OCC).set_boxes(vox, *zip(*edits))
    return vox


def _voxel(k, res):
    """An edit box that sets voxel k (key triple) only."""
    c = tuple((k[a] - K0 + 0.5) * res for a in range(3))
    assert er.box_keys(c, (res,) * 3, res) == [cr.pack(*k)]
    return c, (res,) * 3


# ---- CPU: the restatements agree ------------------------------------------------------------------------------------
def _random_map(rng, res, radius):
    """Known voxels within `radius` m of the origin, mostly free, with sparse occupied voxels and unknown holes."""
    r = int(radius / res)
    ks = np.arange(K0 - r, K0 + r)
    g = np.stack(np.meshgrid(ks, ks, ks, indexing="ij"), -1).reshape(-1, 3)
    scale = (res / 0.075) ** 3  # about as many occupied voxels and holes per m^3 at every resolution
    keep = rng.random(len(g)) > 0.0015 * scale
    occ = rng.random(keep.sum()) < 0.002 * scale
    vals = np.where(occ, L_MAX, rng.choice([L_MIN, F32(-0.4), F32(0.2)], keep.sum())).astype(F32)
    keys = g[keep, 0] | (g[keep, 1] << 16) | (g[keep, 2] << 32)
    return keys.astype(np.uint64), vals


def _random_boxes(rng, res, n, max_work=30000):
    out = []
    while len(out) < n:
        c = rng.uniform(-0.8, 0.8, 3)
        s = rng.uniform(0.0, 3.0 if rng.random() < 0.5 else 0.6, 3)
        s[rng.random(3) < 0.15] = 0.0  # zero axes
        if np.prod(s / res + 2) <= max_work:
            out.append((c, s))
    return out


@pytest.mark.parametrize("res", [0.075, 0.1, 0.25, 1 / 30])
def test_literal_equals_grid_and_any_order(res):
    rng = np.random.default_rng(int(res * 1e4))
    keys, vals = _random_map(rng, res, 1.2)
    vox = cr.as_dict(keys, vals)
    boxes = _random_boxes(rng, res, 60)
    lo, shape = cr.BoxGrid.covering([b[0] for b in boxes], [b[1] for b in boxes], res)
    grid = cr.BoxGrid(keys, vals, L_OCC, lo, shape)
    seen = set()
    for i, (c, s) in enumerate(boxes):
        want = cr.box_status(vox, c, s, res, L_OCC)
        assert grid.status(c, s, res) == want, (c, s)
        if i < 20:
            assert cr.box_status(vox, c, s, res, L_OCC, order="reverse") == want
            assert cr.box_status(vox, c, s, res, L_OCC, order=np.random.default_rng(i)) == want
        seen.add(want)
    assert seen == {FREE, OCC, UNK}


# ---- CPU: answers derived by hand (res 0.1) -------------------------------------------------------------------------
RES = 0.1
OCC_A = (K0, K0, K0)               # the voxel at (0.05, 0.05, 0.05)
OCC_FACE = (K0 + 5, K0 - 5, K0 - 5)  # centre (0.55, -0.45, -0.45)
OCC_END = (K0 + 20, K0 - 5, K0 - 5)  # centre (2.05, -0.45, -0.45)
OCC_EDGE = (65534, K0 + 1, K0)     # near the key space's upper x edge
HAND_EDITS = [((0.0, 0.0, 0.0), (5.0, 2.0, 2.0), False),       # x keys K0-25 ... K0+25, y and z K0-10 ... K0+10 free
              ((3276.5, 0.0, 0.0), (1.0, 2.0, 2.0), False)]    # x keys 65528 ... 65535 free
HAND_EDITS += [_voxel(k, RES) + (True,) for k in (OCC_A, OCC_FACE, OCC_END, OCC_EDGE)]
FREE_BOX = ((-0.45, -0.45, -0.45), (0.5, 0.5, 0.5))
HAND = {
    "occupied centre": (((0.05, 0.05, 0.05), (0.3, 0.3, 0.3)), OCC),
    "unknown centre": (((8.05, 0.05, 0.05), (0.3, 0.3, 0.3)), UNK),
    "all free": (FREE_BOX, FREE),
    "occupied one key inside a face": (((0.35, -0.45, -0.45), (0.4, 0.4, 0.4)), OCC),
    "occupied one key outside a face": (((0.25, -0.45, -0.45), (0.4, 0.4, 0.4)), FREE),
    "size 0 beside an occupied voxel": (((0.55, -0.45, -0.35), (0.0, 0.0, 0.0)), FREE),
    "size 0 on an occupied voxel": (((0.55, -0.45, -0.45), (0.0, 0.0, 0.0)), OCC),
    "nan centre": (((float("nan"), 0.05, 0.05), (1.0, 1.0, 1.0)), UNK),
    "infinite centre": (((0.05, float("inf"), 0.05), (1.0, 1.0, 1.0)), UNK),
    "crossing the key space's edge": (((3276.65, 0.05, 0.05), (0.6, 0.3, 0.3)), UNK),
}


@pytest.fixture(scope="module")
def hand_vox():
    return _vox(HAND_EDITS, RES)


def test_hand_map_preconditions(hand_vox):
    assert all(cr.state(hand_vox, cr.pack(*k), L_OCC) == OCC for k in (OCC_A, OCC_FACE, OCC_END, OCC_EDGE))
    # one key inside the face: the box's x corner keys end at OCC_FACE's key and its cube passes; outside: they end before
    (c, s), _ = HAND["occupied one key inside a face"]
    assert cr.key_f(cr.corners(c[0], s[0])[1], RES) == OCC_FACE[0]
    assert cr.cube_passes(OCC_FACE[0], *cr.corners(c[0], s[0]), RES)
    (c, s), _ = HAND["occupied one key outside a face"]
    assert cr.key_f(cr.corners(c[0], s[0])[1], RES) == OCC_FACE[0] - 1
    # the edge box: its x max corner has an invalid key, so the occupied voxel inside it is not seen, and a loop point
    # keys outside the key space
    (c, s), _ = HAND["crossing the key space's edge"]
    lo, hi = zip(*(cr.corners(c[a], s[a]) for a in range(3)))
    assert cr.key_f(hi[0], RES) is None and all(cr.key_f(lo[a], RES) <= OCC_EDGE[a] <= cr.key_f(hi[a], RES) for a in (1, 2))
    assert cr.key_f(lo[0], RES) <= OCC_EDGE[0] and cr.state(hand_vox, cr.pack(*[cr.key_d(x, RES) for x in c]), L_OCC) == FREE


@pytest.mark.parametrize("name", sorted(HAND))
def test_hand_answers(hand_vox, name):
    (c, s), want = HAND[name]
    assert cr.box_status(hand_vox, c, s, RES, L_OCC) == want


def test_collision_modes():
    assert [cr.collides(s, True) for s in (FREE, OCC, UNK)] == [False, True, True]
    assert [cr.collides(s, False) for s in (FREE, OCC, UNK)] == [False, True, False]


P_FREE, P_OCC, P_UNK = (-0.45, -0.45, -0.45), (0.05, 0.05, 0.05), (8.05, 0.05, 0.05)
PATHS = [[P_OCC, P_FREE, P_FREE], [P_FREE, P_OCC, P_FREE], [P_FREE, P_FREE, P_OCC], [P_FREE, P_FREE], [],
         [P_FREE, P_UNK, P_OCC], [P_UNK]]
PATHS_WANT = {True: [0, 1, 2, -1, -1, 1, 0], False: [0, 1, 2, -1, -1, 2, -1]}
ROBOT = (0.2, 0.2, 0.2)


def _flat(paths):
    pos = np.array([p for path in paths for p in path], np.float64).reshape(-1, 3)
    return pos, np.concatenate([[0], np.cumsum([len(p) for p in paths])]).astype(np.int64)


@pytest.mark.parametrize("unknown_occ", [True, False])
def test_hand_paths(hand_vox, unknown_occ):
    pos, off = _flat(PATHS)
    got = cr.check_paths(hand_vox, pos, off, ROBOT, RES, L_OCC, unknown_occ)
    assert got.tolist() == PATHS_WANT[unknown_occ]


# ---- CPU: cases found by search -------------------------------------------------------------------------------------
def _search_unreached(vox):
    """A box in the free region whose x key range ends at an unknown voxel no loop point reaches."""
    kmax_free = max(k & 0xffff for k in vox if (k >> 16) & 0xffff == K0 - 5 and k >> 32 == K0 - 5 and (k & 0xffff) < 60000)
    for p in np.arange(2.2, 2.7, 0.0037):
        for s in (0.1, 0.2, 0.3, 0.4):
            lo, hi = cr.corners(p, s)
            keys = [cr.key_f(x, RES) for x in cr.loop_points(lo, hi, RES)]
            if cr.key_f(hi, RES) == kmax_free + 1 and keys[-1] == kmax_free and cr.key_f(lo, RES) > OCC_END[0]:
                return (float(p), -0.45, -0.45), (s, 0.3, 0.3)
    raise AssertionError("no box found")


def _search_end_key():
    """A box whose x max corner is exactly on a key boundary: its end key OCC_END[0] fails the cube test."""
    for p in np.arange(1.5, 1.9, 0.05):  # the box stays clear of OCC_FACE
        s = 2 * (2.0 - p)
        lo, hi = cr.corners(p, s)
        if cr.key_f(hi, RES) == OCC_END[0] and not cr.cube_passes(OCC_END[0], lo, hi, RES):
            return (float(p), -0.45, -0.45), (s, 0.3, 0.3)
    raise AssertionError("no box found")


def _search_float_centre():
    """A centre whose x key is valid by the double rule and invalid by the float rule."""
    for x in np.linspace(3276.7999, 3276.80001, 2001):
        if cr.key_d(x, RES) is not None and cr.key_f(x, RES) is None:
            return (float(x), 0.05, 0.05), (0.2, 0.2, 0.2)
    raise AssertionError("no centre found")


def _searched(vox):
    return {"unreached unknown voxel": (_search_unreached(vox), FREE), "end key fails the cube test": (_search_end_key(), FREE),
            "float centre invalid": (_search_float_centre(), UNK)}


def test_searched_cases(hand_vox):
    cases = _searched(hand_vox)
    (c, s), want = cases["unreached unknown voxel"]
    lo, hi = cr.corners(c[0], s[0])
    k = cr.key_f(hi, RES)
    assert cr.pack(k, K0 - 5, K0 - 5) not in hand_vox  # the voxel in the key range is unknown ...
    assert k not in [cr.key_f(x, RES) for x in cr.loop_points(lo, hi, RES)]  # ... and no loop point reaches it
    assert cr.box_status(hand_vox, c, s, RES, L_OCC) == want
    (c, s), want = cases["end key fails the cube test"]
    lo, hi = cr.corners(c[0], s[0])
    assert cr.key_f(hi, RES) == OCC_END[0] and not cr.cube_passes(OCC_END[0], lo, hi, RES)  # occupied, in the key range
    assert cr.state(hand_vox, cr.pack(*OCC_END), L_OCC) == OCC
    assert cr.box_status(hand_vox, c, s, RES, L_OCC) == want
    (c, s), want = cases["float centre invalid"]
    assert cr.state(hand_vox, cr.pack(*[cr.key_d(x, RES) for x in c]), L_OCC) == FREE  # step 1 passes: free
    assert cr.key_f(c[0], RES) is None
    assert cr.box_status(hand_vox, c, s, RES, L_OCC) == want


def test_work_bound_of_the_restatement():
    w = cr.work_items((0.05, 0.05, 0.05), (200.0,) * 3, RES)
    assert w == 251 ** 3  # 2000 keys per axis from a brick boundary on: 251 bricks
    assert cr.check_call([(0.05, 0.05, 0.05)] * 4000, [(200.0,) * 3] * 4000, RES) == 4000 * w <= cr.MAX_WORK
    with pytest.raises(cr.Refused):
        cr.check_call([(0.05, 0.05, 0.05)] * 5000, [(200.0,) * 3] * 5000, RES)
    assert cr.work_items((float("nan"), 0.0, 0.0), (200.0,) * 3, RES) == 0  # an invalid centre spans no work


def test_refusals_of_the_restatement():
    with pytest.raises(cr.Refused):
        cr.box_status({}, (0, 0, 0), (-0.1, 0, 0), RES, L_OCC)
    with pytest.raises(cr.Refused):
        cr.box_status({}, (0, 0, 0), (1e5, 0, 0), RES, L_OCC)  # 10^6 loop points
    assert cr.box_status({}, (float("nan"), 0, 0), (1e5, 0, 0), RES, L_OCC) == UNK  # an invalid centre is not counted


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.fixture
def keep():
    opened = []

    def add(h):
        opened.append(h)
        return h

    yield add
    for h in reversed(opened):
        h.close()


def _dev_map(ctx, edits, res, keep):
    om = keep(ls.OccupancyMap(ctx, resolution=res))
    om.set_boxes(*zip(*edits))
    k, v, _ = om.download(ls.OCC_KNOWN)
    vox = cr.as_dict(k, v)
    assert vox == _vox(edits, res)
    return om, vox


@pytest.mark.gpu
def test_hand_and_searched_cases_on_the_device(gpu_ctx, keep):
    om, vox = _dev_map(gpu_ctx, HAND_EDITS, RES, keep)
    cases = dict(HAND, **_searched(vox))
    names = sorted(cases)
    c = np.array([cases[n][0][0] for n in names], np.float64)
    s = np.array([cases[n][0][1] for n in names], np.float64)
    got = om.box_status(c, s)
    assert got.tolist() == [cases[n][1] for n in names]
    assert om.last_query.keys_visited > 0
    for unknown_occ in (True, False):
        pos, off = _flat(PATHS)
        assert om.check_paths(pos, off, ROBOT, unknown_occ).tolist() == PATHS_WANT[unknown_occ]
    assert om.check_paths(np.zeros((0, 3)), [0, 0, 0], ROBOT).tolist() == [-1, -1]  # empty paths only, no launch
    assert len(om.box_status(np.zeros((0, 3)), np.zeros((0, 3)))) == 0


def _around(poses, rng, n, spread, size_max, spread_z=3.0):
    m = n // len(poses) + 1
    c = np.concatenate([p[:3, 3] + rng.uniform(-1.0, 1.0, (m, 3)) * (spread, spread, spread_z) for p in poses])[:n]
    return c.astype(np.float64), rng.uniform(0.0, size_max, (n, 3))


def _ragged_paths(poses, rng, n):
    """n paths: along the trajectory (waypoints between consecutive poses) and along random lines, 0 ... 40 poses."""
    out = []
    for i in range(n):
        m = int(rng.integers(0, 41))
        a = poses[rng.integers(0, len(poses))][:3, 3].astype(np.float64)
        if i % 2 == 0:
            b = poses[rng.integers(0, len(poses))][:3, 3].astype(np.float64)
        else:
            b = a + rng.uniform(-8.0, 8.0, 3) * (1.0, 1.0, 0.2)
        t = np.linspace(0.0, 1.0, max(m, 1))[:m, None]
        out.append(a + t * (b - a) + rng.normal(0.0, 0.05, (m, 3)))
    return out


def _check_map(om, res, rng, poses):
    """Boxes, robot boxes and paths on om against the grid restatement of its download."""
    k, v, _ = om.download(ls.OCC_KNOWN)
    c, s = _around(poses, rng, 20000, 10.0, 3.0)
    robot = np.array([0.6, 0.6, 0.3])
    rc, _ = _around(poses, rng, 3000, 15.0, 0.0)
    paths = _ragged_paths(poses, rng, 2000)
    pos, off = _flat([p.tolist() for p in paths])
    allc = np.concatenate([c, rc, pos])
    lo, shape = cr.BoxGrid.covering(allc, np.concatenate([s, np.broadcast_to(robot, (len(rc) + len(pos), 3))]), res)
    grid = cr.BoxGrid(k, v, L_OCC, lo, shape)
    bmin, bmax = om.bounds()
    rc[:50, 0] = np.nan
    far = bmax + rng.uniform(1.0, 3000.0, (50, 3))  # outside the map's bounds (unknown), some outside the key space
    assert (far > (lo + shape - K0) * res).any(1).all()  # outside the grid too: the grid's outside is unknown
    rc[50:100] = far
    want = grid.statuses(c, s, res)
    got = om.box_status(c, s)
    assert np.array_equal(got, want)
    assert len(set(want.tolist())) == 3
    assert np.array_equal(om.box_status(rc, robot), grid.statuses(rc, robot, res))
    st = grid.statuses(pos, robot, res)
    for unknown_occ in (True, False):
        want_p = cr.first_collisions(st, off, unknown_occ)
        assert np.array_equal(om.check_paths(pos, off, robot, unknown_occ), want_p)
        assert (want_p >= 0).any() and (want_p == -1).any()
        # one path of one pose per box: checkCollisionWithRobot
        single = om.check_paths(rc, np.arange(len(rc) + 1), robot, unknown_occ)
        assert np.array_equal(single == 0, np.array([cr.collides(x, unknown_occ) for x in grid.statuses(rc, robot, res)]))
    return k, v


PARAMS = {"defaults": {}, "res01_unlimited": dict(resolution=0.1, max_range=-1.0)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PARAMS))
def test_twelve_scan_map(gpu_ctx, full_scans, name, keep):
    scans, poses = full_scans
    prm = PARAMS[name]
    res = prm.get("resolution", 0.075)
    ring = keep(gpu_ctx.create_map(2, 131072))
    om = keep(ls.OccupancyMap(gpu_ctx, **prm))
    nrm = np.zeros((131072, 3), F32)
    for j in range(len(scans)):
        om.insert_scan(ring, ring.push_scan(scans[j], nrm), poses[j])
    _check_map(om, res, np.random.default_rng(7), poses)
    _check_strides(om, res, np.random.default_rng(17), poses)


VOXEL_STRIDE = (1 << 16) * 8  # items one pass of the voxel kernel's grid covers


def _check_strides(om, res, rng, poses):
    """Boxes and robot boxes of 40 voxels a side near the sensor (where centres are mostly free, so most boxes reach the
    voxel pass) whose items take the pass's warps several strides, against the grid."""
    c, _ = _around(poses, rng, 16000, 5.0, 0.0, spread_z=1.5)
    size = np.full(3, 40 * res)
    k, v, _ = om.download(ls.OCC_KNOWN)
    lo, shape = cr.BoxGrid.covering(c, size, res)
    grid = cr.BoxGrid(k, v, L_OCC, lo, shape)
    undecided = [grid._state([cr.key_d(x, res) for x in ci]) == FREE and None not in [cr.key_f(x, res) for x in ci]
                 for ci in c]
    items = sum(cr.work_items(ci, size, res) for ci, u in zip(c, undecided) if u)
    assert items > 2 * VOXEL_STRIDE  # precondition: every warp of the grid takes more than two items
    want = grid.statuses(c, size, res)
    assert np.array_equal(om.box_status(c, size), want) and {OCC, UNK} <= set(want.tolist())
    off = np.arange(0, len(c) + 1, 80)
    for unknown_occ in (True, False):
        assert np.array_equal(om.check_paths(c, off, size, unknown_occ), cr.first_collisions(want, off, unknown_occ))


@pytest.mark.gpu
def test_after_edits_a_read_and_clear(gpu_ctx, full_scans, tmp_path, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    nrm = np.zeros((131072, 3), F32)
    om = keep(ls.OccupancyMap(gpu_ctx, resolution=0.1))
    for j in range(3):
        om.insert_scan(ring, ring.push_scan(scans[j], nrm), poses[j])
    p = poses[1][:3, 3].astype(np.float64)
    om.set_occupied([p + (1.0, 0, 0), p + (0, 2.0, 0)], [(0.5, 0.5, 0.5), (1.0, 0.3, 0.3)])
    om.set_free([p, p + (0, 0, 1.0)], [(2.0, 2.0, 1.0), (1.0, 1.0, 1.0)])
    _check_map(om, 0.1, np.random.default_rng(8), poses[:3])
    path = str(tmp_path / "m.ot")
    om.save_octomap_full(path)
    other = keep(ls.OccupancyMap(gpu_ctx))  # 0.075 m until the read
    other.read_octomap_full(path)
    assert other.params.resolution == 0.1
    _check_map(other, 0.1, np.random.default_rng(9), poses[:3])
    om.clear()
    c, s = _around(poses[:3], np.random.default_rng(10), 2000, 10.0, 3.0)
    assert (om.box_status(c, s) == UNK).all()
    pos, off = _flat([[tuple(x) for x in c[:10]], [tuple(x) for x in c[10:30]]])
    assert om.check_paths(pos, off, (0.5, 0.5, 0.5), True).tolist() == [0, 0]
    assert om.check_paths(pos, off, (0.5, 0.5, 0.5), False).tolist() == [-1, -1]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.gpu
def test_calls_change_nothing(gpu_ctx, full_scans, tmp_path, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    nrm = np.zeros((131072, 3), F32)
    maps = [keep(ls.OccupancyMap(gpu_ctx, initial_capacity=64)) for _ in range(2)]
    rng = np.random.default_rng(11)
    for j in range(4):
        sid = ring.push_scan(scans[j], nrm)
        stats = [m.insert_scan(ring, sid, poses[j]) for m in maps]
        # device_bytes counts the query staging, which the calls grow; every count of the insert itself is equal
        d = [{f: getattr(st, f) for f, _ in st._fields_ if f not in ("device_ms", "device_bytes")} for st in stats]
        assert d[0] == d[1] and stats[0].device_bytes >= stats[1].device_bytes
        c, s = _around(poses[:j + 1], rng, 5000, 10.0, 3.0)
        maps[0].box_status(c, s)
        pos, off = _flat([[tuple(x) for x in c[:100]], [tuple(x) for x in c[100:300]]])
        maps[0].check_paths(pos, off, (0.6, 0.6, 0.3), j % 2 == 0)
    for which in (ls.OCC_KNOWN, ls.OCC_OCCUPIED):
        a, b = maps[0].download(which), maps[1].download(which)
        assert np.array_equal(a[0], b[0]) and np.array_equal(_bits(a[1]), _bits(b[1]))
    for m, name in zip(maps, "ab"):
        m.save_octomap(str(tmp_path / f"{name}.bt"))
    assert (tmp_path / "a.bt").read_bytes() == (tmp_path / "b.bt").read_bytes()


def _raw_box_status(om, c, s, n=None):
    c = np.ascontiguousarray(c, np.float64).reshape(-1, 3)
    s = np.ascontiguousarray(s, np.float64).reshape(-1, 3)
    st = np.full(max(len(c), 1), 7, np.int8)
    return ls.lib().ls_occupancy_box_status(om._h, c.ctypes.data, s.ctypes.data, len(c) if n is None else n,
                                            st.ctypes.data, None), st


def _raw_paths(om, pos, off, robot, n=None):
    pos = np.ascontiguousarray(pos, np.float64).reshape(-1, 3)
    off = np.ascontiguousarray(off, np.int64)
    robot = np.ascontiguousarray(robot, np.float64)
    first = np.full(max(len(off) - 1, 1), 7, np.int64)
    return ls.lib().ls_occupancy_check_paths(om._h, pos.ctypes.data, off.ctypes.data, len(off) - 1 if n is None else n,
                                             robot.ctypes.data, 1, first.ctypes.data, None), first


@pytest.mark.gpu
def test_refusals(gpu_ctx, keep):
    om, vox = _dev_map(gpu_ctx, HAND_EDITS, RES, keep)
    good_c = np.array([P_FREE, P_OCC], np.float64)
    for bad in ((-0.1, 0.3, 0.3), (np.nan, 0.3, 0.3), (np.inf, 0.3, 0.3), (2e4, 0.3, 0.3)):
        rc, st = _raw_box_status(om, good_c, [(0.3, 0.3, 0.3), bad])
        assert rc == ls.LS_ERR_ARG and (st == 7).all()  # the whole call, before any result
        rc, first = _raw_paths(om, good_c, [0, 2], bad)
        assert rc == ls.LS_ERR_ARG and (first == 7).all()
    rc, st = _raw_box_status(om, [(np.nan, 0, 0), (0, np.inf, 0)], [(2e4, 0.3, 0.3)] * 2)
    assert rc == 0 and st[:2].tolist() == [UNK, UNK]  # invalid centres are unknown, never refused
    assert _raw_box_status(om, good_c, [(0.3,) * 3] * 2, n=-1)[0] == ls.LS_ERR_ARG
    assert ls.lib().ls_occupancy_box_status(om._h, None, None, 2, None, None) == ls.LS_ERR_ARG
    for off in ([1, 2], [0, 2, 1]):  # not from 0, decreasing
        assert _raw_paths(om, good_c, off, (0.2,) * 3)[0] == ls.LS_ERR_ARG
    with pytest.raises(ValueError):  # offsets past the positions: the wrapper refuses before the call
        om.check_paths(good_c, [0, 3], (0.2,) * 3)
    for bad in ((-0.1, 0.3, 0.3), (np.nan, 0.3, 0.3)):  # a bad robot size is refused even when every path is empty
        rc, first = _raw_paths(om, np.zeros((0, 3)), [0, 0, 0], bad)
        assert rc == ls.LS_ERR_ARG and (first == 7).all()
    # more than 2^36 (box, brick) items in all: one box that spans them, and many boxes that do only together
    with pytest.raises(cr.Refused):
        cr.check_call([(0.05, 0.05, 0.05)], [(6000.0,) * 3], RES)
    rc, st = _raw_box_status(om, [(0.05, 0.05, 0.05)], [(6000.0,) * 3])
    assert rc == ls.LS_ERR_ARG and st[0] == 7
    rc, first = _raw_paths(om, [P_FREE], [0, 1], (6000.0,) * 3)
    assert rc == ls.LS_ERR_ARG and first[0] == 7
    w = cr.work_items(P_OCC, (200.0,) * 3, RES)  # the box's centre is occupied: the bound counts it all the same
    assert w <= cr.MAX_WORK < 5000 * w
    rc, st = _raw_box_status(om, np.tile(P_OCC, (5000, 1)), [(200.0,) * 3] * 5000)
    assert rc == ls.LS_ERR_ARG and (st == 7).all()
    big = np.array([0, 1 << 31], np.int64)
    assert _raw_paths(om, good_c, big, (0.2,) * 3)[0] == ls.LS_ERR_ARG
    assert _raw_paths(om, good_c, [0, 2], (0.2,) * 3, n=-1)[0] == ls.LS_ERR_ARG
    k, v, _ = om.download(ls.OCC_KNOWN)
    assert cr.as_dict(k, v) == vox  # the map is unchanged
    assert om.box_status(good_c, (0.3, 0.3, 0.3)).tolist() == [FREE, OCC]  # and answers as before


@pytest.mark.gpu
def test_calls_between_batch_begin_and_end(full_scans, keep):
    scans, poses = full_scans
    ctx = keep(ls.Context(0))
    ring = keep(ctx.create_map(4, 131072))
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(2)]
    om = keep(ls.OccupancyMap(ctx, resolution=0.1))
    om.insert_scan(ring, ids[0], poses[0])
    c, s = _around(poses[:1], np.random.default_rng(12), 3000, 8.0, 2.0)
    pos, off = _flat([[tuple(x) for x in c[:40]], [tuple(x) for x in c[40:100]]])
    want = om.box_status(c, s), om.check_paths(pos, off, (0.5, 0.5, 0.5))
    end = ring.begin_batch([(ids[1], [ids[0]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[0]) @ poses[1])])
    try:
        got = om.box_status(c, s), om.check_paths(pos, off, (0.5, 0.5, 0.5))
    finally:
        end()
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


@pytest.mark.gpu
def test_host_layer_equals_the_abi(gpu_ctx, synth_mod, tmp_path, keep):
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    n = 3
    truth, odom = synth_mod.trajectory(3, 2 * n + 2)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 3, k), 8) for k in range(2 * n)]
    odom7 = pg.se3_from_matrix(odom)
    off = pg.se3_from_matrix(np.array([[1, 0, 0, 3.0], [0, 1, 0, 2.0], [0, 0, 1, 0], [0, 0, 0, 1.0]]))
    est = keep(host.Estimator(n_workers=2, nscan_in_sub_map=3))
    times = [[k * 10**8 for k in range(n)], [k * 10**8 + 5 * 10**7 for k in range(n)]]
    for k in range(n):
        data = [scans[k], scans[n + k]]
        feats = [np.ascontiguousarray(d[0]) for d in data]
        nrms = [np.ascontiguousarray(d[1]) for d in data]
        est.step_batch([0, 1], [times[0][k], times[1][k]], [odom7[k], pg.se3_compose(off, odom7[n + k])],
                       [f.ctypes.data for f in feats], [x.ctypes.data for x in nrms], [len(f) for f in feats])
    path = str(tmp_path / "h.ot")
    dev = keep(ls.OccupancyMap(gpu_ctx, resolution=0.1, max_range=15.0))
    rng = np.random.default_rng(13)
    poses = [truth[k] for k in range(n)]
    c, s = _around(poses, rng, 3000, 8.0, 2.0)
    paths = _ragged_paths(poses, rng, 200)
    pos, offs = _flat([p.tolist() for p in paths])
    robot = (0.6, 0.6, 0.3)
    for unknown_occ in (True, False):
        hm = keep(host.OccupancyMap(est, resolution=0.1, max_range=15.0, treat_unknown_as_occupied=unknown_occ))
        assert hm.insert_laser_tracks() == 2 * n
        hm.write_full(path)
        dev.read_octomap_full(path)
        want = dev.box_status(c, s)
        assert len(set(want.tolist())) == 3
        assert np.array_equal(hm.box_status(c, s), want)
        assert np.array_equal(hm.box_status(c[:200], s[:200], single=True), want[:200])
        want_p = dev.check_paths(pos, offs, robot, unknown_occ)
        assert (want_p >= 0).any() and (want_p == -1).any()
        assert np.array_equal(hm.check_paths(pos, offs, robot), want_p)
        assert np.array_equal(hm.check_paths(pos, offs, robot, single=True), want_p)
        one = dev.check_paths(c[:300], np.arange(301), robot, unknown_occ)
        assert np.array_equal(hm.check_paths(c[:300], np.arange(301), robot, single=True), one)
        hm.close()
    dev.close(), est.close()
