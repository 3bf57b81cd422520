"""Edits of the resident occupancy map (ls_occupancy_set_boxes / _clear / _box_voxels / _bounds): volumetric_mapping's
setFree / setOccupied, resetMap, getOccupiedPointcloudInBoundingBox and getMapBounds.  CPU: the restatement
(tests/occupancy_edits_ref.py) against a scalar triple loop, answers derived by hand and cases found by search.  GPU: the
device against the restatement bit for bit, then queries, trees and inserts after an edit, growth, refusals, reset, batches
and laser_slam::OccupancyMap.  The rules are DESIGN.md §4b''''''''."""
import ctypes
import math

import numpy as np
import pytest

import laser_slam_b200 as ls
import occupancy_edits_ref as er
import octomap_full_ref as fr
import octomap_read_ref as rr
from oracle import occupancy as oc
from oracle import octree as ot_oracle
from oracle import queries as oq
from test_occupancy import F32, K0, _bits, full_scans  # noqa: F401  (full_scans: fixture)

L_MIN, L_MAX = rr.clamps()
L_OCC = oc.logodds(0.7)
RESS = [0.075, 0.1, 0.25, 1.0 / 30.0]


def ed(res):
    return er.Edits(res, L_MIN, L_MAX, L_OCC)


# ---- CPU ----------------------------------------------------------------------------------------------------------
def scalar_loop(center, size, res):
    """setLogOddsBoundingBox's triple loop written out: every point cast to float, keyed, invalid keys skipped."""
    def snap(p):
        return res * math.floor(p / res) + res / 2.0

    c = [snap(p) for p in center]
    lo = [(c[a] - size[a] / 2) + 0.001 for a in range(3)]
    hi = [(c[a] + size[a] / 2) - 0.001 for a in range(3)]
    out = []
    x = lo[0]
    while x <= hi[0]:
        y = lo[1]
        while y <= hi[1]:
            z = lo[2]
            while z <= hi[2]:
                k = [math.floor(float(np.float32(v)) * (1.0 / res)) for v in (x, y, z)]
                if all(-K0 <= f < K0 for f in k):
                    out.append((k[0] + K0) | ((k[1] + K0) << 16) | ((k[2] + K0) << 32))
                z += res
            y += res
        x += res
    return out


@pytest.mark.parametrize("res", RESS)
def test_separable_loop_equals_the_triple_loop(res):
    rng = np.random.default_rng(int(res * 1e4))
    for _ in range(40):
        c = rng.uniform(-50, 50, 3) * rng.choice([1e-3, 1, 20])
        s = rng.uniform(0, 8 * res, 3) * rng.choice([0.3, 1])
        assert er.box_keys(c, s, res) == scalar_loop(c, s, res)


def _j(p, res):
    return math.floor(p / res)


KNOWN = {  # name: (res, centre, size, the keys per axis derived by hand)
    "size_res_is_the_voxel": (0.1, (0.23, -1.47, 3.06), (0.1, 0.1, 0.1), [[2 + K0], [-15 + K0], [30 + K0]]),
    "three_res_is_27": (0.1, (0.23, -1.47, 3.06), (0.3,) * 3, [[1 + K0, 2 + K0, 3 + K0], [-16 + K0, -15 + K0, -14 + K0],
                                                               [29 + K0, 30 + K0, 31 + K0]]),
    "two_res_is_j_minus_1_and_j": (0.1, (0.23, -1.47, 3.06), (0.2,) * 3, [[1 + K0, 2 + K0], [-16 + K0, -15 + K0],
                                                                          [29 + K0, 30 + K0]]),
    "size_zero_is_nothing": (0.1, (0.23, -1.47, 3.06), (0.0, 0.0, 0.0), [[], [], []]),
    "just_above_0.002_is_one": (0.1, (0.23, 0.23, 0.23), (0.00201,) * 3, [[2 + K0]] * 3),
    "just_below_0.002_is_none": (0.1, (0.23, 0.23, 0.23), (0.00199, 0.00199, 0.00199), [[], [], []]),
    "on_a_boundary_at_0.25": (0.25, (0.5, -0.5, 0.25), (0.25,) * 3, [[2 + K0], [-2 + K0], [1 + K0]]),
    "negative_coordinates": (0.1, (-0.35, -7.05, -0.01), (0.1,) * 3, [[-4 + K0], [-71 + K0], [-1 + K0]]),
    "straddling_the_key_space_edge": (1.0, (32767.5, -32767.5, 0.5), (3.0, 3.0, 1.0), [[65534, 65535], [0, 1], [K0]]),
}


@pytest.mark.parametrize("name", sorted(KNOWN))
def test_known_answers_of_the_loop(name):
    res, c, s, want = KNOWN[name]
    assert [er.axis_keys(c[a], s[a], res) for a in range(3)] == want
    assert er.box_keys(c, s, res) == [er.pack(x, y, z) for x in want[0] for y in want[1] for z in want[2]]


def division_case():
    """(p, res) with floor(p / res) != floor(p * (1/res))."""
    for res in (0.1, 0.075, 0.3, 1.0 / 30.0):
        for i in range(-4000, 4000):
            p = i * res
            if _j(p, res) != math.floor(p * (1.0 / res)):
                return p, res
    raise AssertionError("no case")


def float_cast_case():
    """(p, s, res): s not a multiple of res, with a loop point whose double and float keys differ."""
    rng = np.random.default_rng(5)
    res = 0.075
    for _ in range(200000):
        p, s = float(rng.uniform(200, 2000)), float(rng.uniform(0.1, 0.5))
        if abs(s / res - round(s / res)) < 1e-3:
            continue
        for x in er.axis_points(p, s, res):
            if math.floor(x * (1.0 / res)) != math.floor(float(np.float32(x)) * (1.0 / res)):
                return p, s, res
    raise AssertionError("no case")


def bounds_order_case():
    """(k, res): ((double)c - h) + res != (double)c + h for the float centre c of key k, h = res / 2."""
    res = 0.075
    for k in range(K0, K0 + 40000):
        c = float(er.centre(k, res))
        if (c - res / 2.0) + res != c + res / 2.0:
            return k, res
    raise AssertionError("no case")


def bound_case():
    """(p, s, res): the loop's last point lands exactly on hi = (c + s/2) - 0.001, so only `<=` keeps it."""
    for res in (0.25, 0.1, 0.075):
        for p in (0.1, 0.37, -1.3, 2.06):
            c = res * math.floor(p / res) + res / 2.0
            for m in range(1, 12):
                s = m * res + 0.002
                lo, hi = (c - s / 2) + 0.001, (c + s / 2) - 0.001
                x = lo
                while x < hi:
                    x += res
                if x == hi and er.key_of(np.float32(x), res) is not None:
                    return p, s, res
    raise AssertionError("no case")


def _precondition(name, res, c, s):
    """Assert that a searched case reaches the branch it was found for."""
    p = c[0]
    if name == "division":
        assert _j(p, res) != math.floor(p * (1.0 / res))
    elif name == "float_cast":
        pts = er.axis_points(p, s[0], res)
        assert [math.floor(x * (1.0 / res)) for x in pts] != [math.floor(float(np.float32(x)) * (1.0 / res)) for x in pts]
    elif name == "inclusive_bound":
        cc = res * math.floor(p / res) + res / 2.0
        lo, hi = (cc - s[0] / 2) + 0.001, (cc + s[0] / 2) - 0.001
        x = lo
        while x < hi:
            x += res
        assert x == hi
    else:  # bounds_order: the box is the one voxel of key k on every axis
        k = er.axis_keys(p, res, res)
        assert len(k) == 1
        cf = float(er.centre(k[0], res))
        assert (cf - res / 2.0) + res != cf + res / 2.0


def searched(name):
    """(res, centre, size) of a searched case, the same value on every axis, its precondition checked."""
    if name == "division":
        p, res = division_case()
        s = res
    elif name == "float_cast":
        p, s, res = float_cast_case()
    elif name == "inclusive_bound":
        p, s, res = bound_case()
    else:
        k, res = bounds_order_case()
        p, s = float(er.centre(k, res)), res
    c, sz = (p, p, p), (s, s, s)
    _precondition(name, res, c, sz)
    return res, c, sz


SEARCHED = ["bounds_order", "division", "float_cast", "inclusive_bound"]


@pytest.mark.parametrize("name", SEARCHED)
def test_searched_cases_equal_the_triple_loop(name):
    res, c, s = searched(name)
    assert er.box_keys(c, s, res) == scalar_loop(c, s, res) and len(er.box_keys(c, s, res)) > 0


def test_loop_bound_is_inclusive():
    p, s, res = bound_case()
    cc = res * math.floor(p / res) + res / 2.0
    hi = (cc + s / 2) - 0.001
    assert er.axis_points(p, s, res)[-1] == hi
    assert er.axis_keys(p, s, res)[-1] == er.key_of(np.float32(hi), res)


def test_snap_divides():
    p, res = division_case()
    assert _j(p, res) != math.floor(p * (1.0 / res))  # the precondition: the case reaches its branch
    assert er.axis_keys(p, res, res) == [_j(p, res) + K0]


def test_points_are_cast_to_float():
    p, s, res = float_cast_case()
    pts = er.axis_points(p, s, res)
    double_keys = [math.floor(x * (1.0 / res)) + K0 for x in pts]
    assert er.axis_keys(p, s, res) != double_keys  # precondition
    assert er.axis_keys(p, s, res) == [math.floor(float(np.float32(x)) * (1.0 / res)) + K0 for x in pts]


def test_bounds_max_adds_res_to_the_lower_corner():
    k, res = bounds_order_case()
    c = float(er.centre(k, res))
    assert (c - res / 2.0) + res != c + res / 2.0  # precondition
    lo, hi = ed(res).bounds({er.pack(k, k, k): F32(1)})
    assert (lo == c - res / 2.0).all() and (hi == (c - res / 2.0) + res).all()


@pytest.mark.parametrize("order", ["free_then_occupied", "occupied_then_free"])
def test_overlapping_boxes_the_last_wins(order):
    e, vox = ed(0.1), {}
    occ = [False, True] if order == "free_then_occupied" else [True, False]
    n, new = e.set_boxes(vox, [(0, 0, 0), (0.15, 0, 0)], [(0.3,) * 3, (0.3,) * 3], occ)
    assert (n, new) == (54, 36)
    overlap = set(er.box_keys((0, 0, 0), (0.3,) * 3, 0.1)) & set(er.box_keys((0.15, 0, 0), (0.3,) * 3, 0.1))
    assert len(overlap) == 18
    assert all(vox[k] == (L_MAX if occ[1] else L_MIN) for k in overlap)


def test_crop_order_and_which():
    e = ed(0.1)
    keys = er.box_keys((0, 0, 0), (0.3,) * 3, 0.1)
    vox = {k: (L_MAX if i % 3 == 0 else L_MIN) for i, k in enumerate(keys) if i % 2 == 0}
    k, v, c = e.crop(vox, (0, 0, 0), (0.3,) * 3, True)
    assert list(k) == [kk for i, kk in enumerate(keys) if i % 6 == 0] and (v == L_MAX).all()
    k, v, c = e.crop(vox, (0, 0, 0), (0.3,) * 3, False)
    assert list(k) == keys[::2] and np.array_equal(c, er.centres(k, 0.1))


def test_bounds_cases():
    e, res = ed(0.1), 0.1
    assert [list(x) for x in e.bounds({})] == [[0, 0, 0], [0, 0, 0]]
    one = er.pack(K0, K0 + 1, K0 - 1)
    lo, hi = e.bounds({one: F32(0)})
    assert np.allclose(lo, [0, 0.1, -0.1]) and np.allclose(hi, [0.1, 0.2, 0.0])
    lo, hi = e.bounds({er.pack(K0 - 500, K0 + 7, K0): F32(0), er.pack(K0 + 900, K0 - 3, K0 + 2): F32(0)})
    assert np.allclose(lo, [-50.0, -0.3, 0.0]) and np.allclose(hi, [90.1, 0.8, 0.3])


# ---- GPU ----------------------------------------------------------------------------------------------------------
@pytest.fixture
def keep():
    """keep(h) returns h and closes it when the test ends, in reverse order, even when the test fails: no map, ring or
    context outlives the test (or the session's context)."""
    opened = []

    def add(h):
        opened.append(h)
        return h

    yield add
    for h in reversed(opened):
        h.close()


def _known(dev):
    k, v, c = dev.download(ls.OCC_KNOWN)
    return k, v, c


def _same_as(dev, vox, res):
    k, v, c = _known(dev)
    wk, wv = er.as_arrays(vox)
    assert np.array_equal(k, wk) and np.array_equal(_bits(v), _bits(wv))
    assert np.array_equal(_bits(c), _bits(er.centres(wk, res)))


def _same_crop(dev, e, vox, center, size):
    for which, occ in ((ls.OCC_OCCUPIED, True), (ls.OCC_KNOWN, False)):
        k, v, c = dev.box_voxels(center, size, which)
        wk, wv, wc = e.crop(vox, center, size, occ)
        assert np.array_equal(k, wk) and np.array_equal(_bits(v), _bits(wv)) and np.array_equal(_bits(c), _bits(wc))


def _same_bounds(dev, e, vox):
    lo, hi = dev.bounds()
    wlo, whi = e.bounds(vox)
    assert np.array_equal(lo, wlo) and np.array_equal(hi, whi)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(KNOWN) + ["searched_" + n for n in SEARCHED])
def test_known_answers_on_the_device(gpu_ctx, name, keep):
    res, c, s = searched(name[9:]) if name.startswith("searched_") else KNOWN[name][:3]
    e, vox = ed(res), {}
    dev = keep(ls.OccupancyMap(gpu_ctx, resolution=res))
    for occ in (True, False):
        st = dev.set_boxes([c], [s], [occ])
        n, new = e.set_boxes(vox, [c], [s], [occ])
        assert (st.voxels_set, st.new_known, st.known_voxels) == (n, new, len(vox))
        _same_as(dev, vox, res)
        _same_crop(dev, e, vox, c, s)
        _same_bounds(dev, e, vox)
    dev.close()


def _same_queries(dev, vox, params, poses, rng):
    k, v = er.as_arrays(vox)
    o = oq.KnownVoxels(k, v, **params)
    cen = er.centres(k, params["resolution"])[:, :3].astype(np.float64)
    pts = np.concatenate([cen[::7], rng.uniform(cen.min(axis=0), cen.max(axis=0), (50_000, 3))])
    a, b = dev.cell_status(pts), o.cell_status(pts)
    assert np.array_equal(a[0], b[0]) and np.array_equal(_bits(a[1]), _bits(b[1]))
    p = np.array([poses[i][:3, 3] for i in rng.integers(0, len(poses), 20_000)], np.float64)
    s = p + rng.uniform(-3.0, 3.0, p.shape) * [1, 1, 0.3]
    d = rng.normal(size=p.shape)
    e = s + d / np.linalg.norm(d, axis=1)[:, None] * rng.uniform(1.0, 10.0, (len(p), 1))
    for stop in (True, False):
        a, b = dev.line_status(s, e, stop_at_unknown=stop), o.line_status(s, e, stop_at_unknown=stop)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    a, b = dev.line_status(s[:200], e[:200], box=(0.6, 0.6, 0.3)), o.line_status(s[:200], e[:200], box=(0.6, 0.6, 0.3))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    origins = np.repeat(poses[0][:3, 3][None], 20_000, axis=0).astype(F32)
    dirs = rng.normal(size=(20_000, 3)).astype(F32)
    for ignore in (False, True):
        a, b = dev.cast_rays(origins, dirs, ignore, 20.0), o.cast_rays(origins, dirs, ignore, 20.0)
        assert np.array_equal(a[0], b[0]) and np.array_equal(_bits(a[1]), _bits(b[1]))


def _same_trees(dev, vox, res):
    k, v = er.as_arrays(vox)
    t, wt = dev.octree(), ot_oracle.octree(k, v, res)
    assert (t.nodes, t.payload) == (wt.nodes, wt.payload)
    f, wf = dev.full_octree(), fr.full_octree(k, v, res)
    assert (f.nodes, f.payload) == (wf.nodes, wf.payload)


@pytest.mark.gpu
def test_edits_of_the_twelve_scan_map(gpu_ctx, full_scans, keep):
    scans, poses = full_scans
    params = dict(oc.DEFAULTS)
    res = params["resolution"]
    ring = keep(gpu_ctx.create_map(2, 131072))
    dev = keep(ls.OccupancyMap(gpu_ctx))
    nrm = np.zeros((131072, 3), F32)
    for k in range(len(scans)):
        dev.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
    dev.octree(), dev.full_octree()  # cached builds an edit must invalidate
    e = ed(res)
    vox = er.as_dict(*_known(dev)[:2])
    rng = np.random.default_rng(7)
    p0 = poses[0][:3, 3].astype(np.float64)
    lo, hi = e.bounds(vox)
    edits = [([p0], [(4.0, 4.0, 4.0)], [False]),
             ([p0 + [3.0, 1.0, 0.5]], [(1.0, 1.0, 2.0)], [True]),
             (rng.uniform(lo, hi, (64, 3)), rng.uniform(0.0, 3.0, (64, 3)), rng.integers(0, 2, 64).astype(bool))]
    for c, s, o in edits:
        st = dev.set_boxes(c, s, o)
        n, new = e.set_boxes(vox, c, s, o)
        assert (st.voxels_set, st.new_known, st.known_voxels) == (n, new, len(vox)) and n > 0
        _same_as(dev, vox, res)
        _same_queries(dev, vox, params, poses, rng)
        _same_trees(dev, vox, res)
        _same_crop(dev, e, vox, c[0], (20.0, 20.0, 20.0) if len(c) == 1 else s[0])
        _same_bounds(dev, e, vox)
    o = rr.seed(oc.OccupancyMap(**params), *er.as_arrays(vox))
    for k in (2, 5, 9):
        a = dev.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
        b = o.insert_scan(scans[k], poses[k])
        assert (a.free_updates, a.occupied_updates, a.known_voxels) == (
            b["free_updates"], b["occupied_updates"], b["known_voxels"])
    (k, v, _), (wk, wv) = _known(dev), o.download()
    assert np.array_equal(k, wk) and np.array_equal(_bits(v), _bits(wv))
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_growth(gpu_ctx, keep):
    res = 0.075
    e, vox = ed(res), {}
    dev = keep(ls.OccupancyMap(gpu_ctx, initial_capacity=16))
    c0, s0 = (1.0, 2.0, 0.5), (0.5, 0.5, 0.5)
    st0 = dev.set_boxes([c0], [s0], [False])
    e.set_boxes(vox, [c0], [s0], [False])
    c, s = (30.0, 0.0, 1.0), (12.0, 12.0, 6.0)  # 20 x 20 x 10 bricks: the pool of 16 grows past 4x, the table of 1024 past half
    st = dev.set_boxes([c], [s], [True])
    e.set_boxes(vox, [c], [s], [True])
    assert st0.bricks <= 16 and st.bricks >= 4 * 16 and 2 * st.bricks > 1024 and st.device_bytes > st0.device_bytes
    _same_as(dev, vox, res)
    _same_bounds(dev, e, vox)
    dev.close()
    empty = keep(ls.OccupancyMap(gpu_ctx, initial_capacity=16))
    vox = {}
    empty.set_boxes([c], [s], [False])
    e.set_boxes(vox, [c], [s], [False])
    _same_as(empty, vox, res)
    _same_bounds(empty, e, vox)
    empty.close()


def _snapshot(dev):
    return _known(dev), dev.octree().payload, dev.full_octree().payload, dev.size(ls.OCC_KNOWN)


def _same_snapshot(a, b):
    assert all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(a[0], b[0])) and a[1:] == b[1:]


@pytest.mark.gpu
def test_refusals_change_nothing(gpu_ctx, full_scans, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    dev = keep(ls.OccupancyMap(gpu_ctx))
    dev.insert_scan(ring, ring.push_scan(scans[0], np.zeros((131072, 3), F32)), poses[0])
    before = _snapshot(dev)
    bytes0 = dev.set_boxes([(0, 0, 0)], [(0, 0, 0)], [False]).device_bytes
    good = ([poses[0][:3, 3]], [(1.0, 1.0, 1.0)])
    bad = [((np.nan, 0, 0), (1, 1, 1)), ((np.inf, 0, 0), (1, 1, 1)), ((0, 0, 0), (1, np.nan, 1)),
           ((0, 0, 0), (1, np.inf, 1)), ((0, 0, 0), (1, 1, -0.5)), ((0, 0, 0), (1, 1, 0.075 * (1 << 17) + 1.0))]
    for c, s in bad:
        with pytest.raises(ls.LsError, match="rc=-1"):
            dev.set_boxes(good[0] + [c] + good[0], good[1] + [s] + good[1], [True, True, True])
        with pytest.raises(ls.LsError, match="rc=-1"):
            dev.box_voxels(c, s)
        _same_snapshot(before, _snapshot(dev))
    with pytest.raises(ls.LsError, match="rc=-3"):  # (9000 / 8)^3 bricks > 2^29
        dev.set_boxes(good[0] + [(0, 0, 0)], good[1] + [(9000 * 0.075,) * 3], [True, True])
    _same_snapshot(before, _snapshot(dev))
    assert dev.set_boxes([(0, 0, 0)], [(0, 0, 0)], [False]).device_bytes == bytes0
    L, c3, o = ls.lib(), np.zeros(3), np.zeros(1, np.int8)
    assert L.ls_occupancy_set_boxes(dev._h, c3.ctypes.data, c3.ctypes.data, o.ctypes.data, -1, None) == ls.LS_ERR_ARG
    assert L.ls_occupancy_set_boxes(dev._h, None, c3.ctypes.data, o.ctypes.data, 1, None) == ls.LS_ERR_ARG
    assert L.ls_occupancy_set_boxes(dev._h, c3.ctypes.data, c3.ctypes.data, None, 1, None) == ls.LS_ERR_ARG
    assert L.ls_occupancy_box_voxels(dev._h, c3.ctypes.data, c3.ctypes.data, 3, None, None, None, 0, None) == ls.LS_ERR_ARG
    assert L.ls_occupancy_bounds(dev._h, None, c3.ctypes.data) == ls.LS_ERR_ARG
    with pytest.raises(ls.LsError, match="rc=-1"):  # 1300^3 loop points > 2^31 - 1
        dev.box_voxels((0, 0, 0), (1300 * 0.075,) * 3, ls.OCC_KNOWN)
    n = ctypes.c_int64(-1)
    s3 = np.full(3, 4.0)
    p3 = np.ascontiguousarray(poses[0][:3, 3], np.float64)
    assert L.ls_occupancy_box_voxels(dev._h, p3.ctypes.data, s3.ctypes.data, ls.OCC_KNOWN, None, None, None, 0,
                                     ctypes.byref(n)) == ls.LS_ERR_ARG
    assert n.value == len(dev.box_voxels(p3, s3, ls.OCC_KNOWN)[0]) > 0
    _same_snapshot(before, _snapshot(dev))
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_reset(gpu_ctx, full_scans, tmp_path, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    nrm = np.zeros((131072, 3), F32)
    dev = keep(ls.OccupancyMap(gpu_ctx, initial_capacity=64))
    for k in range(3):
        dev.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
    dev.set_occupied(poses[0][:3, 3], (2.0, 2.0, 2.0))
    cen = _known(dev)[2][:, :3].astype(np.float64)
    dev.octree(), dev.full_octree()
    bytes0 = dev.set_boxes([(0, 0, 0)], [(0, 0, 0)], [False]).device_bytes
    dev.clear()
    assert dev.size(ls.OCC_KNOWN) == 0 and [list(x) for x in dev.bounds()] == [[0, 0, 0], [0, 0, 0]]
    assert dev.set_boxes([(0, 0, 0)], [(0, 0, 0)], [False]).device_bytes == bytes0
    assert dev.save_octomap(str(tmp_path / "empty.bt")) == 0 and b"\nsize 0\n" in (tmp_path / "empty.bt").read_bytes()
    assert (dev.cell_status(cen)[0] == ls.CELL_UNKNOWN).all()
    fresh = keep(ls.OccupancyMap(gpu_ctx, initial_capacity=64))
    for k in (5, 6):
        sid = ring.push_scan(scans[k], nrm)
        a, b = dev.insert_scan(ring, sid, poses[k]), fresh.insert_scan(ring, sid, poses[k])
        assert (a.free_updates, a.occupied_updates, a.known_voxels, a.bricks) == (
            b.free_updates, b.occupied_updates, b.known_voxels, b.bricks)
        assert all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(_known(dev), _known(fresh)))
    dev.close()
    fresh.close()
    ring.close()


@pytest.mark.gpu
def test_edits_between_batch_begin_and_end(full_scans, keep):
    scans, poses = full_scans
    ctx = keep(ls.Context(0))
    ring = keep(ctx.create_map(4, 131072))
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(3)]
    dev = keep(ls.OccupancyMap(ctx, resolution=0.1))
    dev.insert_scan(ring, ids[0], poses[0])
    e, vox = ed(0.1), er.as_dict(*_known(dev)[:2])
    c, s = [poses[0][:3, 3], poses[0][:3, 3] + 1.0], [(2.0, 2.0, 1.0), (1.0, 1.0, 1.0)]
    end = ring.begin_batch([(ids[1], [ids[0]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[0]) @ poses[1])])
    try:  # the batch always ends, so a failed comparison cannot leave it open
        dev.set_boxes(c, s, [False, True])
        known = _known(dev)
        crops = [dev.box_voxels(c[0], (6.0, 6.0, 6.0), w) for w in (ls.OCC_OCCUPIED, ls.OCC_KNOWN)]
        bounds = dev.bounds()
        dev.clear()
        cleared = dev.size(ls.OCC_KNOWN)
    finally:
        end()
    e.set_boxes(vox, c, s, [False, True])
    wk, wv = er.as_arrays(vox)
    assert np.array_equal(known[0], wk) and np.array_equal(_bits(known[1]), _bits(wv))
    for got, occ in zip(crops, (True, False)):
        want = e.crop(vox, c[0], (6.0, 6.0, 6.0), occ)
        assert np.array_equal(got[0], want[0]) and np.array_equal(_bits(got[1]), _bits(want[1]))
        assert np.array_equal(_bits(got[2]), _bits(want[2]))
    assert all(np.array_equal(x, y) for x, y in zip(bounds, e.bounds(vox))) and cleared == 0
    dev.close()
    ring.close()
    ctx.close()


@pytest.mark.gpu
def test_host_layer_equals_the_abi(synth_mod, keep):
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
    e = ed(0.1)
    vox = er.as_dict(*hm.voxels(1))
    c = [truth[0][:3, 3], truth[1][:3, 3] + 0.5]
    s = [(3.0, 3.0, 1.0), (1.0, 1.0, 2.0)]
    hm.set_boxes(c, s, [False, True], single=True)
    e.set_boxes(vox, c, s, [False, True])
    k, v = hm.voxels(1)
    wk, wv = er.as_arrays(vox)
    assert np.array_equal(k, wk) and np.array_equal(_bits(v), _bits(wv))
    c2, s2, o2 = [truth[2][:3, 3]], [(2.0, 2.0, 2.0)], [True]
    n, new = e.set_boxes(vox, c2, s2, o2)
    assert hm.set_boxes(c2, s2, o2) == (n, new, len(vox))
    cloud = hm.occupied_cloud_in_box(truth[1][:3, 3], (8.0, 8.0, 4.0))
    assert np.array_equal(_bits(cloud), _bits(e.crop(vox, truth[1][:3, 3], (8.0, 8.0, 4.0), True)[2]))
    lo, hi, size, centre = hm.map_bounds()
    wlo, whi = e.bounds(vox)
    assert np.array_equal(lo, wlo) and np.array_equal(hi, whi)
    assert np.array_equal(size, whi - wlo) and np.array_equal(centre, wlo + (whi - wlo) / 2.0)
    hm.reset_map()
    assert len(hm.voxels(1)[0]) == 0 and [list(x) for x in hm.map_bounds()[:2]] == [[0, 0, 0], [0, 0, 0]]
    hm.close()
    est.close()
