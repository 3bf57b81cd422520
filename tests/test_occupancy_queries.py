"""Queries of the occupancy map (volumetric_mapping's WorldBase and octomap's castRay): known answers for every rule of
oracle/QUERIES.md and the oracle against a pure-Python restatement on the CPU; the device queries (ls_occupancy_cell_status /
_line_status / _cast_rays), the Python wrapper and laser_slam::OccupancyMap bit for bit against the oracle on the GPU."""
import ctypes
import math

import numpy as np
import pytest

from oracle import occupancy as oc
from oracle import queries as oq
from test_occupancy import K0, _pack, _rel, _tie_free_cloud, _translate, segment_cells

F32 = np.float32
FREE, OCC, UNK = oq.CELL_FREE, oq.CELL_OCCUPIED, oq.CELL_UNKNOWN
NONE = int(oq.NO_KEY)
NAN_BITS = 0x7FC00000


def _bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def _centre(k, res):
    return float(F32(((k - K0) + 0.5) * res))


def _centre3(key, res):
    return [_centre((key >> s) & 0xFFFF, res) for s in (0, 16, 32)]


# ---- hand-built maps (res 0.1, unlimited range) ----------------------------------------------------------------------
# A: sensor at (0.05, 0.05, 0.05); rays along +x to 0.55 and 1.05 and along +y to 0.55.  Free (0..9, 0, 0) but for the
#    occupied (5, 0, 0) and (10, 0, 0); free (0, 0..4, 0), occupied (0, 5, 0).
# B: the same sensor; rays to (0.15, 0.25, 0.05) and (0.15, 0.25, 0.25).  Free (0,0,0) (0,1,0) (1,1,0) (0,0,1) (0,1,1)
#    (1,1,1) (1,1,2); occupied (1, 2, 0) and (1, 2, 2): the paths the tie-breaking lines below take.
PARAMS = dict(resolution=0.1, max_range=-1.0)
_T = _translate([0.05, 0.05, 0.05])
SCANS = {
    "A": [(np.array([[0.5, 0, 0, 1], [1.0, 0, 0, 1], [0, 0.5, 0, 1]], F32), _T)],
    "B": [(np.array([[0.1, 0.2, 0.0, 1], [0.1, 0.2, 0.2, 1]], F32), _T)],
}
O = (0.05, 0.05, 0.05)


def _oracle_map(name):
    m = oq.OccupancyMap(**PARAMS)
    for c, T in SCANS[name]:
        m.insert_scan(c, T)
    return m


def test_hand_maps_hold_what_the_answers_assume():
    ka, va = _oracle_map("A").download()
    want_a = {_rel(i, 0, 0) for i in range(11)} | {_rel(0, i, 0) for i in range(6)}
    assert set(int(k) for k in ka) == want_a
    occ_a = {int(k) for k, v in zip(ka, va) if v >= oc.logodds(0.7)}
    assert occ_a == {_rel(5, 0, 0), _rel(10, 0, 0), _rel(0, 5, 0)}
    kb, vb = _oracle_map("B").download()
    free_b = {(0, 0, 0), (0, 1, 0), (1, 1, 0), (0, 0, 1), (0, 1, 1), (1, 1, 1), (1, 1, 2)}
    assert {int(k): bool(v >= oc.logodds(0.7)) for k, v in zip(kb, vb)} == \
        {**{_rel(*k): False for k in free_b}, _rel(1, 2, 0): True, _rel(1, 2, 2): True}


# Known answers: (map, kind, inputs, expected).  kind cell: points -> [(status, log-odds or None)]; line: (starts, ends,
# box, stop_at_unknown) -> [(status, first key)]; ray: (origins, directions, ignore_unknown, max_range) -> [(result, end
# key or None)].
L_HIT, L_MISS = oc.logodds(0.9), oc.logodds(0.4)
INF, NAN = float("inf"), float("nan")
CASES = {
    "cell_states": ("A", "cell", [O, (0.55, 0.05, 0.05), (0.95, 0.05, 0.05), (-3.0, -3.0, -3.0)],
                    [(FREE, L_MISS), (OCC, L_HIT), (FREE, L_MISS), (UNK, None)]),
    "cell_neighbour_in_a_known_brick": ("A", "cell", [(0.15, 0.15, 0.05), (0.05, 0.05, 0.15)], [(UNK, None), (UNK, None)]),
    "cell_invalid_keys": ("A", "cell", [(NAN, 0.05, 0.05), (0.05, INF, 0.05), (0.05, 0.05, -INF), (5000.0, 0.05, 0.05),
                                        (-3276.81, 0.05, 0.05)], [(UNK, None)] * 5),
    # 0.5 - 1e-12 is in voxel 4 as a double, in voxel 5 once cast to float: the cell query keys the double
    "cell_keys_the_double": ("A", "cell", [(0.5 - 1e-12, 0.05, 0.05)], [(FREE, L_MISS)]),
    "line_occupied": ("A", "line", ([O], [(0.95, 0.05, 0.05)], None, True), [(OCC, _rel(5, 0, 0))]),
    "line_free": ("A", "line", ([O], [(0.45, 0.05, 0.05)], None, True), [(FREE, NONE)]),
    "line_end_voxel_not_checked": ("A", "line", ([O], [(0.55, 0.05, 0.05)], None, True), [(FREE, NONE)]),
    "line_in_one_voxel": ("A", "line", ([(0.51, 0.05, 0.05)], [(0.59, 0.05, 0.05)], None, True), [(FREE, NONE)]),
    "line_leaving_the_key_space": ("A", "line", ([(0.55, 0.05, 0.05)], [(5000.0, 0.05, 0.05)], None, True), [(FREE, NONE)]),
    "line_nan_end": ("A", "line", ([(0.55, 0.05, 0.05)], [(NAN, 0.05, 0.05)], None, True), [(FREE, NONE)]),
    "line_unknown_before_occupied": ("A", "line", ([(-0.15, 0.05, 0.05)], [(0.95, 0.05, 0.05)], None, True),
                                     [(UNK, _rel(-2, 0, 0))]),
    "line_unknown_passed_without_stop": ("A", "line", ([(-0.15, 0.05, 0.05)], [(0.95, 0.05, 0.05)], None, False),
                                         [(OCC, _rel(5, 0, 0))]),
    "line_unknown_only_without_stop": ("A", "line", ([(-0.15, -0.25, 0.05)], [(-0.95, -0.25, 0.05)], None, False),
                                       [(FREE, NONE)]),
    # equal tMax in x and y: y steps first, along (0,1,0) (1,1,0) to the occupied (1,2,0); x first would meet unknown
    "line_tie_two_axes": ("B", "line", ([O], [(0.25, 0.25, 0.05)], None, True), [(OCC, _rel(1, 2, 0))]),
    # three-way ties: z, y, x, then z, y: along B's second ray to the occupied (1,2,2)
    "line_tie_three_axes": ("B", "line", ([O], [(0.25, 0.25, 0.25)], None, True), [(OCC, _rel(1, 2, 2))]),
    # box (0, 0.2, 0): y offsets -0.1, -0.0333, 0.0333, 0.1 (x and z: one zero offset).  Segment on y = 0.05: line 0 runs
    # at y = -0.05 (unknown), line 1 on the x row (occupied): the unknown line 0 wins; without the stop line 0 is free and
    # line 1 decides
    "box_lower_line_wins_unknown": ("A", "line", ([O], [(0.95, 0.05, 0.05)], (0.0, 0.2, 0.0), True),
                                    [(UNK, _rel(0, -1, 0))]),
    "box_without_stop": ("A", "line", ([O], [(0.95, 0.05, 0.05)], (0.0, 0.2, 0.0), False), [(OCC, _rel(5, 0, 0))]),
    # segment on y = 0.15: line 0 on the x row (occupied), line 1 at y = 0.1167 meets the unknown (1,1,0): line 0 wins
    "box_lower_line_wins_occupied": ("A", "line", ([(0.05, 0.15, 0.05)], [(0.95, 0.15, 0.05)], (0.0, 0.2, 0.0), True),
                                     [(OCC, _rel(5, 0, 0))]),
    "box_of_size_zero_is_the_line": ("A", "line", ([O, (-0.15, 0.05, 0.05)], [(0.95, 0.05, 0.05), (0.45, 0.05, 0.05)],
                                                   (0.0, 0.0, 0.0), True), [(OCC, _rel(5, 0, 0)), (UNK, _rel(-2, 0, 0))]),
    "box_all_free": ("A", "line", ([O], [(0.45, 0.05, 0.05)], (0.05, 0.0, 0.05), True), [(FREE, NONE)]),
    "ray_hit": ("A", "ray", ([O], [(1.0, 0.0, 0.0)], False, -1.0), [(oq.RAY_HIT, _rel(5, 0, 0))]),
    "ray_occupied_origin": ("A", "ray", ([(0.55, 0.05, 0.05)], [(1.0, 0.0, 0.0)], False, -1.0), [(oq.RAY_HIT, _rel(5, 0, 0))]),
    "ray_unknown_origin": ("A", "ray", ([(0.15, 0.15, 0.05)], [(1.0, 0.0, 0.0)], False, -1.0),
                           [(oq.RAY_UNKNOWN, _rel(1, 1, 0))]),
    "ray_unknown_origin_ignored": ("A", "ray", ([(-0.05, 0.05, 0.05)], [(3.0, 0.0, 0.0)], True, -1.0),
                                   [(oq.RAY_HIT, _rel(5, 0, 0))]),
    "ray_unknown_ahead": ("A", "ray", ([O], [(-1.0, 0.0, 0.0)], False, -1.0), [(oq.RAY_UNKNOWN, _rel(-1, 0, 0))]),
    "ray_zero_direction": ("A", "ray", ([O, (0.15, 0.05, 0.05)], [(0.0, 0.0, 0.0), (NAN, 0.0, 0.0)], False, -1.0),
                           [(oq.RAY_INVALID, None)] * 2),
    "ray_zero_direction_at_occupied_origin": ("A", "ray", ([(0.55, 0.05, 0.05)], [(0.0, 0.0, 0.0)], False, -1.0),
                                              [(oq.RAY_HIT, _rel(5, 0, 0))]),
    "ray_invalid_origin": ("A", "ray", ([(5000.0, 0.0, 0.0), (NAN, 0.0, 0.0)], [(1.0, 0.0, 0.0)] * 2, True, -1.0),
                           [(oq.RAY_INVALID, None)] * 2),
    # centres 0.15, 0.25, 0.35: the third is 0.3 from the origin, past 0.25
    "ray_max_range": ("A", "ray", ([O], [(2.0, 0.0, 0.0)], False, 0.25), [(oq.RAY_MAX_RANGE, _rel(3, 0, 0))]),
    "ray_key_bound": ("A", "ray", ([(3276.65, 0.05, 0.05), (-3276.75, 0.05, 0.05)], [(1.0, 0.0, 0.0), (-1.0, 0.0, 0.0)],
                                   True, -1.0), [(oq.RAY_KEY_BOUND, _pack((65535, K0, K0))),
                                                 (oq.RAY_KEY_BOUND, _pack((0, K0, K0)))]),
    "ray_diagonal_ties": ("B", "ray", ([O], [(1.0, 1.0, 1.0)], False, -1.0), [(oq.RAY_HIT, _rel(1, 2, 2))]),
}


def run_case(m, kind, inputs):
    """(status / result int8, second output) of one case on an oracle or device map."""
    if kind == "cell":
        return m.cell_status(np.array(inputs, np.float64))
    if kind == "line":
        s, e, box, stop = inputs
        return m.line_status(np.array(s, np.float64), np.array(e, np.float64), box=box, stop_at_unknown=stop)
    o, d, ign, mr = inputs
    return m.cast_rays(np.array(o, F32), np.array(d, F32), ignore_unknown=ign, max_range=mr)


def check_case(kind, got, want):
    st, out = got
    assert [int(x) for x in st] == [w[0] for w in want]
    for j, (_, w) in enumerate(want):
        if kind == "cell":
            if w is None:
                assert _bits(out[j : j + 1])[0] == NAN_BITS
            else:
                assert _bits(out[j : j + 1])[0] == _bits(np.array([w], F32))[0]
        elif kind == "line":
            assert int(out[j]) == w
        elif w is None:
            assert (_bits(out[j]) == NAN_BITS).all()
        else:
            assert np.array_equal(_bits(out[j]), _bits(np.array(_centre3(w, PARAMS["resolution"]), F32)))


@pytest.mark.parametrize("name", sorted(CASES))
def test_known_answers(name):
    mname, kind, inputs, want = CASES[name]
    check_case(kind, run_case(_oracle_map(mname), kind, inputs), want)


def test_box_offsets_as_the_answers_assume():
    assert box_offsets((0.0, 0.2, 0.0), 0.1)[1] == pytest.approx([-0.1, -0.1 / 3, 0.1 / 3, 0.1])
    assert box_offsets((0.0, 0.0, 0.0), 0.1) == [[-0.0], [-0.0], [-0.0]]
    assert [len(a) for a in box_offsets((0.6, 0.6, 0.3), 0.075)] == [10, 10, 6]


# ---- restatement: float64 segment-voxel intersection, float64 ray traversal, the box loop in Python ---------------------
def box_offsets(size, res):
    """getLineStatusBoundingBox's offsets per axis (double, accumulated as its loop does)."""
    out = []
    for s in size:
        disc = s / math.ceil((s + 0.001) / res)
        if disc <= 0.0:
            disc = 1.0
        vals, x = [], -(s * 0.5)
        while x <= s * 0.5:
            vals.append(x)
            x += disc
        out.append(vals)
    return out


def _states(m):
    k, v = m.download()
    lo = oc.logodds(0.7)
    return {int(a): (OCC if b >= lo else FREE) for a, b in zip(k, v)}


def _occupied_centre(rng, states, res):
    occ = [k for k, v in states.items() if v == OCC]
    return np.array(_centre3(occ[rng.integers(len(occ))], res), np.float64)


def _restated_line(states, s, e, res, stop):
    cells = segment_cells(np.asarray(s, F32), np.asarray(e, F32), res, margin=1e-6)
    if cells is None:
        return None
    for c in cells:
        st = states.get(_pack(c), UNK)
        if st == OCC or (st == UNK and stop):
            return st, _pack(c)
    return FREE, NONE


def _random_map(rng, res):
    origin = np.array([0.013, -0.021, 0.037], F32)
    m = oq.OccupancyMap(resolution=res, max_range=-1.0)
    for _ in range(2):
        cloud = _tie_free_cloud(rng, 150, res, origin, -1.0)
        m.insert_scan(cloud - np.array([*origin, 0], F32), _translate(origin))
    return m, origin


@pytest.mark.parametrize("res", [0.1, 0.075])
def test_line_status_equals_segment_voxel_intersection(res):
    rng = np.random.default_rng(21)
    m, origin = _random_map(rng, res)
    states = _states(m)
    seen = {FREE: 0, OCC: 0, UNK: 0}
    checked = 0
    while checked < 400:
        s = origin + rng.uniform(-1.0, 1.0, 3)
        e = s + rng.uniform(-2.5, 2.5, 3)
        if rng.integers(2):  # half of them through an occupied voxel
            e = s + (_occupied_centre(rng, states, res) - s) * rng.uniform(1.1, 1.5)
        stop = bool(rng.integers(2))
        want = _restated_line(states, s, e, res, stop)
        if want is None:
            continue
        st, fk = m.line_status(s[None], e[None], stop_at_unknown=stop)
        assert (int(st[0]), int(fk[0])) == want, (s, e, stop)
        seen[want[0]] += 1
        checked += 1
    assert min(seen.values()) > 10


def _restated_ray(states, o, d, res, ignore, length=8.0):
    """castRay in float64 geometry: the voxels the ray o + t * d / |d| crosses for t in (0, length); None on a near tie
    or when it does not stop within length."""
    o = np.asarray(o, F32).astype(np.float64)
    d = np.asarray(d, F32).astype(np.float64)
    e = o + d / np.linalg.norm(d) * length
    cells = segment_cells(o, e, res, margin=1e-6)
    if cells is None or not cells:
        return None
    for c in cells:
        st = states.get(_pack(c), UNK)
        if st == OCC:
            return oq.RAY_HIT, _pack(c)
        if st == UNK and not ignore:
            return oq.RAY_UNKNOWN, _pack(c)
    return None


@pytest.mark.parametrize("res", [0.1, 0.075])
def test_rays_equal_float64_traversal(res):
    rng = np.random.default_rng(22)
    m, origin = _random_map(rng, res)
    states = _states(m)
    seen = {oq.RAY_HIT: 0, oq.RAY_UNKNOWN: 0}
    checked = 0
    while checked < 400:
        o = (origin + rng.uniform(-0.5, 0.5, 3)).astype(F32)
        d = rng.normal(size=3).astype(F32)
        if rng.integers(2):
            d = (_occupied_centre(rng, states, res) - o).astype(F32)
        ignore = bool(rng.integers(2))
        want = _restated_ray(states, o, d, res, ignore)
        if want is None:
            continue
        r, ends = m.cast_rays(o[None], d[None], ignore_unknown=ignore)
        assert int(r[0]) == want[0], (o, d, ignore)
        assert np.array_equal(_bits(ends[0]), _bits(np.array(_centre3(want[1], res), F32)))
        seen[want[0]] += 1
        checked += 1
    assert min(seen.values()) > 10


@pytest.mark.parametrize("size", [(0.6, 0.6, 0.3), (0.0, 0.35, 0.2), (0.25, 0.0, 0.0)])
def test_box_equals_the_restated_offset_loop(size):
    rng = np.random.default_rng(23)
    res = 0.1
    m, origin = _random_map(rng, res)
    offs = box_offsets(size, res)
    seen = set()
    states = _states(m)
    for _ in range(80):
        s = origin + rng.uniform(-1.0, 1.0, 3)
        e = s + rng.uniform(-2.0, 2.0, 3)
        if rng.integers(2):
            e = s + (_occupied_centre(rng, states, res) - s) * rng.uniform(1.1, 1.5)
        stop = bool(rng.integers(2))
        want = (FREE, NONE)
        for x in offs[0]:
            for y in offs[1]:
                for z in offs[2]:
                    st, fk = m.line_status((s + [x, y, z])[None], (e + [x, y, z])[None], stop_at_unknown=stop)
                    if st[0] != FREE:
                        want = (int(st[0]), int(fk[0]))
                        break
                if want[0] != FREE:
                    break
            if want[0] != FREE:
                break
        st, fk = m.line_status(s[None], e[None], box=size, stop_at_unknown=stop)
        assert (int(st[0]), int(fk[0])) == want
        seen.add(want[0])
    assert seen == {FREE, OCC, UNK}


def test_oracle_cell_status_of_known_voxels_and_keys_visited():
    m = _oracle_map("A")
    k, v = m.download()
    st, lo = m.cell_status(oc.centres(k, 0.1).astype(np.float64))
    assert m.keys_visited == len(k)
    assert np.array_equal(st, np.where(v >= oc.logodds(0.7), OCC, FREE)) and np.array_equal(_bits(lo), _bits(v))


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _device_map(ls, ctx, name):
    ring = ctx.create_map(2, 1024)
    dev = ls.OccupancyMap(ctx, **PARAMS)
    for c, T in SCANS[name]:
        dev.insert_scan(ring, ring.push_scan(c, np.zeros((len(c), 3), F32)), T)
    return ring, dev


def _same(a, b):
    """Bit-equality of (status, second output) pairs."""
    if not np.array_equal(a[0], b[0]):
        return False
    x, y = np.asarray(a[1]), np.asarray(b[1])
    if x.dtype == np.float32:
        return np.array_equal(_bits(x), _bits(y))
    return np.array_equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_known_answers_on_the_device(gpu_ctx, name):
    import laser_slam_b200 as ls
    mname, kind, inputs, want = CASES[name]
    ring, dev = _device_map(ls, gpu_ctx, mname)
    o = _oracle_map(mname)
    got = run_case(dev, kind, inputs)
    check_case(kind, got, want)
    assert _same(got, run_case(o, kind, inputs))
    if "box" not in name:
        assert dev.last_query.keys_visited == o.keys_visited
    dev.close()
    ring.close()


N_FULL = 12


@pytest.fixture(scope="module", params=[dict(), dict(resolution=0.1, max_range=-1.0)], ids=["defaults", "res0.1_unlimited"])
def full_maps(request, gpu_ctx, synth_mod):
    import laser_slam_b200 as ls
    params = request.param
    truth, _ = synth_mod.trajectory(0, N_FULL)
    scans = [synth_mod.scan(truth[k], 0, k)[0] for k in range(N_FULL)]
    poses = [truth[k].astype(F32) for k in range(N_FULL)]
    ring = gpu_ctx.create_map(2, 131072)
    dev = ls.OccupancyMap(gpu_ctx, **params)
    o = oq.OccupancyMap(**params)
    nrm = np.zeros((131072, 3), F32)
    for k in range(N_FULL):
        dev.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
        o.insert_scan(scans[k], poses[k])
    yield dict(ls=ls, dev=dev, o=o, scans=scans, poses=poses, res=dev.params.resolution)
    dev.close()
    ring.close()


def _segments(rng, poses, n, lo=1.0, hi=10.0):
    p = np.array([poses[k][:3, 3] for k in rng.integers(0, len(poses), n)], np.float64)
    s = p + rng.uniform(-3.0, 3.0, (n, 3)) * [1, 1, 0.3]
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    return s, s + d * rng.uniform(lo, hi, (n, 1))


@pytest.mark.gpu
def test_full_map_cells_match_the_oracle(full_maps):
    ls, dev, o, res = full_maps["ls"], full_maps["dev"], full_maps["o"], full_maps["res"]
    keys, lo = o.download()
    rng = np.random.default_rng(31)
    cen = oc.centres(keys, res).astype(np.float64)
    box_lo, box_hi = cen.min(axis=0), cen.max(axis=0)
    extra = np.array([[NAN, 0, 0], [0, INF, 0], [0, 0, -INF], [4000.0, 0, 0], [0, -4000.0, 0], [1e30, 1e30, 1e30]])
    pts = np.concatenate([cen, rng.uniform(box_lo, box_hi, (200_000, 3)), cen[:5000] + rng.uniform(-res, res, (5000, 3)),
                          extra])
    got = dev.cell_status(pts)
    want = o.cell_status(pts)
    assert _same(got, want) and dev.last_query.keys_visited == o.keys_visited
    st = got[0]
    assert (st[:len(keys)] != UNK).all() and np.array_equal(_bits(got[1][:len(keys)]), _bits(lo))
    assert (st[-len(extra):] == UNK).all() and set(np.unique(st[len(keys):])) == {FREE, OCC, UNK}
    # every known voxel's status is what the occupied download implies
    occ_keys = dev.download(ls.OCC_OCCUPIED)[0]
    assert np.array_equal(np.isin(keys, occ_keys), st[:len(keys)] == OCC)


@pytest.mark.gpu
@pytest.mark.parametrize("stop", [True, False])
def test_full_map_lines_match_the_oracle(full_maps, stop):
    dev, o = full_maps["dev"], full_maps["o"]
    rng = np.random.default_rng(32 + stop)
    s, e = _segments(rng, full_maps["poses"], 100_000)
    got = dev.line_status(s, e, stop_at_unknown=stop)
    want = o.line_status(s, e, stop_at_unknown=stop)
    assert _same(got, want) and dev.last_query.keys_visited == o.keys_visited
    assert set(np.unique(got[0])) == ({FREE, OCC, UNK} if stop else {FREE, OCC})  # no stop: an unknown key is passed


@pytest.mark.gpu
@pytest.mark.parametrize("box", [(0.6, 0.6, 0.3), (0.3, 0.0, 0.45)])
def test_full_map_boxes_match_the_oracle(full_maps, box):
    dev, o = full_maps["dev"], full_maps["o"]
    rng = np.random.default_rng(34)
    s, e = _segments(rng, full_maps["poses"], 300, 0.5, 4.0)
    for stop in (True, False):
        got = dev.line_status(s, e, box=box, stop_at_unknown=stop)
        assert _same(got, o.line_status(s, e, box=box, stop_at_unknown=stop))
        assert len(set(np.unique(got[0]))) >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("ignore", [False, True])
def test_full_map_rays_match_the_oracle(full_maps, ignore):
    dev, o = full_maps["dev"], full_maps["o"]
    for k in (0, 5, 11):
        T = full_maps["poses"][k].astype(np.float64)
        origins = np.repeat(full_maps["poses"][k][:3, 3][None], 131072, axis=0).astype(F32)
        dirs = (full_maps["scans"][k][:, :3].astype(np.float64) @ T[:3, :3].T).astype(F32)
        for mr in (20.0, 7.5):
            got = dev.cast_rays(origins, dirs, ignore_unknown=ignore, max_range=mr)
            want = o.cast_rays(origins, dirs, ignore_unknown=ignore, max_range=mr)
            assert _same(got, want) and dev.last_query.keys_visited == o.keys_visited
            assert oq.RAY_HIT in got[0] and oq.RAY_MAX_RANGE in got[0]


@pytest.mark.gpu
def test_host_layer_queries_equal_the_abi(synth_mod):
    """laser_slam::OccupancyMap's WorldBase names and castRay, single and batched, against the Python ABI on the same
    map; probabilities follow 1 - 1 / (1 + exp(v)) and -1 when unknown."""
    import laser_slam_b200 as ls
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    n = 4
    truth, odom = synth_mod.trajectory(3, n + 1)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 3, k), 8) for k in range(n)]
    est = host.Estimator(n_workers=1, nscan_in_sub_map=3)
    odom7 = pg.se3_from_matrix(odom)
    for k in range(n):
        f, nr = np.ascontiguousarray(scans[k][0]), np.ascontiguousarray(scans[k][1])
        est.step_batch([0], [k * 10**8], [odom7[k]], [f.ctypes.data], [nr.ctypes.data], [len(f)])
    params = dict(resolution=0.1, max_range=15.0)
    occ = host.OccupancyMap(est, **params)
    assert occ.insert_laser_tracks() == n
    keys, lo = occ.voxels(1)
    ctx = ls.Context(0)
    ring = ctx.create_map(n, 131072)
    dev = ls.OccupancyMap(ctx, **params)
    ts, traj = est.trajectory(0)
    from test_local_map import _float_matrix
    for k in range(n):
        dev.insert_scan(ring, ring.push_scan(scans[k][0], np.zeros((len(scans[k][0]), 3), F32)), _float_matrix(traj[k]))
    dk, dlo, _ = dev.download(ls.OCC_KNOWN)
    assert np.array_equal(dk, keys) and np.array_equal(_bits(dlo), _bits(lo))
    rng = np.random.default_rng(41)
    cen = oc.centres(keys, 0.1).astype(np.float64)
    pts = np.concatenate([cen[::50], rng.uniform(cen.min(0), cen.max(0), (300, 3)), [[NAN, 0, 0]]])
    st, pr = occ.cell_probability(pts)
    dst, dlo2 = dev.cell_status(pts)
    assert np.array_equal(st, dst)
    want = np.array([-1.0 if s == UNK else 1.0 - 1.0 / (1.0 + math.exp(float(v))) for s, v in zip(dst, dlo2)])
    assert np.array_equal(pr, want)
    p0 = truth[0][:3, 3]
    s, e = _segments(rng, [truth[k] for k in range(n)], 400)
    for box in (None, (0.4, 0.2, 0.0)):
        for stop in (True, False):
            if box is not None and not stop:
                continue
            want = dev.line_status(s, e, box=box, stop_at_unknown=stop)
            got = occ.line_status(s, e, box=box, stop_at_unknown=stop)
            assert _same(got, want)
            assert np.array_equal(occ.line_status(s[:60], e[:60], box=box, stop_at_unknown=stop, single=True), want[0][:60])
    dirs = rng.normal(size=(500, 3))
    origins = np.repeat(p0[None], 500, axis=0)
    for ign in (False, True):
        r, ends = dev.cast_rays(origins, dirs, ignore_unknown=ign, max_range=10.0)
        hr, hends = occ.cast_rays(origins, dirs, ignore_unknown=ign, max_range=10.0)
        assert np.array_equal(hr, r) and np.array_equal(hends, ends.astype(np.float64))
        sr, sends = occ.cast_rays(origins[:80], dirs[:80], ignore_unknown=ign, max_range=10.0, single=True,
                                  ends_in=np.full((80, 3), 7.0))
        assert np.array_equal(sr, (r[:80] == oq.RAY_HIT).astype(np.int32))
        valid = r[:80] != oq.RAY_INVALID
        assert np.array_equal(sends[valid], ends[:80][valid].astype(np.float64)) and (sends[~valid] == 7.0).all()
    dev.close()
    ring.close()
    ctx.close()
    occ.close()
    est.close()


@pytest.mark.gpu
def test_queries_between_batch_begin_and_end(synth_mod):
    import laser_slam_b200 as ls
    truth, _ = synth_mod.trajectory(0, 4)
    scans = [synth_mod.scan(truth[k], 0, k)[0] for k in range(4)]
    poses = [truth[k].astype(F32) for k in range(4)]
    ctx = ls.Context(0)
    ring = ctx.create_map(16, 131072)
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(4)]
    dev = ls.OccupancyMap(ctx)
    o = oq.OccupancyMap()
    for k in range(2):
        dev.insert_scan(ring, ids[k], poses[k])
        o.insert_scan(scans[k], poses[k])
    problems = [(ids[k + 1], [ids[k]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[k]) @ poses[k + 1]) for k in range(3)]
    p = ls.default_params(max_iterations=5)
    alone = ring.register_batch(problems, p)
    rng = np.random.default_rng(51)
    s, e = _segments(rng, poses[:2], 2000)
    origins = np.repeat(poses[0][:3, 3][None], 4096, axis=0)
    dirs = rng.normal(size=(4096, 3)).astype(F32)
    end = ring.begin_batch(problems, p)
    cells = dev.cell_status(s)
    lines = dev.line_status(s, e)
    boxes = dev.line_status(s[:100], e[:100], box=(0.6, 0.6, 0.3))
    rays = dev.cast_rays(origins, dirs, max_range=20.0)
    res = end()
    for a, b in zip(res, alone):
        assert a["rc"] == b["rc"] and np.array_equal(a["T"], b["T"])
    assert _same(cells, o.cell_status(s)) and _same(lines, o.line_status(s, e))
    assert _same(boxes, o.line_status(s[:100], e[:100], box=(0.6, 0.6, 0.3)))
    assert _same(rays, o.cast_rays(origins, dirs, max_range=20.0))
    dev.close()
    ring.close()
    ctx.close()


@pytest.mark.gpu
def test_errors_return_their_code_and_leave_the_map_unchanged(gpu_ctx, synth_mod):
    import laser_slam_b200 as ls
    truth, _ = synth_mod.trajectory(0, 1)
    ring = gpu_ctx.create_map(2, 131072)
    dev = ls.OccupancyMap(gpu_ctx)
    dev.insert_scan(ring, ring.push_scan(synth_mod.scan(truth[0], 0, 0)[0], np.zeros((131072, 3), F32)), truth[0].astype(F32))
    before = [dev.download(w) for w in (ls.OCC_KNOWN, ls.OCC_OCCUPIED)]
    L, h = ls.lib(), dev._h
    p = np.zeros((4, 3), np.float64)
    f = np.zeros((4, 3), F32)
    st = np.zeros(4, np.int8)
    fk = np.zeros(4, np.uint64)
    qs = ls.OccupancyQueryStats()
    ARG = -1
    assert L.ls_occupancy_cell_status(h, p.ctypes.data, -1, st.ctypes.data, None, None) == ARG
    assert L.ls_occupancy_cell_status(h, None, 4, st.ctypes.data, None, None) == ARG
    assert L.ls_occupancy_cell_status(h, p.ctypes.data, 4, None, None, None) == ARG
    assert L.ls_occupancy_line_status(h, p.ctypes.data, p.ctypes.data, -2, None, 1, st.ctypes.data, None, None) == ARG
    assert L.ls_occupancy_line_status(h, p.ctypes.data, None, 4, None, 1, st.ctypes.data, None, None) == ARG
    assert L.ls_occupancy_line_status(h, p.ctypes.data, p.ctypes.data, 4, None, 1, None, None, None) == ARG
    launches = gpu_ctx.launch_count
    for box in ((-0.1, 0.1, 0.1), (0.1, NAN, 0.1), (0.1, 0.1, INF), (300.0, 300.0, 300.0), (1e300, 0.0, 0.0)):
        b = np.array(box, np.float64)
        assert L.ls_occupancy_line_status(h, p.ctypes.data, p.ctypes.data, 4, b.ctypes.data, 1, st.ctypes.data,
                                          fk.ctypes.data, None) == ARG
    assert gpu_ctx.launch_count == launches          # refused before any launch
    assert L.ls_occupancy_cast_rays(h, f.ctypes.data, f.ctypes.data, -1, 0, 20.0, st.ctypes.data, None, None) == ARG
    assert L.ls_occupancy_cast_rays(h, None, f.ctypes.data, 4, 0, 20.0, st.ctypes.data, None, None) == ARG
    assert L.ls_occupancy_cast_rays(h, f.ctypes.data, f.ctypes.data, 4, 0, 20.0, None, None, None) == ARG
    # n = 0: LS_OK without a launch, NULL buffers allowed
    qs.keys_visited = 99
    assert L.ls_occupancy_cell_status(h, None, 0, None, None, ctypes.byref(qs)) == 0 and qs.keys_visited == 0
    assert L.ls_occupancy_line_status(h, None, None, 0, None, 1, None, None, None) == 0
    assert L.ls_occupancy_cast_rays(h, None, None, 0, 0, -1.0, None, None, None) == 0
    assert gpu_ctx.launch_count == launches
    # valid queries, the optional outputs NULL
    assert L.ls_occupancy_cell_status(h, p.ctypes.data, 4, st.ctypes.data, None, None) == 0
    assert L.ls_occupancy_line_status(h, p.ctypes.data, p.ctypes.data, 4, None, 1, st.ctypes.data, None, None) == 0
    assert L.ls_occupancy_cast_rays(h, f.ctypes.data, f.ctypes.data, 4, 0, 20.0, st.ctypes.data, None, None) == 0
    after = [dev.download(w) for w in (ls.OCC_KNOWN, ls.OCC_OCCUPIED)]
    for a, b in zip(before, after):
        assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
    dev.close()
    ring.close()
