"""Change detection of the resident occupancy map (ls_occupancy_track_changes / _changes; DESIGN.md §4b'''''''''').
CPU: octomap's event rule (tests/occupancy_changes_ref.py's EventLog) equals the snapshot diff on random update sequences,
the oracle's per-scan maps and box edits, and known answers.  GPU: every result bit for bit against the diff of two
downloads and against the event rule, after inserts, edits, growth, clear and .bt / .ot reads; tracking leaves everything
else as it was; refusals keep the baseline; calls inside a batch; the C++ layer against the ABI."""
import ctypes

import numpy as np
import pytest

import laser_slam_b200 as ls
import occupancy_changes_ref as cr
import occupancy_edits_ref as er
from oracle import occupancy as oc
from test_occupancy import F32, full_scans  # noqa: F401  (full_scans: fixture)

L_OCC = oc.logodds(0.7)
L_MIN, L_MAX = F32(oc.logodds(0.12)), F32(oc.logodds(0.97))
FREE, OCC, UNK = cr.CELL_FREE, cr.CELL_OCCUPIED, cr.CELL_UNKNOWN


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _same(got, want):
    """(keys, status, previous) equal, and the centres bit for bit when both have them."""
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
    if len(got) > 3 and len(want) > 3:
        assert np.array_equal(_bits(got[3]), _bits(want[3]))


def _with_centres(d, res_now, res_base):
    return d + (cr.centres(d[0], d[1], res_now, res_base),)


# ---- CPU: the event rule equals the diff rule --------------------------------------------------------------------
def test_event_rule_equals_diff_rule_on_random_sequences():
    rng = np.random.default_rng(0)
    values = np.array([L_MIN, F32(-0.3), F32(0.4), F32(L_OCC), F32(1.2), L_MAX], F32)  # 3 free, 3 occupied
    seen = dict(created=0, flip=0, flip_back=0, created_flipped=0, same_state=0)
    for trial in range(200):
        keys = rng.integers(0, 40, 20).tolist()
        base = {k: values[rng.integers(0, 6)] for k in keys[:10]}
        now = dict(base)
        log = cr.EventLog(L_OCC)
        flips = {}
        for _ in range(rng.integers(1, 80)):
            k = int(rng.integers(0, 40))
            v = values[rng.integers(0, 6)]
            before = now.get(k)
            if before is None:
                seen["created"] += 1
            elif (before >= F32(L_OCC)) != (v >= F32(L_OCC)):
                flips[k] = flips.get(k, 0) + 1
                seen["flip"] += 1
                seen["flip_back"] += flips[k] == 2 and k in base
                seen["created_flipped"] += k not in base
            else:
                seen["same_state"] += 1
            log.update(k, before, v)
            now[k] = v
        _same(log.result(now), cr.diff(base, now, L_OCC))
        _same(cr.diff(base, now, L_OCC), cr.diff_arrays(*_arrays(base), *_arrays(now), L_OCC))
    assert all(v > 10 for v in seen.values()), seen  # every branch of the rule was reached


def _arrays(vox):
    keys = np.array(sorted(vox), np.uint64)
    return keys, np.array([vox[int(k)] for k in keys], F32)


def test_event_rule_equals_diff_rule_on_the_oracles_per_scan_maps(synth_mod):
    truth, _ = synth_mod.trajectory(0, 8)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 0, k), 16)[0] for k in range(8)]
    o = oc.OccupancyMap(resolution=0.2, max_range=10.0)
    arrays = [(np.zeros(0, np.uint64), np.zeros(0, F32))]
    for k in range(8):
        o.insert_scan(scans[k], truth[k])
        arrays.append(o.download())
    o.close()
    snaps = [cr.as_dict(*a) for a in arrays]
    flipped = 0
    for b in (0, 1, 4):
        log, log_a = cr.EventLog(L_OCC), cr.EventLog(L_OCC)
        for j in range(b, 8):
            log.apply(snaps[j], snaps[j + 1])
            log_a.apply_arrays(*arrays[j], *arrays[j + 1])
        got, want = log.result(snaps[8]), cr.diff(snaps[b], snaps[8], L_OCC)
        _same(got, want)
        _same(log_a.result_arrays(*arrays[8]), want)  # the vectorised steps the GPU tests use
        _same(cr.diff_arrays(*arrays[b], *arrays[8], L_OCC), want)
        flipped += int((want[2] != UNK).sum())
        assert len(want[0]) > 1000
    assert flipped > 0  # known voxels that changed state, not only new ones


def test_event_rule_equals_diff_rule_on_box_edits():
    e = er.Edits(0.1, L_MIN, L_MAX, L_OCC)
    base = {}
    e.set_boxes(base, [(0.0, 0.0, 0.0), (0.5, 0.2, 0.0)], [(1.0, 1.0, 1.0), (0.6, 0.6, 0.6)], [False, True])
    sequences = [
        ([(0.3, 0.3, 0.3)], [(0.6, 0.6, 0.6)], [True]),                   # free -> occupied, plus new voxels
        ([(0.3, 0.3, 0.3)], [(0.4, 0.4, 0.4)], [False]),                  # some of them back
        ([(0.5, 0.2, 0.0), (0.5, 0.2, 0.0)], [(0.4,) * 3, (0.2,) * 3], [False, True]),  # occupied -> free -> occupied
        ([(2.0, 2.0, 2.0)], [(0.5, 0.5, 0.5)], [True]),                   # created
        ([(2.0, 2.0, 2.0)], [(0.3, 0.3, 0.3)], [False]),                  # created, then flipped
    ]
    now = dict(base)
    log = cr.EventLog(L_OCC)
    for centres, sizes, occupied in sequences:
        for c, s, o in zip(centres, sizes, occupied):  # box by box, voxel by voxel, as setNodeValue
            v = L_MAX if o else L_MIN
            for k in er.box_keys(c, s, 0.1):
                log.update(k, now.get(k), v)
                now[k] = v
    d = cr.diff(base, now, L_OCC)
    _same(log.result(now), d)
    assert ((d[2] == FREE) & (d[1] == OCC)).any() and ((d[2] == OCC) & (d[1] == FREE)).any() and (d[2] == UNK).any()


# ---- CPU: known answers ----------------------------------------------------------------------------------------
def test_a_voxel_flipped_twice_is_absent():
    base = {1: L_MIN, 2: L_MIN}
    log = cr.EventLog(L_OCC)
    now = dict(base)
    for v in (L_MAX, L_MIN):
        log.update(1, now[1], v)
        now[1] = v
    log.update(2, now[2], L_MAX)
    now[2] = L_MAX
    assert log.changed == {2: False}  # precondition: voxel 1 flipped and came back
    assert cr.diff(base, now, L_OCC)[0].tolist() == [2]


def test_a_created_voxel_stays_baseline_unknown_after_flipping():
    log = cr.EventLog(L_OCC)
    log.update(5, None, L_MIN)
    log.update(5, L_MIN, L_MAX)
    assert log.changed == {5: True}
    k, st, prev = cr.diff({}, {5: L_MAX}, L_OCC)
    assert (k.tolist(), st.tolist(), prev.tolist()) == ([5], [OCC], [UNK])


def test_a_state_preserving_log_odds_change_is_absent():
    base, now = {7: F32(0.9), 8: F32(-0.5)}, {7: F32(1.4), 8: F32(-1.5)}
    assert base[7] != now[7] and base[8] != now[8]  # precondition: the values changed, the states did not
    log = cr.EventLog(L_OCC)
    for k in base:
        log.update(k, base[k], now[k])
    assert log.changed == {} and len(cr.diff(base, now, L_OCC)[0]) == 0


def test_after_a_clear_every_baseline_voxel_is_now_unknown():
    base = {1: L_MIN, 2 << 16: L_MAX, 3 << 32: F32(0.2)}
    k, st, prev = cr.diff(base, {}, L_OCC)
    assert k.tolist() == [1, 2 << 16, 3 << 32] and (st == UNK).all() and prev.tolist() == [FREE, OCC, FREE]


def test_centres_after_a_read_at_a_foreign_resolution():
    key = np.uint64(32770 | (32760 << 16) | (32768 << 32))
    c = cr.centres([key, key], [UNK, FREE], 0.2, 0.05)  # unknown now: the baseline's 0.05; known now: the map's 0.2
    assert c[0, :3].tolist() == [F32(2.5 * 0.05), F32(-7.5 * 0.05), F32(0.5 * 0.05)]
    assert c[1, :3].tolist() == [F32(2.5 * 0.2), F32(-7.5 * 0.2), F32(0.5 * 0.2)] and (c[:, 3] == 1).all()


# ---- GPU ----------------------------------------------------------------------------------------------------------
PARAMS = {"defaults": {}, "res01_unlimited": dict(resolution=0.1, max_range=-1.0)}
BASELINES = (1, 5, 9)  # tracking enabled after scan k


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


def _known(om):
    k, v, _ = om.download(ls.OCC_KNOWN)
    return k, v


def _raw_changes(om, cap, reset):
    """The ABI call with buffers of cap: (rc, n, keys, status, previous, centres)."""
    n = ctypes.c_int64(-1)
    m = max(cap, 1)
    k, s, p, c = np.zeros(m, np.uint64), np.zeros(m, np.int8), np.zeros(m, np.int8), np.zeros((m, 4), F32)
    rc = ls.lib().ls_occupancy_changes(om._h, k.ctypes.data, s.ctypes.data, p.ctypes.data, c.ctypes.data, cap,
                                       ctypes.byref(n), int(reset), None)
    return rc, n.value, k, s, p, c


@pytest.fixture(scope="module")
def oracle_events(full_scans):
    """Per PARAMS entry: {k: the event rule's result over scans k ... 11 of the oracle's per-scan maps}."""
    scans, poses = full_scans
    out = {}
    for name, prm in PARAMS.items():
        o = oc.OccupancyMap(**prm)
        logs = {k: cr.EventLog(L_OCC) for k in BASELINES}
        before = (np.zeros(0, np.uint64), np.zeros(0, F32))
        for j in range(len(scans)):
            o.insert_scan(scans[j], poses[j])
            after = o.download()
            for k, log in logs.items():
                if j >= k:
                    log.apply_arrays(*before, *after)
            before = after
        out[name] = {k: log.result_arrays(*before) for k, log in logs.items()}
        o.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PARAMS))
def test_twelve_scan_map(gpu_ctx, full_scans, oracle_events, name, keep):
    scans, poses = full_scans
    prm = PARAMS[name]
    res = prm.get("resolution", 0.075)
    ring = keep(gpu_ctx.create_map(2, 131072))
    nrm = np.zeros((131072, 3), F32)
    for k in BASELINES:
        om = keep(ls.OccupancyMap(gpu_ctx, **prm))
        for j in range(len(scans)):
            if j == k:
                om.track_changes()
                base = _known(om)
            om.insert_scan(ring, ring.push_scan(scans[j], nrm), poses[j])
        want = _with_centres(cr.diff_arrays(*base, *_known(om), L_OCC), res, res)
        assert (want[2] == UNK).any() and (want[2] != UNK).any()  # new voxels and flipped ones
        got = om.changes()
        _same(got, want)
        _same(got, oracle_events[name][k])
        st = om.last_changes
        assert st.changed == len(want[0]) and st.bricks_compared > 0 and st.baseline_bricks > 0
        if k == BASELINES[0]:
            rc, n, *_ = _raw_changes(om, 0, 1)  # the count: refused without a copy and without a reset
            assert rc == ls.LS_ERR_ARG and n == len(want[0])
            got = om.changes(reset=True)
            _same(got, want)
            assert all(len(a) == 0 for a in om.changes())  # the map is the baseline now
            rc, n, *_ = _raw_changes(om, 0, 0)
            assert rc == 0 and n == 0
        om.close()
    ring.close()


@pytest.mark.gpu
def test_edits_flip_known_voxels_both_ways_and_back(gpu_ctx, full_scans, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    om = keep(ls.OccupancyMap(gpu_ctx, resolution=0.1))
    nrm = np.zeros((131072, 3), F32)
    for j in range(3):
        om.insert_scan(ring, ring.push_scan(scans[j], nrm), poses[j])
    p = poses[1][:3, 3].astype(np.float64)
    om.track_changes()
    base = _known(om)
    vox = cr.as_dict(*base)
    e = er.Edits(0.1, L_MIN, L_MAX, L_OCC)
    log = cr.EventLog(L_OCC)
    occ = base[0][base[1] >= F32(L_OCC)]
    oc_c = oc.centres(occ, 0.1).astype(np.float64)
    q = oc_c[np.argmin(np.linalg.norm(oc_c - p, axis=1))]  # the occupied voxel nearest the sensor
    steps = [([p], [(4.0, 4.0, 1.0)], [True]),                  # free -> occupied, and new voxels
             ([p + 0.5], [(2.0, 2.0, 1.0)], [False]),            # some of them back
             ([q], [(1.0, 1.0, 1.0)], [False]),                  # occupied -> free
             ([q, q + 0.3], [(0.5, 0.5, 0.5), (0.3, 0.3, 0.3)], [True, False]),  # back, and out again
             ([p + (0, 3.0, 0)], [(1.0, 1.0, 1.0)], [True])]
    for c, s, o in steps:
        om.set_boxes(c, s, o)
        for ci, si, oi in zip(c, s, o):
            v = L_MAX if oi else L_MIN
            for k in er.box_keys(ci, si, 0.1):
                log.update(k, vox.get(k), v)
                vox[k] = v
    now = _known(om)
    assert np.array_equal(now[0], er.as_arrays(vox)[0])  # the edits are the restatement's
    want = _with_centres(cr.diff_arrays(*base, *now, L_OCC), 0.1, 0.1)
    assert ((want[2] == FREE) & (want[1] == OCC)).any() and ((want[2] == OCC) & (want[1] == FREE)).any()
    base_vox = cr.as_dict(*base)
    flipped_back = [k for k in er.box_keys(q, (0.5, 0.5, 0.5), 0.1) if cr.state(base_vox, k, L_OCC) == OCC]
    assert flipped_back and not np.isin(flipped_back, want[0]).any()  # flipped twice: absent
    got = om.changes()
    _same(got, want)
    _same(got, log.result(vox))
    om.close(), ring.close()


@pytest.mark.gpu
def test_growth_from_sixteen_bricks(gpu_ctx, full_scans, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    om = keep(ls.OccupancyMap(gpu_ctx, resolution=0.1, initial_capacity=16))
    nrm = np.zeros((131072, 3), F32)
    om.set_free(poses[0][:3, 3], (1.0, 1.0, 1.0))
    om.track_changes()
    base = _known(om)
    for j in range(4):
        st = om.insert_scan(ring, ring.push_scan(scans[j], nrm), poses[j])
    assert st.bricks > 1024  # the pool doubled and the hash was rebuilt several times
    got = om.changes()
    _same(got, _with_centres(cr.diff_arrays(*base, *_known(om), L_OCC), 0.1, 0.1))
    assert 0 < om.last_changes.baseline_bricks <= 27  # the 1 m box's bricks only
    om.close(), ring.close()


@pytest.mark.gpu
def test_clear_and_reads_after_a_baseline(gpu_ctx, full_scans, tmp_path, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    nrm = np.zeros((131072, 3), F32)
    a = keep(ls.OccupancyMap(gpu_ctx, resolution=0.1))
    b = keep(ls.OccupancyMap(gpu_ctx))  # 0.075 m
    for j in range(3):
        sid = ring.push_scan(scans[j], nrm)
        a.insert_scan(ring, sid, poses[j])
        b.insert_scan(ring, sid, poses[j + 1])
    a_ot, b_bt = str(tmp_path / "a.ot"), str(tmp_path / "b.bt")
    a.save_octomap_full(a_ot)
    b.save_octomap(b_bt)
    # clear: every baseline voxel is now unknown, centred at the baseline's resolution
    a.track_changes()
    base = _known(a)
    a.clear()
    got = a.changes(reset=True)
    assert len(got[0]) == len(base[0]) > 0 and (got[1] == UNK).all()
    _same(got, _with_centres(cr.diff_arrays(*base, *_known(a), L_OCC), 0.1, 0.1))
    # a .bt read at 0.075 m over the empty baseline, then a .ot read back at 0.1 m over a 0.075 m baseline
    a.read_octomap_full(a_ot)
    a.changes(reset=True)
    base = _known(a)
    a.read_octomap(b_bt)
    assert a.params.resolution == 0.075
    got = a.changes(reset=True)
    want = _with_centres(cr.diff_arrays(*base, *_known(a), L_OCC), 0.075, 0.1)
    assert (want[1] == UNK).any() and (want[1] != UNK).any()  # centres at both resolutions
    _same(got, want)
    base = _known(a)
    a.read_octomap_full(a_ot)
    _same(a.changes(), _with_centres(cr.diff_arrays(*base, *_known(a), L_OCC), 0.1, 0.075))
    a.close(), b.close(), ring.close()


def _query_points(poses, rng):
    return np.concatenate([poses[k][:3, 3] + rng.uniform(-12.0, 12.0, (5000, 3)) for k in range(4)])


@pytest.mark.gpu
def test_tracking_changes_nothing_else(gpu_ctx, full_scans, tmp_path, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    nrm = np.zeros((131072, 3), F32)
    maps = [keep(ls.OccupancyMap(gpu_ctx, initial_capacity=64)) for _ in range(2)]
    maps[0].track_changes()
    pts = _query_points(poses, np.random.default_rng(3))
    for j in range(4):
        sid = ring.push_scan(scans[j], nrm)
        stats = [m.insert_scan(ring, sid, poses[j]) for m in maps]
        d = [{f: getattr(s, f) for f, _ in s._fields_ if f != "device_ms"} for s in stats]
        assert d[0] == d[1]
        if j == 1:
            for m in maps:
                m.set_boxes([poses[1][:3, 3], poses[1][:3, 3] + 1.0], [(2.0, 2.0, 1.0), (1.0, 1.0, 1.0)], [True, False])
        maps[0].changes(reset=j % 2 == 0)
    assert maps[0].last_changes.changed > 0
    k0, k1 = maps[0].download(ls.OCC_KNOWN), maps[1].download(ls.OCC_KNOWN)
    assert all(np.array_equal(_bits(x) if x.dtype == F32 else x, _bits(y) if y.dtype == F32 else y) for x, y in zip(k0, k1))
    assert maps[0].octree().payload == maps[1].octree().payload
    assert maps[0].full_octree().payload == maps[1].full_octree().payload
    for m, name in zip(maps, "ab"):
        m.save_octomap(str(tmp_path / f"{name}.bt"))
    assert (tmp_path / "a.bt").read_bytes() == (tmp_path / "b.bt").read_bytes()
    q0, q1 = maps[0].cell_status(pts), maps[1].cell_status(pts)
    assert np.array_equal(q0[0], q1[0]) and np.array_equal(_bits(q0[1]), _bits(q1[1]))
    l0 = maps[0].line_status(pts[:2000], pts[2000:4000])
    l1 = maps[1].line_status(pts[:2000], pts[2000:4000])
    assert np.array_equal(l0[0], l1[0]) and np.array_equal(l0[1], l1[1])
    for m in maps:
        m.close()
    ring.close()


@pytest.mark.gpu
def test_refusals_keep_the_baseline(gpu_ctx, full_scans, keep):
    scans, poses = full_scans
    ring = keep(gpu_ctx.create_map(2, 131072))
    nrm = np.zeros((131072, 3), F32)
    om = keep(ls.OccupancyMap(gpu_ctx, resolution=0.1))
    om.insert_scan(ring, ring.push_scan(scans[0], nrm), poses[0])
    L = ls.lib()
    with pytest.raises(ls.LsError, match="rc=-4"):
        om.changes()
    rc, n, *_ = _raw_changes(om, 10, 0)
    assert rc == ls.LS_ERR_STATE and n == 0
    om.track_changes()
    base = _known(om)
    occ0 = base
    om.insert_scan(ring, ring.push_scan(scans[1], nrm), poses[1])
    after = _known(om)
    want = _with_centres(cr.diff_arrays(*base, *after, L_OCC), 0.1, 0.1)
    assert len(want[0]) > 2
    for cap in (0, 1, len(want[0]) - 1):
        rc, n, k, *_ = _raw_changes(om, cap, 1)
        assert rc == ls.LS_ERR_ARG and n == len(want[0]) and (cap == 0 or k[0] == 0)  # nothing copied, no reset
    assert L.ls_occupancy_changes(om._h, None, None, None, None, 10, None, 0, None) == ls.LS_ERR_ARG
    n = ctypes.c_int64(-1)
    assert L.ls_occupancy_changes(om._h, None, None, None, None, -1, ctypes.byref(n), 0, None) == ls.LS_ERR_ARG
    assert n.value == 0
    _same(om.changes(), want)  # the same set: the baseline is as it was
    rc, n, k, s, p, c = _raw_changes(om, len(want[0]), 0)
    assert rc == 0 and n == len(want[0])
    _same((k, s, p, c), want)
    k1, v1 = _known(om)
    assert np.array_equal(k1, after[0]) and np.array_equal(_bits(v1), _bits(after[1]))  # the map too
    # re-enabling takes a fresh baseline; disabling refuses again
    om.track_changes(True)
    assert all(len(a) == 0 for a in om.changes())
    om.track_changes(False)
    with pytest.raises(ls.LsError, match="rc=-4"):
        om.changes()
    assert len(occ0[0]) > 0
    om.close(), ring.close()


@pytest.mark.gpu
def test_calls_between_batch_begin_and_end(full_scans, keep):
    scans, poses = full_scans
    ctx = keep(ls.Context(0))
    ring = keep(ctx.create_map(4, 131072))
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(2)]
    om = keep(ls.OccupancyMap(ctx, resolution=0.1))
    om.insert_scan(ring, ids[0], poses[0])
    base = _known(om)
    end = ring.begin_batch([(ids[1], [ids[0]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[0]) @ poses[1])])
    try:  # the batch always ends, so a failed comparison cannot leave it open
        om.track_changes()
        om.insert_scan(ring, ids[1], poses[1])
        got = om.changes(reset=True)
        empty = om.changes()
    finally:
        end()
    _same(got, _with_centres(cr.diff_arrays(*base, *_known(om), L_OCC), 0.1, 0.1))
    assert len(got[0]) > 0 and len(empty[0]) == 0
    om.close(), ring.close(), ctx.close()


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
    hm = keep(host.OccupancyMap(est, resolution=0.1, max_range=15.0))
    assert hm.insert_laser_tracks() == 2 * n
    assert hm.num_changes() == 0 and len(hm.changed_points(10)[0]) == 0  # off: nothing, as octomap's empty set
    assert hm.reset_change_detection() is False
    path = str(tmp_path / "h.ot")
    hm.write_full(path)
    dev = keep(ls.OccupancyMap(gpu_ctx, resolution=0.1, max_range=15.0))
    dev.read_octomap_full(path)
    assert hm.enable_change_detection(True) is True
    dev.track_changes()
    p = truth[1][:3, 3]
    boxes = ([p, p + 0.5, p + (0, 2.0, 0)], [(3.0, 3.0, 1.0), (1.0, 1.0, 1.0), (2.0, 2.0, 2.0)], [True, False, True])
    hm.set_boxes(*boxes)
    dev.set_boxes(*boxes)
    want = dev.changes()
    assert len(want[0]) > 0 and (want[2] != UNK).any()
    m = hm.num_changes()
    assert m == len(want[0])
    _same(hm.changed_keys(), want[:3])
    pts, occ = hm.changed_points(m)
    assert np.array_equal(pts, want[3][:, :3].astype(np.float64)) and np.array_equal(occ, want[1] == OCC)
    assert hm.num_changes() == 0  # getChangedPoints reset
    assert hm.reset_change_detection() is True and hm.enable_change_detection(False) is False
    assert hm.num_changes() == 0
    hm.close(), dev.close(), est.close()
