"""The occupancy map's leaves as boxes (ls_occupancy_build_leaves / _download_leaves / _marker_cubes): volumetric_mapping's
getAllFreeBoxes / getAllOccupiedBoxes and generateMarkerArray's cube lists.  CPU: the reference (tests/leaf_boxes_ref.py)
tiles the known voxels, lies inside the .bt tree, matches hand-derived answers, and its region and colour rules match brute
force and hand values.  GPU: the device against the reference bit for bit, caching, invalidation, refusals and batches.
The rules are DESIGN.md §4b''''''''''''."""
import ctypes

import numpy as np
import pytest

import laser_slam_b200 as ls
import leaf_boxes_ref as lr
import octomap_full_ref as fr
from oracle import occupancy as oc
from oracle import octree as ot_oracle
from test_occupancy import F32, K0, _bits, full_scans  # noqa: F401  (full_scans: fixture)
from test_octomap import C, RES, block
from test_octomap_full import KA, V, W, _arrays, _load, _random_voxels, unpruned
from test_occupancy_collision import keep  # noqa: F401  (fixture)
from test_octomap_read import _download, _full_map, _same_downloads

L_OCC = oc.logodds(0.7)
L_MIN, L_MAX = oc.logodds(0.12), oc.logodds(0.97)


def _ref(vox, res=RES, l_occ=L_OCC):
    return lr.leaves(fr.full_octree(*_arrays(vox), res).payload, res, l_occ)


def _tiles(lv, keys, values, l_occ=L_OCC):
    """The leaves tile the known voxels: each voxel in exactly one leaf, of the voxel's state; volumes sum to the count."""
    assert int(sum(8 ** (16 - int(d)) for d in lv["depths"])) == len(keys)
    p = dict(keys=lv["keys"], depths=lv["depths"], values=lv["values"])
    ek, ev = fr.expand(p)
    assert np.array_equal(ek, np.sort(keys))  # sorted and equal: each voxel exactly once
    order = np.argsort(keys, kind="stable")
    assert np.array_equal(ev >= l_occ, values[order] >= l_occ)


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(KA))
def test_leaves_tile_the_known_answers(name):
    vox = KA[name][0]
    lv = _ref(vox)
    _tiles(lv, *_arrays(vox))


def test_leaves_tile_random_voxel_sets():
    rng = np.random.default_rng(7)
    for _ in range(200):
        vox = _random_voxels(rng, int(rng.integers(1, 12)))
        _tiles(_ref(vox), *_arrays(vox))


def test_leaves_tile_the_12_scan_map(full_scans):
    scans, poses = full_scans
    o = oc.OccupancyMap()
    for k in range(len(scans)):
        o.insert_scan(scans[k], poses[k])
    k, v = o.download()
    lv = _ref_kv(k, v, o.params["resolution"])
    _tiles(lv, k, v)
    assert len(lv["depths"]) > 100_000 and (lv["depths"] < 16).any()


def _ref_kv(k, v, res, l_occ=L_OCC):
    return lr.leaves(fr.full_octree(k, v, res).payload, res, l_occ)


def _bt_leaves(k, v, res, tmp_path, threshold=0.7):
    path = str(tmp_path / "t.bt")
    ot_oracle.octree(k, v, res, threshold).write(path)
    p = ls.read_octomap(path)
    return p["keys"], p["depths"], p["states"]


def _inside_bt(lv, bt):
    """Each value-pruned leaf lies inside exactly one .bt leaf of its state."""
    bk, bd, bs = bt
    state = {(int(d), int(x), int(y), int(z)): int(s) for (x, y, z), d, s in zip(bk, bd, bs)}
    bt_occ = {1: lr.CELL_FREE, 2: lr.CELL_OCCUPIED}  # the .bt bit pairs: 10 free, 01 occupied
    for k, d, s in zip(lv["keys"], lv["depths"], lv["states"]):
        hits = []
        for dd in range(1, int(d) + 1):
            sh = 16 - dd
            key = (dd, (int(k[0]) >> sh) << sh, (int(k[1]) >> sh) << sh, (int(k[2]) >> sh) << sh)
            if key in state:
                hits.append(state[key])
        assert len(hits) == 1 and bt_occ[hits[0]] == s


def test_the_bt_tree_is_never_finer(full_scans, tmp_path):
    rng = np.random.default_rng(3)
    sets = [KA[n][0] for n in sorted(KA) if KA[n][0]] + [_random_voxels(rng, 30) for _ in range(5)]
    for vox in sets:
        k, v = _arrays(vox)
        _inside_bt(_ref(vox), _bt_leaves(k, v, RES, tmp_path))
    scans, poses = full_scans
    o = oc.OccupancyMap()
    for j in range(4):
        o.insert_scan(scans[j], poses[j])
    k, v = o.download()
    lv = _ref_kv(k, v, o.params["resolution"])
    bt = _bt_leaves(k, v, o.params["resolution"], tmp_path)
    _inside_bt(lv, bt)
    assert len(lv["depths"]) > len(bt[1])  # finer here


def test_on_clamped_values_the_two_leaf_lists_are_equal(tmp_path):
    rng = np.random.default_rng(11)
    for _ in range(20):
        vox = {key: F32(L_MAX if val >= L_OCC else L_MIN) for key, val in _random_voxels(rng, 25).items()}
        k, v = _arrays(vox)
        lv = _ref(vox)
        bk, bd, bs = _bt_leaves(k, v, RES, tmp_path)
        assert np.array_equal(lv["keys"], bk) and np.array_equal(lv["depths"], bd)
        assert np.array_equal(lv["states"], np.where(bs == 2, lr.CELL_OCCUPIED, lr.CELL_FREE))


def test_hand_derived_answers():
    c = F32((0.5) * RES)
    lv = _ref({C: V})  # one voxel: one occupied leaf at depth 16, centred half a voxel above the origin
    assert lv["keys"].tolist() == [list(C)] and lv["depths"].tolist() == [16] and lv["states"].tolist() == [1]
    assert _bits(lv["centres"]).tolist() == [[_bits(c)] * 3] and lv["edges"].tolist() == [RES]
    lv = _ref({k: V for k in block(C, 8, 0)})  # a uniform brick collapses to depth 13
    assert lv["depths"].tolist() == [13] and lv["edges"].tolist() == [RES * 8]
    assert _bits(lv["centres"]).tolist() == [[_bits(F32(4 * RES))] * 3]
    # one voxel one ulp apart, same state: the .bt tree collapses the brick, the value-pruned tree keeps 7 + 7 + 8 leaves
    vox = {k: V for k in block(C, 8, 0)}
    vox[C] = W
    lv = _ref(vox)
    assert sorted(lv["depths"].tolist()) == [14] * 7 + [15] * 7 + [16] * 8 and (lv["states"] == 1).all()
    assert lv["depths"].tolist() == [16] * 8 + [15] * 7 + [14] * 7  # pre-order: the octet of C first
    bt = ot_oracle.octree(*_arrays(vox), RES)
    assert bt.nodes == 14  # root, 12 inner nodes, one leaf at depth 13
    # negative keys: the voxel below the origin on every axis
    lv = _ref({(K0 - 1, K0 - 1, K0 - 1): F32(-1.0)})
    assert _bits(lv["centres"]).tolist() == [[_bits(F32(-0.5 * RES))] * 3] and lv["states"].tolist() == [0]
    # the ends of the key range
    lv = _ref(KA["both_ends_of_the_key_space"][0])
    assert lv["keys"].tolist() == [[0, 0, 0], [65535] * 3] and lv["states"].tolist() == [1, 0]
    assert _bits(lv["centres"]).tolist() == [[_bits(F32(-32767.5 * RES))] * 3, [_bits(F32(32767.5 * RES))] * 3]


def _brute_region(lv, region, res):
    """The region rule by brute force: a leaf is listed iff one of its voxel keys lies in the clamped corner keys' box."""
    lo = [lr.corner_key(float(region[0][a]), res) for a in range(3)]
    hi = [lr.corner_key(float(region[1][a]), res) for a in range(3)]
    keep = []
    for k, d in zip(lv["keys"], lv["depths"]):
        side = 1 << (16 - int(d))
        keep.append(all(any(lo[a] <= int(k[a]) + j <= hi[a] for j in range(side)) for a in range(3)))
    return np.array(keep, bool)


REGION_RES = 0.125  # a power of two, so leaf faces are exact coordinates


def _regions():
    b = lambda k: (k - K0) * REGION_RES  # noqa: E731  the low face of key k
    return [
        ((b(K0), b(K0), b(K0)), (b(K0 + 8), b(K0 + 8), b(K0 + 8))),  # faces on brick boundaries: the far face keys K0 + 8
        ((b(K0 + 8) - 1e-9, b(K0), b(K0)), (b(K0 + 8) - 1e-9, b(K0 + 2), b(K0 + 1))),  # just below a boundary
        ((b(K0 - 16), b(K0 - 16), b(K0 - 16)), (b(K0 - 16), b(K0 - 16), b(K0 - 16))),  # one point
        ((-1e9, -1e9, -1e9), (1e9, 1e9, 1e9)),  # corners outside the key range clamp: everything
        ((-1e9, b(K0 + 3), -1e9), (b(K0 - 40), 1e9, 1e9)),
        ((1e9, 1e9, 1e9), (2e9, 2e9, 2e9)),  # clamps to key 65535
    ]


def test_region_rule_against_brute_force():
    rng = np.random.default_rng(5)
    sets = [_random_voxels(rng, 40) for _ in range(4)] + [KA["both_ends_of_the_key_space"][0]]
    for vox in sets:
        lv = _ref(vox, REGION_RES)
        for region in _regions():
            sel = lr.select(lv, region, REGION_RES)
            want = _brute_region(lv, region, REGION_RES)
            assert np.array_equal(sel["keys"], lv["keys"][want]) and np.array_equal(sel["depths"], lv["depths"][want])
    lv = _ref(KA["both_ends_of_the_key_space"][0], REGION_RES)
    assert len(lr.select(lv, _regions()[3], REGION_RES)["keys"]) == 2
    assert lr.select(lv, _regions()[5], REGION_RES)["keys"].tolist() == [[65535] * 3]
    assert lr.corner_key(-1e9, REGION_RES) == 0 and lr.corner_key(REGION_RES * 8, REGION_RES) == K0 + 8


def test_height_map_color_by_hand():
    want = [(1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 1, 1), (0, 0, 1), (1, 0, 1), (1, 0, 0)]
    for k in range(7):
        h = k / 6
        assert h * 6 == k  # precondition: each sector boundary is hit exactly
        assert lr.height_map_color(h) == tuple(F32(x) for x in want[k]) + (F32(1),)
    assert lr.height_map_color(0.8) == (F32(0.8), F32(0), F32(1), F32(1))
    # z below min_z, at min_z, at max_z and above it; color_factor 0.8
    assert lr.cube_color(-5.0, -1.0, 3.0, 0.8) == lr.cube_color(-1.0, -1.0, 3.0, 0.8) == lr.height_map_color(0.8)
    assert lr.cube_color(3.0, -1.0, 3.0, 0.8) == lr.cube_color(9.0, -1.0, 3.0, 0.8) == (F32(1), F32(0), F32(0), F32(1))


# ---- GPU ------------------------------------------------------------------------------------------------------------
L = ls.lib
MARK = (-1.0, 3.0, 0.8)


def _same(dev, lv, region=None, res=None):
    """Every output of the device's listing equals the reference's: leaves per `which`, stats and marker cubes."""
    res = dev.params.resolution if res is None else res
    want = lr.select(lv, region, res)
    st = dev.build_leaves(region)
    cen, dep, sta = dev.download_leaves(ls.LEAVES_ALL)
    assert np.array_equal(_bits(cen[:, :3]), _bits(want["centres"])) and (cen[:, 3] == 1).all()
    assert np.array_equal(dep, want["depths"]) and np.array_equal(sta, want["states"])
    for which, s in ((ls.LEAVES_FREE, lr.CELL_FREE), (ls.LEAVES_OCCUPIED, lr.CELL_OCCUPIED)):
        c, d, t = dev.download_leaves(which)
        sel = want["states"] == s
        assert np.array_equal(_bits(c[:, :3]), _bits(want["centres"][sel])) and np.array_equal(d, want["depths"][sel])
        assert (t == s).all()
    for d in range(17):
        assert st.occupied_by_depth[d] == int(((want["depths"] == d) & (want["states"] == 1)).sum())
        assert st.free_by_depth[d] == int(((want["depths"] == d) & (want["states"] == 0)).sum())
    lists, colors = lr.marker_cubes(want, *MARK)
    m = dev.marker_cubes(*MARK, region=region)
    got_colors = np.concatenate([c.colors for c in m.occupied])
    assert np.array_equal(_bits(got_colors), _bits(colors))
    for part in ("occupied", "free"):
        for d in range(17):
            cl = getattr(m, part)[d]
            assert cl.size == res * 2.0 ** (16 - d)
            assert np.array_equal(_bits(cl.points), _bits(want["centres"][lists[part][d]].reshape(-1, 3)))
    return len(want["depths"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(KA))
def test_known_answers_on_the_device(gpu_ctx, name):
    vox = KA[name][0]
    dev = _load(gpu_ctx, vox)
    assert _same(dev, _ref(vox)) == len(_ref(vox)["depths"])
    b = lambda k: (k - K0) * RES  # noqa: E731
    _same(dev, _ref(vox), ((b(K0), b(K0), b(K0)), (b(K0 + 1), b(K0), b(K0))))
    dev.close()


@pytest.mark.gpu
def test_random_voxel_sets_and_regions_on_the_device(gpu_ctx):
    rng = np.random.default_rng(21)
    for _ in range(6):
        vox = _random_voxels(rng, 60)
        dev = ls.OccupancyMap(gpu_ctx, resolution=REGION_RES)
        dev.read_full_octree(unpruned(vox)[1], unpruned(vox)[0], REGION_RES)
        lv = _ref(vox, REGION_RES)
        for region in [None] + _regions():
            _same(dev, lv, region)
        dev.close()


def _three_regions(dev):
    lo, hi = dev.bounds()
    mid = (lo + hi) / 2
    return [(lo, mid), (mid - 2.0, mid + 2.0), ((mid[0], lo[1] - 5, -1e9), (hi[0] + 1, mid[1], 1e9))]


@pytest.mark.gpu
@pytest.mark.parametrize("params", [dict(), dict(resolution=0.1, max_range=-1.0)], ids=["defaults", "res0.1_unlimited"])
def test_the_12_scan_maps_equal_the_reference(gpu_ctx, full_scans, params):
    scans, _ = full_scans
    dev, ring = _full_map(gpu_ctx, full_scans, params, len(scans))
    k, v, _ = dev.download(ls.OCC_KNOWN)
    res = dev.params.resolution
    lv = _ref_kv(k, v, res)
    assert _same(dev, lv) > 100_000
    for region in _three_regions(dev):
        assert 0 < _same(dev, lv, region) < len(lv["depths"])
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_edits_reads_empty_and_growth(gpu_ctx, full_scans, tmp_path):
    scans, poses = full_scans
    dev, ring = _full_map(gpu_ctx, full_scans, dict(initial_capacity=16), 4)  # grows from 16 bricks
    res = dev.params.resolution
    lo, hi = dev.bounds()
    mid = (lo + hi) / 2
    dev.set_boxes([mid, mid + 1.0, lo + 0.5], [[2.0, 2.0, 1.0], [0.6, 0.6, 0.6], [1.0, 0.3, 2.0]], [1, 0, 1])
    k, v, _ = dev.download(ls.OCC_KNOWN)
    _same(dev, _ref_kv(k, v, res))
    # a .bt read: the list equals the .bt tree's leaves
    bt = str(tmp_path / "m.bt")
    dev.save_octomap(bt)
    back = ls.OccupancyMap(gpu_ctx)
    back.read_octomap(bt)
    k, v, _ = back.download(ls.OCC_KNOWN)
    _same(back, _ref_kv(k, v, res))
    p = ls.read_octomap(bt)
    cen, dep, sta = back.download_leaves(ls.LEAVES_ALL)
    assert np.array_equal(dep, p["depths"]) and np.array_equal(sta, np.where(p["states"] == 2, 1, 0))
    assert np.array_equal(_bits(cen[:, :3]), _bits(ls.leaf_centres(p["keys"], p["depths"], res)))
    # a .ot read at a foreign resolution
    vox = _random_voxels(np.random.default_rng(2), 50)
    size, payload = unpruned(vox)
    back.read_full_octree(payload, size, 0.3)
    _same(back, _ref(vox, 0.3))
    # empty: a new map, and a map after clear
    empty = ls.OccupancyMap(gpu_ctx)
    assert _same(empty, _ref({})) == 0
    back.clear()
    assert _same(back, _ref({})) == 0
    for m in (dev, back, empty):
        m.close()
    ring.close()


def _leaf_call(dev, which=ls.LEAVES_ALL):
    """The count-only download: (LS_ERR_ARG, the count) while the list is current, (LS_ERR_STATE, 0) after a change."""
    n = ctypes.c_int64(-1)
    rc = L().ls_occupancy_download_leaves(dev._h, which, None, None, None, 0, ctypes.byref(n))
    return rc, n.value


@pytest.mark.gpu
def test_listing_changes_nothing_and_an_insert_invalidates(gpu_ctx, full_scans):
    scans, poses = full_scans
    dev, ring = _full_map(gpu_ctx, full_scans, dict(), 3)
    before = _download(dev)
    t, ft = dev.octree(), dev.full_octree()
    launches = gpu_ctx.launch_count
    dev.build_leaves()
    dev.marker_cubes(*MARK)
    dev.build_leaves(_three_regions(dev)[1])
    # both cached builds are still current: their downloads need no rebuild
    pay = np.empty(max(len(t.payload), 1), np.uint8)
    assert L().ls_occupancy_download_octree(dev._h, pay.ctypes.data, len(t.payload), None, None, 0) == 0
    assert pay[:len(t.payload)].tobytes() == t.payload
    fpay = np.empty(max(len(ft.payload), 1), np.uint8)
    assert L().ls_occupancy_download_full_octree(dev._h, fpay.ctypes.data, len(ft.payload)) == 0
    assert fpay[:len(ft.payload)].tobytes() == ft.payload
    assert gpu_ctx.launch_count > launches
    assert _same_downloads(_download(dev), before)
    assert dev.octree().payload == t.payload and dev.full_octree().payload == ft.payload
    assert _leaf_call(dev)[0] == ls.LS_ERR_ARG and _leaf_call(dev)[1] > 0
    nrm = np.zeros((131072, 3), F32)
    dev.insert_scan(ring, ring.push_scan(scans[3], nrm), poses[3])
    assert _leaf_call(dev)[0] == ls.LS_ERR_STATE
    off = np.zeros(18, np.int64)
    n = ctypes.c_int64(0)
    assert L().ls_occupancy_marker_cubes(dev._h, *MARK, None, None, off.ctypes.data, off.ctypes.data, 0,
                                         ctypes.byref(n)) == ls.LS_ERR_STATE
    for change in (lambda: dev.set_free([0.0, 0.0, 0.0], [1.0, 1.0, 1.0]), dev.clear):
        dev.build_leaves()
        assert _leaf_call(dev)[0] == ls.LS_ERR_ARG
        change()
        assert _leaf_call(dev)[0] == ls.LS_ERR_STATE
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_refusals_leave_everything_unchanged(gpu_ctx, full_scans):
    dev, ring = _full_map(gpu_ctx, full_scans, dict(), 3)
    before = _download(dev)
    t, ft = dev.octree(), dev.full_octree()
    region = _three_regions(dev)[1]
    dev.build_leaves(region)
    listed = dev.download_leaves()
    nan, inf = float("nan"), float("inf")
    lo = np.zeros(3)
    bad_regions = [(np.array([nan, 0, 0]), np.ones(3)), (lo, np.array([1, inf, 1])), (np.ones(3), np.zeros(3))]
    for r in bad_regions:
        lo_, hi_ = (np.ascontiguousarray(x, np.float64) for x in r)
        assert L().ls_occupancy_build_leaves(dev._h, lo_.ctypes.data, hi_.ctypes.data, None) == ls.LS_ERR_ARG
    assert L().ls_occupancy_build_leaves(dev._h, lo.ctypes.data, None, None) == ls.LS_ERR_ARG
    n = ctypes.c_int64(0)
    m = len(listed[1])
    buf = np.empty((m, 4), np.float32)
    dep, sta = np.empty(m, np.uint8), np.empty(m, np.int8)
    assert L().ls_occupancy_download_leaves(dev._h, 3, None, dep.ctypes.data, sta.ctypes.data, m, ctypes.byref(n)) == ls.LS_ERR_ARG
    assert L().ls_occupancy_download_leaves(dev._h, 4, buf.ctypes.data, dep.ctypes.data, sta.ctypes.data, m,
                                            ctypes.byref(n)) == ls.LS_ERR_ARG
    assert L().ls_occupancy_download_leaves(dev._h, 3, buf.ctypes.data, dep.ctypes.data, sta.ctypes.data, m - 1,
                                            ctypes.byref(n)) == ls.LS_ERR_ARG and n.value == m
    off = np.zeros(18, np.int64)
    for args in ((nan, 1.0, 0.8), (0.0, inf, 0.8), (1.0, 1.0, 0.8), (2.0, 1.0, 0.8), (0.0, 1.0, nan), (-1e308, 1e308, 0.8)):
        assert L().ls_occupancy_marker_cubes(dev._h, *args, None, None, off.ctypes.data, off.ctypes.data, 0,
                                             ctypes.byref(n)) == ls.LS_ERR_ARG
    assert L().ls_occupancy_marker_cubes(dev._h, *MARK, buf.ctypes.data, buf.ctypes.data, off.ctypes.data,
                                         off.ctypes.data, m - 1, ctypes.byref(n)) == ls.LS_ERR_ARG and n.value == m
    after = dev.download_leaves()
    assert all(np.array_equal(_bits(a) if a.dtype == np.float32 else a, _bits(b) if b.dtype == np.float32 else b)
               for a, b in zip(after, listed))
    assert _same_downloads(_download(dev), before)
    assert dev.octree().payload == t.payload and dev.full_octree().payload == ft.payload
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_leaf_calls_between_batch_begin_and_end(full_scans):
    scans, poses = full_scans
    ctx = ls.Context(0)
    ring = ctx.create_map(16, 131072)
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(4)]
    problems = [(ids[k + 1], [ids[k]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[k]) @ poses[k + 1]) for k in range(3)]
    p = ls.default_params(max_iterations=5)
    alone = ring.register_batch(problems, p)
    dev = ls.OccupancyMap(ctx)
    dev.insert_scan(ring, ids[0], poses[0])
    k, v, _ = dev.download(ls.OCC_KNOWN)
    lv = _ref_kv(k, v, dev.params.resolution)
    end = ring.begin_batch(problems, p)
    boxes = dev.leaf_boxes(ls.LEAVES_ALL)
    cubes = dev.marker_cubes(*MARK)
    res = end()
    for a, b in zip(res, alone):
        assert a["rc"] == b["rc"] and np.array_equal(a["T"], b["T"])
    assert np.array_equal(_bits(boxes.centres), _bits(lv["centres"])) and np.array_equal(boxes.depths, lv["depths"])
    assert sum(len(c.points) for c in cubes.occupied + cubes.free) == len(lv["depths"])
    dev.close()
    ring.close()
    ctx.close()


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
    hm = keep(host.OccupancyMap(est, resolution=0.1, max_range=15.0))
    assert hm.insert_laser_tracks() == 2 * n
    hm.write_full(path)
    dev = keep(ls.OccupancyMap(gpu_ctx, resolution=0.1, max_range=15.0))
    dev.read_octomap_full(path)
    lo, hi = dev.bounds()
    region = (lo + 1.0, (lo + hi) / 2)
    for r in (None, region):
        for which, occupied in ((ls.LEAVES_FREE, False), (ls.LEAVES_OCCUPIED, True)):
            want = dev.leaf_boxes(which, r)
            c, e = hm.boxes(occupied, r)
            assert len(c) > 0 and np.array_equal(c, want.centres.astype(np.float64)) and np.array_equal(e, want.edges)
    want = dev.marker_cubes(*MARK)
    occ, free = hm.marker_array(*MARK)
    for got, ref in ((occ, want.occupied), (free, want.free)):
        for (size, pts, rgba), cl in zip(got, ref):
            assert size == cl.size and np.array_equal(pts, cl.points.astype(np.float64))
            assert np.array_equal(_bits(rgba), _bits(cl.colors))
    with pytest.raises(ls.LsError):
        hm.marker_array(1.0, 1.0)
    with pytest.raises(ls.LsError):
        hm.boxes(True, ((1.0, 0, 0), (0.0, 0, 0)))
    one = np.zeros(3)
    assert host.lib().lsh_occupancy_boxes(hm._h, 1, one.ctypes.data, None, None, None, 0) == ls.LS_ERR_STATE
    assert "both corners" in host.lib().lsh_occupancy_last_error(hm._h).decode()
    hm.close()
    dev.close(), est.close()


def test_product_never_imports_the_reference():
    """tests/leaf_boxes_ref.py is test infrastructure: nothing under laser_slam_b200/ may reference it."""
    import os
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "laser_slam_b200")
    for d, _, files in os.walk(root):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".hpp")):
                assert "leaf_boxes_ref" not in open(os.path.join(d, f), errors="replace").read(), f
