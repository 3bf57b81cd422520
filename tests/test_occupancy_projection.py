"""The occupancy map projected onto octomap_server's 2D occupancy grid (ls_occupancy_build_projection /
_download_projection) and saved as map_saver saves it.  CPU: the reference (tests/projected_map_ref.py) equals an
independent per-voxel projection, hand-derived answers, the grid geometry and the map_saver bytes.  GPU: the device
against the reference bit for bit, caching, invalidation, refusals and batches.  The rules are DESIGN.md
§4b'''''''''''''."""
import ctypes
import math

import numpy as np
import pytest

import laser_slam_b200 as ls
import projected_map_ref as pr
from oracle import occupancy as oc
from oracle import octree as ot_oracle
from test_octomap import block
from test_octomap_full import _arrays, unpruned

K0 = 32768
F32 = np.float32
RES = 0.125  # a power of two: every face below is an exact coordinate
V = F32(oc.logodds(0.9))  # occupied (>= L_occ = logodds(0.7))
FREE = F32(-V)
INF = math.inf
N_SCANS = 12


@pytest.fixture(scope="module")
def scans12(synth_mod):
    truth, _ = synth_mod.trajectory(0, N_SCANS)
    return [synth_mod.scan(truth[k], 0, k)[0] for k in range(N_SCANS)], [truth[k].astype(F32) for k in range(N_SCANS)]


def _bt(vox, res=RES):
    """The .bt leaves of a voxel set {key: float32 log-odds}, from the oracle's writeBinary payload."""
    if not vox:
        return pr.bt_leaves(b"")
    return pr.bt_leaves(ot_oracle.octree(*_arrays(vox), res).payload)


def _project(vox, res=RES, **band):
    return pr.project(_bt(vox, res), res, **band)


def _unpack(keys):
    k = np.asarray(keys, np.uint64)
    return np.stack([(k >> np.uint64(16 * a)) & np.uint64(0xFFFF) for a in range(3)], 1).astype(np.int64)


def _independent(keys3, occupied, res, band):
    """The per-voxel projection with its own geometry: the padded key range is the known keys' [min, max + 1], widened to
    key 32768 (the padded corners with no minimum size)."""
    kmin = [min(int(keys3[:, a].min()), K0) for a in range(2)]
    kmax = [max(int(keys3[:, a].max()) + 1, K0) for a in range(2)]
    shape = (kmax[1] - kmin[1] + 1, kmax[0] - kmin[0] + 1)
    return pr.per_voxel(keys3, occupied, res, band[0], band[1], kmin, shape), kmin


def _random_set(rng, n_blocks):
    vox = {}
    for _ in range(n_blocks):
        n = int(rng.choice([1, 2, 4, 8, 16]))
        k0 = tuple(int(x) // n * n for x in rng.integers(K0 - 60, K0 + 60, 3))
        value = V if rng.random() < 0.4 else FREE
        for k in block(k0, n, 0):
            vox[k] = value
    return vox


# bands whose edges are not voxel faces at RES (faces are multiples of 0.125)
BANDS = [(-INF, INF), (-0.3, 0.7), (0.01, 2.2), (-3.1, -0.4), (5.06, 1.01)]


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_reference_equals_the_per_voxel_projection_on_random_sets():
    rng = np.random.default_rng(11)
    for _ in range(60):
        vox = _random_set(rng, int(rng.integers(1, 10)))
        keys3 = np.array(list(vox), np.int64)
        occ = np.array([vox[k] >= F32(oc.logodds(0.7)) for k in vox])
        for band in BANDS:
            grid, info = _project(vox, min_z=band[0], max_z=band[1])
            want, kmin = _independent(keys3, occ, RES, band)
            assert np.array_equal(grid, want)
            assert info["origin_x"] == (kmin[0] - K0) * RES and info["origin_y"] == (kmin[1] - K0) * RES


def test_reference_equals_the_per_voxel_projection_on_the_12_scan_map(scans12):
    scans, poses = scans12
    o = oc.OccupancyMap(resolution=RES)
    for k in range(len(scans)):
        o.insert_scan(scans[k], poses[k])
    k, v = o.download()
    leaves = pr.bt_leaves(ot_oracle.octree(k, v, RES).payload)
    assert len(leaves[1]) > 10_000 and (leaves[1] < 16).any()
    keys3 = _unpack(k)
    occ = v >= F32(oc.logodds(0.7))
    for band in [(-INF, INF), (0.3, 2.0), (-1.01, 0.33)]:
        grid, info = pr.project(leaves, RES, *band)
        want, _ = _independent(keys3, occ, RES, band)
        assert np.array_equal(grid, want)
        assert info["free"] > 0 and info["occupied"] > 0


def test_hand_derived_answers():
    # one occupied voxel at key (K0 + 2, K0 + 3, K0): x [0.25, 0.375], y [0.375, 0.5]; the padded corners reach key K0
    # (min(0.25, -0.0) = -0.0), so the grid is 4 x 5 from key K0 and the voxel is cell (2, 3)
    grid, info = _project({(K0 + 2, K0 + 3, K0): V})
    want = np.full((5, 4), -1, np.int8)
    want[3, 2] = 100
    assert np.array_equal(grid, want)
    assert (info["width"], info["height"], info["origin_x"], info["origin_y"]) == (4, 5, 0.0, 0.0)
    assert (info["unknown"], info["free"], info["occupied"]) == (19, 0, 1)
    # a free depth-13 leaf (an 8^3 block at x key K0 + 8) paints its 8 x 8 square; x to key K0 + 16 (its far face)
    coarse = {k: FREE for k in block((K0 + 8, K0, K0), 8, 0)}
    grid, info = _project(coarse)
    want = np.full((9, 17), -1, np.int8)
    want[0:8, 8:16] = 0
    assert np.array_equal(grid, want) and _bt(coarse)[1].tolist() == [13]
    # occupied over free in one column, whichever comes first in the leaf order
    for zf, zo in ((K0, K0 + 5), (K0 + 5, K0)):
        grid, _ = _project({(K0 + 1, K0 + 1, zf): FREE, (K0 + 1, K0 + 1, zo): V, (K0 + 2, K0 + 1, zf): FREE})
        assert grid[1, 1] == 100 and grid[1, 2] == 0
    # a band that excludes everything keeps the geometry
    g_all, i_all = _project({(K0 + 2, K0 + 3, K0): V})
    grid, info = _project({(K0 + 2, K0 + 3, K0): V}, min_z=10.0, max_z=20.0)
    assert (grid == -1).all() and grid.shape == g_all.shape and info["origin_x"] == i_all["origin_x"]
    # band edges exactly on the voxel's faces (z in [0, 0.125]): strict comparisons exclude a band touching one face
    one = {(K0, K0, K0): V}
    assert _project(one, min_z=0.125)[0].max() == -1 and _project(one, max_z=0.0)[0].max() == -1
    assert _project(one, min_z=0.0, max_z=0.125)[0].max() == 100
    # an inverted band still takes a leaf that spans it, and nothing when it lies above the leaf
    assert _project(one, min_z=0.124, max_z=0.001)[0].max() == 100 and _project(one, min_z=0.2, max_z=0.15)[0].max() == -1
    # padding larger than the map: 10 m in x is keys K0 - 40 ... K0 + 40
    grid, info = _project({(K0 + 2, K0 + 3, K0): V}, min_size_x=10.0)
    assert (info["width"], info["height"], info["origin_x"]) == (81, 5, -5.0) and grid[3, 42] == 100
    # negative coordinates: x [-1, -0.875], y [-2.25, -2.125]; the far corners reach key K0
    grid, info = _project({(K0 - 8, K0 - 18, K0 - 3): FREE})
    assert (info["width"], info["height"], info["origin_x"], info["origin_y"]) == (9, 19, -1.0, -2.25)
    assert grid[0, 0] == 0 and (grid == 0).sum() == 1
    # the empty map
    grid, info = _project({})
    assert grid.shape == (0, 0) and info["width"] == info["height"] == 0


def test_refusals():
    one = {(K0, K0, K0): V}
    for kw in (dict(min_z=math.nan), dict(max_z=math.nan), dict(min_size_x=-1.0), dict(min_size_y=math.nan),
               dict(min_size_x=INF), dict(min_size_x=1e6)):  # 1e6 m: a padded corner outside the key space
        with pytest.raises(pr.Refused):
            _project(one, **kw)
    with pytest.raises(pr.Refused):  # the far face of key 65535 has no key
        _project({(65535, K0, K0): V})
    with pytest.raises(pr.Refused):  # 65536 x 65536 cells
        _project({(0, 0, K0): V, (65534, 65534, K0): FREE})


def test_cell_centres_are_key_centres():
    # paddedMinKey by hand: min(0.25, -0.0) keys to K0; y min(-2.25, -1.5) = -2.25; x min(12.5, -0.65) = -0.65, keyed as
    # floor(-5.2) = -6
    for vox, kw, kmin in (({(K0 + 2, K0 + 3, K0): V}, {}, (K0, K0)),
                          ({(K0 - 8, K0 - 18, K0): FREE}, dict(min_size_y=3.0), (K0 - 8, K0 - 18)),
                          ({(K0 + 100, K0 - 7, K0): V}, dict(min_size_x=1.3), (K0 - 6, K0 - 7))):
        grid, info = pr.project(_bt(vox), RES, **kw)
        for i, j in ((0, 0), (info["width"] - 1, info["height"] - 1), (info["width"] // 2, 1)):
            assert info["origin_x"] + (i + 0.5) * RES == pr.centre(kmin[0] + i, 16, RES)
            assert info["origin_y"] + (j + 0.5) * RES == pr.centre(kmin[1] + j, 16, RES)


def test_map_saver_files_by_hand(tmp_path):
    grid = np.array([[0, 100, -1], [-1, 0, 100]], np.int8)
    stem = str(tmp_path / "m")
    ls.save_map(stem, grid, 0.125, -1.5, 2.25)
    pgm = b"P5\n# CREATOR: map_saver.cpp 0.125 m/pix\n3 2\n255\n" + bytes([205, 254, 0, 254, 0, 205])
    yaml = (f"image: {stem}.pgm\nresolution: 0.125000\norigin: [-1.500000, 2.250000, 0.000000]\nnegate: 0\n"
            "occupied_thresh: 0.65\nfree_thresh: 0.196\n\n")
    assert open(stem + ".pgm", "rb").read() == pgm
    assert open(stem + ".yaml").read() == yaml
    assert pr.map_saver_bytes(grid, 0.125, -1.5, 2.25, stem + ".pgm") == (pgm, yaml)
    # the resolution is the message's float32: 0.05 prints from 0.0500000007
    ls.save_map(stem, grid[:1, :1], 0.05, 0.0, -0.0)
    assert open(stem + ".pgm", "rb").read() == b"P5\n# CREATOR: map_saver.cpp 0.050 m/pix\n1 1\n255\n\xfe"
    assert "resolution: 0.050000\norigin: [0.000000, -0.000000, 0.000000]\n" in open(stem + ".yaml").read()


# ---- GPU ------------------------------------------------------------------------------------------------------------
L = ls.lib


def _load(ctx, vox, res=RES, **kw):
    dev = ls.OccupancyMap(ctx, resolution=res, **kw)
    if vox:
        size, payload = unpruned(vox)
        dev.read_full_octree(payload, size, res)
    return dev


def _same(dev, **band):
    """The device projection (the .bt build not cached when the map just changed) equals the reference over the device's
    .bt tree, bit for bit; returns the grid."""
    grid, info = dev.projected_map(**band)
    res = dev.params.resolution
    try:
        want, w = pr.project(pr.bt_leaves(dev.octree().payload), res, **band)
    except pr.Refused:
        raise AssertionError("the reference refuses what the device accepted")
    assert grid.dtype == np.int8 and np.array_equal(grid, want)
    assert (info.width, info.height, info.unknown_cells, info.free_cells, info.occupied_cells) == (
        w["width"], w["height"], w["unknown"], w["free"], w["occupied"])
    assert info.resolution == res and info.origin_x == w["origin_x"] and info.origin_y == w["origin_y"]
    return grid


HAND = {
    "one_voxel": ({(K0 + 2, K0 + 3, K0): V}, {}),
    "free_coarse_leaf": ({k: FREE for k in block((K0 + 8, K0, K0), 8, 0)}, {}),
    "occupied_over_free": ({(K0 + 1, K0 + 1, K0): FREE, (K0 + 1, K0 + 1, K0 + 5): V, (K0 + 2, K0 + 1, K0): FREE}, {}),
    "band_excludes_all": ({(K0 + 2, K0 + 3, K0): V}, dict(min_z=10.0, max_z=20.0)),
    "band_on_faces_out": ({(K0, K0, K0): V}, dict(min_z=0.125)),
    "band_on_faces_in": ({(K0, K0, K0): V}, dict(min_z=0.0, max_z=0.125)),
    "padding": ({(K0 + 2, K0 + 3, K0): V}, dict(min_size_x=10.0, min_size_y=0.3)),
    "negative": ({(K0 - 8, K0 - 18, K0 - 3): FREE}, {}),
    "empty": ({}, {}),
    "coarse_free_wide": ({k: FREE for k in block((K0 - 64, K0 - 32, K0), 32, 0)}, dict(min_size_x=40.0)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(HAND))
def test_hand_cases_on_the_device(gpu_ctx, name):
    vox, band = HAND[name]
    dev = _load(gpu_ctx, vox)
    want = _project(vox, **band)[0]
    assert np.array_equal(_same(dev, **band), want)
    dev.close()


@pytest.mark.gpu
def test_random_sets_on_the_device(gpu_ctx):
    rng = np.random.default_rng(5)
    for t in range(25):
        vox = _random_set(rng, int(rng.integers(1, 14)))
        dev = _load(gpu_ctx, vox, res=[RES, 0.1, 0.05][t % 3])
        for band in BANDS[:3]:
            _same(dev, min_z=band[0], max_z=band[1], min_size_x=float(rng.choice([0.0, 3.3])))
        dev.close()


def _scan_map(ctx, scans12, params, n=N_SCANS):
    scans, poses = scans12
    ring = ctx.create_map(2, 131072)
    dev = ls.OccupancyMap(ctx, **params)
    nrm = np.zeros((131072, 3), F32)
    for k in range(n):
        dev.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
    return dev, ring


@pytest.mark.gpu
@pytest.mark.parametrize("params", [dict(), dict(resolution=0.1, max_range=-1.0)], ids=["defaults", "res0.1_unlimited"])
def test_the_12_scan_maps_equal_the_reference(gpu_ctx, scans12, params):
    dev, ring = _scan_map(gpu_ctx, scans12, params)
    for band in [dict(), dict(min_z=0.3, max_z=2.0), dict(min_z=-1.0, max_z=0.5), dict(min_size_x=250.0, min_size_y=90.0)]:
        g = _same(dev, **band)
        assert (g == 0).any() and (g == 100).any()
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_edits_reads_and_growth(gpu_ctx, scans12, tmp_path):
    dev, ring = _scan_map(gpu_ctx, scans12, dict(initial_capacity=16), 4)  # grows from 16 bricks
    _same(dev)
    lo, hi = dev.bounds()
    mid = (lo + hi) / 2
    dev.set_free([mid, lo + 0.5], [[6.0, 4.0, 1.0], [1.0, 0.3, 2.0]])
    _same(dev, min_z=0.3, max_z=2.0)
    dev.set_occupied([mid + 1.0], [[0.6, 0.6, 0.6]])
    _same(dev)
    bt = str(tmp_path / "m.bt")
    dev.save_octomap(bt)
    back = ls.OccupancyMap(gpu_ctx)
    back.read_octomap(bt)
    g = _same(back)
    assert np.array_equal(g, dev.projected_map()[0])  # the .bt tree of a map read from it is the same tree
    size, payload = unpruned(_random_set(np.random.default_rng(3), 30))
    back.read_full_octree(payload, size, 0.3)  # a foreign resolution
    _same(back, min_z=-1.0, max_z=4.0)
    back.clear()
    assert _same(back).shape == (0, 0)
    dev.close(), back.close(), ring.close()


def _download_rc(dev, cap=0):
    buf = np.empty(max(cap, 1), np.int8)
    return L().ls_occupancy_download_projection(dev._h, buf.ctypes.data, cap)


@pytest.mark.gpu
def test_projecting_changes_nothing_and_changes_invalidate(gpu_ctx, scans12):
    scans, poses = scans12
    dev, ring = _scan_map(gpu_ctx, scans12, dict(), 3)
    known = [dev.download(w) for w in (ls.OCC_KNOWN, ls.OCC_OCCUPIED)]
    t, ft = dev.octree(), dev.full_octree()
    leaves = dev.leaf_boxes()
    grid, info = dev.projected_map(min_z=0.3, max_z=2.0)
    assert info.width * info.height == grid.size > 0
    for a, b in zip([dev.download(w) for w in (ls.OCC_KNOWN, ls.OCC_OCCUPIED)], known):
        assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
    pay = np.empty(len(t.payload), np.uint8)
    assert L().ls_occupancy_download_octree(dev._h, pay.ctypes.data, len(t.payload), None, None, 0) == 0
    assert pay.tobytes() == t.payload
    fpay = np.empty(len(ft.payload), np.uint8)
    assert L().ls_occupancy_download_full_octree(dev._h, fpay.ctypes.data, len(ft.payload)) == 0
    assert fpay.tobytes() == ft.payload
    cen, dep, st = dev.download_leaves()  # the leaf list is still current and unchanged
    assert np.array_equal(cen[:, :3].view(np.uint32), leaves.centres.view(np.uint32)) and np.array_equal(dep, leaves.depths)
    assert _download_rc(dev, grid.size) == 0 and _download_rc(dev, grid.size - 1) == ls.LS_ERR_ARG
    nrm = np.zeros((131072, 3), F32)
    one = unpruned({(K0, K0, K0): V})
    changes = [lambda: dev.insert_scan(ring, ring.push_scan(scans[3], nrm), poses[3]),
               lambda: dev.set_free([0.0, 0.0, 0.0], [1.0, 1.0, 1.0]),
               lambda: dev.read_full_octree(one[1], one[0], 0.1), dev.clear]
    for change in changes:
        g, i = dev.projected_map()
        assert _download_rc(dev, g.size) == 0
        change()
        assert _download_rc(dev, max(g.size, 1)) == ls.LS_ERR_STATE
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_refusals_leave_everything_unchanged(gpu_ctx, scans12):
    dev, ring = _scan_map(gpu_ctx, scans12, dict(), 3)
    t, ft = dev.octree(), dev.full_octree()
    leaves = dev.leaf_boxes()
    known = dev.download(ls.OCC_KNOWN)
    grid, info = dev.projected_map(min_z=0.3, max_z=2.0)
    nan = math.nan
    g = ls.GridInfo()
    for args in ((nan, 1.0, 0.0, 0.0), (0.0, nan, 0.0, 0.0), (-INF, INF, -1.0, 0.0), (-INF, INF, 0.0, nan),
                 (-INF, INF, INF, 0.0), (-INF, INF, 1e7, 0.0)):
        assert L().ls_occupancy_build_projection(dev._h, *args, ctypes.byref(g)) == ls.LS_ERR_ARG
    assert L().ls_occupancy_build_projection(dev._h, 0.0, 1.0, 0.0, 0.0, None) == ls.LS_ERR_ARG
    out = np.empty(grid.size, np.int8)
    assert L().ls_occupancy_download_projection(dev._h, out.ctypes.data, grid.size) == 0
    assert np.array_equal(out.reshape(grid.shape), grid)  # the last projection survives the refusals
    assert dev.octree().payload == t.payload and dev.full_octree().payload == ft.payload
    assert np.array_equal(dev.download(ls.OCC_KNOWN)[0], known[0])
    cen, dep, _ = dev.download_leaves()
    assert np.array_equal(dep, leaves.depths)
    # a grid over 2^31 - 1 cells: voxels at both ends of the key space
    far = _load(gpu_ctx, {(0, 0, K0): V, (65534, 65534, K0): FREE})
    assert L().ls_occupancy_build_projection(far._h, -INF, INF, 0.0, 0.0, ctypes.byref(g)) == ls.LS_ERR_ARG
    assert _download_rc(far) == ls.LS_ERR_STATE
    far.close()
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_a_grid_just_under_the_cell_cap(gpu_ctx):
    """One voxel at 0.075 m padded to 3474 m: a 46321 x 46321 grid of 2 145 635 041 cells, under 2^31 - 1 but within one
    grid stride (2^21 threads) of it, so the cell pass's index must not wrap.  Every cell is written once."""
    res = 0.075
    dev = _load(gpu_ctx, {(K0, K0, K0): V}, res=res)
    kmin = pr.coord_key_checked(float(F32(-1737.0)), res)
    w = pr.coord_key_checked(float(F32(1737.0)), res) - kmin + 1
    assert w == 46321 and 2**31 - 2**21 < w * w <= 2**31 - 1
    grid, info = dev.projected_map(min_size_x=3474.0, min_size_y=3474.0)
    assert (info.width, info.height) == (w, w)
    assert (info.occupied_cells, info.free_cells, info.unknown_cells) == (1, 0, w * w - 1)
    assert grid[K0 - kmin, K0 - kmin] == 100 and grid[0, 0] == -1 and grid[-1, -1] == -1
    del grid
    dev.close()


@pytest.mark.gpu
def test_projection_between_batch_begin_and_end(scans12):
    scans, poses = scans12
    ctx = ls.Context(0)
    ring = ctx.create_map(16, 131072)
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(4)]
    problems = [(ids[k + 1], [ids[k]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[k]) @ poses[k + 1]) for k in range(3)]
    p = ls.default_params(max_iterations=5)
    alone = ring.register_batch(problems, p)
    dev = ls.OccupancyMap(ctx)
    dev.insert_scan(ring, ids[0], poses[0])  # the .bt build is stale: the call builds it inside the batch
    end = ring.begin_batch(problems, p)
    grid, _ = dev.projected_map(min_z=0.3, max_z=2.0)
    res = end()
    for a, b in zip(res, alone):
        assert a["rc"] == b["rc"] and np.array_equal(a["T"], b["T"])
    want = pr.project(pr.bt_leaves(dev.octree().payload), dev.params.resolution, 0.3, 2.0)[0]
    assert np.array_equal(grid, want) and (want == 0).any()
    dev.close()
    ring.close()
    ctx.close()


@pytest.mark.gpu
def test_host_layer_and_saved_files(gpu_ctx, synth_mod, tmp_path):
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    n = 3
    truth, odom = synth_mod.trajectory(3, 2 * n + 2)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 3, k), 8) for k in range(2 * n)]
    odom7 = pg.se3_from_matrix(odom)
    off = pg.se3_from_matrix(np.array([[1, 0, 0, 3.0], [0, 1, 0, 2.0], [0, 0, 1, 0], [0, 0, 0, 1.0]]))
    est = host.Estimator(n_workers=2, nscan_in_sub_map=3)
    times = [[k * 10**8 for k in range(n)], [k * 10**8 + 5 * 10**7 for k in range(n)]]
    for k in range(n):
        data = [scans[k], scans[n + k]]
        feats = [np.ascontiguousarray(d[0]) for d in data]
        nrms = [np.ascontiguousarray(d[1]) for d in data]
        est.step_batch([0, 1], [times[0][k], times[1][k]], [odom7[k], pg.se3_compose(off, odom7[n + k])],
                       [f.ctypes.data for f in feats], [x.ctypes.data for x in nrms], [len(f) for f in feats])
    hm = host.OccupancyMap(est, resolution=0.1, max_range=15.0)
    assert hm.insert_laser_tracks() == 2 * n
    path = str(tmp_path / "h.ot")
    hm.write_full(path)
    dev = ls.OccupancyMap(gpu_ctx, resolution=0.1, max_range=15.0)
    dev.read_octomap_full(path)
    for band in (dict(), dict(min_z=0.3, max_z=2.0, min_x_size=60.0)):
        kw = dict(band)
        kw["min_size_x"] = kw.pop("min_x_size", 0.0)
        want, info = dev.projected_map(**kw)
        got, geo = hm.projected_map(**band)
        assert np.array_equal(got, want) and (want == 100).any()
        assert geo == (info.width, info.height, info.resolution, info.origin_x, info.origin_y)
        stem = str(tmp_path / "cpp")
        assert hm.save_projected_map(stem, **band)
        pstem = str(tmp_path / "py")
        dev.save_projected_map(pstem, **kw)
        pgm, yaml = pr.map_saver_bytes(want, info.resolution, info.origin_x, info.origin_y, stem + ".pgm")
        assert open(stem + ".pgm", "rb").read() == pgm and open(stem + ".yaml").read() == yaml
        assert open(pstem + ".pgm", "rb").read() == pgm
        assert open(pstem + ".yaml").read() == yaml.replace(stem + ".pgm", pstem + ".pgm")
    with pytest.raises(ls.LsError):
        hm.projected_map(min_z=math.nan)
    assert not hm.save_projected_map(str(tmp_path / "no" / "such" / "dir"))
    hm.close()
    dev.close(), est.close()
