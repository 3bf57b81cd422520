"""Reading octomap binary files (.bt) into the resident occupancy map (ls_occupancy_read_octree / _read_octomap): the
pruned tree parsed and expanded on the device, then queried or mapped into.  CPU: the reference expansion
(tests/octomap_read_ref.py) against the known answers of test_octomap.py and hand-made foreign payloads, and the seeded
oracle map.  GPU: the device read against that reference bit for bit, the round trip of full-scan maps, mapping after a
read, and refusals that leave the map unchanged.  The rules are DESIGN.md §4b''''''."""
import ctypes

import numpy as np
import pytest

import laser_slam_b200 as ls
import octomap_read_ref as rr
from oracle import occupancy as oc
from oracle import octree as ot_oracle
from test_occupancy import F32, K0, _bits, _pack, full_scans  # noqa: F401  (full_scans: fixture)
from test_octomap import FREE, INNER, KA, OCC, RES, _oracle_tree, block, child, pair

L_MIN, L_MAX = rr.clamps()
HEAD = ("# Octomap OcTree binary file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
        "id OcTree\nsize {}\nres {}\ndata\n")


def bt_bytes(size, payload, res_text="0.1"):
    return HEAD.format(size, res_text).encode() + payload


def tree_of(items):
    """(size, payload) of the tree holding `items` as given, unpruned: (first key, depth, FREE / OCC) leaves and
    (first key, depth, INNER) inner nodes without children."""
    root = {}
    for k, d, s in items:
        node = root
        for dd in range(d - 1):
            node = node.setdefault(child(k, dd), {})
        node[child(k, d - 1)] = {} if s == INNER else s

    def write(n, out):
        out += pair({i: INNER if isinstance(c, dict) else c for i, c in n.items()})
        for i in sorted(n):
            if isinstance(n[i], dict):
                write(n[i], out)

    def count(n):
        return 1 + sum(count(c) if isinstance(c, dict) else 1 for c in n.values())

    if not items:
        return 0, b""
    out = bytearray()
    write(root, out)
    return count(root), bytes(out)


def _leaf_voxels(k, d, s):
    return block(k, 1 << (16 - d), s)


C = (K0, K0, K0)
_B = (K0 + 64, K0, K0)  # a brick-aligned depth-12 node: 64 voxels per axis
FOREIGN = {  # name: (items, voxels {key: FREE / OCC})
    "unpruned_2x2x2": ([((C[0] + (i & 1), C[1] + ((i >> 1) & 1), C[2] + (i >> 2)), 16, FREE) for i in range(8)],
                       block(C, 2, FREE)),
    "inner_node_without_children": ([((0, 0, 0), 1, INNER), ((K0, 0, K0), 5, INNER)] +
                                    [((C[0] + (i & 1), C[1] + ((i >> 1) & 1), C[2] + (i >> 2)), 16, FREE) for i in range(8)],
                                    block(C, 2, FREE)),
    "free_leaf_at_depth_9": ([(C, 9, FREE)], _leaf_voxels(C, 9, FREE)),
    "mixed_leaves_at_depths_13_to_16": (
        [(_B, 13, FREE), ((_B[0] + 8, _B[1], _B[2]), 14, OCC), ((_B[0] + 12, _B[1], _B[2]), 15, FREE),
         ((_B[0] + 14, _B[1] + 2, _B[2]), 16, OCC), ((_B[0] + 15, _B[1] + 3, _B[2] + 1), 16, FREE),
         ((_B[0] + 12, _B[1] + 4, _B[2] + 4), 14, FREE), ((_B[0] + 32, _B[1] + 32, _B[2] + 32), 13, OCC)],
        {**_leaf_voxels(_B, 13, FREE), **_leaf_voxels((_B[0] + 8, _B[1], _B[2]), 14, OCC),
         **_leaf_voxels((_B[0] + 12, _B[1], _B[2]), 15, FREE), (_B[0] + 14, _B[1] + 2, _B[2]): OCC,
         (_B[0] + 15, _B[1] + 3, _B[2] + 1): FREE, **_leaf_voxels((_B[0] + 12, _B[1] + 4, _B[2] + 4), 14, FREE),
         **_leaf_voxels((_B[0] + 32, _B[1] + 32, _B[2] + 32), 13, OCC)}),
    "both_ends_of_the_key_space": (
        [((0, 0, 0), 16, OCC), ((65535, 65535, 65535), 16, FREE), ((65532, 0, 65532), 14, OCC), ((0, 65528, 0), 13, FREE)],
        {(0, 0, 0): OCC, (65535, 65535, 65535): FREE, **_leaf_voxels((65532, 0, 65532), 14, OCC),
         **_leaf_voxels((0, 65528, 0), 13, FREE)}),
}
CASES = sorted(["ka_" + n for n in KA]) + sorted("foreign_" + n for n in FOREIGN)


def case(name):
    """(size, payload, voxels {key: FREE / OCC}) of a known answer or a foreign payload."""
    if name.startswith("ka_"):
        vox, size, payload, _, _ = KA[name[3:]]
        return size, payload, vox
    items, vox = FOREIGN[name[8:]]
    size, payload = tree_of(items)
    return size, payload, vox


def want_voxels(vox, l_min=L_MIN, l_max=L_MAX):
    keys = np.array(sorted(_pack(k) for k in vox), np.uint64)
    by_key = {_pack(k): s for k, s in vox.items()}
    return keys, np.array([l_max if by_key[int(k)] == OCC else l_min for k in keys], F32)


def _parse(tmp_path, size, payload, res_text="0.1", name="in.bt"):
    path = tmp_path / name
    path.write_bytes(bt_bytes(size, payload, res_text))
    return str(path), ls.read_octomap(str(path))


# ---- CPU ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_reference_expansion_equals_the_voxels(name, tmp_path):
    size, payload, vox = case(name)
    _, p = _parse(tmp_path, size, payload)
    k, v = rr.expand(p, L_MIN, L_MAX)
    wk, wv = want_voxels(vox)
    assert np.array_equal(k, wk) and np.array_equal(_bits(v), _bits(wv))


def test_foreign_payloads_are_what_they_say():
    for name in ("unpruned_2x2x2", "inner_node_without_children"):  # not what writeBinary writes
        size, payload, vox = case("foreign_" + name)
        assert (size, payload) != (_oracle_tree(vox, False).nodes, _oracle_tree(vox, False).payload)
    for name in ("free_leaf_at_depth_9", "mixed_leaves_at_depths_13_to_16", "both_ends_of_the_key_space"):  # pruned
        size, payload, vox = case("foreign_" + name)
        t = _oracle_tree(vox, False)
        assert (size, payload) == (t.nodes, t.payload)
    assert len(case("foreign_free_leaf_at_depth_9")[2]) == 4096 * 512


def test_seeded_oracle_map_inserts_as_one_built_voxel_by_voxel(synth_mod):
    truth, _ = synth_mod.trajectory(0, 3)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 0, k), 8)[0] for k in range(3)]
    params = dict(resolution=0.1, max_range=15.0)
    built = oc.OccupancyMap(**params)
    for k in range(2):
        built.insert_scan(scans[k], truth[k].astype(F32))
    seeded = rr.seed(oc.OccupancyMap(**params), *built.download())
    assert all(np.array_equal(a, b) for a, b in zip(seeded.download(), built.download()))
    sa = built.insert_scan(scans[2], truth[2].astype(F32))
    sb = seeded.insert_scan(scans[2], truth[2].astype(F32))
    assert sa == sb
    (ka, va), (kb, vb) = built.download(), seeded.download()
    assert np.array_equal(ka, kb) and np.array_equal(_bits(va), _bits(vb)) and len(ka) > 10000


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _download(dev):
    return tuple(dev.download(w) for w in (ls.OCC_KNOWN, ls.OCC_OCCUPIED))


def _same_downloads(a, b):
    return all(np.array_equal(x[0], y[0]) and np.array_equal(_bits(x[1]), _bits(y[1])) and
               np.array_equal(_bits(x[2]), _bits(y[2])) for x, y in zip(a, b))


def _check_loaded(dev, st, p, res, l_min=L_MIN, l_max=L_MAX, l_occ=oc.logodds(0.7)):
    k, v = rr.expand(p, l_min, l_max)
    known, occ = _download(dev)
    assert np.array_equal(known[0], k) and np.array_equal(_bits(known[1]), _bits(v))
    assert np.array_equal(_bits(known[2][:, :3]), _bits(oc.centres(k, res))) and (known[2][:, 3] == 1).all()
    sel = v >= l_occ
    assert np.array_equal(occ[0], k[sel]) and np.array_equal(_bits(occ[1]), _bits(v[sel]))
    bricks = len(np.unique(((k & np.uint64(0xFFFF)) >> np.uint64(3)) | (((k >> np.uint64(16)) & np.uint64(0xFFFF)) >> np.uint64(3)) << np.uint64(13) |
                           ((k >> np.uint64(32)) >> np.uint64(3)) << np.uint64(26)))
    leaves = p["states"]
    assert (st.nodes, st.inner_nodes, st.free_leaves, st.occupied_leaves) == (
        p["nodes"], len(p["payload"]) // 2, int((leaves == FREE).sum()), int((leaves == OCC).sum()))
    assert (st.known_voxels, st.bricks, st.resolution) == (len(k), bricks, res) and dev.params.resolution == res
    assert st.device_ms > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_read_equals_the_reference(gpu_ctx, name, tmp_path):
    size, payload, vox = case(name)
    path, p = _parse(tmp_path, size, payload)
    oracle_file = tmp_path / "oracle.bt"
    k, v = rr.expand(p, L_MIN, L_MAX)
    ot_oracle.octree(k, v, RES).write(str(oracle_file))
    for how in ("file", "payload"):
        dev = ls.OccupancyMap(gpu_ctx, resolution=0.075)
        st = dev.read_octomap(path) if how == "file" else dev.read_octree(payload, size, 0.1)
        _check_loaded(dev, st, p, RES)
        dev.save_octomap(str(tmp_path / "back.bt"))
        back = (tmp_path / "back.bt").read_bytes()
        assert back == oracle_file.read_bytes()
        if name.startswith("ka_") or name[8:] not in ("unpruned_2x2x2", "inner_node_without_children"):
            assert back == open(path, "rb").read()
        dev.close()


def _segments(rng, poses, n, lo=1.0, hi=10.0):
    p = np.array([poses[k][:3, 3] for k in rng.integers(0, len(poses), n)], np.float64)
    s = p + rng.uniform(-3.0, 3.0, (n, 3)) * [1, 1, 0.3]
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    return s, s + d * rng.uniform(lo, hi, (n, 1))


def _same_queries(a, b, scans, poses, res):
    rng = np.random.default_rng(41)
    keys = a.download(ls.OCC_KNOWN)[0]
    cen = oc.centres(keys, res).astype(np.float64)
    pts = np.concatenate([cen, rng.uniform(cen.min(axis=0), cen.max(axis=0), (200_000, 3))])
    assert np.array_equal(a.cell_status(pts)[0], b.cell_status(pts)[0])
    for stop in (True, False):
        s, e = _segments(rng, poses, 100_000)
        ga, gb = a.line_status(s, e, stop_at_unknown=stop), b.line_status(s, e, stop_at_unknown=stop)
        assert np.array_equal(ga[0], gb[0]) and np.array_equal(ga[1], gb[1])
    s, e = _segments(rng, poses, 300, 0.5, 4.0)
    for box in ((0.6, 0.6, 0.3), (0.3, 0.0, 0.45)):
        for stop in (True, False):
            ga, gb = a.line_status(s, e, box=box, stop_at_unknown=stop), b.line_status(s, e, box=box, stop_at_unknown=stop)
            assert np.array_equal(ga[0], gb[0]) and np.array_equal(ga[1], gb[1])
    for ignore in (False, True):
        for k in (0, 5, 11):
            T = poses[k].astype(np.float64)
            origins = np.repeat(poses[k][:3, 3][None], 131072, axis=0).astype(F32)
            dirs = (scans[k][:, :3].astype(np.float64) @ T[:3, :3].T).astype(F32)
            ga, gb = a.cast_rays(origins, dirs, ignore, 20.0), b.cast_rays(origins, dirs, ignore, 20.0)
            assert np.array_equal(ga[0], gb[0]) and np.array_equal(_bits(ga[1]), _bits(gb[1]))
            assert ls.RAY_HIT in ga[0]


def _full_map(ctx, full_scans, params, n):
    scans, poses = full_scans
    ring = ctx.create_map(2, 131072)
    dev = ls.OccupancyMap(ctx, **params)
    nrm = np.zeros((131072, 3), F32)
    for k in range(n):
        dev.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
    return dev, ring


@pytest.mark.gpu
@pytest.mark.parametrize("params", [dict(), dict(resolution=0.1, max_range=-1.0)], ids=["defaults", "res0.1_unlimited"])
def test_full_scan_maps_round_trip(gpu_ctx, full_scans, params, tmp_path):
    scans, poses = full_scans
    orig, ring = _full_map(gpu_ctx, full_scans, params, len(scans))
    bt = str(tmp_path / "orig.bt")
    orig.save_octomap(bt)
    ok, ov, _ = orig.download(ls.OCC_KNOWN)
    l_occ = oc.logodds(0.7)
    for cap in (0, 16):
        dev = ls.OccupancyMap(gpu_ctx, initial_capacity=cap, **params)
        st = dev.read_octomap(bt)
        assert cap == 0 or st.bricks > 16
        dev.save_octomap(str(tmp_path / "back.bt"))
        assert (tmp_path / "back.bt").read_bytes() == open(bt, "rb").read()
        k, v, _ = dev.download(ls.OCC_KNOWN)
        assert np.array_equal(k, ok) and np.array_equal(_bits(v), _bits(np.where(ov >= l_occ, L_MAX, L_MIN).astype(F32)))
        assert st.known_voxels == len(ok) > 1_000_000
        _same_queries(dev, orig, scans, poses, orig.params.resolution)
        dev.close()
    orig.close()
    ring.close()


@pytest.mark.gpu
def test_mapping_continues_after_a_read(gpu_ctx, full_scans, tmp_path):
    scans, poses = full_scans
    params = dict(resolution=0.1, max_range=15.0)
    first, ring = _full_map(gpu_ctx, full_scans, params, 6)
    bt = str(tmp_path / "six.bt")
    first.save_octomap(bt)
    first.close()
    dev = ls.OccupancyMap(gpu_ctx, **params)
    dev.read_octomap(bt)
    o = rr.seed(oc.OccupancyMap(**params), *rr.expand(ls.read_octomap(bt), L_MIN, L_MAX))
    nrm = np.zeros((131072, 3), F32)
    for k in range(6, 12):
        st = dev.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
        ost = o.insert_scan(scans[k], poses[k])
        assert (st.free_updates, st.occupied_updates, st.known_voxels) == (
            ost["free_updates"], ost["occupied_updates"], ost["known_voxels"])
    (k, v, _), (wk, wv) = dev.download(ls.OCC_KNOWN), o.download()
    assert np.array_equal(k, wk) and np.array_equal(_bits(v), _bits(wv))
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_read_into_a_used_map_equals_a_read_into_a_new_one(gpu_ctx, full_scans, tmp_path):
    scans, poses = full_scans
    params = dict(resolution=0.1, max_range=12.0)
    src, ring = _full_map(gpu_ctx, full_scans, params, 2)
    bt = str(tmp_path / "two.bt")
    src.save_octomap(bt)
    src.close()
    used = ls.OccupancyMap(gpu_ctx, initial_capacity=16, **params)
    nrm = np.zeros((131072, 3), F32)
    for k in (7, 8, 9):  # grows the pool and the hash past what the file needs
        used.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
    with pytest.raises(ls.LsError):
        used.read_octree(b"\x03", 5, 0.1)
    fresh = ls.OccupancyMap(gpu_ctx, **params)
    for m in (used, fresh):
        m.read_octomap(bt)
    assert _same_downloads(_download(used), _download(fresh))
    sid = ring.push_scan(scans[3], nrm)
    a, b = used.insert_scan(ring, sid, poses[3]), fresh.insert_scan(ring, sid, poses[3])
    assert (a.free_updates, a.occupied_updates, a.known_voxels) == (b.free_updates, b.occupied_updates, b.known_voxels)
    assert _same_downloads(_download(used), _download(fresh))
    used.close()
    fresh.close()
    ring.close()


@pytest.mark.gpu
def test_the_file_resolution_becomes_the_maps(gpu_ctx, full_scans, tmp_path):
    scans, poses = full_scans
    res = 1.0 / 30.0
    o = oc.OccupancyMap(resolution=res, max_range=6.0)
    o.insert_scan(scans[0], poses[0])
    bt = str(tmp_path / "fine.bt")
    ot_oracle.of_map(o).write(bt)
    assert b"\nres 0.0333333\n" in open(bt, "rb").read()
    dev = ls.OccupancyMap(gpu_ctx, max_range=6.0)
    st = dev.read_octomap(bt)
    assert st.resolution == 0.0333333 and dev.params.resolution == 0.0333333
    p = ls.read_octomap(bt)
    _check_loaded(dev, st, p, 0.0333333)
    ref = rr.seed(oc.OccupancyMap(resolution=0.0333333, max_range=6.0), *rr.expand(p, L_MIN, L_MAX))
    ring = gpu_ctx.create_map(2, 131072)
    dev.insert_scan(ring, ring.push_scan(scans[1], np.zeros((131072, 3), F32)), poses[1])
    ref.insert_scan(scans[1], poses[1])
    (k, v, c), (wk, wv) = dev.download(ls.OCC_KNOWN), ref.download()
    assert np.array_equal(k, wk) and np.array_equal(_bits(v), _bits(wv))
    assert np.array_equal(_bits(c[:, :3]), _bits(oc.centres(wk, 0.0333333)))
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_clamp_max_below_the_threshold_loads_occupied_leaves_as_free(gpu_ctx, tmp_path):
    size, payload, vox = case("ka_uniform_brick")
    path, p = _parse(tmp_path, size, payload)
    dev = ls.OccupancyMap(gpu_ctx, clamp_max=0.6)
    st = dev.read_octomap(path)
    l_max = oc.logodds(0.6)
    _check_loaded(dev, st, p, RES, l_max=l_max)
    assert dev.size(ls.OCC_OCCUPIED) == 0 and dev.size(ls.OCC_KNOWN) == 512
    assert (dev.cell_status(dev.download()[2][:, :3].astype(np.float64))[0] == ls.CELL_FREE).all()
    dev.close()


@pytest.mark.gpu
def test_size_0_empties_the_map(gpu_ctx, full_scans, tmp_path):
    dev, ring = _full_map(gpu_ctx, full_scans, dict(), 1)
    path = tmp_path / "empty.bt"
    path.write_bytes(bt_bytes(0, b"", "0.2"))
    st = dev.read_octomap(str(path))
    assert (st.nodes, st.known_voxels, st.bricks, st.resolution) == (0, 0, 0, 0.2)
    assert dev.size(ls.OCC_KNOWN) == 0 and dev.size(ls.OCC_OCCUPIED) == 0 and dev.octree().nodes == 0
    assert (dev.cell_status([[0.1, 0.1, 0.1]])[0] == ls.CELL_UNKNOWN).all()
    dev.close()
    ring.close()


def _malformed(tmp_path):
    good = tmp_path / "good.bt"
    _oracle_tree(block((K0, K0, K0), 2, FREE), False).write(str(good))
    data = good.read_bytes()
    head, payload = data[: -30], data[-30:]
    return {
        "first_line": data.replace(b"# Octomap OcTree binary file", b"# Octomap OcTree file", 1),
        "tree_type": data.replace(b"id OcTree", b"id ColorOcTree"),
        "no_size": data.replace(b"size 16\n", b""),
        "bad_res": data.replace(b"res 0.1", b"res x"),
        "no_data_line": head.replace(b"data\n", b""),
        "truncated": head + payload[:-2],
        "size_too_large": data.replace(b"size 16", b"size 17"),
        "size_too_small": data.replace(b"size 16", b"size 15"),
        "inner_at_depth_16": head + payload[:-2] + b"\x03\x00\x03\x00",
        "res_0": data.replace(b"res 0.1", b"res 0"),
        "res_inf": data.replace(b"res 0.1", b"res inf"),
        "depth_1_free_leaf": bt_bytes(2, pair({0: FREE})),
    }


@pytest.mark.gpu
def test_refusals_leave_the_map_and_its_tree_unchanged(gpu_ctx, full_scans, tmp_path):
    dev, ring = _full_map(gpu_ctx, full_scans, dict(resolution=0.1, max_range=10.0), 2)
    before, tree = _download(dev), dev.octree()
    L = ls.lib()
    pay = np.zeros(len(tree.payload), np.uint8)
    for name, blob in _malformed(tmp_path).items():
        path = tmp_path / (name + ".bt")
        path.write_bytes(blob)
        st = ls.OctomapReadStats()
        rc = L.ls_occupancy_read_octomap(dev._h, str(path).encode(), ctypes.byref(st))
        assert rc == (ls.LS_ERR_NOMEM if name == "depth_1_free_leaf" else ls.LS_ERR_ARG), name
        if name not in ("res_inf", "depth_1_free_leaf"):  # the CPU parser refuses the same files
            with pytest.raises(ValueError):
                ls.read_octomap(str(path))
        # the tree built before is still current and unchanged
        assert L.ls_occupancy_download_octree(dev._h, pay.ctypes.data, len(pay), None, None, 0) == 0, name
        assert pay.tobytes() == tree.payload
    for args in ((b"", 5, 0.1), (pair({0: FREE}), 2, 0.0), (pair({0: FREE}), 2, float("nan")), (pair({0: FREE}), -1, 0.1)):
        with pytest.raises(ls.LsError):
            dev.read_octree(*args)
    assert dev.params.resolution == 0.1
    assert _same_downloads(_download(dev), before)
    t = dev.octree()
    assert (t.nodes, t.payload) == (tree.nodes, tree.payload) and np.array_equal(_bits(t.centres), _bits(tree.centres))
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_read_between_batch_begin_and_end(full_scans, tmp_path):
    scans, poses = full_scans
    ctx = ls.Context(0)
    ring = ctx.create_map(16, 131072)
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(4)]
    problems = [(ids[k + 1], [ids[k]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[k]) @ poses[k + 1]) for k in range(3)]
    p = ls.default_params(max_iterations=5)
    alone = ring.register_batch(problems, p)
    src = ls.OccupancyMap(ctx)
    src.insert_scan(ring, ids[0], poses[0])
    bt = str(tmp_path / "one.bt")
    src.save_octomap(bt)
    dev = ls.OccupancyMap(ctx)
    end = ring.begin_batch(problems, p)
    st = dev.read_octomap(bt)
    dev.save_octomap(str(tmp_path / "back.bt"))
    res = end()
    for a, b in zip(res, alone):
        assert a["rc"] == b["rc"] and np.array_equal(a["T"], b["T"])
    _check_loaded(dev, st, ls.read_octomap(bt), 0.075)
    assert (tmp_path / "back.bt").read_bytes() == open(bt, "rb").read()
    for m in (src, dev):
        m.close()
    ring.close()
    ctx.close()


@pytest.mark.gpu
def test_host_layer_read_binary_equals_the_abi(gpu_ctx, synth_mod, tmp_path):
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    truth, odom = synth_mod.trajectory(3, 4)
    scans = [synth_mod.subsample(*synth_mod.scan(truth[k], 3, k), 8) for k in range(3)]
    est = host.Estimator(n_workers=1, nscan_in_sub_map=3)
    odom7 = pg.se3_from_matrix(odom)
    for k in range(3):
        f, n = np.ascontiguousarray(scans[k][0]), np.ascontiguousarray(scans[k][1])
        est.step_batch([0], [k * 10**8], [odom7[k]], [f.ctypes.data], [n.ctypes.data], [len(f)])
    params = dict(resolution=0.1, max_range=15.0)
    occ = host.OccupancyMap(est, **params)
    assert occ.insert_laser_tracks() == 3
    bt = str(tmp_path / "h.bt")
    occ.write_binary(bt)
    other = host.OccupancyMap(est, resolution=0.2, max_range=15.0)
    bad = tmp_path / "bad.bt"
    bad.write_bytes(b"# not octomap\n")
    assert other.read_binary(str(bad)) is False
    assert other.read_binary(bt) is True
    dev = ls.OccupancyMap(gpu_ctx, resolution=0.2, max_range=15.0)
    dev.read_octomap(bt)
    k, v, _ = dev.download(ls.OCC_KNOWN)
    hk, hv = other.voxels(1)
    assert np.array_equal(hk, k) and np.array_equal(_bits(hv), _bits(v)) and len(k) > 0
    other.write_binary(str(tmp_path / "h2.bt"))
    assert (tmp_path / "h2.bt").read_bytes() == open(bt, "rb").read()
    other.close()
    occ.close()
    est.close()
    dev.close()
