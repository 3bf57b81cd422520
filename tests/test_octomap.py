"""Octree export of the occupancy map: the map as octomap's pruned binary tree (.bt) and its occupied leaves, what
octomap_to_point_cloud writes.  CPU: the oracle's writer against bytes derived by hand, a recursive pure-Python
restatement and the .bt parser; a round trip through the parser; malformed files.  GPU: the device export
(ls_occupancy_build_octree / _download_octree / _write_octomap), the Python wrapper and laser_slam::OccupancyMap against
the oracle, byte for byte.  The rules are oracle/OCTREE.md."""
import ctypes

import numpy as np
import pytest

import laser_slam_b200 as ls
from oracle import occupancy as oc
from oracle import octree as ot_oracle
from test_occupancy import F32, K0, _bits, _pack, _translate, full_scans  # noqa: F401  (full_scans: fixture)

FREE, OCC, INNER = 1, 2, 3
RES = 0.1
L_HIT, L_MISS = oc.logodds(0.9), oc.logodds(0.4)


def pair(children):
    """The two payload bytes of an inner node: {child index: FREE / OCC / INNER}."""
    m = sum(bits << (2 * i) for i, bits in children.items())
    return bytes([m & 0xFF, m >> 8])


def child(k, d):
    """Child index of key k (kx, ky, kz) below a node at depth d."""
    b = 15 - d
    return ((k[0] >> b) & 1) | (((k[1] >> b) & 1) << 1) | (((k[2] >> b) & 1) << 2)


def block(k0, n, state):
    """An aligned n^3 block of voxels from key k0, all in one state."""
    return {(k0[0] + x, k0[1] + y, k0[2] + z): state for x in range(n) for y in range(n) for z in range(n)}


# ---- pure-Python restatement: a recursive tree of nested lists ------------------------------------------------------
def restate(vox):
    """(nodes, payload, [(first-voxel key, depth) of each occupied leaf in pre-order]) of {key: FREE / OCC}."""
    def build(d, items):
        if d == 16:
            return items[0][1]
        groups = [[] for _ in range(8)]
        for k, s in items:
            groups[child(k, d)].append((k, s))
        ch = [build(d + 1, g) if g else None for g in groups]
        if d > 0 and all(isinstance(c, int) for c in ch) and len(set(ch)) == 1:
            return ch[0]
        return ch

    def write(n, out):
        out += pair({i: (INNER if isinstance(c, list) else c) for i, c in enumerate(n) if c is not None})
        for c in n:
            if isinstance(c, list):
                write(c, out)

    def count(n):
        return 1 + sum(count(c) if isinstance(c, list) else 1 for c in n if c is not None)

    def leaves(n, d, k0, out):
        for i, c in enumerate(n):
            sh = 15 - d
            ck = (k0[0] | ((i & 1) << sh), k0[1] | (((i >> 1) & 1) << sh), k0[2] | (((i >> 2) & 1) << sh))
            if isinstance(c, list):
                leaves(c, d + 1, ck, out)
            elif c == OCC:
                out.append((ck, d + 1))

    if not vox:
        return 0, b"", []
    root = build(0, sorted(vox.items()))
    out, lv = bytearray(), []
    write(root, out)
    leaves(root, 0, (0, 0, 0), lv)
    return count(root), bytes(out), lv


# ---- known answers: voxel sets and their hand-derived (size, payload, occupied leaves as (first key, depth)) ----------
C = (K0, K0, K0)
KA = {}


def _lo(vox, different=False):
    """Log-odds the oracle map would hold: L_hit for occupied, L_miss for free (the first occupied voxel twice hit)."""
    lo = {k: (L_HIT if s == OCC else L_MISS) for k, s in vox.items()}
    if different:
        k = min(vox)
        lo[k] = min(F32(L_HIT + L_HIT), oc.logodds(0.97))
    return lo


def known(name, vox, size, payload, leaves, different=False):
    KA[name] = (vox, size, payload, leaves, different)


known("empty", {}, 0, b"", [])
known("one_occupied_voxel", {C: OCC}, 17, b"\x00\xC0" + b"\x03\x00" * 14 + b"\x02\x00", [(C, 16)])
known("free_2x2x2", block(C, 2, FREE), 16, b"\x00\xC0" + b"\x03\x00" * 13 + b"\x01\x00", [])
_seven = {k: OCC for k in block(C, 2, OCC) if k != (K0 + 1, K0 + 1, K0 + 1)}
known("seven_occupied_one_free", {**_seven, (K0 + 1, K0 + 1, K0 + 1): FREE}, 24,
      b"\x00\xC0" + b"\x03\x00" * 14 + bytes([0b10101010, 0b01101010]), [(k, 16) for k in sorted(_seven, key=lambda k: child(k, 15))])
known("seven_known_one_unknown", _seven, 23, b"\x00\xC0" + b"\x03\x00" * 14 + bytes([0b10101010, 0b00101010]),
      [(k, 16) for k in sorted(_seven, key=lambda k: child(k, 15))])
known("eight_occupied_different_log_odds", block(C, 2, OCC), 16, b"\x00\xC0" + b"\x03\x00" * 13 + b"\x02\x00", [(C, 15)],
      different=True)
known("uniform_brick", block(C, 8, OCC), 14, b"\x00\xC0" + b"\x03\x00" * 11 + b"\x02\x00", [(C, 13)])
known("free_16_cubed_across_8_bricks", block(C, 16, FREE), 13, b"\x00\xC0" + b"\x03\x00" * 10 + b"\x01\x00", [])


def _both_sides():
    lo, hi = (K0 - 1,) * 3, (65534,) * 3
    vox = {**block(lo, 2, OCC), **block((0, 0, 0), 2, FREE), **block(hi, 2, OCC)}
    corner = lambda c: (K0 - 1 + (c & 1), K0 - 1 + ((c >> 1) & 1), K0 - 1 + ((c >> 2) & 1))  # noqa: E731
    pay = pair({i: INNER for i in range(8)})
    # root child 0: the free block at key 0 (child 0 down to a depth-15 leaf), the voxel 32767^3 (child 7 all the way)
    pay += pair({0: INNER, 7: INNER}) + b"\x03\x00" * 12 + pair({0: FREE}) + pair({7: INNER}) * 13 + pair({7: OCC})
    leaves = [(corner(0), 16)]
    # root children 1 ... 6: one voxel each, whose lower key bits are the complement of the root child's bits
    for c in range(1, 7):
        pay += pair({7 - c: INNER}) * 14 + pair({7 - c: OCC})
        leaves.append((corner(c), 16))
    # root child 7: the voxel 32768^3 (child 0 all the way), the occupied block at 65534 (child 7 down to depth 15)
    pay += pair({0: INNER, 7: INNER}) + b"\x03\x00" * 13 + pair({0: OCC}) + pair({7: INNER}) * 12 + pair({7: OCC})
    leaves += [(corner(7), 16), (hi, 15)]
    return vox, 1 + 30 + 6 * 16 + 30, pay, leaves


known("both_sides_of_the_origin_and_the_key_ends", *_both_sides())


def _centres(leaves, res):
    keys = np.array([k for k, _ in leaves], np.int64).reshape(-1, 3)
    return ls.leaf_centres(keys, np.array([d for _, d in leaves], np.uint8), res)


def _oracle_tree(vox, different, res=RES):
    lo = _lo(vox, different)
    keys = np.array([_pack(k) for k in sorted(lo, key=_pack)], np.uint64)
    return ot_oracle.octree(keys, np.array([lo[k] for k in sorted(lo, key=_pack)], F32), res)


def _parse(t, tmp_path, name="o.bt"):
    path = str(tmp_path / name)
    t.write(path)
    return path, ls.read_octomap(path)


@pytest.mark.parametrize("name", sorted(KA))
def test_oracle_writer_known_answers(name, tmp_path):
    vox, size, payload, leaves, different = KA[name]
    t = _oracle_tree(vox, different)
    assert (t.nodes, t.payload) == (size, payload)
    assert np.array_equal(t.depths, [d for _, d in leaves])
    assert np.array_equal(_bits(t.centres[:, :3]), _bits(_centres(leaves, RES))) and (t.centres[:, 3] == 1).all()
    # the restatement
    assert restate(vox) == (size, payload, leaves)
    # the parser: header, size, payload, and the occupied leaves in order
    path, p = _parse(t, tmp_path)
    head = open(path, "rb").read()[: -len(payload) or None]
    assert head.decode().endswith(f"id OcTree\nsize {size}\nres 0.1\ndata\n")
    assert (p["nodes"], p["payload"], p["resolution"]) == (size, payload, RES)
    occ = p["states"] == OCC
    assert [tuple(k) for k in p["keys"][occ]] == [k for k, _ in leaves] and list(p["depths"][occ]) == [d for _, d in leaves]
    out = str(tmp_path / "leaves.ply")
    assert ls.octomap_to_point_cloud(path, out) == len(leaves)
    lines = open(out).read().splitlines()
    body = lines[lines.index("end_header") + 1:]
    back = np.loadtxt(body, dtype=F32, ndmin=2).reshape(-1, 3) if body else np.zeros((0, 3), F32)
    assert np.array_equal(_bits(back), _bits(_centres(leaves, RES)))


def test_single_voxel_centre():
    t = _oracle_tree({C: OCC}, False)
    assert np.array_equal(t.centres[0], np.array([0.05, 0.05, 0.05, 1], F32))
    assert np.array_equal(_bits(t.centres[:, :3]), _bits(oc.centres([_pack(C)], RES)))


@pytest.mark.parametrize("res,text", [(0.075, "0.075"), (1.0 / 30.0, "0.0333333"), (0.1, "0.1"), (2.0, "2")])
def test_res_line_is_formatted_as_a_stream_prints_a_double(res, text, tmp_path):
    path = str(tmp_path / "r.bt")
    _oracle_tree({C: OCC}, False, res).write(path)
    assert f"\nres {text}\ndata\n" in open(path, "rb").read().decode(errors="replace")


def test_round_trip_expands_to_the_oracle_voxels(synth_mod, tmp_path):
    truth, _ = synth_mod.trajectory(0, 3)
    m = oc.OccupancyMap(resolution=0.1, max_range=-1.0)
    for k in range(3):
        m.insert_scan(synth_mod.scan(truth[k], 0, k)[0], truth[k].astype(F32))
    path = str(tmp_path / "map.bt")
    ot_oracle.of_map(m).write(path)
    p = ls.read_octomap(path)
    known_keys, occ_keys = [], []
    for s in (FREE, OCC):
        sel = p["states"] == s
        for d in np.unique(p["depths"][sel]):
            k0 = p["keys"][sel][p["depths"][sel] == d]
            n = 1 << (16 - int(d))
            off = np.stack(np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 3)
            k = (k0[:, None, :] + off[None]).reshape(-1, 3).astype(np.uint64)
            packed = k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32))
            known_keys.append(packed)
            if s == OCC:
                occ_keys.append(packed)
    assert np.array_equal(np.sort(np.concatenate(known_keys)), m.download(oc.KNOWN)[0])
    assert np.array_equal(np.sort(np.concatenate(occ_keys)), m.download(oc.OCCUPIED)[0])
    assert p["nodes"] < len(m.download(oc.KNOWN)[0])


def test_parser_rejects_malformed_files(tmp_path):
    good = tmp_path / "good.bt"
    _oracle_tree(block(C, 2, FREE), False).write(str(good))
    data = good.read_bytes()
    head, payload = data[: -30], data[-30:]
    bad = {
        "first_line": data.replace(b"# Octomap OcTree binary file", b"# Octomap OcTree file", 1),
        "tree_type": data.replace(b"id OcTree", b"id ColorOcTree"),
        "no_size": data.replace(b"size 16\n", b""),
        "bad_res": data.replace(b"res 0.1", b"res x"),
        "no_data_line": head.replace(b"data\n", b""),
        "truncated": head + payload[:-2],
        "size_too_large": data.replace(b"size 16", b"size 17"),
        "size_too_small": data.replace(b"size 16", b"size 15"),
        "inner_at_depth_16": head + payload[:-2] + b"\x03\x00\x03\x00",
    }
    for name, blob in bad.items():
        path = tmp_path / (name + ".bt")
        path.write_bytes(blob)
        with pytest.raises(ValueError):
            ls.octomap_to_point_cloud(str(path), str(tmp_path / "x.pcd"))
    assert ls.read_octomap(str(good))["nodes"] == 16


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _voxel_scans(vox, different):
    """One scan per voxel at resolution 0.1 with a 0.05 m range: an occupied voxel from a point 0.017 m from an origin
    inside it (no free cell), a free one from a point 10 m away whose ray is cut in the next voxel (the origin's voxel is
    its only free cell).  The first occupied voxel is hit twice when `different`."""
    scans = []
    for k, s in sorted(vox.items(), key=lambda e: _pack(e[0])):
        c = (np.array(k, np.float64) - K0 + 0.5) * RES
        if s == OCC:
            scans.append((np.array([[0.01, 0.01, 0.01, 1]], F32), _translate(c.astype(F32))))
        else:
            sx = 1.0 if k[0] < K0 else -1.0
            scans.append((np.array([[10.0 * sx, 0, 0, 1]], F32), _translate((c + [0.04 * sx, 0, 0]).astype(F32))))
    if different:
        scans.append(scans[[s for _, s in sorted(vox.items(), key=lambda e: _pack(e[0]))].index(OCC)])
    return scans


KA_PARAMS = dict(resolution=RES, max_range=0.05)


def _insert_both(ctx, scans, params, dev=None, o=None):
    ring = ctx.create_map(2, 1024)
    dev = dev or ls.OccupancyMap(ctx, **params)
    o = o or oc.OccupancyMap(**params)
    for cloud, T in scans:
        sid = ring.push_scan(cloud, np.zeros((len(cloud), 3), F32))
        dev.insert_scan(ring, sid, T)
        o.insert_scan(cloud, T)
    ring.close()
    return dev, o


def _same_tree(dev_tree, o_tree):
    return (dev_tree.nodes == o_tree.nodes and dev_tree.payload == o_tree.payload and
            np.array_equal(_bits(dev_tree.centres), _bits(o_tree.centres)) and np.array_equal(dev_tree.depths, o_tree.depths))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(KA))
def test_known_answers_on_the_device(gpu_ctx, name, tmp_path):
    vox, size, payload, leaves, different = KA[name]
    dev, o = _insert_both(gpu_ctx, _voxel_scans(vox, different), KA_PARAMS)
    k, v = o.download()
    assert {int(x): s for x, s in zip(k, np.where(v >= oc.logodds(0.7), OCC, FREE))} == {_pack(x): s for x, s in vox.items()}
    t, ot = dev.octree(), ot_oracle.of_map(o)
    assert _same_tree(t, ot)
    assert (t.nodes, t.payload) == (size, payload) and list(t.depths) == [d for _, d in leaves]
    assert np.array_equal(_bits(t.centres[:, :3]), _bits(_centres(leaves, RES)))
    dev.save_octomap(str(tmp_path / "d.bt"))
    ot.write(str(tmp_path / "o.bt"))
    assert (tmp_path / "d.bt").read_bytes() == (tmp_path / "o.bt").read_bytes()
    dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("params", [dict(), dict(resolution=0.1, max_range=-1.0)], ids=["defaults", "res0.1_unlimited"])
def test_full_scans_write_the_oracle_file(gpu_ctx, full_scans, params, tmp_path):
    scans, poses = full_scans
    ring = gpu_ctx.create_map(4, 131072)
    dev, o = ls.OccupancyMap(gpu_ctx, **params), oc.OccupancyMap(**params)
    nrm = np.zeros((131072, 3), F32)
    for k in range(len(scans)):
        dev.insert_scan(ring, ring.push_scan(scans[k], nrm), poses[k])
        o.insert_scan(scans[k], poses[k])
        if k + 1 not in (1, 6, 12):
            continue
        nodes = dev.save_octomap(str(tmp_path / "d.bt"))
        ot = ot_oracle.of_map(o)
        ot.write(str(tmp_path / "o.bt"))
        assert (tmp_path / "d.bt").read_bytes() == (tmp_path / "o.bt").read_bytes() and nodes == ot.nodes > 1000
        assert _same_tree(dev.octree(), ot)
        for ext in (".pcd", ".ply"):
            assert dev.save_pruned_point_cloud(str(tmp_path / ("d" + ext))) == len(ot.depths)
            ls.octomap_to_point_cloud(str(tmp_path / "d.bt"), str(tmp_path / ("p" + ext)))
            assert (tmp_path / ("d" + ext)).read_bytes() == (tmp_path / ("p" + ext)).read_bytes()
        ot.close()
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_grown_map_exports_the_same_bytes(gpu_ctx, full_scans):
    scans, poses = full_scans
    params = dict(resolution=0.1, max_range=12.0)
    trees = []
    for cap in (16, 0):
        ring = gpu_ctx.create_map(2, 131072)
        dev = ls.OccupancyMap(gpu_ctx, initial_capacity=cap, **params)
        for k in range(3):
            st = dev.insert_scan(ring, ring.push_scan(scans[k], np.zeros((131072, 3), F32)), poses[k])
        trees.append(dev.octree())
        assert cap == 0 or st.bricks > 16
        dev.close()
        ring.close()
    assert _same_tree(*trees) and trees[0].nodes > 1000


@pytest.mark.gpu
def test_export_leaves_the_map_unchanged_and_an_insert_invalidates_it(gpu_ctx, full_scans):
    scans, poses = full_scans
    ring = gpu_ctx.create_map(2, 131072)
    nrm = np.zeros((131072, 3), F32)
    dev = ls.OccupancyMap(gpu_ctx)
    dev.insert_scan(ring, ring.push_scan(scans[0], nrm), poses[0])
    before = (dev.download(ls.OCC_KNOWN), dev.download(ls.OCC_OCCUPIED))
    t = dev.octree()
    after = (dev.download(ls.OCC_KNOWN), dev.download(ls.OCC_OCCUPIED))
    for a, b in zip(before, after):
        assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))
    L = ls.lib()
    pay = np.full(len(t.payload), 0xAB, np.uint8)
    cen = np.full((len(t.depths), 4), -7, F32)
    dep = np.full(len(t.depths), 0xCD, np.uint8)
    n_pay, n_leaf = len(t.payload), len(t.depths)
    # caps one short: LS_ERR_ARG, nothing written
    assert L.ls_occupancy_download_octree(dev._h, pay.ctypes.data, n_pay - 1, None, None, 0) == ls.LS_ERR_ARG
    assert L.ls_occupancy_download_octree(dev._h, pay.ctypes.data, n_pay, cen.ctypes.data, dep.ctypes.data,
                                          n_leaf - 1) == ls.LS_ERR_ARG
    assert L.ls_occupancy_download_octree(dev._h, pay.ctypes.data, n_pay, None, dep.ctypes.data, n_leaf - 1) == ls.LS_ERR_ARG
    assert (pay == 0xAB).all() and (cen == -7).all() and (dep == 0xCD).all()
    # the payload alone, then everything
    assert L.ls_occupancy_download_octree(dev._h, pay.ctypes.data, n_pay, None, None, 0) == 0
    assert pay.tobytes() == t.payload and (cen == -7).all()
    assert L.ls_occupancy_download_octree(dev._h, pay.ctypes.data, n_pay, cen.ctypes.data, dep.ctypes.data, n_leaf) == 0
    assert np.array_equal(_bits(cen), _bits(t.centres)) and np.array_equal(dep, t.depths)
    dev.insert_scan(ring, ring.push_scan(scans[1], nrm), poses[1])
    assert L.ls_occupancy_download_octree(dev._h, pay.ctypes.data, n_pay, None, None, 0) == ls.LS_ERR_STATE
    st = ls.OctreeStats()
    assert L.ls_occupancy_build_octree(dev._h, ctypes.byref(st)) == 0 and st.device_ms > 0
    assert st.nodes > 0 and (st.nodes, st.payload_bytes) != (t.nodes, len(t.payload))
    want = 0 if st.payload_bytes <= n_pay else ls.LS_ERR_ARG  # the rebuilt tree is current again
    assert L.ls_occupancy_download_octree(dev._h, pay.ctypes.data, n_pay, None, None, 0) == want
    fresh = ls.OccupancyMap(gpu_ctx)
    assert L.ls_occupancy_download_octree(fresh._h, pay.ctypes.data, n_pay, None, None, 0) == ls.LS_ERR_STATE
    empty = fresh.octree()
    assert (empty.nodes, empty.payload, len(empty.depths)) == (0, b"", 0)
    fresh.close()
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_export_between_batch_begin_and_end(full_scans):
    scans, poses = full_scans
    ctx = ls.Context(0)
    ring = ctx.create_map(16, 131072)
    nrm = np.zeros((131072, 3), F32)
    ids = [ring.push_scan(scans[k], nrm) for k in range(4)]
    problems = [(ids[k + 1], [ids[k]], [np.eye(4, dtype=F32)], np.linalg.inv(poses[k]) @ poses[k + 1]) for k in range(3)]
    p = ls.default_params(max_iterations=5)
    alone = ring.register_batch(problems, p)
    dev, o = ls.OccupancyMap(ctx), oc.OccupancyMap()
    end = ring.begin_batch(problems, p)
    for k in range(2):
        dev.insert_scan(ring, ids[k], poses[k])
        o.insert_scan(scans[k], poses[k])
    t = dev.octree()
    res = end()
    for a, b in zip(res, alone):
        assert a["rc"] == b["rc"] and np.array_equal(a["T"], b["T"])
    assert _same_tree(t, ot_oracle.of_map(o))
    dev.close()
    ring.close()
    ctx.close()


@pytest.mark.gpu
def test_host_layer_write_binary(synth_mod, tmp_path):
    """laser_slam::OccupancyMap::writeBinary after insertLaserTracks on two workers: the oracle's file for the same scan
    order; getOccupiedLeafCloud: its occupied leaves."""
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    from test_local_map import _float_matrix
    n = 4
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
    params = dict(resolution=0.1, max_range=15.0)
    occ = host.OccupancyMap(est, **params)
    assert occ.insert_laser_tracks() == 2 * n
    o = oc.OccupancyMap(**params)
    entries = []
    for w in range(2):
        ts, traj = est.trajectory(w)
        entries += [(int(ts[k]), w, k, _float_matrix(traj[k])) for k in range(n)]
    for t, w, k, T in sorted(entries, key=lambda e: e[:3]):
        o.insert_scan(scans[w * n + k][0], T)
    occ.write_binary(str(tmp_path / "h.bt"))
    ot = ot_oracle.of_map(o)
    ot.write(str(tmp_path / "o.bt"))
    assert (tmp_path / "h.bt").read_bytes() == (tmp_path / "o.bt").read_bytes()
    cloud = occ.occupied_leaf_cloud()
    assert np.array_equal(_bits(cloud), _bits(ot.centres)) and len(cloud) > 0
    occ.close()
    est.close()
