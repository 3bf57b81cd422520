"""The occupancy map as octomap's full tree (.ot, OcTree::write / AbstractOcTree::read): every node's float log-odds,
pruned by value, written and read on the device (ls_occupancy_build_full_octree / _download_full_octree /
_write_octomap_full / _read_full_octree / _read_octomap_full).  CPU: the full-tree oracle (tests/octomap_full_ref.py)
against bytes derived by hand, a recursive pure-Python restatement and the CPU parser; refusals; the tie to the .bt tree.
GPU: the device against the oracle bit for bit, round trips, resuming a saved map, foreign payloads, refusals and caching,
and laser_slam::OccupancyMap.  The rules are DESIGN.md §4b'''''''."""
import ctypes

import numpy as np
import pytest

import laser_slam_b200 as ls
import octomap_full_ref as fr
import octomap_read_ref as rr
from oracle import occupancy as oc
from oracle import octree as ot_oracle
from test_occupancy import F32, K0, _bits, _pack, full_scans  # noqa: F401  (full_scans: fixture)
from test_octomap import C, FREE, INNER, OCC, RES, _voxel_scans, block, child, pair
from test_octomap_read import _download, _full_map, _same_downloads, _same_queries

HEAD = ("# Octomap OcTree file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
        "id OcTree\nsize {}\nres {}\ndata\n")
L_OCC = oc.logodds(0.7)
V = oc.logodds(0.9)
W = np.nextafter(V, F32(np.inf), dtype=F32)  # one ulp above V
NEG0, POS0 = F32(-0.0), F32(0.0)


def nb(v, mask=0):
    """One node of the payload: its float32 value (little-endian), then the byte of its existing children."""
    return np.array([v], "<f4").tobytes() + bytes([mask])


def ot_bytes(size, payload, res_text="0.1"):
    return HEAD.format(size, res_text).encode() + payload


def _octet(base, values):
    """{key: value} of the voxels below one depth-15 node whose first voxel is `base`: {child index: value}."""
    return {(base[0] + (i & 1), base[1] + ((i >> 1) & 1), base[2] + (i >> 2)): F32(v) for i, v in values.items()}


# ---- pure-Python restatement: a recursive tree of nested lists -----------------------------------------------------
def restate(vox):
    """(nodes, payload) of {key: float32 log-odds}: value pruning, inner nodes holding their largest child, pre-order."""
    def build(d, items):
        if d == 16:
            return items[0][1]
        groups = [[] for _ in range(8)]
        for k, v in items:
            groups[child(k, d)].append((k, v))
        ch = [build(d + 1, g) if g else None for g in groups]
        if d > 0 and all(c is not None and not isinstance(c, list) for c in ch) and all(c == ch[0] for c in ch):
            return ch[0]  # child 0's bits
        return ch

    def value(n):
        if not isinstance(n, list):
            return n
        best = None
        for c in n:
            if c is not None and (best is None or value(c) > best):
                best = value(c)
        return best

    def write(n, out):
        if not isinstance(n, list):
            out += nb(n)
            return 1
        out += nb(value(n), sum(1 << i for i, c in enumerate(n) if c is not None))
        return 1 + sum(write(c, out) for c in n if c is not None)

    if not vox:
        return 0, b""
    out = bytearray()
    size = write(build(0, sorted(vox.items())), out)
    return size, bytes(out)


def unpruned(vox, inner=F32(123.0)):
    """(size, payload) of {key: float32} with every voxel a leaf at depth 16 and every inner node holding `inner`."""
    root = {}
    for k, v in vox.items():
        node = root
        for d in range(15):
            node = node.setdefault(child(k, d), {})
        node[child(k, 15)] = F32(v)

    def write(n, out):
        if not isinstance(n, dict):
            out += nb(n)
            return 1
        out += nb(inner, sum(1 << i for i in n))
        return 1 + sum(write(n[i], out) for i in sorted(n))

    if not vox:
        return 0, b""
    out = bytearray()
    return write(root, out), bytes(out)


def tree_of(items, inner=None):
    """(size, payload) of leaves given as (first key, depth, float32 value), unpruned; inner nodes hold `inner`, or their
    largest child when None."""
    root = {}
    for k, d, v in items:
        node = root
        for dd in range(d - 1):
            node = node.setdefault(child(k, dd), {})
        node[child(k, d - 1)] = F32(v)

    def value(n):
        if not isinstance(n, dict):
            return n
        best = None
        for i in sorted(n):
            if best is None or value(n[i]) > best:
                best = value(n[i])
        return best

    def write(n, out):
        if not isinstance(n, dict):
            out += nb(n)
            return 1
        out += nb(value(n) if inner is None else inner, sum(1 << i for i in n))
        return 1 + sum(write(n[i], out) for i in sorted(n))

    if not items:
        return 0, b""
    out = bytearray()
    return write(root, out), bytes(out)


# ---- known answers: {key: value} and the hand-derived (size, payload) ------------------------------------------------
KA = {}
KA["empty"] = ({}, 0, b"")
KA["one_voxel"] = ({C: V}, 17, nb(V, 0x80) + nb(V, 0x01) * 15 + nb(V))  # 85 bytes
KA["eight_equal_pruned_at_depth_15"] = ({k: V for k in block(C, 2, 0)}, 16, nb(V, 0x80) + nb(V, 0x01) * 14 + nb(V))
_ulp = _octet(C, {i: (W if i == 5 else V) for i in range(8)})
KA["eight_one_ulp_apart_not_pruned"] = (_ulp, 24, nb(W, 0x80) + nb(W, 0x01) * 14 + nb(W, 0xFF) +
                                        b"".join(nb(W if i == 5 else V) for i in range(8)))
KA["signed_zeros_keep_child_0"] = (_octet(C, {i: (NEG0 if i == 0 else POS0) for i in range(8)}), 16,
                                   nb(NEG0, 0x80) + nb(NEG0, 0x01) * 14 + nb(NEG0))
KA["signed_zeros_reversed"] = (_octet(C, {i: (POS0 if i == 0 else NEG0) for i in range(8)}), 16,
                               nb(POS0, 0x80) + nb(POS0, 0x01) * 14 + nb(POS0))
KA["uniform_brick_leaf_at_depth_13"] = ({k: V for k in block(C, 8, 0)}, 14, nb(V, 0x80) + nb(V, 0x01) * 12 + nb(V))
# one depth-14 node with three depth-15 children: A {1: -1, 2: -0.0, 5: +0.0} holds -0.0 (the earliest of the tie), B at
# x + 2 {0: 0.25, 7: 0.25} holds 0.25, D at y + 2 {3: +0.0, 4: -0.0} holds +0.0; the depth-14 node and above hold 0.25
_ties = {**_octet(C, {1: -1.0, 2: NEG0, 5: POS0}), **_octet((K0 + 2, K0, K0), {0: 0.25, 7: 0.25}),
         **_octet((K0, K0 + 2, K0), {3: POS0, 4: NEG0})}
KA["inner_values_are_the_largest_child_earliest_on_ties"] = (
    _ties, 25, nb(0.25, 0x80) + nb(0.25, 0x01) * 13 + nb(0.25, 0x07) + nb(NEG0, 0x26) + nb(-1.0) + nb(NEG0) + nb(POS0) +
    nb(0.25, 0x81) + nb(0.25) + nb(0.25) + nb(POS0, 0x18) + nb(POS0) + nb(NEG0))
KA["both_ends_of_the_key_space"] = ({(0, 0, 0): F32(1.5), (65535, 65535, 65535): F32(-2.0)}, 33,
                                    nb(1.5, 0x81) + nb(1.5, 0x01) * 15 + nb(1.5) + nb(-2.0, 0x80) * 15 + nb(-2.0))


def _arrays(vox):
    keys = sorted(vox, key=_pack)
    return np.array([_pack(k) for k in keys], np.uint64), np.array([vox[k] for k in keys], F32)


def _oracle(vox, res=RES):
    return fr.full_octree(*_arrays(vox), res)


def _write_parse(t, tmp_path, name="o.ot"):
    path = str(tmp_path / name)
    t.write(path)
    return path, ls.read_octomap_full(path)


def _random_voxels(rng, n_blocks):
    """Aligned blocks of 1, 2, 4 or 8 voxels per axis, each of one value or of values drawn from a few (so that some
    octets compare equal and some do not), some with signed zeros."""
    vox = {}
    choices = np.array([V, W, -V, 0.0, -0.0, 1.0, 2.5], F32)
    for _ in range(n_blocks):
        n = int(rng.choice([1, 2, 4, 8]))
        k0 = tuple(int(x) // n * n for x in rng.integers(K0 - 40, K0 + 40, 3))
        mode = rng.integers(0, 3)
        for k in block(k0, n, 0):
            if mode == 0:
                vox[k] = choices[0]
            elif mode == 1:
                vox[k] = choices[rng.integers(3, 5)]
            else:
                vox[k] = choices[rng.integers(0, len(choices))]
    return vox


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(KA))
def test_oracle_known_answers(name, tmp_path):
    vox, size, payload = KA[name]
    t = _oracle(vox)
    assert (t.nodes, t.payload) == (size, payload)
    assert restate(vox) == (size, payload)
    path, p = _write_parse(t, tmp_path)
    assert open(path, "rb").read() == ot_bytes(size, payload)
    assert (p["nodes"], p["payload"], p["resolution"]) == (size, payload, RES)
    assert t.leaves == len(p["values"])
    k, v = fr.expand(p)
    wk, wv = _arrays(vox)
    # the voxels come back equal as floats; bit for bit except below a collapsed octet of signed zeros (child 0's bits)
    assert np.array_equal(k, wk) and np.array_equal(v, wv)
    assert np.array_equal(_bits(v), _bits(wv)) == (not name.startswith("signed_zeros"))


def test_one_voxel_is_85_bytes():
    assert len(KA["one_voxel"][2]) == 85


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_restatement_on_random_voxels(seed, tmp_path):
    vox = _random_voxels(np.random.default_rng(seed), 60)
    t = _oracle(vox)
    assert (t.nodes, t.payload) == restate(vox)
    _, p = _write_parse(t, tmp_path)
    k, v = fr.expand(p)
    wk, wv = _arrays(vox)
    assert np.array_equal(k, wk) and np.array_equal(v, wv)
    assert p["nodes"] < len(vox) + 16 * 60  # pruning happened


def test_oracle_on_the_12_scan_map(full_scans, tmp_path):
    """The occupancy oracle's map of the 12 scans at the defaults (0.075 m, 20 m); the GPU tests compare the device with
    the oracle at 0.1 m unlimited too."""
    scans, poses = full_scans
    o = oc.OccupancyMap()
    for k in range(len(scans)):
        o.insert_scan(scans[k], poses[k])
    k, v = o.download()
    t = fr.of_map(o)
    path, p = _write_parse(t, tmp_path)
    assert p["nodes"] == t.nodes and p["payload"] == t.payload and len(t.payload) == 5 * t.nodes
    ek, ev = fr.expand(p)
    assert np.array_equal(ek, k) and np.array_equal(_bits(ev), _bits(v)) and len(k) > 1_000_000
    # the restatement on a part of the map: the voxels of the depth-12 node (16 voxels per axis) of the middle voxel
    node = lambda x: (x & np.uint64(0xFFFF)) >> np.uint64(4) | ((x >> np.uint64(20)) & np.uint64(0xFFF)) << np.uint64(12) | (  # noqa
        (x >> np.uint64(36)) << np.uint64(24))
    sel = node(k) == node(k[len(k) // 2])
    part = {(int(x) & 0xFFFF, (int(x) >> 16) & 0xFFFF, int(x) >> 32): F32(y) for x, y in zip(k[sel], v[sel])}
    assert len(part) > 100
    assert (_oracle(part).nodes, _oracle(part).payload) == restate(part)


def _bt_of_full_leaves(p, l_occ):
    """The .bt (size, payload) of a parsed .ot: its leaves thresholded at l_occ, then pruned by state."""
    root = {}
    for k, d, v in zip(p["keys"], p["depths"], p["values"]):
        k = tuple(int(x) for x in k)
        node = root
        for dd in range(int(d) - 1):
            node = node.setdefault(child(k, dd), {})
        node[child(k, int(d) - 1)] = OCC if v >= l_occ else FREE

    def prune(n, d):
        for i in list(n):
            if isinstance(n[i], dict):
                n[i] = prune(n[i], d + 1)
        if d > 0 and len(n) == 8 and all(not isinstance(c, dict) for c in n.values()) and len(set(n.values())) == 1:
            return n[0]
        return n

    def write(n, out):
        out += pair({i: INNER if isinstance(c, dict) else c for i, c in n.items()})
        for i in sorted(n):
            if isinstance(n[i], dict):
                write(n[i], out)

    def count(n):
        return 1 + sum(count(c) if isinstance(c, dict) else 1 for c in n.values())

    if not len(p["values"]):
        return 0, b""
    root = prune(root, 0)
    out = bytearray()
    write(root, out)
    return count(root), bytes(out)


@pytest.mark.parametrize("name", sorted(KA) + [f"random_{s}" for s in range(3)])
def test_thresholded_leaves_give_the_bt_tree(name, tmp_path):
    vox = KA[name][0] if name in KA else _random_voxels(np.random.default_rng(100 + int(name[7:])), 60)
    _, p = _write_parse(_oracle(vox), tmp_path)
    for threshold in (0.7, 0.5, 0.56):  # the defaults, zero (between the signed zeros and 0.25), between 0.25 and 1.0
        bt = ot_oracle.octree(*_arrays(vox), RES, threshold)
        assert _bt_of_full_leaves(p, oc.logodds(threshold)) == (bt.nodes, bt.payload)


def _malformed(tmp_path):
    vox = KA["eight_one_ulp_apart_not_pruned"][0]
    good = tmp_path / "good.ot"
    _oracle(vox).write(str(good))
    data = good.read_bytes()
    head, payload = data[: -24 * 5], data[-24 * 5:]
    assert head.endswith(b"data\n") and b"size 24\n" in head
    leaf = payload[:-5]
    return {
        "first_line": data.replace(b"# Octomap OcTree file", b"# Octomap OcTree binary file", 1),
        "tree_type": data.replace(b"id OcTree", b"id ColorOcTree"),
        "stamped_tree_type": data.replace(b"id OcTree", b"id OcTreeStamped"),
        "no_size": data.replace(b"size 24\n", b""),
        "bad_res": data.replace(b"res 0.1", b"res x"),
        "no_data_line": head.replace(b"data\n", b""),
        "truncated": head + payload[:-2],
        "size_too_large": data.replace(b"size 24", b"size 25"),
        "size_too_small": data.replace(b"size 24", b"size 23"),
        "children_at_depth_16": head.replace(b"size 24", b"size 25") + leaf + nb(V, 0x01) + nb(V),
        "res_0": data.replace(b"res 0.1", b"res 0"),
        "res_negative": data.replace(b"res 0.1", b"res -0.1"),
        "res_inf": data.replace(b"res 0.1", b"res inf"),
        "res_nan": data.replace(b"res 0.1", b"res nan"),
        "leaf_nan": head + leaf + nb(F32(np.nan)),
        "leaf_inf": head + leaf + nb(F32(np.inf)),
        "leaf_minus_inf": head + leaf + nb(F32(-np.inf)),
    }


def test_parser_round_trips_and_refuses_malformed_files(tmp_path):
    good = tmp_path / "good.ot"
    _oracle(KA["eight_one_ulp_apart_not_pruned"][0]).write(str(good))
    p = ls.read_octomap_full(str(good))
    assert p["nodes"] == 24 and p["payload"] == KA["eight_one_ulp_apart_not_pruned"][2]
    (tmp_path / "trailing.ot").write_bytes(good.read_bytes() + b"\x00" * 7)  # bytes after the tree are ignored
    assert ls.read_octomap_full(str(tmp_path / "trailing.ot"))["payload"] == p["payload"]
    (tmp_path / "nan_inner.ot").write_bytes(ot_bytes(*tree_of([(C, 16, V)], inner=F32(np.nan))))
    assert np.array_equal(ls.read_octomap_full(str(tmp_path / "nan_inner.ot"))["values"], [V])  # inner values unused
    for name, blob in _malformed(tmp_path).items():
        path = tmp_path / (name + ".ot")
        path.write_bytes(blob)
        with pytest.raises(ValueError):
            ls.read_octomap_full(str(path))
    with pytest.raises(ValueError):  # a .bt is not a .ot
        ot_oracle.octree(*_arrays(KA["one_voxel"][0]), RES).write(str(tmp_path / "x.bt"))
        ls.read_octomap_full(str(tmp_path / "x.bt"))


# ---- GPU ------------------------------------------------------------------------------------------------------------
L = ls.lib


def _load(ctx, vox, params=None, **kw):
    """A device map holding exactly the voxels {key: float32}: an unpruned payload read into it."""
    dev = ls.OccupancyMap(ctx, **dict(resolution=RES, **(params or {})), **kw)
    size, payload = unpruned(vox)
    dev.read_full_octree(payload, size, RES)
    return dev


def _known(dev):
    k, v, _ = dev.download(ls.OCC_KNOWN)
    return k, v


def _same_known(dev, k, v):
    dk, dv = _known(dev)
    return np.array_equal(dk, k) and np.array_equal(_bits(dv), _bits(v))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(KA))
def test_known_answers_on_the_device(gpu_ctx, name, tmp_path):
    vox, size, payload = KA[name]
    dev = _load(gpu_ctx, vox)
    assert _same_known(dev, *_arrays(vox))
    t = dev.full_octree()
    assert (t.nodes, t.payload) == (size, payload) and (size == 0 or t.device_ms > 0)
    assert dev.save_octomap_full(str(tmp_path / "d.ot")) == size
    _oracle(vox).write(str(tmp_path / "o.ot"))
    assert (tmp_path / "d.ot").read_bytes() == (tmp_path / "o.ot").read_bytes() == ot_bytes(size, payload)
    st = ls.FullOctreeStats()
    assert L().ls_occupancy_build_full_octree(dev._h, ctypes.byref(st)) == 0
    p = ls.read_octomap_full(str(tmp_path / "d.ot"))
    assert (st.nodes, st.leaves, st.payload_bytes) == (size, len(p["values"]), 5 * size)
    dev.close()


@pytest.mark.gpu
def test_known_answer_inserted_as_scans(gpu_ctx, tmp_path):
    """A map built by inserts (not by a read): two occupied octets, one hit twice, and a free voxel."""
    params = dict(resolution=RES, max_range=0.05)
    vox = {**block(C, 2, OCC), **block((K0 + 2, K0, K0), 2, OCC), (K0 - 1, K0, K0): FREE}
    ring = gpu_ctx.create_map(2, 1024)
    dev, o = ls.OccupancyMap(gpu_ctx, **params), oc.OccupancyMap(**params)
    for cloud, T in _voxel_scans(vox, True):
        dev.insert_scan(ring, ring.push_scan(cloud, np.zeros((len(cloud), 3), F32)), T)
        o.insert_scan(cloud, T)
    k, v = o.download()
    assert _same_known(dev, k, v)
    t, ot = dev.full_octree(), fr.of_map(o)
    assert (t.nodes, t.payload) == (ot.nodes, ot.payload) and t.nodes > 16
    ring.close()
    dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("params", [dict(), dict(resolution=0.1, max_range=-1.0)], ids=["defaults", "res0.1_unlimited"])
def test_full_scan_maps_match_the_oracle_and_round_trip(gpu_ctx, full_scans, params, tmp_path):
    scans, poses = full_scans
    orig, ring = _full_map(gpu_ctx, full_scans, params, len(scans))
    k, v = _known(orig)
    res = orig.params.resolution
    t = orig.full_octree()
    ot = fr.full_octree(k, v, res)
    assert (t.nodes, t.payload) == (ot.nodes, ot.payload)
    path, bt = str(tmp_path / "orig.ot"), str(tmp_path / "orig.bt")
    orig.save_octomap_full(path)
    ot.write(str(tmp_path / "oracle.ot"))
    assert open(path, "rb").read() == (tmp_path / "oracle.ot").read_bytes()
    orig.save_octomap(bt)
    p = ls.read_octomap_full(path)
    for cap in (0, 16):
        for how in ("file", "payload"):
            dev = ls.OccupancyMap(gpu_ctx, initial_capacity=cap, **params)
            st = dev.read_octomap_full(path) if how == "file" else dev.read_full_octree(p["payload"], p["nodes"], res)
            assert cap == 0 or st.bricks > 16
            assert _same_known(dev, k, v) and st.known_voxels == len(k) > 1_000_000
            assert (st.nodes, st.inner_nodes, st.free_leaves + st.occupied_leaves) == (
                t.nodes, t.nodes - len(p["values"]), len(p["values"]))
            assert st.occupied_leaves == int((p["values"] >= L_OCC).sum()) and dev.params.resolution == res
            dev.save_octomap_full(str(tmp_path / "back.ot"))
            assert (tmp_path / "back.ot").read_bytes() == open(path, "rb").read()
            dev.save_octomap(str(tmp_path / "back.bt"))
            assert (tmp_path / "back.bt").read_bytes() == open(bt, "rb").read()
            if how == "file":
                _same_queries(dev, orig, scans, poses, res)
            dev.close()
    orig.close()
    ring.close()


@pytest.mark.gpu
@pytest.mark.parametrize("params", [dict(), dict(resolution=0.1, max_range=15.0)], ids=["defaults", "res0.1"])
def test_a_saved_map_resumes_mapping_exactly(gpu_ctx, full_scans, params, tmp_path):
    scans, poses = full_scans
    a, ring = _full_map(gpu_ctx, full_scans, params, 6)
    path = str(tmp_path / "six.ot")
    a.save_octomap_full(path)
    a.close()
    b = ls.OccupancyMap(gpu_ctx, initial_capacity=64, **params)
    b.read_octomap_full(path)
    c = ls.OccupancyMap(gpu_ctx, **params)
    nrm = np.zeros((131072, 3), F32)
    for k in range(12):
        sid = ring.push_scan(scans[k], nrm)
        if k >= 6:
            sb = b.insert_scan(ring, sid, poses[k])
        sc = c.insert_scan(ring, sid, poses[k])
        if k >= 6:
            assert (sb.free_updates, sb.occupied_updates, sb.known_voxels) == (
                sc.free_updates, sc.occupied_updates, sc.known_voxels)
    assert _same_known(b, *_known(c))
    assert b.full_octree()[:2] == c.full_octree()[:2]
    tb, tc = b.octree(), c.octree()
    assert (tb.nodes, tb.payload) == (tc.nodes, tc.payload)
    for m in (b, c):
        m.save_octomap_full(str(tmp_path / f"{id(m)}.ot"))
    assert (tmp_path / f"{id(b)}.ot").read_bytes() == (tmp_path / f"{id(c)}.ot").read_bytes()
    b.close()
    c.close()
    ring.close()


@pytest.mark.gpu
def test_one_hit_then_four_misses_ends_free_through_ot_and_occupied_through_bt(gpu_ctx, tmp_path):
    params = dict(resolution=RES, max_range=0.05)
    hit, = _voxel_scans({C: OCC}, False)
    miss, = _voxel_scans({C: FREE}, False)
    ring = gpu_ctx.create_map(2, 1024)
    push = lambda s: ring.push_scan(s[0], np.zeros((len(s[0]), 3), F32))  # noqa: E731
    never = ls.OccupancyMap(gpu_ctx, **params)
    never.insert_scan(ring, push(hit), hit[1])
    never.save_octomap_full(str(tmp_path / "one.ot"))
    never.save_octomap(str(tmp_path / "one.bt"))
    assert _known(never)[1][0] == oc.logodds(0.9)
    via_ot, via_bt = ls.OccupancyMap(gpu_ctx, **params), ls.OccupancyMap(gpu_ctx, **params)
    via_ot.read_octomap_full(str(tmp_path / "one.ot"))
    via_bt.read_octomap(str(tmp_path / "one.bt"))
    assert _known(via_bt)[1][0] == oc.logodds(0.97)
    sid = push(miss)
    for _ in range(4):
        for m in (never, via_ot, via_bt):
            m.insert_scan(ring, sid, miss[1])
    want = F32(oc.logodds(0.9))
    for _ in range(4):
        want = F32(want + F32(oc.logodds(0.4)))
    assert _bits(_known(never)[1]) == _bits(_known(via_ot)[1]) == _bits(np.array([want], F32))
    assert abs(float(want) - 0.575) < 1e-3 and abs(float(_known(via_bt)[1][0]) - 1.854) < 1e-3
    centre = oc.centres([_pack(C)], RES).astype(np.float64)
    assert via_ot.cell_status(centre)[0][0] == ls.CELL_FREE == never.cell_status(centre)[0][0]
    assert via_bt.cell_status(centre)[0][0] == ls.CELL_OCCUPIED
    for m in (never, via_ot, via_bt):
        m.close()
    ring.close()


_B = (K0 + 64, K0, K0)  # a brick-aligned depth-12 node: 64 voxels per axis
FOREIGN = {  # name: leaves (first key, depth, value) and the value of every inner node (None: the largest child)
    "unpruned_equal_octet": ([(k, 16, V) for k in block(C, 2, 0)], None),
    "values_outside_the_clamps": ([(C, 16, F32(5.0)), ((K0 + 1, K0, K0), 16, F32(-3.0)), ((K0 - 8, K0, K0), 13, F32(4.5))],
                                  None),
    "inconsistent_inner_values": ([(C, 16, V), ((K0 + 1, K0 + 1, K0), 16, -V), (_B, 13, W)], F32(np.nan)),
    "leaf_at_depth_9": ([(C, 9, F32(-0.5))], None),
    "mixed_leaves_at_depths_13_to_16": ([(_B, 13, F32(0.5)), ((_B[0] + 8, _B[1], _B[2]), 14, V),
                                         ((_B[0] + 12, _B[1], _B[2]), 15, NEG0), ((_B[0] + 14, _B[1] + 2, _B[2]), 16, W),
                                         ((_B[0] + 15, _B[1] + 3, _B[2] + 1), 16, POS0),
                                         ((_B[0] + 32, _B[1] + 32, _B[2] + 32), 13, -V)], None),
    "both_ends_of_the_key_space": ([((0, 0, 0), 16, V), ((65535, 65535, 65535), 16, -V), ((65532, 0, 65532), 14, W),
                                    ((0, 65528, 0), 13, F32(1.0))], F32(7.0)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FOREIGN))
def test_foreign_payloads_load_as_the_reference_expands_them(gpu_ctx, name, tmp_path):
    items, inner = FOREIGN[name]
    size, payload = tree_of(items, inner)
    path = tmp_path / "in.ot"
    path.write_bytes(ot_bytes(size, payload))
    p = ls.read_octomap_full(str(path))
    k, v = fr.expand(p)
    params = dict(resolution=RES, max_range=0.05)
    for how in ("file", "payload"):
        dev = ls.OccupancyMap(gpu_ctx, **params)
        st = dev.read_octomap_full(str(path)) if how == "file" else dev.read_full_octree(payload, size, 0.1)
        assert _same_known(dev, k, v) and st.known_voxels == len(k)
        occ = v >= L_OCC
        ok, ov, _ = dev.download(ls.OCC_OCCUPIED)
        assert np.array_equal(ok, k[occ]) and np.array_equal(_bits(ov), _bits(v[occ]))
        assert (st.free_leaves, st.occupied_leaves) == (int((p["values"] < L_OCC).sum()), int((p["values"] >= L_OCC).sum()))
        t, ot = dev.full_octree(), fr.full_octree(k, v, RES)
        assert (t.nodes, t.payload) == (ot.nodes, ot.payload)
        if inner is None and name != "unpruned_equal_octet":  # a file as this library writes it comes back byte for byte
            assert t.payload == payload
        dev.close()
    # mapping on: the next insert clamps the loaded values, as the seeded oracle does
    dev = ls.OccupancyMap(gpu_ctx, **params)
    dev.read_octomap_full(str(path))
    o = rr.seed(oc.OccupancyMap(**params), k, v)
    ring = gpu_ctx.create_map(2, 1024)
    targets = {tuple(int(x) for x in it[0]): (OCC if i % 2 == 0 else FREE) for i, it in enumerate(items[:2])}
    for cloud, T in _voxel_scans(targets, False):
        sid = ring.push_scan(cloud, np.zeros((len(cloud), 3), F32))
        st = dev.insert_scan(ring, sid, T)
        ost = o.insert_scan(cloud, T)
        assert (st.free_updates, st.occupied_updates, st.known_voxels) == (
            ost["free_updates"], ost["occupied_updates"], ost["known_voxels"])
    assert _same_known(dev, *o.download())
    if name == "values_outside_the_clamps":
        lo = dict(zip(_known(dev)[0].tolist(), _known(dev)[1].tolist()))
        assert lo[_pack(C)] == F32(oc.logodds(0.97)) and lo[_pack((K0 + 1, K0, K0))] == F32(oc.logodds(0.12))
        assert lo[_pack((K0 - 8, K0, K0))] == F32(4.5)  # not touched: still verbatim
    ring.close()
    dev.close()


@pytest.mark.gpu
def test_refusals_leave_the_map_and_both_builds_unchanged(gpu_ctx, full_scans, tmp_path):
    dev, ring = _full_map(gpu_ctx, full_scans, dict(resolution=0.1, max_range=10.0), 2)
    before, tree, full = _download(dev), dev.octree(), dev.full_octree()
    bt_pay, ot_pay = np.zeros(len(tree.payload), np.uint8), np.zeros(len(full.payload), np.uint8)
    blobs = _malformed(tmp_path)
    blobs["depth_1_leaf"] = ot_bytes(2, nb(V, 0x01) + nb(V))  # 8^12 bricks
    for name, blob in blobs.items():
        path = tmp_path / (name + ".ot")
        path.write_bytes(blob)
        st = ls.OctomapReadStats()
        rc = L().ls_occupancy_read_octomap_full(dev._h, str(path).encode(), ctypes.byref(st))
        assert rc == (ls.LS_ERR_NOMEM if name == "depth_1_leaf" else ls.LS_ERR_ARG), name
        assert L().ls_occupancy_download_octree(dev._h, bt_pay.ctypes.data, len(bt_pay), None, None, 0) == 0, name
        assert L().ls_occupancy_download_full_octree(dev._h, ot_pay.ctypes.data, len(ot_pay)) == 0, name
        assert bt_pay.tobytes() == tree.payload and ot_pay.tobytes() == full.payload
    for args in ((b"", 5, 0.1), (nb(V), 1, 0.0), (nb(V), 1, float("nan")), (nb(V), -1, 0.1), (nb(V), 1, float("inf"))):
        with pytest.raises(ls.LsError):
            dev.read_full_octree(*args)
    assert dev.params.resolution == 0.1
    assert _same_downloads(_download(dev), before)
    assert dev.full_octree()[:2] == full[:2]
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_the_two_builds_are_cached_apart(gpu_ctx, full_scans, tmp_path):
    scans, poses = full_scans
    dev, ring = _full_map(gpu_ctx, full_scans, dict(resolution=0.1, max_range=10.0), 1)
    buf = np.zeros(1 << 26, np.uint8)  # outlives every download below

    def full_dl(f):
        return L().ls_occupancy_download_full_octree(dev._h, buf.ctypes.data, len(f.payload))

    def bt_dl(t):
        return L().ls_occupancy_download_octree(dev._h, buf.ctypes.data, len(t.payload), None, None, 0)

    assert full_dl(dev.full_octree()) == 0
    tree = dev.octree()
    full = dev.full_octree()
    assert len(tree.payload) < len(buf) and len(full.payload) < len(buf)
    assert bt_dl(tree) == 0 and full_dl(full) == 0  # the full build left the .bt build current, and the reverse
    tree = dev.octree()
    assert full_dl(full) == 0 and buf[:len(full.payload)].tobytes() == full.payload
    dev.insert_scan(ring, ring.push_scan(scans[1], np.zeros((131072, 3), F32)), poses[1])
    assert bt_dl(tree) == ls.LS_ERR_STATE and full_dl(full) == ls.LS_ERR_STATE
    for read in ("bt", "ot"):
        tree, full = dev.octree(), dev.full_octree()
        path = str(tmp_path / ("m." + read))
        (dev.save_octomap if read == "bt" else dev.save_octomap_full)(path)
        (dev.read_octomap if read == "bt" else dev.read_octomap_full)(path)
        assert bt_dl(tree) == ls.LS_ERR_STATE and full_dl(full) == ls.LS_ERR_STATE, read
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_full_tree_calls_between_batch_begin_and_end(full_scans, tmp_path):
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
    ot = str(tmp_path / "one.ot")
    src.save_octomap_full(ot)
    dev = ls.OccupancyMap(ctx)
    end = ring.begin_batch(problems, p)
    dev.read_octomap_full(ot)
    t = dev.full_octree()
    dev.save_octomap_full(str(tmp_path / "back.ot"))
    res = end()
    for a, b in zip(res, alone):
        assert a["rc"] == b["rc"] and np.array_equal(a["T"], b["T"])
    assert (tmp_path / "back.ot").read_bytes() == open(ot, "rb").read()
    assert t.payload == ls.read_octomap_full(ot)["payload"]
    assert _same_known(dev, *_known(src))
    for m in (src, dev):
        m.close()
    ring.close()
    ctx.close()


@pytest.mark.gpu
def test_host_layer_write_and_read_equal_the_abi(gpu_ctx, synth_mod, tmp_path):
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
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
    hk, hv = occ.voxels(1)
    path = str(tmp_path / "h.ot")
    occ.write_full(path)
    o = fr.full_octree(hk, hv, 0.1)
    o.write(str(tmp_path / "o.ot"))
    assert open(path, "rb").read() == (tmp_path / "o.ot").read_bytes() and len(hk) > 0
    nodes, payload = occ.write_data()
    assert (nodes, payload) == (o.nodes, o.payload)
    other = host.OccupancyMap(est, resolution=0.2, max_range=15.0)
    bad = tmp_path / "bad.ot"
    bad.write_bytes(b"# not octomap\n")
    assert other.read_full(str(bad)) is False and other.read_data(b"\x00", 1, 0.1) is False
    assert other.read_full(path) is True
    dev = ls.OccupancyMap(gpu_ctx, resolution=0.2, max_range=15.0)
    dev.read_octomap_full(path)
    k, v = _known(dev)
    ok, ov = other.voxels(1)
    assert np.array_equal(ok, k) and np.array_equal(_bits(ov), _bits(v)) and np.array_equal(k, hk)
    other.write_full(str(tmp_path / "h2.ot"))
    assert (tmp_path / "h2.ot").read_bytes() == open(path, "rb").read()
    third = host.OccupancyMap(est, resolution=0.3, max_range=15.0)
    assert third.read_data(payload, nodes, 0.1) is True
    tk, tv = third.voxels(1)
    assert np.array_equal(tk, hk) and np.array_equal(_bits(tv), _bits(hv))
    for m in (other, third, occ):
        m.close()
    est.close()
    dev.close()
