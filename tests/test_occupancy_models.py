"""The occupancy map under the sensor models it accepts: hit and miss probabilities, clamps, occupancy threshold,
resolution and max range other than laser_to_octomap's defaults.  Each named model is checked, on the CPU reference, to
reach the regime it is named for: log-odds landing exactly on the threshold, updates clamped against their direction,
maps where every known voxel is occupied or none is.  CPU: the oracle against an independent restatement that takes every
parameter, known answers, and the oracle's octree against a property check.  GPU: the device insert, queries, export and
.bt read bit for bit against the oracle at every model, laser_slam::OccupancyMap with seven distinct values, and the
parameter checks of ls_occupancy_create.  The rules are oracle/OCCUPANCY.md and oracle/OCTREE.md."""
import collections
import ctypes
import functools
import inspect
import math
import os
import re

import numpy as np
import pytest

import laser_slam_b200 as ls
import octomap_read_ref as rr
from oracle import occupancy as oc
from oracle import octree as ot_oracle
from oracle import queries as oq
from test_occupancy import (F32, K0, _bits, _key3, _pack, _rel, _same_map, _stats_dict, _tie_free_cloud, _translate,
                            cut_end, segment_cells)
from test_occupancy_queries import _same, _segments
from test_octomap import _same_tree
from test_octomap_read import _check_loaded

FREE, OCC = 1, 2  # the .bt leaf states
INF = float("inf")


# ---- the models ------------------------------------------------------------------------------------------------------
class Model(collections.namedtuple("Model", "hit miss clamp_min clamp_max threshold resolution max_range")):
    def params(self):
        """Keyword arguments of laser_slam_b200.OccupancyMap and oracle.occupancy.OccupancyMap."""
        return dict(resolution=self.resolution, prob_hit=self.hit, prob_miss=self.miss, clamp_min=self.clamp_min,
                    clamp_max=self.clamp_max, occupancy_threshold=self.threshold, max_range=self.max_range)


def M(hit=0.9, miss=0.4, clamp_min=0.12, clamp_max=0.97, threshold=0.7, resolution=0.1, max_range=15.0):
    return Model(hit, miss, clamp_min, clamp_max, threshold, resolution, max_range)


MODELS = {
    "defaults": M(),
    "hit_at_threshold": M(hit=0.7),
    "clamp_max_at_threshold": M(clamp_max=0.8, threshold=0.8),
    "clamp_min_at_threshold": M(miss=0.2, clamp_min=0.3, threshold=0.3),
    "return_to_zero": M(hit=0.75, miss=0.25, threshold=0.5),
    "inverted": M(hit=0.3, miss=0.8, clamp_min=0.05, clamp_max=0.95, threshold=0.6),
    "clamp_min_above_half": M(hit=0.52, clamp_min=0.55),
    "equal_clamps_free": M(clamp_min=0.6, clamp_max=0.6, threshold=0.7),
    "equal_clamps_occupied": M(clamp_min=0.6, clamp_max=0.6, threshold=0.6),
    "threshold_above_clamps": M(threshold=0.99),
    "res_0.05": M(resolution=0.05, max_range=8.0),
    "res_0.2": M(resolution=0.2),
    "res_1_30": M(resolution=1.0 / 30.0, max_range=6.0),
    "res_1.0": M(resolution=1.0, max_range=40.0),
    "range_0": M(max_range=0.0),
    "range_inf": M(resolution=0.2, max_range=INF),
    "range_unlimited": M(resolution=0.2, max_range=-1.0),
}
# models whose maps hold voxels with v == L_occ exactly: `>` in place of `>=` changes their answers
EQUALITY = ("hit_at_threshold", "clamp_max_at_threshold", "clamp_min_at_threshold", "return_to_zero",
            "equal_clamps_occupied")
FULL_SCANS = ("clamp_min_at_threshold", "equal_clamps_occupied")  # uniform regions: leaves at depth 12 and above
N_SCANS = {True: 2, False: 3}


def L(p):
    """Log-odds as the rules define them, computed here in Python: (float)log(p / (1 - p))."""
    return F32(math.log(p / (1.0 - p)))


def logodds_of(m):
    return dict(hit=L(m.hit), miss=L(m.miss), min=L(m.clamp_min), max=L(m.clamp_max), occ=L(m.threshold))


# ---- independent restatement of the sensor model: every parameter, float32 updates, clamps both ways ------------------
class Restated:
    def __init__(self, m):
        self.m, self.l = m, logodds_of(m)
        self.vox = {}

    def insert(self, pts, origin):
        """pts (n,4) in the world frame, origin the sensor position; returns the stats as oracle.occupancy does."""
        m, l = self.m, self.l
        occ, free = set(), set()
        o = np.asarray(origin, F32)
        cast = skipped = 0
        for p in np.asarray(pts, F32)[:, :3]:
            if not np.isfinite(p).all():
                skipped += 1
                continue
            k = _key3(p, m.resolution)
            if k is not None and k in occ:
                skipped += 1
                continue
            cast += 1
            d = (p - o).astype(F32)
            if m.max_range < 0 or math.sqrt(float(np.sum(d.astype(np.float64) ** 2))) <= m.max_range:
                free.update(segment_cells(o, p, m.resolution))
                if k is not None:
                    occ.add(k)
            else:
                free.update(segment_cells(o, cut_end(o, p, m.max_range), m.resolution))
        for k in occ | free:
            v = F32(self.vox.get(k, F32(0)) + (l["hit"] if k in occ else l["miss"]))
            if v < l["min"]:
                v = l["min"]
            if v > l["max"]:
                v = l["max"]
            self.vox[k] = v
        return dict(rays_cast=cast, rays_skipped=skipped, free_updates=len(free - occ), occupied_updates=len(occ),
                    known_voxels=len(self.vox))

    def download(self, which=oc.KNOWN):
        ks = sorted((k for k, v in self.vox.items() if which == oc.KNOWN or v >= self.l["occ"]),
                    key=lambda k: (k[2], k[1], k[0]))
        return np.array([_pack(k) for k in ks], np.uint64), np.array([self.vox[k] for k in ks], F32)


# ---- the scans and the oracle maps every model is checked on -----------------------------------------------------------
@functools.lru_cache(maxsize=None)
def scans(full):
    """(clouds, poses): synthetic scans of sequence 0, every eighth azimuth unless `full`.  The last point of each cloud
    is the sensor origin itself, so a zero max range still makes the origin voxel known."""
    from laser_slam_b200 import synth
    synth.build()
    n = N_SCANS[full]
    truth, _ = synth.trajectory(0, n + 1)
    clouds = []
    for k in range(n):
        c = synth.scan(truth[k], 0, k)
        c = c[0] if full else synth.subsample(*c, 8)[0]
        c = c.copy()
        c[-1] = (0.0, 0.0, 0.0, 1.0)
        clouds.append(c)
    return clouds, [truth[k].astype(F32) for k in range(n)]


def scans_of(name):
    return scans(name in FULL_SCANS)


@functools.lru_cache(maxsize=None)
def oracle_map(name):
    """(oracle.queries.OccupancyMap after the model's scans, the stats of each insert)."""
    o = oq.OccupancyMap(**MODELS[name].params())
    clouds, poses = scans_of(name)
    return o, [o.insert_scan(c, T) for c, T in zip(clouds, poses)]


def equality_keys(name):
    k, v = oracle_map(name)[0].download()
    return k[v == logodds_of(MODELS[name])["occ"]]


def _bricks(keys):
    k = np.asarray(keys, np.uint64)
    return np.unique(((k & np.uint64(0xFFFF)) >> np.uint64(3)) | (((k >> np.uint64(16)) & np.uint64(0xFFFF)) >> np.uint64(3))
                     << np.uint64(13) | ((k >> np.uint64(32)) >> np.uint64(3)) << np.uint64(26))


# What each model reaches on its scans, from the CPU reference: (keys, log-odds, occupied keys, the model's L, stats)
def _reaches(name, k, v, occ, l, st):
    n = len(k)
    if name == "defaults":
        assert 0 < len(occ) < n and not (v == l["occ"]).any()
    elif name == "hit_at_threshold":
        assert l["hit"] == l["occ"] and (v == l["occ"]).sum() > 100 and len(occ) < n
    elif name == "clamp_max_at_threshold":
        assert l["max"] == l["occ"] and (v == l["occ"]).sum() > 100 and (v[np.isin(k, occ)] == l["occ"]).all()
    elif name == "clamp_min_at_threshold":
        assert l["min"] == l["occ"] and len(occ) == n and (v == l["occ"]).sum() > n // 2
    elif name == "return_to_zero":
        assert l["occ"] == 0 and l["hit"] == -l["miss"] and (v == 0).sum() > 100
        assert len(occ) == (v >= 0).sum() < n
    elif name == "inverted":
        assert l["hit"] < l["occ"] <= l["miss"]
        assert (v == l["max"]).sum() > 100 and (v == l["hit"]).sum() > 100 and 0 < len(occ) < n
    elif name == "clamp_min_above_half":
        assert 0 < l["hit"] < l["min"] and (v == l["min"]).sum() > 100 and v.min() == l["min"]
        assert (v > l["min"]).any()
    elif name == "equal_clamps_free":
        assert l["min"] == l["max"] < l["occ"] and (v == l["min"]).all() and len(occ) == 0
    elif name == "equal_clamps_occupied":
        assert l["min"] == l["max"] == l["occ"] and (v == l["occ"]).all() and len(occ) == n
    elif name == "threshold_above_clamps":
        assert l["occ"] > l["max"] and (v == l["max"]).any() and len(occ) == 0
    elif name.startswith("res_"):
        assert len(occ) > 100 and len(_bricks(k)) > (20 if name == "res_1.0" else 500)
        ks = np.stack([(k >> np.uint64(s)) & np.uint64(0xFFFF) for s in (0, 16)], 1).astype(np.int64)
        assert (ks < K0).any() and (ks >= K0).any()  # keys on both sides of the origin
    elif name == "range_0":  # the origin voxel of each scan, nothing free
        assert n == len(occ) == len({_key3(T[:3, 3], 0.1) for T in scans_of(name)[1]}) and n > 0
        assert all(s["free_updates"] == 0 and s["rays_cast"] > 10000 for s in st)
    elif name == "range_inf":   # behaves as unlimited
        kk, vv = oracle_map("range_unlimited")[0].download()
        assert np.array_equal(k, kk) and np.array_equal(_bits(v), _bits(vv)) and n > 100000
        limited = oc.OccupancyMap(**MODELS["range_inf"]._replace(max_range=15.0).params())
        for c, T in zip(*scans_of(name)):
            limited.insert_scan(c, T)
        assert limited.size() < n
    elif name == "range_unlimited":
        assert n > 100000 and 0 < len(occ) < n
    else:
        raise AssertionError(f"no regime check for {name}")


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_every_model_has_a_regime_check():
    assert set(EQUALITY) <= set(MODELS) and set(FULL_SCANS) <= set(MODELS)
    for name, m in MODELS.items():
        assert 0 < m.clamp_min <= m.clamp_max < 1 and m.resolution > 0, name


@pytest.mark.parametrize("name", sorted(MODELS))
def test_models_reach_their_regimes(name):
    o, st = oracle_map(name)
    k, v = o.download()
    occ = o.download(oc.OCCUPIED)[0]
    l = logodds_of(MODELS[name])
    assert np.array_equal(occ, k[v >= l["occ"]])
    _reaches(name, k, v, occ, l, st)
    if name in EQUALITY:
        assert len(equality_keys(name)) > 0


@pytest.mark.parametrize("name", sorted(MODELS))
def test_oracle_matches_restatement(name):
    m = MODELS[name]
    rng = np.random.default_rng(71)
    origin = np.array([0.013, -0.021, 0.037], F32)
    T = _translate(origin)
    o, r = oc.OccupancyMap(**m.params()), Restated(m)
    at_origin = np.array([[origin[0], origin[1], origin[2], 1.0]], F32)
    n_eq = 0
    for _ in range(3):
        cloud = _tie_free_cloud(rng, 150, m.resolution, origin, m.max_range)
        cloud = np.concatenate([cloud, cloud[:10], at_origin])   # repeated endpoints, a point at the sensor
        st = o.insert_scan(cloud - np.array([*origin, 0], F32), T)
        assert st == r.insert(cloud, origin)
        assert _same_map(o.download(), r.download())
        assert _same_map(o.download(oc.OCCUPIED), r.download(oc.OCCUPIED))
        n_eq += int((o.download()[1] == r.l["occ"]).sum())
    assert o.size() > (0 if name == "range_0" else 100)
    if name in ("hit_at_threshold", "clamp_max_at_threshold", "clamp_min_at_threshold", "equal_clamps_occupied"):
        assert n_eq > 0


# Known answers at resolution 0.1, unlimited range: a ray from the corner (0, 0, 0) to (0.35, 0.05, 0.05) misses voxels
# x = 0, 1, 2 and hits x = 3.  Expected per model: (value of a missed voxel, its state), (value of the hit voxel, its state),
# the values named by the model's log-odds.
ONE = {
    "defaults": (("miss", FREE), ("hit", OCC)),
    "hit_at_threshold": (("miss", FREE), ("hit", OCC)),
    "clamp_max_at_threshold": (("miss", FREE), ("max", OCC)),
    "clamp_min_at_threshold": (("min", OCC), ("hit", OCC)),
    "return_to_zero": (("miss", FREE), ("hit", OCC)),
    "inverted": (("miss", OCC), ("hit", FREE)),
    "clamp_min_above_half": (("min", FREE), ("min", FREE)),
    "equal_clamps_free": (("min", FREE), ("max", FREE)),
    "equal_clamps_occupied": (("min", OCC), ("max", OCC)),
    "threshold_above_clamps": (("miss", FREE), ("hit", FREE)),
}


def _known(o):
    """{packed key: (log-odds, FREE / OCC as the OCCUPIED download says)}."""
    k, v = o.download()
    occ = set(int(x) for x in o.download(oc.OCCUPIED)[0])
    return {int(a): (b, OCC if int(a) in occ else FREE) for a, b in zip(k, v)}


@pytest.mark.parametrize("name", sorted(ONE))
def test_one_hit_and_one_miss(name):
    m = MODELS[name]._replace(resolution=0.1, max_range=-1.0)
    l = logodds_of(m)
    o = oc.OccupancyMap(**m.params())
    st = o.insert_scan(np.array([[0.35, 0.05, 0.05, 1]], F32), np.eye(4, dtype=F32))
    assert st["free_updates"] == 3 and st["occupied_updates"] == 1
    (mv, ms), (hv, hs) = ONE[name]
    want = {_rel(i, 0, 0): (l[mv], ms) for i in range(3)}
    want[_rel(3, 0, 0)] = (l[hv], hs)
    got = _known(o)
    assert {k: (_bits(np.array([v]))[0], s) for k, (v, s) in got.items()} == \
        {k: (_bits(np.array([v]))[0], s) for k, (v, s) in want.items()}


def test_return_to_zero_two_scans():
    m = MODELS["return_to_zero"]._replace(max_range=-1.0)
    o = oc.OccupancyMap(**m.params())
    o.insert_scan(np.array([[0.35, 0.05, 0.05, 1]], F32), np.eye(4, dtype=F32))   # hits x = 3
    o.insert_scan(np.array([[0.55, 0.05, 0.05, 1]], F32), np.eye(4, dtype=F32))   # misses it
    got = _known(o)
    v, s = got[_rel(3, 0, 0)]
    assert _bits(np.array([v]))[0] == 0 and s == OCC   # +0.0 exactly, occupied: 0 >= L_occ = 0
    l = logodds_of(m)
    assert F32(l["miss"] + l["miss"]) < l["min"]   # missed twice: clamped
    assert all(got[_rel(i, 0, 0)] == (l["min"], FREE) for i in range(3)) and got[_rel(5, 0, 0)] == (l["hit"], OCC)
    assert got[_rel(4, 0, 0)] == (l["miss"], FREE) and len(got) == 6


def test_zero_max_range_at_the_origin_and_one_metre_away():
    l_hit = L(0.9)
    o = oc.OccupancyMap(resolution=0.1, max_range=0.0)
    T = _translate([0.05, 0.05, 0.05])
    st = o.insert_scan(np.array([[0, 0, 0, 1]], F32), T)   # at the sensor: in range, occupied, no free cell
    assert st == dict(rays_cast=1, rays_skipped=0, free_updates=0, occupied_updates=1, known_voxels=1)
    assert _known(o) == {_rel(0, 0, 0): (l_hit, OCC)}
    o = oc.OccupancyMap(resolution=0.1, max_range=0.0)
    st = o.insert_scan(np.array([[1.0, 0, 0, 1]], F32), T)  # cut to a zero-length ray: cast, nothing known
    assert st == dict(rays_cast=1, rays_skipped=0, free_updates=0, occupied_updates=0, known_voxels=0)


def _leaf_states(bt):
    """(the parsed file, keys and FREE / OCC states of every voxel below a leaf, ascending keys)."""
    p = ls.read_octomap(bt)
    k, s = rr.expand(p, F32(FREE), F32(OCC))
    return p, k, s.astype(np.uint8)


def _fully_pruned(p):
    """No node at depth 1..15 has eight leaf children of one state (the root is never pruned)."""
    keys, depths, states = p["keys"].astype(np.uint64), p["depths"].astype(np.int64), p["states"]
    sel = depths >= 2
    shift = (17 - depths[sel]).astype(np.uint64)
    mask = ~((np.uint64(1) << shift) - np.uint64(1))
    kk = keys[sel] & mask[:, None]
    parent = (kk[:, 0] | (kk[:, 1] << np.uint64(16)) | (kk[:, 2] << np.uint64(32)) |
              ((depths[sel] - 1).astype(np.uint64) << np.uint64(48)))
    u, inv, n = np.unique(parent, return_inverse=True, return_counts=True)
    n_free = np.bincount(inv, weights=(states[sel] == FREE), minlength=len(u))
    return not ((n == 8) & ((n_free == 0) | (n_free == 8))).any()


@pytest.mark.parametrize("name", sorted(MODELS))
def test_oracle_octree_properties(name, tmp_path):
    o, _ = oracle_map(name)
    m = MODELS[name]
    k, v = o.download()
    bt = str(tmp_path / "o.bt")
    t = ot_oracle.of_map(o)
    t.write(bt)
    p, lk, ls_ = _leaf_states(bt)
    assert np.array_equal(lk, k)                                       # covered voxels == known voxels
    assert np.array_equal(ls_, np.where(v >= L(m.threshold), OCC, FREE))  # every leaf's state is its voxels' state
    assert _fully_pruned(p)
    assert p["nodes"] == t.nodes and len(p["depths"]) > 0
    if name in FULL_SCANS:
        assert (p["depths"] <= 12).any()


def test_default_parameters_agree():
    p = ls.OccupancyParams()
    ls.lib().ls_occupancy_default_params(ctypes.byref(p))
    assert {f: getattr(p, f) for f in oc.DEFAULTS} == oc.DEFAULTS and p.initial_capacity == 0
    from laser_slam_b200 import host
    sig = inspect.signature(host.OccupancyMap.__init__).parameters
    assert {f: sig[f].default for f in oc.DEFAULTS} == oc.DEFAULTS
    hpp = open(os.path.join(os.path.dirname(ls.__file__), "..", "include", "laser_slam", "occupancy_map.hpp")).read()
    cxx = {n: float(v) for n, v in re.findall(r"double (\w+) = ([0-9.]+);", hpp)}
    names = dict(resolution="resolution", prob_hit="probability_hit", prob_miss="probability_miss",
                 clamp_min="clamping_thres_min", clamp_max="clamping_thres_max", occupancy_threshold="occupancy_thres",
                 max_range="sensor_max_range")
    assert {f: cxx[names[f]] for f in oc.DEFAULTS} == oc.DEFAULTS


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=sorted(MODELS))
def model_maps(request, gpu_ctx):
    """The device map and the oracle map of a model after its scans, and both inserts' stats."""
    name = request.param
    m = MODELS[name]
    clouds, poses = scans_of(name)
    o, ostats = oracle_map(name)
    ring = gpu_ctx.create_map(2, 131072)
    dev = ls.OccupancyMap(gpu_ctx, **m.params())
    stats = [_stats_dict(dev.insert_scan(ring, ring.push_scan(c, np.zeros((len(c), 3), F32)), T))
             for c, T in zip(clouds, poses)]
    yield dict(name=name, m=m, dev=dev, o=o, stats=stats, ostats=ostats, poses=poses, clouds=clouds)
    dev.close()
    ring.close()


@pytest.mark.gpu
def test_insert_matches_the_oracle(model_maps):
    dev, o, m = model_maps["dev"], model_maps["o"], model_maps["m"]
    assert model_maps["stats"] == model_maps["ostats"]
    k, v, cen = dev.download(ls.OCC_KNOWN)
    assert _same_map((k, v), o.download())
    assert np.array_equal(_bits(cen[:, :3]), _bits(oc.centres(k, m.resolution))) and (cen[:, 3] == 1).all()
    k, v, cen = dev.download(ls.OCC_OCCUPIED)
    assert _same_map((k, v), o.download(oc.OCCUPIED))
    assert np.array_equal(_bits(cen[:, :3]), _bits(oc.centres(k, m.resolution)))
    assert dev.size(ls.OCC_KNOWN) == o.size() and dev.size(ls.OCC_OCCUPIED) == o.size(oc.OCCUPIED)


@pytest.mark.gpu
def test_queries_match_the_oracle(model_maps):
    name, dev, o, m = model_maps["name"], model_maps["dev"], model_maps["o"], model_maps["m"]
    poses = model_maps["poses"]
    rng = np.random.default_rng(81)
    keys, _ = o.download()
    eq = equality_keys(name)
    eq_set = set(int(x) for x in eq)
    assert (name in EQUALITY) == (len(eq) > 0)
    cen = oc.centres(keys, m.resolution).astype(np.float64)
    # cells: up to 200 000 known voxels, every voxel on the threshold up to as many, random points around them
    pick = lambda a: a if len(a) <= 200_000 else a[rng.choice(len(a), 200_000, replace=False)]  # noqa: E731
    pts = np.concatenate([pick(cen), pick(oc.centres(eq, m.resolution).astype(np.float64)),
                          rng.uniform(cen.min(axis=0) - 1.0, cen.max(axis=0) + 1.0, (50_000, 3))])
    got = dev.cell_status(pts)
    assert _same(got, o.cell_status(pts)) and dev.last_query.keys_visited == o.keys_visited
    # lines: random segments, and from near the sensor (its own voxel is occupied) through voxels on the threshold
    s, e = _segments(rng, poses, 20_000)
    if len(eq):
        tgt = oc.centres(eq[rng.integers(0, len(eq), 5000)], m.resolution).astype(np.float64)
        s0 = np.array([poses[k][:3, 3] for k in rng.integers(0, len(poses), 5000)], np.float64)
        s0 += rng.uniform(-1.5, 1.5, (5000, 3)) * [1, 1, 0.2]
        s, e = np.concatenate([s, s0]), np.concatenate([e, s0 + (tgt - s0) * 1.25])
    on_eq = 0
    size = (6 * m.resolution, 6 * m.resolution, 3 * m.resolution)   # one box of 6 x 6 x 3 voxels
    for stop in (True, False):
        got = dev.line_status(s, e, stop_at_unknown=stop)
        assert _same(got, o.line_status(s, e, stop_at_unknown=stop)) and dev.last_query.keys_visited == o.keys_visited
        on_eq += sum(int(x) in eq_set for x in got[1][got[0] == oq.CELL_OCCUPIED])
        box = dev.line_status(s[:300], e[:300], box=size, stop_at_unknown=stop)
        assert _same(box, o.line_status(s[:300], e[:300], box=size, stop_at_unknown=stop))
    # rays: from around each pose along its scan's points, and from voxels on the threshold (an occupied origin voxel is
    # the hit)
    hits_eq, results = 0, set()
    eq_centres = {tuple(r) for r in _bits(oc.centres(eq, m.resolution)).tolist()}
    for T, c in zip(poses, model_maps["clouds"]):
        dirs = (c[::4, :3].astype(np.float64) @ T[:3, :3].astype(np.float64).T).astype(F32)
        origins = (T[:3, 3] + rng.uniform(-1.5, 1.5, (len(dirs), 3)) * [1, 1, 0.2]).astype(F32)
        if len(eq):
            origins = np.concatenate([origins, oc.centres(eq[rng.integers(0, len(eq), 2000)], m.resolution)])
            dirs = np.concatenate([dirs, rng.normal(size=(2000, 3)).astype(F32)])
        for ignore in (False, True):
            got = dev.cast_rays(origins, dirs, ignore_unknown=ignore, max_range=20.0)
            assert _same(got, o.cast_rays(origins, dirs, ignore_unknown=ignore, max_range=20.0))
            assert dev.last_query.keys_visited == o.keys_visited
            hits_eq += len({tuple(r) for r in _bits(got[1][got[0] == oq.RAY_HIT]).tolist()} & eq_centres)
            results |= set(np.unique(got[0]).tolist())
    assert (oq.RAY_HIT in results) == (o.size(oc.OCCUPIED) > 0) and (name == "range_0" or oq.RAY_MAX_RANGE in results)
    if name in EQUALITY:  # the queries met voxels whose log-odds is exactly L_occ, as occupied
        assert on_eq > 0 and hits_eq > 0


@pytest.mark.gpu
def test_export_matches_the_oracle_tree(model_maps, tmp_path):
    name, dev, o = model_maps["name"], model_maps["dev"], model_maps["o"]
    t, ot = dev.octree(), ot_oracle.of_map(o)
    assert _same_tree(t, ot) and t.nodes > 0
    dev.save_octomap(str(tmp_path / "d.bt"))
    ot.write(str(tmp_path / "o.bt"))
    assert (tmp_path / "d.bt").read_bytes() == (tmp_path / "o.bt").read_bytes()
    if name in FULL_SCANS:   # whole uniform nodes above the brick level
        assert (t.depths <= 12).any()


FILE_MODELS = ("defaults", "inverted")
READ_MODELS = ("defaults", "clamp_max_at_threshold", "clamp_min_at_threshold", "threshold_above_clamps",
               "equal_clamps_free", "equal_clamps_occupied")


@pytest.fixture(scope="module")
def bt_files(tmp_path_factory):
    """.bt files of the oracle maps of FILE_MODELS, and their parse."""
    out = {}
    for name in FILE_MODELS:
        path = str(tmp_path_factory.mktemp("bt") / (name + ".bt"))
        ot_oracle.of_map(oracle_map(name)[0]).write(path)
        out[name] = (path, ls.read_octomap(path))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("reader", READ_MODELS)
@pytest.mark.parametrize("writer", FILE_MODELS)
def test_read_under_every_model(gpu_ctx, bt_files, writer, reader, tmp_path):
    path, p = bt_files[writer]
    r = MODELS[reader]
    l = logodds_of(r)
    dev = ls.OccupancyMap(gpu_ctx, **r._replace(resolution=0.075).params())
    st = dev.read_octomap(path)
    _check_loaded(dev, st, p, p["resolution"], l_min=l["min"], l_max=l["max"], l_occ=l["occ"])
    assert 0 < st.free_leaves and 0 < st.occupied_leaves
    dev.save_octomap(str(tmp_path / "back.bt"))
    back, orig = (tmp_path / "back.bt").read_bytes(), open(path, "rb").read()
    if r.clamp_min < r.threshold <= r.clamp_max:
        assert back == orig
    else:  # every voxel takes one state: the tree of the expanded voxels at the map's threshold
        ot_oracle.octree(*rr.expand(p, l["min"], l["max"]), p["resolution"], r.threshold).write(str(tmp_path / "o.bt"))
        assert back == (tmp_path / "o.bt").read_bytes() and back != orig
    dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("reader", ["inverted", "clamp_min_above_half"])
def test_insert_after_a_read_under_another_model(gpu_ctx, bt_files, reader):
    path, p = bt_files["defaults"]
    r = MODELS[reader]
    l = logodds_of(r)
    dev = ls.OccupancyMap(gpu_ctx, **r.params())
    dev.read_octomap(path)
    o = rr.seed(oc.OccupancyMap(**r._replace(resolution=p["resolution"]).params()), *rr.expand(p, l["min"], l["max"]))
    from laser_slam_b200 import synth
    truth, _ = synth.trajectory(0, 6)
    cloud = synth.subsample(*synth.scan(truth[5], 0, 5), 8)[0]
    ring = gpu_ctx.create_map(2, 131072)
    st = dev.insert_scan(ring, ring.push_scan(cloud, np.zeros((len(cloud), 3), F32)), truth[5].astype(F32))
    assert _stats_dict(st) == o.insert_scan(cloud, truth[5].astype(F32))
    assert _same_map(dev.download(ls.OCC_KNOWN)[:2], o.download())
    assert _same_map(dev.download(ls.OCC_OCCUPIED)[:2], o.download(oc.OCCUPIED))
    dev.close()
    ring.close()


# laser_slam::OccupancyMap with every value non-default and the seven pairwise distinct: a swap on the way from
# OccupancyMapParams to ls_occupancy_params changes the map, or is refused (clamp_min > clamp_max)
HOST = dict(resolution=0.05, prob_hit=0.8, prob_miss=0.3, clamp_min=0.2, clamp_max=0.9, occupancy_threshold=0.6,
            max_range=12.0)


def test_host_parameters_are_distinct_and_non_default():
    assert len(set(HOST.values())) == 7 and all(HOST[k] != v for k, v in oc.DEFAULTS.items())


@pytest.mark.gpu
def test_host_layer_under_a_non_default_model(synth_mod, tmp_path):
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    from test_local_map import _float_matrix
    n = 4
    truth, odom = synth_mod.trajectory(3, n + 1)
    scans_ = [synth_mod.subsample(*synth_mod.scan(truth[k], 3, k), 8) for k in range(n)]
    est = host.Estimator(n_workers=1, nscan_in_sub_map=3)
    odom7 = pg.se3_from_matrix(odom)
    for k in range(n):
        f, nr = np.ascontiguousarray(scans_[k][0]), np.ascontiguousarray(scans_[k][1])
        est.step_batch([0], [k * 10**8], [odom7[k]], [f.ctypes.data], [nr.ctypes.data], [len(f)])
    occ = host.OccupancyMap(est, **HOST)
    assert occ.insert_laser_tracks() == n
    ctx = ls.Context(0)
    ring = ctx.create_map(n, 131072)
    dev = ls.OccupancyMap(ctx, **HOST)
    o = oq.OccupancyMap(**HOST)
    _, traj = est.trajectory(0)
    for k in range(n):
        T = _float_matrix(traj[k])
        dev.insert_scan(ring, ring.push_scan(scans_[k][0], np.zeros((len(scans_[k][0]), 3), F32)), T)
        o.insert_scan(scans_[k][0], T)
    for which in (1, 2):
        hk, hv = occ.voxels(which)
        assert _same_map((hk, hv), o.download(which)) and _same_map((hk, hv), dev.download(which)[:2]) and len(hk) > 0
    occ.write_binary(str(tmp_path / "h.bt"))
    ot_oracle.of_map(o).write(str(tmp_path / "o.bt"))
    dev.save_octomap(str(tmp_path / "d.bt"))
    assert (tmp_path / "h.bt").read_bytes() == (tmp_path / "o.bt").read_bytes() == (tmp_path / "d.bt").read_bytes()
    rng = np.random.default_rng(91)
    keys = o.download()[0]
    cen = oc.centres(keys, HOST["resolution"]).astype(np.float64)
    pts = np.concatenate([cen[::40], rng.uniform(cen.min(0), cen.max(0), (300, 3))])
    st, pr = occ.cell_probability(pts)
    ost, olo = o.cell_status(pts)
    assert np.array_equal(st, ost) and set(np.unique(st)) == {oq.CELL_FREE, oq.CELL_OCCUPIED, oq.CELL_UNKNOWN}
    assert np.array_equal(pr, [-1.0 if s == oq.CELL_UNKNOWN else 1.0 - 1.0 / (1.0 + math.exp(float(v))) for s, v in zip(ost, olo)])
    s, e = _segments(rng, [truth[k] for k in range(n)], 400)
    for stop in (True, False):
        assert _same(occ.line_status(s, e, stop_at_unknown=stop), o.line_status(s, e, stop_at_unknown=stop))
    origins = np.repeat(truth[0][:3, 3][None], 500, axis=0)
    dirs = rng.normal(size=(500, 3))
    for ign in (False, True):
        r, ends = o.cast_rays(origins, dirs, ignore_unknown=ign, max_range=10.0)
        hr, hends = occ.cast_rays(origins, dirs, ignore_unknown=ign, max_range=10.0)
        assert np.array_equal(hr, r) and np.array_equal(hends, ends.astype(np.float64)) and oq.RAY_HIT in r
    with pytest.raises(ls.LsError):
        host.OccupancyMap(est, **dict(HOST, clamp_min=HOST["clamp_max"], clamp_max=HOST["clamp_min"]))
    dev.close()
    ring.close()
    ctx.close()
    occ.close()
    est.close()


def _create(ctx, **kw):
    p = ls.OccupancyParams()
    ls.lib().ls_occupancy_default_params(ctypes.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    h = ctypes.c_void_p(0x1234)
    return ls.lib().ls_occupancy_create(ctx._h, ctypes.byref(p), ctypes.byref(h)), h


@pytest.mark.gpu
def test_parameters_accepted_and_refused(gpu_ctx):
    for kw in (dict(clamp_min=0.6, clamp_max=0.6), dict(max_range=0.0), dict(max_range=INF), dict(max_range=-INF),
               dict(occupancy_threshold=0.99), dict(occupancy_threshold=0.01)):
        rc, h = _create(gpu_ctx, **kw)
        assert rc == 0 and h.value not in (None, 0x1234), kw
        ls.lib().ls_occupancy_destroy(h)
    bad = [{f: x} for f in ("prob_hit", "prob_miss", "clamp_min", "clamp_max", "occupancy_threshold") for x in (0.0, 1.0)]
    bad += [dict(clamp_min=0.5, clamp_max=0.4), dict(max_range=float("nan"))]
    for kw in bad:
        rc, h = _create(gpu_ctx, **kw)
        assert rc == ls.LS_ERR_ARG and h.value is None, kw   # and no map
        with pytest.raises(ls.LsError, match="rc=-1"):
            ls.OccupancyMap(gpu_ctx, **kw)
