"""The spatial hash (laser_slam_b200/csrc/ls_grid.cuh) against brute force at the grid shapes its build and its queries
depend on: how grid_setup picks H0 and the level-0 dimensions under the cell budget, how far the occupancy pyramid
reaches, and whether a cell becomes a fine table or stays a leaf (including when the table pool runs out).

The contract is the exact nearest neighbour (and the exact k nearest, for normals) with the lowest index winning ties.
CPU tests run the header through tests/sim/grid_sim.cpp; GPU tests compare the device with the oracle bit for bit.
Every case states the branch it is meant to reach and checks it from the CPU first (`device_grid` restates the geometry
the device derives), so a change of the data cannot quietly turn a case into one that exercises nothing."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_SRC = os.path.join(HERE, "sim", "grid_sim.cpp")
SIM_LIB = os.path.join(HERE, "sim", "libgrid_sim.so")
F32 = np.float32
INT_MAX = np.iinfo(np.int32).max
TOP_CELLS = 4 ** 7          # level-0 cells per axis under one top cell of a full-height (7-level) pyramid
THREADS = min(16, os.cpu_count() or 1)


# ---- simulator ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sim():
    deps = [SIM_SRC] + [os.path.join(HERE, "..", "laser_slam_b200", "csrc", f) for f in ("ls_grid.cuh", "ls_math.cuh")]
    if not os.path.exists(SIM_LIB) or os.path.getmtime(SIM_LIB) < max(os.path.getmtime(d) for d in deps):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared",
                               "-I/usr/local/cuda/include", "-o", SIM_LIB, SIM_SRC])
    L = ctypes.CDLL(SIM_LIB)
    vp, ci, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    L.sim_nn.argtypes = [vp, ci, vp, ci, cf, ci, ci, vp, vp, vp, vp, vp, vp, cf]
    L.sim_knn.argtypes = [vp, ci, vp, ci, cf, ci, ci, ci, vp, vp, vp]
    L.sim_grid.argtypes = [vp, vp, cf, ci, ci, ci, vp, vp]
    L.sim_grid.restype = ci

    class Sim:
        @staticmethod
        def grid(lo, hi, cell=1.0, max_cells=1 << 22, split=32, m=1):
            lo, hi = np.ascontiguousarray(lo, F32), np.ascontiguousarray(hi, F32)
            h0 = np.zeros(1, F32)
            out = np.zeros(6 + 4 * 32, np.int32)
            levels = L.sim_grid(lo.ctypes.data, hi.ctypes.data, cell, max_cells, split, m, h0.ctypes.data, out.ctypes.data)
            lv = out[6:6 + 4 * (levels + 1)].reshape(levels + 1, 4)
            return dict(H0=F32(h0[0]), dim=out[:3].copy(), n_cells0=int(out[3]), n_pyr=int(out[4]),
                        n_pyr_cells=int(out[5]), pdim=lv[:, :3].copy(), poff=lv[:, 3].copy(), levels=levels)

        @staticmethod
        def nn(q, ref, cell=1.0, max_cells=1 << 22, split=32):
            q, ref = np.ascontiguousarray(q, F32), np.ascontiguousarray(ref, F32)
            ids = np.empty(max(len(q), 1), np.int32)
            d2 = np.empty(max(len(q), 1), F32)
            st = np.zeros(8)
            L.sim_nn(q.ctypes.data, len(q), ref.ctypes.data, len(ref), cell, max_cells, split, None, ids.ctypes.data,
                     d2.ctypes.data, st.ctypes.data, None, None, np.inf)
            return ids[:len(q)], d2[:len(q)], dict(n_tab1=int(st[3]), H0=st[4], n_cells0=int(st[5]))

        @staticmethod
        def knn(q, ref, k, cell=1.0, max_cells=1 << 22, split=32):
            q, ref = np.ascontiguousarray(q, F32), np.ascontiguousarray(ref, F32)
            ids = np.empty((max(len(q), 1), k), np.int32)
            d2 = np.empty((max(len(q), 1), k), F32)
            L.sim_knn(q.ctypes.data, len(q), ref.ctypes.data, len(ref), cell, max_cells, split, k, ids.ctypes.data,
                      d2.ctypes.data, None)
            return ids[:len(q)], d2[:len(q)]
    return Sim


# ---- references ---------------------------------------------------------------------------------------------------
def knn_brute(q, ref, k):
    """Exact k nearest by brute force: d2 = fl(fl(fl(dx*dx) + fl(dy*dy)) + fl(dz*dz)) in float32, ascending by
    (d2, index); a map with fewer than k points leaves INT_MAX / +inf in the tail."""
    q, ref = np.asarray(q, F32), np.asarray(ref, F32)
    ids = np.full((len(q), k), INT_MAX, np.int32)
    d2 = np.full((len(q), k), np.inf, F32)
    kk = min(k, len(ref))
    for a in range(0, len(q), 256):
        b = min(len(q), a + 256)
        dx = q[a:b, None, 0] - ref[None, :, 0]
        dy = q[a:b, None, 1] - ref[None, :, 1]
        dz = q[a:b, None, 2] - ref[None, :, 2]
        d = (dx * dx + dy * dy) + dz * dz
        order = np.argsort(d, axis=1, kind="stable")[:, :kk]     # stable: the lower index first among equal d2
        ids[a:b, :kk] = order
        d2[a:b, :kk] = np.take_along_axis(d, order, 1)
    return ids, d2


def check_nn(sim, oracle_mod, q, ref, **kw):
    ib, db = oracle_mod.nn_brute(q, ref)
    ig, dg, st = sim.nn(q, ref, **kw)
    bad = ib != ig
    assert not bad.any(), f"{bad.sum()} of {len(q)} queries differ; first {np.flatnonzero(bad)[:5]}: " \
                          f"d2 {dg[bad][:5]} vs brute force {db[bad][:5]}"
    assert np.array_equal(db, dg)
    return st


def check_knn(sim, q, ref, k, **kw):
    ib, db = knn_brute(q, ref, k)
    ig, dg = sim.knn(q, ref, k, **kw)
    assert np.array_equal(ib, ig), f"{(ib != ig).any(1).sum()} of {len(q)} queries differ"
    assert np.array_equal(db, dg)


def resolve(cell=0.0, max_cells=0, split=0):
    """The device's reading of ls_icp_params (ls_api.cu resolve)."""
    cell = F32(cell) if cell > 0 else F32(1.0)
    split = (16 if split < 16 else split) if split > 0 else 32
    max_cells = min(max(max_cells if max_cells > 0 else 1 << 22, 64), 1 << 22)
    return cell, max_cells, split


def device_grid(sim, oracle_mod, ref3, cell=0.0, max_cells=0, split=0):
    """The grid the device builds over a map: bounding box of the points centred on the oracle's (= the device's) exact
    mean, then grid_setup with the resolved parameters."""
    ref4 = np.ones((len(ref3), 4), F32)
    ref4[:, :3] = ref3
    mu = oracle_mod.mean(ref4)
    c = (np.asarray(ref3, F32) - mu).astype(F32)
    cell, max_cells, split = resolve(cell, max_cells, split)
    g = sim.grid(c.min(0), c.max(0), cell, max_cells, split, len(ref3))
    g.update(centred=c, lo=c.min(0), mu=mu, max_cells=max_cells, split=split)
    return g


def cell_counts(g):
    """Points per level-0 cell of `device_grid`'s grid (coord_top in float32)."""
    inv = F32(1.0) / g["H0"]
    t = np.floor((g["centred"] - g["lo"]) * inv)
    t = np.clip(t, 0, g["dim"] - 1).astype(np.int64)
    key = (t[:, 2] * g["dim"][1] + t[:, 1]) * g["dim"][0] + t[:, 0]
    return np.bincount(key, minlength=g["n_cells0"])


def homog(p3):
    p4 = np.ones((len(p3), 4), F32)
    p4[:, :3] = p3
    return p4


# ---- shapes -------------------------------------------------------------------------------------------------------
def elongated(axis, far_m, seed=0):
    """A 3000-point cluster in a 10 m box, 20 points `far_m` metres away along `axis`, 6 stragglers in between; queries
    spread along the axis plus one outside the bounding box in every octant."""
    rng = np.random.default_rng(seed + axis)
    pts = rng.uniform(0, 10, (3026, 3))
    pts[3000:3020, axis] = far_m + rng.uniform(0, 10, 20)
    pts[3020:, axis] = np.linspace(0.2, 0.8, 6) * far_m
    q = rng.uniform(-20, 30, (400, 3))
    q[:, axis] = np.linspace(-500, far_m + 500, 400)
    lo, hi = pts.min(0), pts.max(0)
    octants = np.array([[(hi if (o >> a) & 1 else lo)[a] + (100 if (o >> a) & 1 else -100) for a in range(3)]
                        for o in range(8)])
    return pts.astype(F32), np.concatenate([q, octants]).astype(F32)


def symmetric_lattice(half, step, dup_seed=None):
    """Lattice points k*step for |k*step| <= half on every axis (exact when step is a power of two), mean exactly 0, so
    centring keeps every coordinate and the level-0 and fine boundaries fall on lattice multiples."""
    r = np.arange(-half, half + step / 2, step, dtype=np.float64)
    g = np.stack(np.meshgrid(r, r, r[(np.abs(r) <= 1.0)], indexing="ij"), -1).reshape(-1, 3)
    if dup_seed is not None:   # duplicates in symmetric pairs: more exact ties, the mean stays 0
        d = g[np.random.default_rng(dup_seed).permutation(len(g))[:200]]
        g = np.concatenate([g, d, -d])
    return g.astype(F32)


def leaf_blocks(split, seed=0):
    """4x4x2 level-0 cells at H0 = 1 holding split-1, split, split+1 or 2*split points (one point at the origin pins the
    lattice so the cells are the unit cubes)."""
    rng = np.random.default_rng(seed + split)
    counts = np.array([split - 1, split, split + 1, 2 * split] * 8)
    pts = [np.zeros((1, 3))]
    for c, n in enumerate(counts):
        corner = np.array([c % 4, (c // 4) % 4, c // 16], np.float64)
        pts.append(corner + rng.uniform(0.05, 0.95, (n - (1 if c == 0 else 0), 3)))
    return np.concatenate(pts).astype(F32), counts


# ---- CPU: geometry --------------------------------------------------------------------------------------------------
CELLS = (0.1, 0.15, 0.3, 0.7, 1.0, 1.3, 2.0, 3.3)
BUDGETS = (64, 125, 1000, 4096, 1 << 16, 1 << 20, 1 << 22)


def _float_dims(ext, H0):
    return (np.floor(ext.astype(F32) * (F32(1.0) / F32(H0))) + 1).astype(np.int64)


def test_budget_is_exact(sim):
    """n_cells0 <= max_cells and dim == floorf(ext * inv0) + 1 on every axis, for cell sizes that are not powers of two
    and extents at exact multiples of H and one ulp either side.  H0 is the first doubling of the cell size that fits."""
    worst = []
    for cell in CELLS:
        c = F32(cell)
        exts = {F32(1.5)}
        for j in (1, 3, 5, 7, 64, 1000):
            e = F32(j) * c
            exts |= {e, np.nextafter(e, F32(np.inf)), np.nextafter(e, F32(0))}
        for e in sorted(exts):
            for shape in ((e, e, e), (e, F32(0), F32(0)), (e, e, F32(0))):
                ext = np.array(shape, F32)
                for mc in BUDGETS:
                    g = sim.grid(np.zeros(3, F32), ext, cell, mc)
                    dims = _float_dims(ext, g["H0"])
                    assert np.array_equal(g["dim"], dims), (cell, ext, mc, g["dim"], dims)
                    assert g["n_cells0"] == int(np.prod(dims)) <= mc, (cell, ext, mc, g["n_cells0"])
                    H, k = c, 0
                    while H != g["H0"]:
                        H, k = F32(H * 2), k + 1
                        assert k < 40, (cell, g["H0"])
                    if k > 0:   # minimal: half of H0 would not have fitted
                        assert np.prod(_float_dims(ext, F32(g["H0"] / 2))) > mc, (cell, ext, mc)
                    assert g["n_pyr_cells"] <= mc // 2 + 4096     # the device's pyramid buffer
                    worst.append(g["n_cells0"] / mc)
    assert max(worst) > 0.9      # the sweep reaches budgets that are nearly full


def test_budget_case_non_power_of_two_cell(sim):
    """Cell 0.3 over 1.5 m per axis: floor(1.5 / 0.3) in double is 4 (5 cells), floorf(1.5f * (1 / 0.3f)) is 5 (6 cells).
    A budget of 125 admitted H = 0.3 with 216 cells before the budget was counted in float."""
    ext = np.full(3, 1.5, F32)
    assert np.prod(np.floor(ext.astype(np.float64) / np.float64(F32(0.3))) + 1) == 125
    assert np.prod(_float_dims(ext, F32(0.3))) == 216
    g = sim.grid(np.zeros(3, F32), ext, 0.3, 125)
    assert g["n_cells0"] <= 125 and g["H0"] == F32(0.6) and list(g["dim"]) == [3, 3, 3]


PYR_SHAPES = [(1 << 22, 1, 1), (1, 1 << 22, 1), (1, 1, 1 << 22), (16384, 1, 1), (16385, 1, 1), (1, 16385, 255),
              (65537, 8, 7), (1 << 20, 4, 1), (2048, 2048, 1), (161, 161, 161), (1, 1, 1), (5, 5, 5), (1000, 1, 4194)]


@pytest.mark.parametrize("dims", PYR_SHAPES)
def test_pyramid_covers_the_grid(sim, dims):
    """Every level is the previous one divided by 4 (rounded up), the levels tile GridView::pyr back to back within the
    device's buffer, and the top level is one cell unless an axis spans more than 4^7 level-0 cells; then the pyramid
    has its full 7 levels and only that axis has several top cells (no two axes can: 16385^2 > 2^22), which
    pyramid_query and seed_query walk one by one."""
    ext = np.array(dims, F32) - 1
    g = sim.grid(np.zeros(3, F32), ext, 1.0, 1 << 22)
    assert list(g["dim"]) == list(dims) and g["n_cells0"] <= 1 << 22
    L = g["n_pyr"]
    off = 0
    for l in range(1, L + 1):
        assert np.array_equal(g["pdim"][l], (g["pdim"][l - 1] + 3) // 4)
        assert g["poff"][l] == off
        off += int(np.prod(g["pdim"][l]))
    assert off == g["n_pyr_cells"] <= (1 << 22) // 2 + 4096
    top = g["pdim"][L]
    assert (top * 4 ** L >= g["dim"]).all()
    if max(dims) <= TOP_CELLS:
        assert list(top) == [1, 1, 1]
    else:
        assert L == g["levels"] == 7 and (top > 1).sum() == 1 and top.max() == -(-max(dims) // TOP_CELLS)


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_sim_wide_ball_reaches_every_top_cell(sim, axis):
    """20 points spread over 2^22 level-0 cells of one axis (256 top cells): the 16 nearest of queries far outside the
    map, and between the points, are found whichever top cell holds them."""
    rng = np.random.default_rng(7 + axis)
    ref = np.zeros((20, 3), F32)
    ref[:, axis] = np.sort(rng.choice((1 << 22) - 1, 18, replace=False)).tolist() + [0, (1 << 22) - 1]
    g = sim.grid(ref.min(0), ref.max(0))
    assert g["dim"][axis] == 1 << 22 and g["pdim"][g["n_pyr"]][axis] == 256
    q = rng.uniform(-50, 50, (64, 3)).astype(F32)
    q[:, axis] = rng.uniform(-3e5, (1 << 22) + 3e5, 64)
    check_knn(sim, q, ref, 16)
    check_knn(sim, q, ref, 3)


# ---- CPU: exactness of the simulated query --------------------------------------------------------------------------
@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("far_m,H0", [(20000.0, 1.0), (34000.0, 1.0), (70000.0, 2.0)])
def test_sim_elongated_maps(sim, oracle_mod, axis, far_m, H0):
    """More than 16384 level-0 cells on one axis: queries along the axis need the top cells beyond the first."""
    ref, q = elongated(axis, far_m)
    g = sim.grid(ref.min(0), ref.max(0))
    assert g["H0"] == F32(H0) and g["dim"][axis] > TOP_CELLS, g["dim"]
    check_nn(sim, oracle_mod, q, ref)
    check_knn(sim, q, ref, 16)
    check_knn(sim, q[::4], ref, 3)


@pytest.mark.parametrize("cell", [0.15, 0.3, 0.7, 1.3, 3.3])
def test_sim_non_power_of_two_cells(sim, oracle_mod, cell):
    """Lattices with spacing = the cell size, extents at exact multiples of it, under budgets that force H0 to grow."""
    rng = np.random.default_rng(int(cell * 100))
    c = F32(cell)
    r = np.arange(6, dtype=F32) * c
    lat = np.stack(np.meshgrid(r, r, r[:4], indexing="ij"), -1).reshape(-1, 3).astype(F32)
    ref = np.concatenate([lat, rng.uniform(0, float(r[-1]), (3000, 3)).astype(F32)])
    q = np.concatenate([lat, (lat + c / 2).astype(F32), rng.uniform(-c, float(r[-1] + c), (1000, 3)).astype(F32)])
    H0s = set()
    for mc in (64, 125, 4096, 1 << 22):
        st = check_nn(sim, oracle_mod, q, ref, cell=cell, max_cells=mc, split=16)
        assert st["n_cells0"] <= mc
        H0s.add(st["H0"])
        check_knn(sim, q[::3], ref, 16, cell=cell, max_cells=mc, split=16)
    assert len(H0s) >= 2


@pytest.mark.parametrize("split", [16, 32, 64])
def test_sim_leaf_split_boundary(sim, oracle_mod, split):
    """Cells holding exactly leaf_split points stay leaves; split+1 points make a fine table."""
    ref, counts = leaf_blocks(split)
    rng = np.random.default_rng(split)
    q = np.concatenate([ref, rng.uniform(-1, 5, (1500, 3)).astype(F32)]).astype(F32)
    g = sim.grid(ref.min(0), ref.max(0))
    assert g["H0"] == 1 and list(g["dim"]) == [4, 4, 2]
    assert (counts == split).any() and (counts == split + 1).any()
    st = check_nn(sim, oracle_mod, q, ref, split=split)
    assert st["n_tab1"] == int((counts > split).sum()) == 16        # split+1 and 2*split cells only
    check_knn(sim, q[::2], ref, 16, split=split)


def test_sim_boundary_lattice(sim, oracle_mod):
    """Points and queries on level-0 and fine-cell boundaries: multiples of H1 = 0.125 m are exact, and the lattice's
    mean is 0, so the lattice origin is a level-0 boundary."""
    ref = symmetric_lattice(2.0, 0.125, dup_seed=1)
    assert oracle_mod.mean(homog(ref)).tolist() == [0, 0, 0]
    rng = np.random.default_rng(3)
    q = np.concatenate([ref[:4000], (rng.integers(-40, 41, (3000, 3)) * 0.0625).astype(F32)]).astype(F32)
    for split in (16, 64):
        st = check_nn(sim, oracle_mod, q, ref, split=split)
        assert st["n_tab1"] > 0
        check_knn(sim, q[::3], ref, 16, split=split)


def test_sim_map_far_from_origin(sim, oracle_mod):
    """A map centred about 1e5 m from the origin (coordinates left uncentred): 1 ulp = 7.8 mm, margin and cell bounds at
    that magnitude."""
    rng = np.random.default_rng(11)
    ref = (np.array([1e5, -1e5, 3e4]) + rng.uniform(0, 20, (5000, 3)) * [1, 1, 0.25]).astype(F32)
    q = (np.array([1e5, -1e5, 3e4]) + rng.uniform(-5, 25, (2000, 3)) * [1, 1, 0.25]).astype(F32)
    q = np.concatenate([q, ref[:500]])
    for cell in (1.0, 0.3):
        check_nn(sim, oracle_mod, q, ref, cell=cell)
        check_knn(sim, q[::4], ref, 16, cell=cell)


# ---- CPU: the oracle's normals against an independent eigensolver --------------------------------------------------
def test_oracle_normals_match_eigh(oracle_mod):
    """On well-conditioned neighbourhoods (eigengap > 1e-3 of the trace) oracle.knn_normals is the +-eigenvector of the
    smallest eigenvalue that numpy.linalg.eigh finds in float64, to |cos| > 1 - 1e-9."""
    rng = np.random.default_rng(5)
    xy = rng.uniform(-3, 3, (1500, 2))
    plane = np.stack([xy[:, 0], xy[:, 1], 0.2 * xy[:, 0] - 0.1 * xy[:, 1] + rng.normal(0, 0.01, 1500) + 4], 1)
    v = rng.normal(size=(1500, 3))
    sphere = 2.0 * v / np.linalg.norm(v, axis=1, keepdims=True) + [10, 0, 1]
    pts = homog(np.concatenate([plane, sphere]).astype(F32))
    checked = 0
    for k in (5, 10, 16):
        n_or = oracle_mod.knn_normals(pts, k).astype(np.float64)
        c = (pts[:, :3] - oracle_mod.mean(pts)).astype(F32)
        ids, d2 = knn_brute(c, c, k + 1)
        for i in range(0, len(pts), 3):
            if d2[i, k - 1] == d2[i, k]:
                continue                              # the k-th neighbour is tied: the set is not unique
            nb = c[ids[i, :k]].astype(np.float64)
            mu = nb.mean(0)
            d = nb - mu
            w, V = np.linalg.eigh(d.T @ d)
            if not (w[1] - w[0] > 1e-3 * w.sum()):
                continue
            n = n_or[i] / np.linalg.norm(n_or[i])
            assert abs(n @ V[:, 0]) > 1 - 1e-9, (k, i, n, V[:, 0])
            checked += 1
    assert checked > 1500


# ---- GPU ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    import laser_slam_b200 as ls
    c = ls.Context(0)
    yield c
    c.close()


def gpu_nn_check(ctx, oracle_mod, q3, ref3, kd=False, **prm):
    """ls_nn_query against brute force (or the oracle's kd-tree) on the map centred on its exact mean."""
    import laser_slam_b200 as ls
    ref4, q4 = homog(ref3), homog(q3)
    mu = oracle_mod.mean(ref4)
    T = np.eye(4, dtype=F32)
    T[:3, 3] = -mu
    qc = oracle_mod.transform_points(T, q4)[:, :3].copy()
    refc = (np.asarray(ref3, F32) - mu).astype(F32)
    ib, db = oracle_mod.nn_kdtree(qc, refc, THREADS) if kd else oracle_mod.nn_brute(qc, refc)
    ig, dg = ctx.nn_query(q4, ref4, None, ls.default_params(**prm) if prm else None)
    bad = ib != ig
    assert not bad.any(), f"{bad.sum()} of {len(q3)} queries differ: d2 {dg[bad][:5]} vs {db[bad][:5]}"
    assert np.array_equal(db, dg)


@pytest.mark.gpu
@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("far_m,H0", [(20000.0, 1.0), (70000.0, 2.0)])
def test_gpu_nn_elongated(ctx, sim, oracle_mod, axis, far_m, H0):
    ref, q = elongated(axis, far_m)
    g = device_grid(sim, oracle_mod, ref)
    assert g["H0"] == F32(H0) and g["dim"][axis] > TOP_CELLS and g["pdim"][g["n_pyr"]][axis] > 1
    gpu_nn_check(ctx, oracle_mod, q, ref)


@pytest.mark.gpu
def test_gpu_nn_grid_shapes(ctx, sim, oracle_mod):
    """Non-power-of-two cells (including the budget case that used to overrun the level-0 arrays), leaf_split
    boundaries and the boundary lattice, through ls_nn_query."""
    rng = np.random.default_rng(21)
    # budget case: extent exactly 1.5 m per axis after centring, cell 0.3, 125 cells
    inner = rng.uniform(-0.74, 0.74, (1500, 3))
    cube = np.concatenate([inner, -inner, [[-0.75] * 3, [0.75] * 3]]).astype(F32)
    g = device_grid(sim, oracle_mod, cube, cell=0.3, max_cells=125)
    assert np.array_equal(g["lo"], [-0.75] * 3) and g["dim"].tolist() == [3, 3, 3] and g["n_cells0"] <= 125
    assert np.prod(_float_dims(np.full(3, 1.5, F32), F32(0.3))) == 216          # what the double count admitted
    qc = rng.uniform(-1, 1, (2000, 3)).astype(F32)
    gpu_nn_check(ctx, oracle_mod, qc, cube, cell_size=0.3, max_cells=125)
    for cell in (0.15, 0.7, 1.3, 3.3):
        for mc in (64, 4096):
            gpu_nn_check(ctx, oracle_mod, qc * 4, cube * 4, cell_size=cell, max_cells=mc, leaf_split=16)
    for split in (16, 32, 64):
        ref, counts = leaf_blocks(split)
        g = device_grid(sim, oracle_mod, ref, split=split)
        cc = cell_counts(g)
        assert (cc == split).sum() == 8 and (cc == split + 1).sum() == 8, "the unit cubes are the level-0 cells"
        q = np.concatenate([ref, rng.uniform(-1, 5, (1500, 3)).astype(F32)]).astype(F32)
        gpu_nn_check(ctx, oracle_mod, q, ref, leaf_split=split)
    lat = symmetric_lattice(2.0, 0.125, dup_seed=1)
    g = device_grid(sim, oracle_mod, lat, split=16)
    assert g["lo"].tolist() == [-2.0, -2.0, -1.0] and (cell_counts(g) > 16).any()
    q = np.concatenate([lat[:4000], (rng.integers(-40, 41, (3000, 3)) * 0.0625).astype(F32)]).astype(F32)
    gpu_nn_check(ctx, oracle_mod, q, lat, leaf_split=16)


def normals_shapes():
    rng = np.random.default_rng(31)
    out = []
    for axis in (0, 2):                       # elongated, with isolated far points (fewer than k neighbours nearby)
        ref, _ = elongated(axis, 20000.0)
        out.append((f"elongated{axis}", ref))
    same = np.concatenate([np.repeat([[1.5, -2.0, 0.25]], 40, 0), rng.uniform(-1, 1, (60, 3))])
    out.append(("identical", same.astype(F32)))   # > k+1 identical points: zero covariance
    t = np.arange(200, dtype=np.float64)[:, None] * 0.1
    line = np.concatenate([t * [1, 0, 0], t * [0.6, 0.8, 0] + [0, 5, 1], t * [0, 0, 1] + [3, 3, 0]])
    out.append(("collinear", line.astype(F32)))
    out.append(("lattice", symmetric_lattice(2.0, 0.125, dup_seed=2)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("k", [3, 16])
def test_gpu_normals_shapes(ctx, sim, oracle_mod, k):
    for name, p3 in normals_shapes():
        if name.startswith("elongated"):
            g = device_grid(sim, oracle_mod, p3)
            assert g["dim"].max() > TOP_CELLS
        pts = homog(p3)
        o = oracle_mod.knn_normals(pts, k, num_threads=THREADS)
        d = ctx.estimate_normals(pts, k)
        bad = (o != d).any(1)
        assert not bad.any(), (name, k, int(bad.sum()))


def far_cluster_problem(small_pair, far_m=20000.0):
    """The small lidar pair cropped to 60 x 20 m (so that H0 stays 1 m), plus a planar patch `far_m` metres along x in
    the map and reading points 5-30 m from it: their nearest neighbours lie in the second top cell, and the empty cells
    around them make the query ball wide."""
    rng = np.random.default_rng(41)
    keep = lambda p: (np.abs(p[:, 0]) < 30) & (np.abs(p[:, 1]) < 10)
    kr, kd = keep(small_pair["ref"]), keep(small_pair["reading"])
    patch = np.stack([np.full(300, far_m) + rng.normal(0, 0.02, 300), rng.uniform(-2, 2, 300), rng.uniform(-2, 2, 300)], 1)
    pn = np.tile([[-1.0, 0.0, 0.0]], (300, 1)) + rng.normal(0, 0.05, (300, 3))
    pn /= np.linalg.norm(pn, axis=1, keepdims=True)
    ref = np.concatenate([small_pair["ref"][kr], homog(patch.astype(F32))])
    nrm = np.concatenate([small_pair["ref_normals"][kr], pn.astype(F32)])
    near = np.stack([np.full(200, far_m) - rng.uniform(5, 30, 200), rng.uniform(-3, 3, 200), rng.uniform(-3, 3, 200)], 1)
    rd = np.concatenate([small_pair["reading"][kd], homog(near.astype(F32))])
    return rd, ref, nrm


@pytest.mark.gpu
def test_gpu_icp_elongated_map(ctx, sim, oracle_mod, small_pair):
    """ICP on a map 20 km long, reading points near the far patch; then the plain pair at cell_size 0.3."""
    import laser_slam_b200 as ls
    o = oracle_mod
    rd, ref, nrm = far_cluster_problem(small_pair)
    g = device_grid(sim, o, ref[:, :3])
    assert g["H0"] == 1 and g["dim"][0] > TOP_CELLS and g["pdim"][g["n_pyr"]][0] == 2
    T0 = small_pair["T0"]
    mu = o.mean(ref)
    Tpre = T0.copy()
    Tpre[:3, 3] -= mu
    qc = o.transform_points(Tpre, rd)[:, :3].copy()
    ids, d2 = o.nn_brute(qc[-200:], (ref[:, :3] - mu).astype(F32))
    assert (ids >= len(ref) - 300).all() and (d2 > 4 * g["H0"] ** 2).all()   # far patch, wide balls
    for prm, ref_, nrm_, rd_ in ((dict(max_iterations=15, use_differential=0), ref, nrm, rd),
                                 (dict(max_iterations=15, use_differential=0, cell_size=0.3),
                                  small_pair["ref"], small_pair["ref_normals"], small_pair["reading"])):
        p = ls.default_params(**prm)
        gr = ctx.icp_register(rd_, ref_, nrm_, T0, p, want_ids=True, want_hist=True)
        kw = {k: v for k, v in prm.items() if k != "cell_size"}
        r = o.icp(rd_, ref_, nrm_, T0, o.default_params(num_threads=THREADS, **kw), want_hist=True)
        assert gr["rc"] == r["rc"] == 0 and gr["stats"].grid_overflow == 0
        assert np.array_equal(gr["T_iter_hist"], r["T_iter_hist"])
        assert np.array_equal(gr["ids"], r["ids_hist"][-1]) and np.array_equal(gr["d2"], r["d2_last"])
        assert np.array_equal(gr["T"], r["T"])
        assert gr["stats"].last_kept == r["stats"].last_kept and gr["stats"].last_limit == r["stats"].last_limit


def pool_block(seed=0):
    """300000 unit cells of a 100 x 100 x 30 m block with 17 points each (one more at the origin, which pins the
    lattice): at leaf_split 16 every cell wants a fine table, more than the pool of 262144 holds."""
    rng = np.random.default_rng(seed)
    ix, iy, iz = np.meshgrid(np.arange(100), np.arange(100), np.arange(30), indexing="ij")
    corner = np.stack([ix.ravel(), iy.ravel(), iz.ravel()], 1).astype(np.float64)
    pts = np.repeat(corner, 17, 0) + rng.uniform(0.05, 0.95, (len(corner) * 17, 3))
    return np.concatenate([[[0.0, 0.0, 0.0]], pts]).astype(F32)


def table_pool(m):
    cap = m + m // 8 + 1024                       # ensure_capacity (ls_api.cu)
    return min(cap // 17 + 1024, (1536 * 1024 * 1024) // (512 * 12))


@pytest.mark.gpu
def test_gpu_table_pool_exhausted(ctx, sim, oracle_mod):
    """More cells over leaf_split than fine tables: the overflow branch of scan_apply_kernel leaves the rest as leaves of
    17-18 points, scattered by the leaf cursors; queries and the reading sort run over those leaves.  Still exact."""
    import torch
    import laser_slam_b200 as ls
    o = oracle_mod
    p3 = pool_block()
    g = device_grid(sim, o, p3, split=16)
    cc = cell_counts(g)
    assert g["H0"] == 1 and (cc > 16).sum() == 300000 > table_pool(len(p3)) == 262144
    rng = np.random.default_rng(3)
    free0 = torch.cuda.mem_get_info(0)[0]
    q = (p3[rng.choice(len(p3), 30000, replace=False)] + rng.normal(0, 0.3, (30000, 3))).astype(F32)
    gpu_nn_check(ctx, o, q, p3, kd=True, leaf_split=16)
    ref4 = homog(p3)
    nrm = rng.normal(size=(len(p3), 3))
    nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(F32)
    rd = homog(p3[rng.choice(len(p3), 20000, replace=False)])
    T0 = np.eye(4, dtype=F32)
    T0[:3, 3] = [0.05, -0.03, 0.02]
    prm = dict(max_iterations=5, use_differential=0)
    gr = ctx.icp_register(rd, ref4, nrm, T0, ls.default_params(leaf_split=16, **prm), want_ids=True, want_hist=True)
    used = free0 - torch.cuda.mem_get_info(0)[0]
    print(f"table-pool exhaustion: device memory in use grew by {used / 2**30:.2f} GiB over the case")
    assert gr["stats"].grid_overflow == 1 and gr["stats"].grid_tables > 262144
    r = o.icp(rd, ref4, nrm, T0, o.default_params(num_threads=THREADS, **prm), want_hist=True)
    assert gr["rc"] == r["rc"] == 0
    assert np.array_equal(gr["T_iter_hist"], r["T_iter_hist"]) and np.array_equal(gr["T"], r["T"])
    assert np.array_equal(gr["ids"], r["ids_hist"][-1])
    assert gr["stats"].last_kept == r["stats"].last_kept and gr["stats"].last_limit == r["stats"].last_limit
