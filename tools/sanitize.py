"""Workload for compute-sanitizer (memcheck / racecheck / synccheck): the smoke registration plus one batched launch of four
small scan-to-sub-map problems, a normals estimate, a pose-graph solve with marginals, the input-side kernels and a short local-map sequence -- every kernel family of the
library on inputs small enough for the tool's ~100x slow-down.  Results are still checked against the oracle."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import laser_slam_b200 as ls
from laser_slam_b200 import synth
import oracle
from oracle import posegraph_oracle as pg

truth, odom = synth.trajectory(0, 6)
sc = [synth.subsample(*synth.scan(truth[k], 0, k), 16) for k in range(6)]
ctx = ls.Context(0)
T0 = (np.linalg.inv(truth[0]) @ odom[1]).astype(np.float32)
p = ls.default_params(max_iterations=8, use_differential=0)
g = ctx.icp_register(sc[1][0], sc[0][0], sc[0][1], T0, p, want_ids=True, want_hist=True)
r = oracle.icp(sc[1][0], sc[0][0], sc[0][1], T0, oracle.default_params(max_iterations=8, use_differential=0), want_hist=True)
assert np.array_equal(g["T"], r["T"]) and np.array_equal(g["ids"], r["ids_hist"][-1])
mp = ctx.create_map(8, 8192)
sid = [mp.push_scan(*sc[k]) for k in range(6)]
probs = []
for ref, rd, ks in [(3, 4, [3, 2, 1, 0]), (4, 5, [4, 3, 2]), (2, 3, [2, 1]), (1, 2, [1, 0])]:
    Ts = [np.eye(4, dtype=np.float32) if k == ref else (np.linalg.inv(truth[ref]) @ truth[k]).astype(np.float32) for k in ks]
    probs.append((sid[rd], [sid[k] for k in ks], Ts, (np.linalg.inv(truth[ref]) @ odom[rd]).astype(np.float32)))
batch = mp.register_batch(probs, p)
single = [mp.register(*pr, p) for pr in probs]
assert all(np.array_equal(b["T"], s["T"]) for b, s in zip(batch, single))
nr = ctx.estimate_normals(sc[0][0][:2048], knn=10)
assert np.array_equal(nr, oracle.knn_normals(sc[0][0][:2048], 10))
keys, init, factors, _ = pg.make_config4(n_poses=60, n_lc=4, lap=20, seed=2)
G = ls.PoseGraph(0)
G.add_poses(keys, init)
G.add_factors(factors)
G.optimize(3)
cov = G.marginals(keys[:10])
assert np.isfinite(cov).all()
# input side (ls_filters.cu): ingest, cylinder, voxel grid, de-skew
pts = sc[0][0][:4096]
rec = np.zeros((len(pts), 8), np.float32)
rec[:, :3] = pts[:, :3]
assert np.array_equal(ls.ingest_pointcloud2(rec.tobytes(), 32, 0, 4, 8, len(pts)), pts)
assert np.array_equal(ls.filter_cylinder(pts, [0, 0, 0], 15.0, 6.0, False), oracle.filter_cylinder(pts, [0, 0, 0], 15.0, 6.0, False))
assert np.array_equal(ls.voxel_grid(pts, 0.5), oracle.voxel_grid(pts, 0.5))
offs = [0, 100, 100, 1500, 4096]
Tp = [np.eye(4, dtype=np.float32)] + [(np.linalg.inv(truth[0]) @ truth[k]).astype(np.float32) for k in (1, 2, 3)]
Tf = oracle.rigid_inverse_f32(Tp[3])
assert np.array_equal(ls.deskew_revolution(pts, offs, Tp, Tf), oracle.deskew_revolution(pts, offs, Tp, Tf))
# resident local map: append, crop, voxel grid with a minimum count, split, transform, queue (one regrowth)
from oracle import local_map as olm
lmp = dict(distance_to_consider_fixed=12.0, voxel_size_m=0.5, minimum_point_number_per_voxel=2, remove_ground_from_local_map=True)
lm, olmap = ls.LocalMap(ctx, initial_capacity_points=4096, **lmp), olm.LocalMap(**lmp)
for k in range(4):
    Tw = ls.correct_rigid(truth[k].astype(np.float32))
    assert lm.add_scan(mp, sid[k], Tw, float(truth[k][2, 3])) == olmap.add_scan(sc[k][0], Tw, float(truth[k][2, 3]))
    if k == 2:
        lm.transform(Tp[1])
        olmap.update_local_map(Tp[1])
        assert len(olmap.local_map_filtered) > 0
        assert np.array_equal(lm.download(ls.LM_LOCAL_FILTERED), olmap.local_map_filtered)
    if k % 2 == 1:
        assert np.array_equal(lm.get_filtered_map(truth[k][:3, 3]), olmap.get_filtered_map(truth[k][:3, 3]))
        assert np.array_equal(lm.download(ls.LM_LOCAL), olmap.local_map)
        q, oq = lm.take_queue(), olmap.get_queued_points()
        assert len(q) == len(oq) and all(np.array_equal(a, b) for a, b in zip(q, oq))
lm.close()
# occupancy map and its octree export (ls_occupancy.cu): two scans, growth from 16 bricks, the pruned tree against the oracle
from oracle import occupancy as oc, octree as oct_oracle
om, oom = ls.OccupancyMap(ctx, resolution=0.2, max_range=10.0, initial_capacity=16), oc.OccupancyMap(resolution=0.2, max_range=10.0)
for k in range(2):
    om.insert_scan(mp, sid[k], truth[k].astype(np.float32))
    oom.insert_scan(sc[k][0], truth[k].astype(np.float32))
tr, otr = om.octree(), oct_oracle.of_map(oom)
assert tr.nodes == otr.nodes > 0 and tr.payload == otr.payload and np.array_equal(tr.centres, otr.centres)
# queries of that map (cells, lines, a bounding box, rays) against the query oracle
from oracle import queries as occ_queries
qo = occ_queries.KnownVoxels(*oom.download(), resolution=0.2, max_range=10.0)
rng = np.random.default_rng(5)
qs = truth[0][:3, 3] + rng.uniform(-4.0, 4.0, (256, 3))
qe = qs + rng.uniform(-4.0, 4.0, (256, 3))
qd = rng.normal(size=(256, 3)).astype(np.float32)
qorg = np.repeat(truth[1][:3, 3][None], 256, axis=0).astype(np.float32)
for got, want in ((om.cell_status(qs), qo.cell_status(qs)), (om.line_status(qs, qe), qo.line_status(qs, qe)),
                  (om.line_status(qs[:32], qe[:32], box=(0.6, 0.6, 0.3)), qo.line_status(qs[:32], qe[:32], box=(0.6, 0.6, 0.3))),
                  (om.cast_rays(qorg, qd, False, 10.0), qo.cast_rays(qorg, qd, False, 10.0)),
                  (om.cast_rays(qorg, qd, True, 10.0), qo.cast_rays(qorg, qd, True, 10.0))):
    assert np.array_equal(got[0], want[0]) and np.array_equal(np.asarray(got[1]).view(np.uint8), np.asarray(want[1]).view(np.uint8))
# that map's .bt and .ot files read back into maps of 16 bricks (parse, growth, expansion) against the reference expansions
import tempfile
sys.path.insert(1, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import octomap_read_ref as rr
with tempfile.TemporaryDirectory() as tmp:
    bt = os.path.join(tmp, "map.bt")
    om.save_octomap(bt)
    rm = ls.OccupancyMap(ctx, resolution=0.05, max_range=10.0, initial_capacity=16)
    rm.read_octomap(bt)
    rk, rv, _ = rm.download(ls.OCC_KNOWN)
    wk, wv = rr.expand(ls.read_octomap(bt), *rr.clamps())
    assert np.array_equal(rk, wk) and np.array_equal(rv.view(np.uint32), wv.view(np.uint32)) and len(rk) > 0
    rm.close()
    # the same map as a full tree: the .ot payload against the full-tree reference, and its file read back
    import octomap_full_ref as fr
    ft, oft = om.full_octree(), fr.of_map(oom)
    assert ft.nodes == oft.nodes > 0 and ft.payload == oft.payload
    oft.close()
    ot = os.path.join(tmp, "map.ot")
    om.save_octomap_full(ot)
    rm = ls.OccupancyMap(ctx, resolution=0.05, max_range=10.0, initial_capacity=16)
    rm.read_octomap_full(ot)
    rk, rv, _ = rm.download(ls.OCC_KNOWN)
    wk, wv = fr.expand(ls.read_octomap_full(ot))
    assert np.array_equal(rk, wk) and np.array_equal(rv.view(np.uint32), wv.view(np.uint32)) and len(rk) > 0
    rm.close()
# edits of that map: a set that grows it from 16 bricks, the crop, the bounds and a reset, against the edit restatement
import occupancy_edits_ref as er
e = er.Edits(0.2, *rr.clamps(), oc.logodds(0.7))
vox = er.as_dict(*oom.download())
bc, bs = [truth[0][:3, 3], truth[0][:3, 3] + 20.0], [(3.0, 3.0, 1.0), (4.0, 4.0, 4.0)]
om.set_boxes(bc, bs, [False, True])
e.set_boxes(vox, bc, bs, [False, True])
ek, ev, _ = om.download(ls.OCC_KNOWN)
assert np.array_equal(ek, er.as_arrays(vox)[0]) and np.array_equal(ev.view(np.uint32), er.as_arrays(vox)[1].view(np.uint32))
assert np.array_equal(om.box_voxels(bc[1], (6.0, 6.0, 6.0))[0], e.crop(vox, bc[1], (6.0, 6.0, 6.0))[0])
assert all(np.array_equal(a, b) for a, b in zip(om.bounds(), e.bounds(vox)))
# the distance map of that map in both modes (ls_distance.cu): one update, the field and one query against the reference
import distance_map_ref as dmr
dk, dv, _ = om.download(ls.OCC_KNOWN)
dlo, dhi = truth[0][:3, 3] - 3.0, truth[0][:3, 3] + 3.0
dq = truth[0][:3, 3] + rng.uniform(-4.0, 4.0, (256, 3))
for unknown in (False, True):
    dm = ls.DistanceMap(ctx, 1.0, dlo, dhi, unknown)
    dm.update(om)
    df = dmr.Field(dk, dv, 0.2, oc.logodds(0.7), 1.0, dlo, dhi, unknown)
    assert np.array_equal(dm.download()[0], df.s) and np.array_equal(dm.query(dq)[1], df.query(dq)[1])
    dm.close()
# change detection of that map (ls_changes.cu): one capture, an edit, one diff with a reset, against two downloads
import occupancy_changes_ref as ocr
om.track_changes()
ck0 = om.download(ls.OCC_KNOWN)[:2]
om.set_boxes([bc[0]], [(2.0, 2.0, 2.0)], [True])
cg = om.changes(reset=True)
cw = ocr.diff_arrays(*ck0, *om.download(ls.OCC_KNOWN)[:2], oc.logodds(0.7))
assert len(cg[0]) > 0 and all(np.array_equal(x, y) for x, y in zip(cg[:3], cw))
# box status and robot collision of that map (ls_collision.cu): one box call and one path call, each in both modes,
# against the restatement
import occupancy_collision_ref as ocl
xk, xv, _ = om.download(ls.OCC_KNOWN)
xvox = ocl.as_dict(xk, xv)
xc = truth[0][:3, 3] + rng.uniform(-4.0, 4.0, (64, 3))
for xs in ((1.0, 1.0, 0.5), (0.0, 0.6, 0.3)):
    assert om.box_status(xc, xs).tolist() == [ocl.box_status(xvox, c, xs, 0.2, oc.logodds(0.7)) for c in xc]
xo = np.array([0, 10, 10, 40, 64], np.int64)
for unknown in (True, False):
    xw = ocl.check_paths(xvox, xc, xo, (1.0, 1.0, 0.5), 0.2, oc.logodds(0.7), unknown)
    assert np.array_equal(om.check_paths(xc, xo, (1.0, 1.0, 0.5), unknown), xw)
# leaf boxes and marker cubes of that map (the leaf kernels in ls_occupancy.cu): a whole-map and a region listing and one
# marker call, against the reference walk of the map's .ot payload
import leaf_boxes_ref as lbr
lv = lbr.leaves(om.full_octree().payload, 0.2, oc.logodds(0.7))
lreg = (truth[0][:3, 3] - 3.0, truth[0][:3, 3] + 3.0)
for r in (None, lreg):
    lw, lg = lbr.select(lv, r, 0.2), om.leaf_boxes(ls.LEAVES_ALL, r)
    assert len(lg.depths) > 0 and np.array_equal(lg.centres.view(np.uint32), lw["centres"].view(np.uint32))
    assert np.array_equal(lg.depths, lw["depths"]) and np.array_equal(lg.states, lw["states"])
lcubes = om.marker_cubes(-1.0, 3.0, 0.8)
assert np.array_equal(np.concatenate([c.colors for c in lcubes.occupied]).view(np.uint32),
                      lbr.marker_cubes(lv, -1.0, 3.0, 0.8)[1].view(np.uint32))
# the 2D projection of that map (ls_projection.cu and the .bt leaf walk in ls_occupancy.cu): the whole map and a padded
# band, against the restatement over the map's .bt payload
import projected_map_ref as pmr
for band in (dict(), dict(min_z=0.3, max_z=2.0, min_size_x=30.0)):
    pg_, pi_ = om.projected_map(**band)
    assert np.array_equal(pg_, pmr.project(pmr.bt_leaves(om.octree().payload), 0.2, **band)[0]) and (pg_ >= 0).any()
om.clear()
assert om.size(ls.OCC_KNOWN) == 0
om.close()
launches = ctx.launch_count
# every handle closed, so a leak check sees only what the library failed to free
mp.close()
ctx.close()
G.close()
print("sanitize workload ok:", g["stats"].iterations, "iterations;", len(batch), "batched problems;", launches, "launches")
