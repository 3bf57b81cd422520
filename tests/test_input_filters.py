"""Per-scan input filters (LaserTrackParams::icp_input_filters_file; reference laser_slam/src/laser_track.cpp:24-30,81,146):
the YAML reader and the oracle's rules on the CPU, the device chain against the oracle bit for bit on the GPU."""
import os
import sys

import numpy as np
import pytest

from oracle import input_filters as fo

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

EGO_BOX = {"xMin": -3.0, "xMax": 3.0, "yMin": -2.0, "yMax": 2.0, "zMin": -3.0, "zMax": 3.0}
CHAIN = [("RemoveNaNDataPointsFilter", {}),
         ("MinDistDataPointsFilter", {"minDist": 1.0}),
         ("MaxDistDataPointsFilter", {"dim": -1, "maxDist": 60.0}),
         ("BoundingBoxDataPointsFilter", EGO_BOX),
         ("RandomSamplingDataPointsFilter", {"prob": 0.5}),
         ("VoxelGridDataPointsFilter", {"vSizeX": 0.1, "vSizeY": 0.1, "vSizeZ": 0.1}),
         ("SurfaceNormalDataPointsFilter", {"knn": 10})]

ALL_YAML = """# every filter this path runs
- RemoveNaNDataPointsFilter
- MaxDistDataPointsFilter:
    dim: 1
    maxDist: 60
- MinDistDataPointsFilter:
    minDist: 0.5
- BoundingBoxDataPointsFilter: {xMin: -3, xMax: 3, yMin: -2, yMax: 2, zMin: -1.5, zMax: 2.5, removeInside: 0}
- RandomSamplingDataPointsFilter:
    prob: 0.25
- FixStepSamplingDataPointsFilter:
    startStep: 3
    endStep: 3
    stepMult: 1
- VoxelGridDataPointsFilter:
    vSizeX: 0.1
    vSizeY: 0.2
    vSizeZ: 0.3
    useCentroid: 1
- SurfaceNormalDataPointsFilter:
    knn: 7
- SamplingSurfaceNormalDataPointsFilter:
    knn: 12
    ratio: 0.6
- SurfaceNormalDataPointsFilter
- RandomSamplingDataPointsFilter
"""


def test_reader_parses_every_filter_and_the_defaults():
    import laser_slam_b200 as ls
    f = ls.point_filters_from_yaml(ALL_YAML)
    assert [x.type for x in f] == [ls.PF_REMOVE_NAN, ls.PF_MAX_DIST, ls.PF_MIN_DIST, ls.PF_BOUNDING_BOX, ls.PF_RANDOM_SAMPLING,
                                   ls.PF_FIX_STEP_SAMPLING, ls.PF_VOXEL_GRID, ls.PF_SURFACE_NORMAL,
                                   ls.PF_SAMPLING_SURFACE_NORMAL, ls.PF_SURFACE_NORMAL, ls.PF_RANDOM_SAMPLING]
    assert (f[1].dim, f[1].dist) == (1, 60.0)
    assert (f[2].dim, f[2].dist) == (-1, 0.5)                               # dim absent: -1
    assert list(f[3].box) == [-3, 3, -2, 2, -1.5, 2.5] and f[3].remove_inside == 0
    assert f[4].prob == np.float32(0.25) and f[5].step == 3
    assert list(f[6].leaf) == [np.float32(0.1), np.float32(0.2), np.float32(0.3)]
    assert f[7].knn == 7 and (f[8].knn, f[8].prob) == (12, np.float32(0.6))
    assert f[9].knn == 10 and f[10].prob == 1.0                              # compat's defaults: knn 10, prob / ratio 1
    d = ls.point_filters_from_yaml("- MaxDistDataPointsFilter\n- BoundingBoxDataPointsFilter\n- VoxelGridDataPointsFilter\n"
                                   "- FixStepSamplingDataPointsFilter\n")
    assert (d[0].dim, d[0].dist) == (-1, 1.0) and list(d[1].box) == [-1, 1, -1, 1, -1, 1] and d[1].remove_inside == 1
    assert list(d[2].leaf) == [1, 1, 1] and d[3].step == 10
    assert ls.point_filters_from_yaml("# nothing\n") == []


@pytest.mark.parametrize("yaml, index", [
    ("- RemoveNaNDataPointsFilter\n- ObservationDirectionDataPointsFilter\n", 1),
    ("- MaxDensityDataPointsFilter\n", 0),
    ("- RemoveNaNDataPointsFilter\n- FixStepSamplingDataPointsFilter:\n    startStep: 2\n    stepMult: 2\n", 1),
    ("- FixStepSamplingDataPointsFilter:\n    startStep: 2\n    endStep: 4\n", 0),
    ("- RemoveNaNDataPointsFilter\n- RemoveNaNDataPointsFilter\n- VoxelGridDataPointsFilter:\n    useCentroid: 0\n", 2),
    ("- MaxDistDataPointsFilter:\n    dim: 3\n", 0),
])
def test_reader_refuses_what_the_path_does_not_run(yaml, index):
    import laser_slam_b200 as ls
    with pytest.raises(ls.LsError, match=f"#{index} "):
        ls.point_filters_from_yaml(yaml)


def test_oracle_filter_rules_on_known_answers(oracle_mod):
    o = oracle_mod
    pts = np.array([[60, 0, 0, 1], [59.99, 0, 0, 1], [0, 1, 0, 1], [0, 0.5, 0, 1], [np.nan, 0, 0, 1], [0, 0, np.inf, 1],
                    [3, 0, 0, 1], [2.5, 1.9, -2.9, 1]], np.float32)
    p, n = fo.apply_filters([("MaxDistDataPointsFilter", {"maxDist": 60.0})], pts)
    assert n is None and np.array_equal(p, pts[[1, 2, 3, 6, 7]])              # at maxDist: dropped; NaN / inf: dropped
    p, _ = fo.apply_filters([("MinDistDataPointsFilter", {"minDist": 1.0})], pts)
    assert np.array_equal(p, pts[[0, 1, 5, 6, 7]])                            # at minDist: dropped; inf: kept
    p, _ = fo.apply_filters([("MaxDistDataPointsFilter", {"dim": 0, "maxDist": 3.0})], pts)
    assert np.array_equal(p, pts[[2, 3, 5, 7]])                               # |x| < 3 only
    p, _ = fo.apply_filters([("RemoveNaNDataPointsFilter", {})], pts)
    assert np.array_equal(p, np.delete(pts, 4, 0))
    box = [("BoundingBoxDataPointsFilter", dict(EGO_BOX, removeInside=1))]
    out, _ = fo.apply_filters(box, pts)
    ins, _ = fo.apply_filters([("BoundingBoxDataPointsFilter", dict(EGO_BOX, removeInside=0))], pts)
    assert [3, 0, 0] in out[:, :3].tolist() and [3, 0, 0] not in ins[:, :3].tolist()    # on a face: outside
    assert np.array_equal(ins, pts[[2, 3, 7]]) and len(out) + len(ins) == len(pts)
    # the fixed step, with normals travelling along
    cloud = np.concatenate([np.arange(30, dtype=np.float32)[:, None] * [1, 0, 0], np.ones((30, 1))], 1).astype(np.float32)
    nrm = np.tile(np.float32([0, 0, 1]), (30, 1)) * np.arange(30, dtype=np.float32)[:, None]
    p, n = fo.apply_filters([("FixStepSamplingDataPointsFilter", {"startStep": 4})], cloud, nrm)
    assert np.array_equal(p[:, 0], np.arange(0, 30, 4)) and np.array_equal(n[:, 2], np.arange(0, 30, 4))
    # RandomSampling draws on the index in the cloud entering it: a crop in front changes which points survive
    rng = np.random.default_rng(1)
    big = np.concatenate([rng.uniform(-20, 20, (4000, 3)), np.ones((4000, 1))], 1).astype(np.float32)
    crop = ("MaxDistDataPointsFilter", {"maxDist": 15.0})
    samp = ("RandomSamplingDataPointsFilter", {"prob": 0.5})
    a, _ = fo.apply_filters([crop, samp], big)
    b, _ = fo.apply_filters([samp, crop], big)
    assert np.array_equal(a, fo.apply_filters([crop], big)[0][o.keep_mask(len(fo.apply_filters([crop], big)[0]), 0x7e11, 0.5)])
    assert not np.array_equal(a, b) and abs(len(a) - len(b)) < 200


def test_oracle_voxel_normals_are_the_exact_mean(oracle_mod):
    rng = np.random.default_rng(4)
    pts = np.concatenate([rng.uniform(-2, 2, (3000, 3)), np.ones((3000, 1))], 1).astype(np.float32)
    nrm = rng.normal(size=(3000, 3)).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    p, n = fo.apply_filters([("VoxelGridDataPointsFilter", {"vSizeX": 0.5, "vSizeY": 0.5, "vSizeZ": 1.0})], pts, nrm)
    assert np.array_equal(p, oracle_mod.voxel_grid(pts, (0.5, 0.5, 1.0)))
    cell = np.floor(pts[:, :3] / np.float32([0.5, 0.5, 1.0])).astype(np.int64)
    key = {tuple(c) for c in cell}
    assert len(p) == len(key)
    for v in range(0, len(p), 37):                                            # every 37th voxel: numpy's exact mean
        c = tuple(np.floor(p[v, :3] / np.float32([0.5, 0.5, 1.0])).astype(np.int64))
        members = (cell == c).all(1)
        want = np.array([float(np.sum([np.rint(np.float64(x) * 2.0 ** 24) for x in nrm[members, a]], dtype=np.float64))
                         for a in range(3)]) / (members.sum() * 2.0 ** 24)
        assert np.array_equal(n[v], want.astype(np.float32))
    assert np.abs(np.linalg.norm(n, axis=1) - 1).max() > 0.1                  # not renormalised


def _raw_scan(scans, k=0):
    """A full 131072-point synthetic scan with injected NaN and far points."""
    p, n = scans[k][0].copy(), scans[k][1].copy()
    p[::97, 0] = np.nan
    p[5::131, 1] = np.nan
    p[7::89, :3] *= 40.0
    return p, n


def _yaml(oracle_mod, chain):
    return fo.filters_yaml(chain)


@pytest.mark.gpu
def test_gpu_each_filter_and_the_chain_equal_the_oracle(gpu_ctx, oracle_mod, scans):
    o = oracle_mod
    raw, nrm = _raw_scan(scans)
    clean = raw[~np.isnan(raw[:, :3]).any(1)]
    singles = [CHAIN[0], CHAIN[1], CHAIN[2], ("MaxDistDataPointsFilter", {"dim": 2, "maxDist": 1.5}), CHAIN[3],
               ("BoundingBoxDataPointsFilter", dict(EGO_BOX, removeInside=0)), CHAIN[4],
               ("FixStepSamplingDataPointsFilter", {"startStep": 3}), CHAIN[5]]
    for f in singles:
        for with_normals in (False, True):
            want = fo.apply_filters([f], raw, nrm if with_normals else None)
            got = gpu_ctx.filter_cloud(_yaml(o, [f]), raw, nrm if with_normals else None)
            assert got[0].shape == want[0].shape and np.array_equal(got[0], want[0], equal_nan=True), f
            if with_normals:
                assert np.array_equal(got[1], want[1]), f
    for f in (CHAIN[6], ("SamplingSurfaceNormalDataPointsFilter", {"knn": 8, "ratio": 0.4})):
        want = fo.apply_filters([f], clean, num_threads=8)
        got = gpu_ctx.filter_cloud(_yaml(o, [f]), clean)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), f
    want = fo.apply_filters(CHAIN, raw, num_threads=8)
    got = gpu_ctx.filter_cloud(_yaml(o, CHAIN), raw)
    assert 10000 < len(want[0]) < len(raw) // 2
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    # the same chain straight into a ring slot: the slot holds the same bits
    mp = gpu_ctx.create_map(4, 131072)
    before = gpu_ctx.launch_count
    sid, kept = mp.push_scan_filtered(_yaml(o, CHAIN), raw)
    launches = gpu_ctx.launch_count - before
    assert kept == len(want[0]) and mp.scan_size(sid) == kept and launches > 0
    pts, nr = mp.assemble([sid], [np.eye(4, dtype=np.float32)])
    assert np.array_equal(pts, want[0]) and np.array_equal(nr, want[1])
    # given normals are carried through the chain when no normal filter follows
    sid2, kept2 = mp.push_scan_filtered(_yaml(o, CHAIN[:5]), raw, nrm)
    want2 = fo.apply_filters(CHAIN[:5], raw, nrm)
    pts, nr = mp.assemble([sid2], [np.eye(4, dtype=np.float32)])
    assert kept2 == len(want2[0]) and np.array_equal(pts, want2[0]) and np.array_equal(nr, want2[1])
    mp.close()


@pytest.mark.gpu
def test_gpu_icp_on_filtered_slots_equals_oracle(gpu_ctx, oracle_mod, scans, traj):
    import laser_slam_b200 as ls
    from conftest import make_submap
    o = oracle_mod
    truth, odom = traj
    mp = gpu_ctx.create_map(8, 131072)
    filt, ids = [], []
    for k in range(5):
        raw, _ = _raw_scan(scans, k)
        filt.append(fo.apply_filters(CHAIN, raw, num_threads=8))
        ids.append(mp.push_scan_filtered(_yaml(o, CHAIN), raw)[0])
    Tparts = [np.eye(4, dtype=np.float32) if k == 3 else (np.linalg.inv(truth[3]) @ truth[k]).astype(np.float32) for k in [3, 2, 1, 0]]
    T0 = (np.linalg.inv(truth[3]) @ odom[4]).astype(np.float32)
    p = ls.default_params(max_iterations=30)
    g = mp.register(ids[4], [ids[3], ids[2], ids[1], ids[0]], Tparts, T0, p)
    ref, nr = make_submap(o, filt, truth, 3, [3, 2, 1, 0])
    po = o.default_params(max_iterations=p.max_iterations, trim_ratio=p.trim_ratio, use_differential=p.use_differential,
                          min_diff_rot=p.min_diff_rot, min_diff_trans=p.min_diff_trans, smooth_length=p.smooth_length)
    r = o.icp(filt[4][0], ref, nr, T0, po)
    assert r["rc"] == 0 and g["rc"] == 0 and g["stats"].iterations == r["stats"].iterations
    assert np.array_equal(g["T"], r["T"])
    rel = np.linalg.inv(truth[3]) @ truth[4]
    assert np.abs(g["T"][:3, 3] - rel[:3, 3]).max() < 0.05
    mp.close()


@pytest.mark.gpu
def test_gpu_empty_result_and_refusals(gpu_ctx, oracle_mod, scans):
    import laser_slam_b200 as ls
    o = oracle_mod
    raw, nrm = _raw_scan(scans)
    mp = gpu_ctx.create_map(4, 131072)
    a = mp.push_scan(scans[1][0], scans[1][1])
    nothing = [("MaxDistDataPointsFilter", {"maxDist": 0.001}), ("SurfaceNormalDataPointsFilter", {})]
    sid, kept = mp.push_scan_filtered(_yaml(o, nothing), raw)
    assert kept == 0 and mp.scan_size(sid) == 0
    T0 = np.eye(4, dtype=np.float32)
    T0[:3, 3] = [0.3, -0.2, 0.1]
    g = mp.register(sid, [a], [np.eye(4, dtype=np.float32)], T0, raise_on_convergence=False)
    assert g["rc"] == ls.LS_ERR_CONVERGENCE and np.array_equal(g["T"], T0)
    n_before = mp.scan_size(a)
    with pytest.raises(ls.LsError, match="normal filter"):                  # a slot must be usable as a reference
        mp.push_scan_filtered(_yaml(o, CHAIN[:5]), raw)
    with pytest.raises(ls.LsError, match="normal filter"):
        gpu_ctx.filter_cloud(_yaml(o, CHAIN[:5]), raw, want_normals=True)
    small = gpu_ctx.create_map(2, 1000)                                      # more points than a slot holds: no slot taken
    with pytest.raises(ls.LsError, match="more than a slot holds"):
        small.push_scan_filtered(_yaml(o, CHAIN[:1]), raw, nrm)
    assert mp.scan_size(a) == n_before
    small.close()
    mp.close()


@pytest.mark.gpu
def test_estimator_with_input_filters_matches_oracle_flow(oracle_mod, synth_mod, tmp_path):
    """host.Estimator handed raw scans (no normals) and a filter file == the restated per-scan flow on oracle-filtered
    scans; the track stores the filtered clouds (buildSubMapAroundTime returns them)."""
    from laser_slam_b200 import host
    from oracle import posegraph_oracle as pg
    from test_host_layer import oracle_flow
    o = oracle_mod
    n_scans, K = 7, 4
    truth, odom = synth_mod.trajectory(2, n_scans)
    raw = [synth_mod.subsample(*synth_mod.scan(truth[k], 2, k), 16)[0].copy() for k in range(n_scans)]
    for k, p in enumerate(raw):
        p[k::53, 2] = np.nan
    chain = [("RemoveNaNDataPointsFilter", {}), ("MaxDistDataPointsFilter", {"maxDist": 60.0}),
             ("RandomSamplingDataPointsFilter", {"prob": 0.8}), ("SurfaceNormalDataPointsFilter", {"knn": 10})]
    path = tmp_path / "input_filters.yaml"
    path.write_text(fo.filters_yaml(chain))
    filt = [fo.apply_filters(chain, p) for p in raw]
    odom7 = pg.se3_from_matrix(odom)
    po = o.default_params(trim_ratio=0.85, min_diff_rot=0.001, min_diff_trans=0.001, smooth_length=3)
    ref_traj, ref_icp = oracle_flow(o, filt, odom7, K, po)
    est = host.Estimator(n_workers=1, nscan_in_sub_map=K, icp_input_filters_path=str(path))
    got_icp = []
    for k in range(n_scans):
        icp7, st = est.step(0, k * 100_000_000, odom7[k], raw[k])
        got_icp.append(icp7)
        if k > 0:
            assert st.iterations >= 1
    times, traj = est.trajectory(0)
    got_icp = np.stack(got_icp)
    assert est.num_scans(0) == n_scans
    assert np.abs(got_icp[:, 4:] - ref_icp[:, 4:]).max() < 1e-6
    assert np.abs(traj[:, 4:] - ref_traj[:, 4:]).max() < 1e-6
    dR = np.swapaxes(pg.quat_to_R(traj[:, :4]), -1, -2) @ pg.quat_to_R(ref_traj[:, :4])
    assert np.abs(pg.so3_log(dR)).max() < 1e-6
    sub, sub_n = est.build_submap(0, 3 * 100_000_000, 1, 3 * len(raw[0]))
    parts = [filt[3]]
    for idx in (2, 4):
        T = pg.se3_to_matrix(pg.se3_compose(pg.se3_inverse(traj[3]), traj[idx])).astype(np.float32)
        parts.append(o.transform_cloud(T, *filt[idx]))
    assert sub.shape[0] == sum(len(f[0]) for f in filt[2:5]) < 3 * len(raw[0])
    assert np.array_equal(sub[:len(filt[3][0])], filt[3][0]) and np.array_equal(sub_n[:len(filt[3][0])], filt[3][1])
    assert np.abs(sub - np.concatenate([p[0] for p in parts])).max() < 1e-4
    est.close()
    # without normals and without a normal filter the scan is refused
    path2 = tmp_path / "no_normals.yaml"
    path2.write_text(fo.filters_yaml(chain[:3]))
    est2 = host.Estimator(n_workers=1, nscan_in_sub_map=K, icp_input_filters_path=str(path2))
    with pytest.raises(Exception, match="normal filter"):
        est2.step(0, 0, odom7[0], raw[0])
    est2.close()
