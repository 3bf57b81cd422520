import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100: pytest -m gpu)")


@pytest.fixture(scope="session")
def oracle_mod():
    import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def synth_mod():
    from laser_slam_b200 import synth
    synth.build()
    return synth


@pytest.fixture(scope="session")
def traj(synth_mod):
    return synth_mod.trajectory(0, 8)


@pytest.fixture(scope="session")
def scans(synth_mod, traj):
    """Six consecutive full HDL-64-shaped scans (131072 points each) of sequence 0."""
    truth, _ = traj
    return [synth_mod.scan(truth[k], 0, k) for k in range(6)]


@pytest.fixture(scope="session")
def small_pair(synth_mod, scans, traj):
    """Two sub-sampled scans (8192 points) + a perturbed initial guess: the CPU-sized parity case."""
    truth, odom = traj
    a, an = synth_mod.subsample(*scans[0], 16)
    b, bn = synth_mod.subsample(*scans[1], 16)
    T0 = (np.linalg.inv(truth[0]) @ odom[1]).astype(np.float32)
    return dict(reading=b, ref=a, ref_normals=an, T0=T0, truth=(np.linalg.inv(truth[0]) @ truth[1]))


def make_submap(oracle_mod, scans, truth, kref, ks):
    """Reference construction of LaserTrack::localScanToSubMap's sub-map (reference laser_track.cpp:476-486)."""
    ref, nr = [], []
    for k in ks:
        if k == kref:
            p, n = scans[k]
        else:
            T = (np.linalg.inv(truth[kref]) @ truth[k]).astype(np.float32)
            p, n = oracle_mod.transform_cloud(T, scans[k][0], scans[k][1])
        ref.append(p)
        nr.append(n)
    return np.concatenate(ref), np.concatenate(nr)


@pytest.fixture(scope="session")
def config2(oracle_mod, scans, traj):
    """Config 2 of BASELINE.json: scan 4 (131072 pts) vs map = scans 3,2,1,0 in the frame of scan 3 (524288 pts)."""
    truth, odom = traj
    ref, nr = make_submap(oracle_mod, scans, truth, 3, [3, 2, 1, 0])
    T0 = (np.linalg.inv(truth[3]) @ odom[4]).astype(np.float32)
    return dict(reading=scans[4][0], ref=ref, ref_normals=nr, T0=T0, truth=(np.linalg.inv(truth[3]) @ truth[4]))


@pytest.fixture(scope="session")
def gpu_ctx():
    import laser_slam_b200 as ls
    ctx = ls.Context(0)
    yield ctx
    ctx.close()
