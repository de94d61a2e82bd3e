"""CPU: slam.buildLoopClosureConstraints over the oracle backend (tests/oracle_backend_ransac.py) on a constructed pair of submaps --
a room of planes and its copy moved by a known rigid transform, with the sparse clouds' features shared, so the proposal is exact:
accepted with the transform recovered, rejected by the correspondence-set gate, rejected by the consistency check (an offset beyond
80 m) -- and the consistency check's RPY restatement."""
import copy

import numpy as np
import pytest

from oracle_backend import OracleCloud, OracleSubmap
from oracle_backend_ransac import RansacOracleBackend
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from test_ransac_oracle import rigid


def room(seed=0, n=6000):
    """floor, two walls and a box: point-to-plane ICP is constrained in every direction"""
    rng = np.random.default_rng(seed)
    parts = []
    k = n // 5
    u = rng.uniform(0, 1, (n, 2))
    parts.append((np.c_[12 * u[:k, 0], 12 * u[:k, 1], np.zeros(k)], [0, 0, 1]))
    parts.append((np.c_[np.zeros(k), 12 * u[k:2 * k, 0], 3 * u[k:2 * k, 1]], [1, 0, 0]))
    parts.append((np.c_[12 * u[2 * k:3 * k, 0], np.zeros(k), 3 * u[2 * k:3 * k, 1]], [0, 1, 0]))
    parts.append((np.c_[4 + 2 * u[3 * k:4 * k, 0], 5 + 3 * u[3 * k:4 * k, 1], np.full(k, 1.5)], [0, 0, 1]))
    parts.append((np.c_[np.full(k, 6.0), 5 + 3 * u[4 * k:5 * k, 0], 1.5 * u[4 * k:5 * k, 1]], [1, 0, 0]))
    xyz = np.vstack([p for p, _ in parts])
    nrm = np.vstack([np.tile(nv, (len(p), 1)) for p, nv in parts]).astype(np.float64)
    return xyz, nrm


def collection(T, seed=0):
    """two submap records: the room, and the room moved by T; sparse clouds = every 10th point, features shared row for row"""
    be = RansacOracleBackend(E.MapperParameters())
    sc = S.SubmapCollection(be, S.SubmapParameters())
    xyz, nrm = room(seed)
    feat = np.random.default_rng(seed + 1).uniform(0, 100, (len(xyz[::10]), 33))
    for k, (x, n) in enumerate([(xyz, nrm), (xyz @ T[:3, :3].T + T[:3, 3], nrm @ T[:3, :3].T)]):
        sm = OracleSubmap(None)
        sm.xyz, sm.nrm = x, n
        rec = S.SubmapRecord(sm, k, 0, np.zeros(3))
        rec.sparse, rec.feature = OracleCloud(x[::10]), feat
        sc.submaps.append(rec)
    return be, sc


P = E.PlaceRecognitionParameters()


def test_accepted_recovers_the_transform():
    T = rigid(0.4, [3.0, -1.5, 0.2], 0.02, -0.01)
    be, sc = collection(T)
    cons, log = S.buildLoopClosureConstraints(be, sc, 0, [1], P, 0.1)
    assert log == [(1, "accepted", len(sc.submaps[0].sparse))]
    (c,) = cons
    assert (c.sourceSubmapIdx, c.targetSubmapIdx, c.isInformationMatrixValid, c.isOdometryConstraint) == (0, 1, True, False)
    assert np.abs(c.sourceToTarget - T).max() < 1e-6
    assert c.informationMatrix.shape == (6, 6) and np.allclose(c.informationMatrix, c.informationMatrix.T)


def test_rejected_by_the_correspondence_gate():
    be, sc = collection(rigid(0.4, [3.0, -1.5, 0.2]))
    p = copy.deepcopy(P)
    p.ransacMinCorrespondenceSetSize = len(sc.submaps[0].sparse) + 1     # more inliers than there are sparse points
    cons, log = S.buildLoopClosureConstraints(be, sc, 0, [1], p, 0.1)
    assert cons == [] and log == [(1, "rejected_correspondences", len(sc.submaps[0].sparse))]


def test_rejected_by_the_consistency_check():
    be, sc = collection(rigid(0.1, [100.0, 0.0, 0.0]))                   # |x| = 100 m > 80 m
    cons, log = S.buildLoopClosureConstraints(be, sc, 0, [1], P, 0.1)
    assert cons == [] and log == [(1, "rejected_ransac_inconsistent", len(sc.submaps[0].sparse))]
    assert S.LoopClosureConsistencyCheck(maxDriftX=200.0).isRegistrationConsistent(rigid(0.1, [100.0, 0.0, 0.0]))


def test_missing_features_and_no_candidates():
    be, sc = collection(np.eye(4))
    assert S.buildLoopClosureConstraints(be, sc, 0, [], P, 0.1) == ([], [])
    sc.submaps[1].feature = None
    with pytest.raises(RuntimeError):
        S.buildLoopClosureConstraints(be, sc, 0, [1], P, 0.1)


@pytest.mark.parametrize("deg,ok", [(29.0, True), (31.0, False)])
def test_rpy_limits(deg, ok):
    """toRPY (src/math.cpp:39-46) against the Z-Y-X angles the rotation was built from; the Lua limit is 30 deg on each"""
    c = S.LoopClosureConsistencyCheck()
    for axis in range(3):
        e = [0.0, 0.0, 0.0]; e[axis] = np.deg2rad(deg)
        T = rigid(e[2], [0, 0, 0], e[1], e[0])
        assert np.allclose(S.toRPY(T[:3, :3]), e, atol=1e-12)
        assert c.isRegistrationConsistent(T) == ok
