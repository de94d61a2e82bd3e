"""-m "not gpu": localisation against a prior map (isUseInitialMap_ / isMergeScansIntoMap_) in slam.py's host flow, over the oracle
backend with the reference's rules restated (tests/oracle_backend_localization.py).  The prior map is the oracle's own map of the first
scans of the closed lap; the localised scans are lap-2 scans of the same poses with another noise seed."""
import copy

import numpy as np
import pytest

from oracle import oracle as O
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W
from oracle_backend import OracleBackend
from oracle_backend_localization import OracleLocalizationBackend

N_MAP = 10


@pytest.fixture(scope="module")
def prior():
    """(closed lap, map xyz): the map an oracle SegmentMapper builds from scans 0 .. N_MAP-1 in one submap"""
    lp = W.ClosedLoop()
    ora = OracleBackend(E.MapperParameters(seed=3), carving=False, dense=False)
    m = S.SegmentMapper(ora, S.SubmapParameters(radius=1e3))
    for k in range(N_MAP):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    xyz, _ = ora.map_cloud(m.submaps.submaps[0].handle)
    return lp, xyz.copy()


def perturbed(T, dxyz=(0.2, -0.15, 0.05), yaw_deg=2.0):
    c, s = np.cos(np.radians(yaw_deg)), np.sin(np.radians(yaw_deg))
    D = np.eye(4)
    D[:2, :2] = [[c, -s], [s, c]]
    D[:3, 3] = dxyz
    return np.asarray(T) @ D


def localiser(merge, dense=True, radius=20.0, minNumRangeData=5):
    p = E.MapperParameters(seed=3, isUseInitialMap=True, isMergeScansIntoMap=merge)
    ora = OracleLocalizationBackend(copy.deepcopy(p), carving=True, dense=dense)
    return ora, S.SegmentMapper(ora, S.SubmapParameters(radius=radius, minNumRangeData=minNumRangeData))


def test_lua_defaults_and_the_mode_switch():
    p = E.MapperParameters()
    assert p.isUseInitialMap is False and p.isMergeScansIntoMap is False
    m = S.SegmentMapper(OracleLocalizationBackend(p))
    with pytest.raises(RuntimeError):
        m.setInitialMap(np.zeros((10, 3)))
    _, m = localiser(False)
    with pytest.raises(RuntimeError):   # the pose slot lives in the submap: the map comes first
        m.setInitialTransform(np.eye(4))


def test_initial_map_is_the_voxelized_map_with_its_normals(prior):
    lp, xyz = prior
    ora, m = localiser(False)
    m.setInitialMap(xyz)
    p = ora.p
    nrm = O.estimate_normals(xyz, p.icp.knn, p.icp.maxDistanceKnn)
    vx, vn = O.voxel_down_sample(xyz, p.mapBuilder.mapVoxelSize, nrm)
    sm = m.submaps.getActiveSubmap().handle
    assert np.array_equal(sm.xyz, vx) and np.array_equal(sm.nrm, vn) and len(vx) < len(xyz)
    sc = m.submaps
    assert len(sc.submaps) == 1 and sc.numScansMergedInActiveSubmap == 1 and len(sc.overlapScansBuffer) == 1
    assert np.array_equal(sc.overlapScansBuffer[0][0].xyz, xyz)                 # the prepared, unvoxelized map is buffered
    assert ora.counters(sm)["inserted_map"] == 0 and m.poses == [] and m.results == []
    with pytest.raises(RuntimeError):
        m.setInitialMap(xyz)


def test_first_step_keeps_T_whatever_the_icp_returned_and_the_next_ignores_odometry(prior):
    lp, xyz = prior
    ora, m = localiser(False)
    m.setInitialMap(xyz)
    k0 = 3
    T = perturbed(lp.map_frame_pose(k0))
    m.setInitialTransform(T)
    sm = m.submaps.getActiveSubmap().handle
    map0 = (sm.xyz.copy(), sm.nrm.copy())
    ks = [k0 + 1, k0 + 2, k0 + 3, k0 + 4]
    for k in ks:
        m.addRangeMeasurement(lp.scan(k + lp.L, seed=100 + k), lp.delta(k))
    r0 = m.results[0]
    assert np.abs(np.asarray(r0.transformation_) - T).max() > 1e-3             # the ICP moved ...
    assert np.array_equal(m.poses[0], T)                                        # ... and its result was discarded
    assert np.array_equal(ora.guesses[0], T)                                    # rule 3: no odometry prediction
    assert np.array_equal(ora.guesses[1], T)                                    # the step after it ignores the odometry too
    assert not np.array_equal(lp.delta(ks[1]), np.eye(4))
    assert np.array_equal(ora.guesses[2], m.poses[1] @ lp.delta(ks[2]))         # then the prediction is back
    for k, P in zip(ks[1:], m.poses[1:]):
        assert np.linalg.norm(P[:3, 3] - lp.map_frame_pose(k)[:3, 3]) < 0.1
    # pure localisation: nothing was carved or inserted, the map is bit-identical, the dense map was fed with every step
    c = ora.counters(sm)
    assert c["inserted_map"] == 0 and c["carve_runs"] == 0 and c["inserted_dense"] == len(ks)
    assert np.array_equal(sm.xyz, map0[0]) and np.array_equal(sm.nrm, map0[1])
    assert m.submaps.numScansMergedInActiveSubmap == 1 and len(m.submaps.overlapScansBuffer) == 1


def test_a_new_initial_value_mid_run_applies_rule_3_again(prior):
    lp, xyz = prior
    ora, m = localiser(False, dense=False)
    m.setInitialMap(xyz)
    m.setInitialTransform(lp.map_frame_pose(2))
    for k in (3, 4):
        m.addRangeMeasurement(lp.scan(k + lp.L, seed=7 + k), lp.delta(k))
    T = perturbed(lp.map_frame_pose(6), (0.1, 0.1, 0.0), -1.5)
    m.setInitialTransform(T)
    m.addRangeMeasurement(lp.scan(7 + lp.L, seed=3), lp.delta(7))
    assert np.array_equal(m.poses[-1], T) and np.array_equal(ora.guesses[-1], T)


def test_merge_mode_merges_and_never_hands_over(prior):
    lp, xyz = prior
    ora, m = localiser(True, dense=False, radius=2.0, minNumRangeData=2)
    m.setInitialMap(xyz)
    sm = m.submaps.getActiveSubmap().handle
    n0 = len(sm.xyz)
    m.setInitialTransform(lp.map_frame_pose(0))
    for k in range(1, 9):
        m.addRangeMeasurement(lp.scan(k + lp.L, seed=50 + k), lp.delta(k))
    assert np.linalg.norm(m.poses[-1][:3, 3] - lp.map_frame_pose(8)[:3, 3]) < 0.1
    assert np.linalg.norm(m.poses[-1][:3, 3]) > 2.0                             # beyond the radius at which a mapping run hands over
    assert len(m.submaps.submaps) == 1 and not any(e[0] == "active_submap_changed" for e in m.submaps.events)
    c = ora.counters(sm)
    assert c["inserted_map"] == 7                                               # every step but the first after the initial value
    assert m.submaps.numScansMergedInActiveSubmap == 8 and len(sm.xyz) != n0
