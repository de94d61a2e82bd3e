"""-m gpu: localisation against a prior map on the device (b2s_submap_set_initial_map / _set_initial_transform / _set_merge_scans) against
the oracle backend with the reference's rules restated (tests/oracle_backend_localization.py).  The prior map is the oracle's map of the
first scans of the closed lap (tests/test_localization_host.py); lap-2 scans of the same poses, with another noise seed, are localised
in it from an initial pose 0.25 m and 2 degrees off.

Tolerances: the voxelized initial map bit-identical to the oracle's, its averaged normals within 1e-6 (the normals' own tolerance,
tests/test_gpu_parity.py); per scan T within 1e-8 and the fitness equal; poses within 0.1 m of the truth."""
import copy

import numpy as np
import pytest

from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S

from oracle_backend_localization import OracleLocalizationBackend
from test_localization_host import perturbed, prior  # noqa: F401  (prior: the module's fixture)

pytestmark = pytest.mark.gpu

TICK = 10_000_000
K0 = 3


def _backends(merge, graph=True):
    p = E.MapperParameters(seed=3, isUseInitialMap=True, isMergeScansIntoMap=merge)
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=graph, submap_capacity=400_000)
    ora = OracleLocalizationBackend(copy.deepcopy(p), carving=True, dense=True)
    sp = S.SubmapParameters(radius=2.0, minNumRangeData=2)   # a mapping run would hand over within a few scans
    return dev, ora, S.SegmentMapper(dev, sp), S.SegmentMapper(ora, sp)


def _sorted(xyz, nrm):
    o = np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0]))
    return xyz[o], nrm[o]


def test_initial_map_load_matches_the_oracle(prior):
    lp, xyz = prior
    dev, ora, md, mo = _backends(False)
    md.setInitialMap(xyz)
    mo.setInitialMap(xyz)
    gx, gn = _sorted(*dev.map_cloud(md.submaps.getActiveSubmap().handle))
    rx, rn = _sorted(*ora.map_cloud(mo.submaps.getActiveSubmap().handle))
    assert len(gx) == len(rx) < len(xyz)
    assert np.array_equal(gx, rx)                                             # voxel means: bit-identical
    assert np.abs(gn - rn).max() < 1e-6                                       # averaged normals
    assert dev.counters(md.submaps.getActiveSubmap().handle)["inserted_map"] == 0
    dev.close()


def _localise(prior, merge, graph, n=10):
    lp, xyz = prior
    dev, ora, md, mo = _backends(merge, graph)
    for m in (md, mo):
        m.setInitialMap(xyz)
    sm = md.submaps.getActiveSubmap().handle
    map0 = dev.map_cloud(sm)
    T = perturbed(lp.map_frame_pose(K0))
    for m in (md, mo):
        m.setInitialTransform(T)
    caps = []
    for i in range(n):
        k = K0 + 1 + i
        raw = lp.scan(k + lp.L, seed=200 + k)
        rd = md.addRangeMeasurement(raw, lp.delta(k))
        ro = mo.addRangeMeasurement(raw, lp.delta(k))
        assert np.abs(np.asarray(rd.transformation_) - np.asarray(ro.transformation_)).max() <= 1e-8, i
        assert rd.fitness_ == ro.fitness_, i
        assert np.abs(md.poses[-1] - mo.poses[-1]).max() <= 1e-8, i
        if i == 0:
            assert np.array_equal(sm.getPose(), T)                             # rule 3 on the device: the pose slot still holds T
        caps.append(dev.eng.graphCaptures)
    assert np.array_equal(md.poses[0], T)                                      # rule 3: the ICP result was discarded
    for i, P in enumerate(md.poses[1:]):
        assert np.linalg.norm(P[:3, 3] - lp.map_frame_pose(K0 + 2 + i)[:3, 3]) < 0.1
    assert len(md.submaps.submaps) == 1
    if graph:   # the chain was captured once (after the eager warm-up) and replayed from then on
        assert caps[-1] == 1 and caps[2] == 1, caps
    return dev, md, sm, map0


@pytest.mark.parametrize("graph", [False, True])
def test_pure_localisation_agrees_with_the_oracle_and_leaves_the_map_alone(prior, graph):
    dev, md, sm, map0 = _localise(prior, merge=False, graph=graph)
    map1 = dev.map_cloud(sm)
    assert np.array_equal(map0[0], map1[0]) and np.array_equal(map0[1], map1[1])
    c = dev.counters(sm)
    assert c["inserted_map"] == 0 and c["carve_runs"] == 0 and c["inserted_dense"] == c["accepted"] == len(md.poses)
    dev.close()


def test_localisation_with_map_building_merges_and_never_hands_over(prior):
    dev, md, sm, map0 = _localise(prior, merge=True, graph=True)
    c = dev.counters(sm)
    assert c["inserted_map"] == len(md.poses) - 1                              # every step but the first after the initial value
    assert not any(e[0] == "active_submap_changed" for e in md.submaps.events)
    assert len(dev.map_cloud(sm)[0]) != len(map0[0])
    dev.close()


def test_merge_switch_drops_the_captured_chain_and_takes_effect(prior):
    """pure localisation, then merge on mid-run: the graph is captured again and the next accepted scans are fused"""
    lp, xyz = prior
    dev, _ora, md, _mo = _backends(False, graph=True)
    md.setInitialMap(xyz)
    sm = md.submaps.getActiveSubmap().handle
    md.setInitialTransform(lp.map_frame_pose(K0))
    for k in range(K0 + 1, K0 + 6):
        md.addRangeMeasurement(lp.scan(k + lp.L, seed=k), lp.delta(k))
    assert dev.counters(sm)["inserted_map"] == 0 and dev.eng.graphCaptures == 1
    sm.setMergeScans(True)
    for k in range(K0 + 6, K0 + 10):
        md.addRangeMeasurement(lp.scan(k + lp.L, seed=k), lp.delta(k))
    c = dev.counters(sm)
    assert c["inserted_map"] == 4 and dev.eng.graphCaptures == 2
    dev.close()


def test_slam_step_follows_rules_3_and_4(prior):
    """SegmentMapper.addRangeScan (b2s_slam_step_host_async, graph-replayed): the first step after the initial value keeps T and pushes it
    into the map-pose buffer at its time; the next step registers from T as well (oracle: the same guesses); then pure localisation"""
    lp, xyz = prior
    dev, ora, md, mo = _backends(False, graph=True)
    for m in (md, mo):
        m.setInitialMap(xyz)
    sm = md.submaps.getActiveSubmap().handle
    map0 = dev.map_cloud(sm)
    T = perturbed(lp.map_frame_pose(K0))
    for m in (md, mo):
        m.setInitialTransform(T)
    times = []
    for i in range(8):
        k = K0 + 1 + i
        t = (10 + i) * TICK
        times.append(t)
        raw = lp.scan(k + lp.L, seed=300 + k)
        rd = md.addRangeScan(raw, t)
        assert dev.last_slam_result.mapperAccepted
        if i == 0:
            assert np.array_equal(sm.getPose(), T)
        if i < 2:   # the two steps that register from the pose alone: the oracle needs no odometry for them
            ro = mo.addRangeMeasurement(raw, np.eye(4))
            assert np.abs(np.asarray(rd.transformation_) - np.asarray(ro.transformation_)).max() <= 1e-8, i
            assert rd.fitness_ == ro.fitness_
    assert np.array_equal(md.poses[0], T)
    odo = dev.odometry()
    assert np.array_equal(odo.getMapToRangeSensor(times[0]), T)                # pushed at the first step's time
    for i, P in enumerate(md.poses[1:]):
        assert np.linalg.norm(P[:3, 3] - lp.map_frame_pose(K0 + 2 + i)[:3, 3]) < 0.1
        assert np.abs(odo.getMapToRangeSensor(times[i + 1]) - P).max() <= 1e-12
    map1 = dev.map_cloud(sm)
    assert np.array_equal(map0[0], map1[0]) and np.array_equal(map0[1], map1[1])
    assert dev.counters(sm)["inserted_map"] == 0
    dev.close()
