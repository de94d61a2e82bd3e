"""CPU: SegmentMapper.getDenseSubmapPointClouds / getActiveDenseMapPointCloud (SubmapCollection::dumpToFile(.., true), publishDenseMap;
DESIGN.md row A2) over the oracle backend on a stretch of the closed lap -- one array per submap in submap order, the active submap's
array, voxels emptied by carving absent, and submaps without a dense map giving empty arrays."""
import copy

import numpy as np
import pytest

from oracle_backend_dense_export import DenseExportOracleBackend, dense_cloud
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W


def rows(a):
    return {tuple(r) for r in np.ascontiguousarray(a).view(np.uint64).reshape(-1, 3)}


@pytest.fixture(scope="module")
def lap():
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    be = DenseExportOracleBackend(copy.deepcopy(p), carving=True, dense=True)
    m = S.SegmentMapper(be, S.SubmapParameters(radius=3.0))
    for k in range(24):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    assert len(m.submaps.submaps) >= 2
    return be, m


def test_one_array_per_submap_in_submap_order(lap):
    be, m = lap
    subs = m.submaps.submaps
    got = m.getDenseSubmapPointClouds()
    assert len(got) == len(subs)
    for g, s in zip(got, subs):
        ref = dense_cloud(s.handle)
        assert g.shape == ref.shape and len(g) > 1000 and np.array_equal(g, ref)
    assert sum(be.counters(s.handle)["dense_carve_runs"] for s in subs) > 0


def test_active_submap_is_the_last_one(lap):
    _be, m = lap
    assert m.submaps.activeSubmapIdx == len(m.submaps.submaps) - 1
    a = m.getActiveDenseMapPointCloud()
    assert np.array_equal(a, m.getDenseSubmapPointClouds()[-1]) and len(a) > 0


def test_emptied_voxels_are_absent():
    """carving a submap's dense map by hand along rays through its own voxels: the export loses as many rows as the carve reports
    voxels removed, and every other voxel keeps its mean"""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    be = DenseExportOracleBackend(copy.deepcopy(p), carving=True, dense=True)
    m = S.SegmentMapper(be, S.SubmapParameters(radius=3.0))
    for k in range(6):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    sm = m.submaps.submaps[0].handle
    before = m.getDenseSubmapPointClouds()[0]
    sensor = before.mean(axis=0)
    scan = sensor + 1.5 * (before[::50] - sensor)   # rays from the sensor through some of its voxels, ending beyond them
    removed = sm.dense.carve(scan, sensor, p.denseMapVoxelSize, 0.1, 0.1, 20.0)
    after = m.getDenseSubmapPointClouds()[0]
    assert removed > 0 and len(after) == len(before) - removed
    assert rows(after) <= rows(before) and len(rows(before) - rows(after)) == removed


def test_submaps_without_a_dense_map_give_empty_arrays(lap):
    be, m = lap
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    nd = DenseExportOracleBackend(copy.deepcopy(p), carving=True, dense=False)
    m2 = S.SegmentMapper(nd, S.SubmapParameters(radius=3.0))
    assert m2.getDenseSubmapPointClouds() == [] and m2.getActiveDenseMapPointCloud().shape == (0, 3)
    for k in range(8):
        m2.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    got = m2.getDenseSubmapPointClouds()
    assert len(got) == len(m2.submaps.submaps) >= 1 and all(g.shape == (0, 3) for g in got)
    assert m2.getActiveDenseMapPointCloud().shape == (0, 3)
    # mixed with dense maps: empty in place, the others unchanged
    a, b = m.submaps.submaps[0].handle, m2.submaps.submaps[0].handle
    mixed = be.dense_map_clouds([a, b, a])
    assert mixed[1].shape == (0, 3) and np.array_equal(mixed[0], dense_cloud(a)) and np.array_equal(mixed[2], mixed[0])
