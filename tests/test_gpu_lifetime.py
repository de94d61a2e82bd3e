"""-m gpu tests of object lifetimes through the C ABI: a create that fails on an allocation reports it once and leaves the engine as
it was, a failed b2s_mapper_graph_enable can be retried, and objects may be destroyed after the engine that made them."""
import numpy as np
import pytest

from open3d_slam_b200 import engine as E
from open3d_slam_b200 import synth
from open3d_slam_b200 import _lib as L
from test_gpu_parity import _keyed, lua_params

pytestmark = pytest.mark.gpu

HUGE = 1 << 40   # points: about 30 TiB of coordinates, so cudaMalloc fails at once and nothing reaches the device


def config1_registration(eng):
    src, tgt, nrm, _ = synth.planar_cloud_config1()
    return E.RegistrationIcpPointToPlane(eng).registerClouds(eng.cloud(src), eng.cloud(tgt, nrm), np.eye(4))


def assert_same_registration(a, b):
    assert a.iters == b.iters and a.n_corr == b.n_corr
    # the ICP kernel's phase-2 queue is drained in atomic order: the fp64 sums agree to the last few bits only
    assert np.abs(a.transformation_ - b.transformation_).max() < 1e-12


def test_failed_create_leaves_the_engine_usable(engine_factory):
    eng = engine_factory(lua_params())
    with pytest.raises(L.B2SError) as err:
        E.Submap(eng, capacity_points=HUGE)
    assert err.value.code == L.E_CUDA
    assert_same_registration(config1_registration(eng), config1_registration(engine_factory(lua_params())))


def test_failed_graph_enable_can_be_retried(engine_factory):
    p = lua_params(seed=3)
    sc = synth.Scene(); poses = synth.loop_trajectory(12)
    e1, e2 = engine_factory(p), engine_factory(p)
    m1, m2 = E.Mapper(e1, 600_000), E.Mapper(e2, 600_000)
    raw0 = synth.lidar_scan(sc, poses[0], seed=50)
    for m, e in ((m1, e1), (m2, e2)):
        m.addRangeMeasurement(e.cloud(raw0), None)
        m.submap.setPose(np.eye(4))
    with pytest.raises(L.B2SError) as err:
        m2.enableGraph(HUGE)
    assert err.value.code == L.E_CUDA
    st = m2.enableGraph(65536)
    for k in range(1, 10):      # steps 1-2 run eagerly (warm-up), step 3 captures, the rest replay
        raw = synth.lidar_scan(sc, poses[k], seed=50 + k)
        delta = np.linalg.inv(poses[k - 1]) @ poses[k]
        m1.addRangeMeasurementAsync(e1.cloud(raw), delta, slot=k)
        st.upload(raw)
        sl = m2.addRangeMeasurementAsync(st, delta)
        r1, r2 = m1.fetchResult(k), m2.fetchResult(sl)
        assert_same_registration(r1, r2)
        assert r1.fitness_ > 0.9
    assert np.abs(m1.submap.getPose() - m2.submap.getPose()).max() < 1e-12
    a = m1.submap.getMapPointCloud()[0]; b = m2.submap.getMapPointCloud()[0]
    assert a.shape == b.shape and np.abs(_keyed(a, a, 0.1)[0] - _keyed(b, b, 0.1)[0]).max() < 1e-11


def test_objects_are_destroyed_after_their_engine(engine_factory):
    """b2s_destroy first, then the clouds, a submap with a dense map and a captured graph, a feature and a voxel map: their destroy
    functions wait for the device and never touch the handle."""
    p = lua_params(seed=3)
    sc = synth.Scene(); poses = synth.loop_trajectory(6)
    eng = engine_factory(p)
    m = E.Mapper(eng, 600_000)
    m.submap.setMapperOptions(dense=True)
    raw = [synth.lidar_scan(sc, poses[k], seed=60 + k) for k in range(5)]
    clouds = [eng.cloud(r) for r in raw]
    m.addRangeMeasurement(clouds[0], None)
    m.submap.setPose(np.eye(4))
    st = m.enableGraph(65536)
    for k in range(1, 5):       # steps 1-2 warm up, step 3 captures, step 4 replays
        st.upload(raw[k])
        m.addRangeMeasurementAsync(st, np.linalg.inv(poses[k - 1]) @ poses[k])
    assert m.submap.denseSize() > 0
    _, tgt, nrm, _ = synth.planar_cloud_config1()
    clouds.append(eng.cloud(tgt, nrm))
    feature = E.computeFPFHFeature(eng, clouds[-1], 0.5, 30)
    vm = E.VoxelMap(eng, 0.25)
    vm.insertCloud("map", clouds[0])
    before = config1_registration(eng)
    eng.synchronize()
    eng.close()
    for c in clouds:
        c.free()
    for obj in (m.submap, feature, vm):
        obj.free()
    assert_same_registration(before, config1_registration(engine_factory(p)))
