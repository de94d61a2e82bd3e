"""-m gpu tests of motion compensation inside the combined device step (b2s_odometry_set_motion_compensation and the mapper's pose
buffer on the odometry object): disabled de-skew changes nothing, the velocities of every step against the numpy estimate over
buffers rebuilt from the fetched poses, the de-skewed clouds against b2s_undistort and the oracle, the chain built on them (eager,
graph-replayed, across a parameter change, and SegmentMapper with hand-overs) against the oracle composition with both de-skews
(tests/motion_compensation.py), the mapper's buffer against the numpy buffer, the argument checks and the lifetime of an object with
de-skew and captured graphs.  The scans are rolling-shutter casts (ClosedLoop.scan_moving): the sensor moves 0.5 m, and up to 0.17 rad
in the corners, during each scan.

The chain comparisons hand the oracle the device's de-skewed clouds of each step (DeskewBackend.inject) after checking them against
the oracle's own de-skew from its own poses.  The device's RandomDownSample selects points by a hash of their bits, so a de-skewed
point one ulp away -- libm's atan2 / sincos, or poses that differ in their last bits (the ICP's reductions are not order-stable between
runs) -- selects another subset; downstream of the de-skew, exact parity needs the same bits.  For the same reason two device runs with
de-skew on are not compared with each other step by step: each is compared with the oracle.

Tolerances: velocities 1e-12 relative, de-skewed clouds bit-identical to b2s_undistort and 1e-12 from the oracle for the same
velocities, 1e-6 m from the oracle's own de-skew (its poses agree with the device's to ~1e-9), discrete outcomes identical,
transforms 1e-8, mapper-buffer lookups 1e-12 against the numpy buffer of the fetched poses."""
import copy

import numpy as np
import pytest

from oracle import oracle as O
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W

from motion_compensation import DeskewBackend, estimate_velocity
from odometry_buffer import TransformInterpolationBuffer
from test_gpu_odometry import canon, check_odometry_step, handle_params, odo_params, rel_rot, rel_trans, sky_scan

pytestmark = pytest.mark.gpu

TICK = 10_000_000


def mc_on(**kw):
    return E.ConstantVelocityMotionCompensationParameters(isUndistortInputCloud=True, **kw)


def _moving_inputs(lp, n):
    """rolling-shutter scans about one scan period apart; scan 20 keeps only returns beyond 13 m (a hole in the buffer of an odometry
    cropped at 12 m), scan 40 is the sky scan (the mapper rejects it)"""
    scans = []
    for k in range(n):
        raw = lp.scan_moving(k, seed=k)
        if k == 20:
            raw = raw[np.linalg.norm(raw.astype(np.float64), axis=1) > 13.0]
        if k == 40:
            raw = sky_scan(seed=40)
        scans.append(raw)
    rng = np.random.default_rng(9)
    times = (12345 + np.cumsum(rng.integers(900_000, 1_100_000, n))).tolist()
    return scans, times


def _close(a, b, rel=1e-12):
    a, b = np.asarray(a), np.asarray(b)
    return np.abs(a - b).max() <= rel * max(np.abs(b).max(), 1.0)


class Run:
    """one odometry object and one submap driven through b2s_slam_step_async from the first scan on"""

    def __init__(self, engine_factory, scans, times, mc=None, graph=False, buffer_size=2000, carve_dense=False):
        p = handle_params()
        self.eng = engine_factory(p)
        self.mapper = E.Mapper(self.eng, 700_000)
        if carve_dense:                                                          # wired as DeviceBackend.new_submap wires them
            self.mapper.submap.setMapperOptions(minMovement=p.minMovementBetweenMappingSteps, carving=p.mapBuilder.carving, dense=True,
                                                denseCarving=p.denseMapCarving, denseCropper=p.denseMapCropper)
        self.odo = E.DeviceLidarOdometry(self.eng, odo_params(rmax=12.0, buffer_size=buffer_size), 65536)
        if mc is not None:
            self.odo.setMotionCompensation(mc)
        self.mapper.addRangeMeasurement(self.eng.cloud(scans[0]), None)       # Mapper.cpp:105-114: both buffers are empty here
        self.mapper.submap.setPose(np.eye(4))
        self.odo.addRangeScan(self.eng.cloud(scans[0]), times[0])
        self.odo.pushMapToRangeSensor(times[0], np.eye(4))                     # Mapper.cpp:112
        self.staging = self.odo.enableGraph(65536) if graph else None
        self.scans, self.times = scans, times

    def step(self, k):
        c = self.eng.cloud(self.scans[k])
        if self.staging is not None:
            L.check(L.lib().b2s_cloud_copy(self.eng._h, c._c, self.staging._c))
            c = self.staging
        before = self.eng.launches
        slot = self.mapper.addRangeMeasurementWithOdometry(self.odo, c, self.times[k], slot=k % 256)
        self.eng.synchronize()
        r = L.SlamResult()
        L.check(L.lib().b2s_slam_result_fetch(self.eng._h, self.odo._o, C_int(slot), L.C.byref(r)))
        return r, self.eng.launches - before

    def free(self):
        self.odo.free()
        self.mapper.submap.free()


def C_int(v):
    return L.C.c_int32(v)


@pytest.mark.parametrize("graph", [False, True])
def test_disabled_motion_compensation_changes_nothing(engine_factory, graph):
    """parameters set with enabled = 0 against an object that never saw them: the same launches and the same results, step by step.
    Two runs of the unchanged chain already differ in the last bits of the ICP's transforms (its reductions are not order-stable
    between runs, ~1e-14), so the transforms are compared to 1e-12 and everything discrete exactly.  In graph mode the parameters
    are set after the capture: the graph is dropped and captured once more, with the same launches and results."""
    lp = W.ClosedLoop()
    scans, times = _moving_inputs(lp, 30)
    off = E.ConstantVelocityMotionCompensationParameters(isUndistortInputCloud=False, scanDuration=0.2, numPosesVelocityEstimation=2)
    runs = [Run(engine_factory, scans, times, graph=graph), Run(engine_factory, scans, times, mc=None if graph else off, graph=graph)]
    for k in range(1, len(scans)):
        if graph and k == 8:
            runs[1].odo.setMotionCompensation(off)
        (ra, la), (rb, lb) = (r.step(k) for r in runs)
        if not graph or k not in (8, 9):                     # 8: eager after the drop, 9: the new capture
            assert la == lb, k
        a, b = E._slam_res(ra), E._slam_res(rb)
        assert (a.odometry.outcome, a.odometry.nPreprocessed, a.odomUsed, a.mapperAccepted) == \
            (b.odometry.outcome, b.odometry.nPreprocessed, b.odomUsed, b.mapperAccepted), k
        for x, y in ((a.odometry.registration, b.odometry.registration), (a.mapper, b.mapper)):
            assert x.iters == y.iters and x.n_corr == y.n_corr, k
            assert np.abs(x.transformation_ - y.transformation_).max() < 1e-12, k
        assert np.abs(a.odometry.odomToRangeSensor - b.odometry.odomToRangeSensor).max() < 1e-12, k
    xa, _ = runs[0].mapper.submap.getMapPointCloud()
    xb, _ = runs[1].mapper.submap.getMapPointCloud()
    assert len(xa) == len(xb) and np.abs(canon(xa) - canon(xb)).max() < 1e-10
    if graph:
        assert [r.eng.graphCaptures for r in runs] == [1, 2]
    for r in runs:
        r.free()


@pytest.mark.parametrize("buffer_size", [2000, 8])
def test_velocities_and_deskewed_clouds(engine_factory, buffer_size):
    """every step: both velocity pairs against the numpy estimate over buffers rebuilt from the fetched odometry poses and the
    accepted mapper poses; at some steps the de-skewed clouds against b2s_undistort (bits) and oracle.undistort (1e-12)"""
    n = 60
    lp = W.ClosedLoop()
    scans, times = _moving_inputs(lp, n)
    run = Run(engine_factory, scans, times, mc=mc_on(), buffer_size=buffer_size)
    eng, odo = run.eng, run.odo
    ob, mb = TransformInterpolationBuffer(buffer_size), TransformInterpolationBuffer(buffer_size)
    ob.push(times[0], np.eye(4)); mb.push(times[0], np.eye(4))
    seen = dict(zero_odo=0, moved_odo=0, zero_map=0, hole=False, rejected=False)
    mc = E.ConstantVelocityMotionCompensation(eng)
    for k in range(1, n):
        vo, wo = estimate_velocity(ob, times[k], 3)
        vm, wm = estimate_velocity(mb, times[k], 3)
        r, _ = run.step(k)
        g = E._slam_res(r)
        m = odo.fetchMotionCompensation(k % 256)
        for got, ref in ((m.odometryLinearVelocity, vo), (m.odometryAngularVelocityRpy, wo), (m.mapLinearVelocity, vm),
                         (m.mapAngularVelocityRpy, wm)):
            assert _close(got, ref), (k, got, ref)
        assert m.odometryApplied == bool(vo.any() or wo.any()) and m.mapApplied == bool(vm.any() or wm.any()), k
        seen["zero_odo"] += not m.odometryApplied
        seen["moved_odo"] += m.odometryApplied
        seen["zero_map"] += not m.mapApplied
        if g.odometry.outcome in (L.ODOM_INIT, L.ODOM_OK):
            ob.push(times[k], g.odometry.odomToRangeSensor)
        else:
            seen["hole"] = True
        if g.mapperAccepted:
            mb.push(times[k], g.mapper.transformation_)
        else:
            seen["rejected"] = True
        if k in (5, 21, 33, 59):
            a, b = odo.undistortedScans()
            oa, _ = a.download(); mbx, _ = b.download()
            raw = scans[k].astype(np.float64)
            for got, v, w in ((oa, m.odometryLinearVelocity, m.odometryAngularVelocityRpy), (mbx, m.mapLinearVelocity, m.mapAngularVelocityRpy)):
                direct, _ = mc.undistortInputPointCloud(eng.cloud(scans[k]), v, w).download()
                assert got.shape == raw.shape and np.array_equal(got, direct), k
                ref = O.undistort(raw, v, w, 0.1, True)
                assert np.abs(got - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1.0), k
            assert np.abs(oa - raw).max() > 0.05                  # the scan really was moved
    assert seen["zero_odo"] >= 3 and seen["moved_odo"] > 40 and seen["zero_map"] >= 3 and seen["hole"] and seen["rejected"], seen
    if buffer_size == 8:
        assert len(ob.entries) == 8 and len(mb.entries) == 8 and ob.entries[0][0] > times[10]   # both rings evicted
    run.free()


def _device_deskewed(odo):
    a, b = odo.undistortedScans()
    return a.download()[0], b.download()[0]


def _compare_step(be, sm, run, k, g, tol=1e-6):
    """the oracle's step k on the device's de-skewed clouds of that step, against the device's result g"""
    inj = _device_deskewed(run.odo)
    be.inject = inj
    res, acc = be.step_with_odometry(sm, run.scans[k], run.times[k])
    assert inj[0].shape == be.odo.deskewed.shape and np.abs(inj[0] - be.odo.deskewed).max() < tol, k   # the oracle's own de-skew
    assert inj[1].shape == be.deskewed.shape and np.abs(inj[1] - be.deskewed).max() < tol, k
    outcome, reg, n_pre = be.odo_result
    check_odometry_step(g.odometry, outcome, reg, n_pre, be.odo.cum)
    assert g.odomUsed == be.odo.buf.has(run.times[k]) and g.mapperAccepted == acc, k
    assert g.mapper.iters == res.iters and g.mapper.n_corr == res.n_corr, k
    assert np.abs(g.mapper.transformation_ - res.T).max() < 1e-8, k
    return acc


def _compare_maps(run, be, sm):
    gx, _ = run.mapper.submap.getMapPointCloud()
    assert len(gx) == len(sm.xyz) and np.abs(canon(gx) - canon(sm.xyz)).max() < 1e-8
    dx, dk = run.mapper.submap.getDenseMap()
    ox, ok = be.dense_map(sm)
    assert len(dx) == len(ox) and len(dx) > 0
    q1, q2 = np.lexsort((dk[:, 2], dk[:, 1], dk[:, 0])), np.lexsort((ok[:, 2], ok[:, 1], ok[:, 0]))
    assert np.array_equal(dk[q1], ok[q2]) and np.abs(dx[q1] - ox[q2]).max() < 1e-8
    c, o = run.mapper.submap.mapperCounters(), be.counters(sm)
    assert {n: c[n] for n in o} == o and o["carve_runs"] >= 1 and o["inserted_dense"] > 10


@pytest.mark.parametrize("graph", [False, True])
def test_deskewed_chain_matches_oracle(engine_factory, graph):
    """the chain with both de-skews, carving and the dense map against the oracle composition: every step's odometry outcome,
    odom_used, mapper acceptance, iterations, correspondences and T; the final sparse map as a keyed set, the dense map, the carving
    counters; b2s_slam_map_lookup against the oracle's mapper buffer; graph-replayed, one capture"""
    n = 50
    lp = W.ClosedLoop()
    scans, times = _moving_inputs(lp, n)
    run = Run(engine_factory, scans, times, mc=mc_on(), graph=graph, carve_dense=True)
    be = DeskewBackend(copy.deepcopy(handle_params()), odo_params(rmax=12.0), mc_on(), carving=True, dense=True)
    sm = be.new_submap()
    be.first_scan_with_odometry(sm, scans[0], times[0])
    acc = []
    for k in range(1, n):
        g = E._slam_res(run.step(k)[0])
        acc.append(_compare_step(be, sm, run, k, g))
    assert not acc[39] and be.odo.velocity[0].any() and be.velocity[0].any()      # the sky scan was rejected; motion was compensated
    _compare_maps(run, be, sm)
    mt = [t for t, _ in be.map_buf.entries]
    for q in mt + [mt[0] - 1, mt[-1] + 5_000_000] + [(a + c) // 2 for a, c in zip(mt[:-1], mt[1:])]:
        T, has = run.odo._map_lookup(q)
        assert has == be.map_buf.has(q)
        assert np.abs(T - be.map_buf.get_transform(q)).max() < 1e-8, q
    assert run.eng.graphCaptures == (1 if graph else 0)
    run.free()


def test_graph_follows_a_scan_duration_change(engine_factory):
    """scan_duration changes before scan 9 of a graph-replayed run: exactly one more capture, and every step -- the replays before and
    after the change -- matches the oracle composition run with the same change (whose own de-skew uses the new duration)"""
    n = 16
    lp = W.ClosedLoop()
    scans, times = _moving_inputs(lp, n)
    run = Run(engine_factory, scans, times, mc=mc_on(), graph=True)
    be = DeskewBackend(copy.deepcopy(handle_params()), odo_params(rmax=12.0), mc_on(), carving=False, dense=False)
    sm = be.new_submap()
    be.first_scan_with_odometry(sm, scans[0], times[0])
    caps = {}
    for k in range(1, n):
        if k == 9:
            new = mc_on(scanDuration=0.12)
            run.odo.setMotionCompensation(new)
            be.mc = be.odo.mc = new
        g = E._slam_res(run.step(k)[0])
        _compare_step(be, sm, run, k, g)
        caps[k] = run.eng.graphCaptures
    assert caps[8] == 1 and caps[9] == 1 and caps[10] == 2 and caps[n - 1] == 2, caps   # dropped at 9, eager at 9, captured at 10
    run.free()


def test_segment_mapper_with_motion_compensation():
    """SegmentMapper.addRangeScan over 200 moving scans with hand-overs: DeviceBackend(motionCompensation=...) (one
    b2s_slam_step_host_async per scan, graph-replayed, carving on) against DeskewBackend with the tolerances of
    test_segment_mapper_from_raw_scans_and_timestamps"""
    N = 200
    p = E.MapperParameters(seed=3)
    op = odo_params()
    lp = W.ClosedLoop()
    sp = S.SubmapParameters(radius=10.0)
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=False, graph=True, odometry=op, motionCompensation=mc_on())
    ora = DeskewBackend(copy.deepcopy(p), op, mc_on(), carving=True, dense=False)
    md, mo = S.SegmentMapper(dev, sp), S.SegmentMapper(ora, sp)
    for k in range(N):
        raw = lp.scan_moving(k, seed=k)
        t = 12345 + k * TICK // 10
        rd = md.addRangeScan(raw, t)
        if k > 0:
            inj = _device_deskewed(dev.odometry())
            ora.inject = inj
        ro = mo.addRangeScan(raw, t)
        if k > 0:
            assert np.abs(inj[0] - ora.odo.deskewed).max() < 1e-5 and np.abs(inj[1] - ora.deskewed).max() < 1e-5, k
        if rd is None:
            assert ro is None
            continue
        assert rd.iters == ro.iters and rd.n_corr == ro.n_corr, k
        assert rel_rot(rd.transformation_, ro.T) < 1e-7 and rel_trans(rd.transformation_, ro.T) < 1e-7, k
        assert md.submaps.activeSubmapIdx == mo.submaps.activeSubmapIdx, k
    ed, eo = md.submaps.events, mo.submaps.events
    assert [e[:2] for e in ed] == [e[:2] for e in eo]
    for a, b in zip(ed, eo):
        if a[0] == "revisit_check":
            assert a[1] == b[1] and abs(a[2] - b[2]) < 1e-12
        else:
            assert a == b
    assert len([e for e in ed if e[0] == "active_submap_changed"]) >= 2
    for q in (12345, 12345 + 50 * TICK // 10 + 7, 12345 + (N - 1) * TICK // 10):   # the first-scan push, an interpolation, the last
        assert np.abs(dev.odometry().getMapToRangeSensor(q) - ora.map_buf.get_transform(q)).max() < 1e-6
    dev.close()


def test_map_lookup_matches_numpy_buffer_of_fetched_poses(engine_factory):
    """b2s_slam_map_lookup at the entries, between them and outside, to 1e-12 against the numpy buffer of the fetched accepted poses"""
    lp = W.ClosedLoop()
    scans, times = _moving_inputs(lp, 45)
    run = Run(engine_factory, scans, times, buffer_size=16)
    mb = TransformInterpolationBuffer(16)
    mb.push(times[0], np.eye(4))
    for k in range(1, len(scans)):
        g = E._slam_res(run.step(k)[0])
        if g.mapperAccepted:
            mb.push(times[k], g.mapper.transformation_)
    mt = [t for t, _ in mb.entries]
    assert len(mt) == 16
    queries = mt + [mt[0] - 1, mt[0] - TICK, mt[-1] + 1, mt[-1] + TICK] + [(a + c) // 2 for a, c in zip(mt[:-1], mt[1:])]
    for q in queries:
        T, has = run.odo._map_lookup(q)
        assert has == mb.has(q)
        assert np.abs(T - mb.get_transform(q)).max() < 1e-12, q
    # an empty buffer: has = 0, T = I; an equal time is accepted, an earlier one ignored
    other = E.DeviceLidarOdometry(run.eng, odo_params(), 1024)
    T, has = other._map_lookup(5)
    assert not has and np.array_equal(T, np.eye(4))
    A, B = np.eye(4), np.eye(4)
    A[0, 3], B[0, 3] = 1.0, 2.0
    other.pushMapToRangeSensor(100, A)
    other.pushMapToRangeSensor(100, B)
    other.pushMapToRangeSensor(50, B)
    assert np.array_equal(other.getMapToRangeSensor(100), A)       # std::find_if: the first of the equal times
    assert np.array_equal(other.getMapToRangeSensor(500), A)       # clamped to lookup(latest_time()) = the same entry
    assert np.array_equal(other.getMapToRangeSensor(10), A)
    other.free()
    run.free()


def test_errors_and_lifetime(engine_factory):
    eng = engine_factory(handle_params())
    odo = E.DeviceLidarOdometry(eng, odo_params(), 65536)
    for bad in (mc_on(scanDuration=0.0), mc_on(scanDuration=-0.1), mc_on(numPosesVelocityEstimation=0)):
        with pytest.raises(L.B2SError) as e:
            odo.setMotionCompensation(bad)
        assert e.value.code == L.E_INVALID
    with pytest.raises(L.B2SError) as e:                        # nothing changed: de-skew was never enabled, so there is nothing to read
        odo.undistortedScans()
    assert e.value.code == L.E_INVALID
    other = engine_factory(handle_params())
    p = mc_on().to_c()
    for call in (lambda: L.lib().b2s_odometry_set_motion_compensation(other._h, odo._o, L.C.byref(p)),
                 lambda: L.lib().b2s_slam_map_pose_push(other._h, odo._o, L.C.c_int64(1), E._pd(np.eye(4))),
                 lambda: L.lib().b2s_slam_map_lookup(other._h, odo._o, L.C.c_int64(1), E._pd(np.zeros(16)), None)):
        with pytest.raises(L.B2SError) as e:
            L.check(call())
        assert e.value.code == L.E_INVALID
    odo.free()
    # destroying an object with de-skew enabled and captured graphs leaves the handle usable
    lp = W.ClosedLoop()
    scans, times = _moving_inputs(lp, 8)
    run = Run(engine_factory, scans, times, mc=mc_on(), graph=True)
    for k in range(1, 6):
        run.step(k)
    assert run.eng.graphCaptures == 1
    run.odo.free()
    r = run.mapper.addRangeMeasurementAsync(run.eng.cloud(lp.scan(6, seed=6)), lp.delta(6), slot=0)
    assert run.mapper.fetchResult(r).fitness_ > 0.5
    run.eng.synchronize()
    run.mapper.submap.free()
