"""-m gpu tests of the device-resident LidarOdometry (b2s_odometry_*) and the combined odometry + mapper step (b2s_slam_*):
the CUDA path against the CPU oracle composition of Odometry.cpp:25-79, the numpy TransformInterpolationBuffer
(tests/odometry_buffer.py) and the oracle mapper.  The odometry runs with parameters deliberately different from the handle's
configuration, so that reading the handle's instead of its own would show.

Tolerances: discrete outcomes (odometry outcomes, iteration / correspondence counts, odom_used, mapper acceptance) IDENTICAL,
transforms 1e-8 relative, cumulative poses and buffer entries 1e-7, buffer lookups 1e-12 against the numpy restatement.
"""
import copy

import numpy as np
import pytest

from oracle import oracle as O
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W

from odometry_buffer import TransformInterpolationBuffer
from oracle_backend import OracleBackend

pytestmark = pytest.mark.gpu

TICK = 10_000_000   # ticks per second


def rel_rot(Ta, Tb):
    return np.linalg.norm(Ta[:3, :3] - Tb[:3, :3]) / np.linalg.norm(Tb[:3, :3])


def rel_trans(Ta, Tb):
    return np.linalg.norm(Ta[:3, 3] - Tb[:3, 3]) / max(np.linalg.norm(Tb[:3, 3]), 1.0)


def canon(xyz, voxel=0.1):
    k = np.floor(xyz / voxel).astype(np.int64)
    return xyz[np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0], k[:, 2], k[:, 1], k[:, 0]))]


def odo_params(seed=7, rmax=30.0, buffer_size=2000):
    """voxel 0.2, ratio 0.5, max_corr 0.8, seed 7: none of them the handle's (0.1, 0.3, 1.0, seed 3)"""
    op = E.OdometryParameters(seed=seed, bufferSize=buffer_size)
    op.scanMatcher.icp = E.IcpParameters(maxNumIter=40, maxCorrespondenceDistance=0.8, knn=15, maxDistanceKnn=2.0)
    op.scanProcessing = E.ScanProcessingParameters(voxelSize=0.2, downSamplingRatio=0.5,
                                                   cropper=E.ScanCroppingParameters("MinMaxRadius", 2.0, rmax, -50.0, 50.0))
    return op


def sky_scan(n=4000, seed=0):
    """a non-empty scan with no correspondence anywhere: points 15-25 m above every surface of the synthetic scene"""
    rng = np.random.default_rng(seed)
    return np.c_[rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(15, 25, n)].astype(np.float32)


class OracleOdometry:
    """Odometry.cpp:25-79 over the oracle + the numpy buffer"""

    def __init__(self, op: E.OdometryParameters):
        self.op = op
        sp = op.scanProcessing
        self.crop = O.cropper(sp.cropper.cropperName, sp.cropper.croppingMinRadius, sp.cropper.croppingMaxRadius, sp.cropper.croppingMinZ,
                              sp.cropper.croppingMaxZ)
        self.prev = (np.zeros((0, 3)), np.zeros((0, 3)))
        self.cum = np.eye(4)
        self.buf = TransformInterpolationBuffer(op.bufferSize)
        self.pending = None

    def preprocess(self, raw):
        sp, ic = self.op.scanProcessing, self.op.scanMatcher.icp
        cx, _ = O.crop(self.crop, np.asarray(raw, dtype=np.float32).astype(np.float64))
        if len(cx) == 0:
            return np.zeros((0, 3)), np.zeros((0, 3))
        vx, _ = O.voxel_down_sample(cx, sp.voxelSize)
        vn = O.estimate_normals(vx, ic.knn, ic.maxDistanceKnn)
        return O.random_down_sample(vx, sp.downSamplingRatio, self.op.seed, vn)

    def setInitialTransform(self, T):
        self.cum = np.array(T, dtype=np.float64)
        self.pending = self.cum.copy()

    def step(self, raw, t):
        """-> (outcome, registration or None, n_pre)"""
        pre = self.preprocess(raw)
        if len(self.prev[0]) == 0:
            self.prev = pre
            self.buf.push(t, self.cum)
            return L.ODOM_INIT, None, len(pre[0])
        reg = None
        if len(pre[0]) > 0:
            ic = self.op.scanMatcher.icp
            reg = O.registration_icp_p2plane(self.prev[0], pre[0], pre[1], ic.maxCorrespondenceDistance, np.eye(4), max_iter=ic.maxNumIter)
        if reg is None or not reg.fitness > self.op.minFitness:
            if len(pre[0]) > 0:
                self.prev = pre
                return L.ODOM_FAILED, reg, len(pre[0])
            return L.ODOM_FAILED_KEPT_PREV, reg, 0
        if self.pending is not None:
            self.cum = self.pending; self.pending = None
        else:
            self.cum = self.cum @ np.linalg.inv(reg.T)
        self.prev = pre
        self.buf.push(t, self.cum)
        return L.ODOM_OK, reg, len(pre[0])


def check_odometry_step(g: E.OdometryStepResult, outcome, reg, n_pre, cum):
    assert g.outcome == outcome and g.nPreprocessed == n_pre
    if reg is not None and outcome != L.ODOM_INIT:
        r = g.registration
        assert r.iters == reg.iters and r.n_corr == reg.n_corr
        assert rel_rot(r.transformation_, reg.T) < 1e-8 and rel_trans(r.transformation_, reg.T) < 1e-8
    assert np.abs(g.odomToRangeSensor - cum).max() < 1e-7


def handle_params():
    return E.MapperParameters(seed=3)


# ----------------------------------------------------------------------------------------------------------------------
# the odometry on its own
# ----------------------------------------------------------------------------------------------------------------------
def test_device_odometry_matches_oracle_composition_and_host_odometry(engine_factory):
    """>= 30 scans of the closed loop: every step against the oracle composition and the host-composed engine.LidarOdometry (the
    latter on an engine configured with the odometry's parameters); then the handle's own registrations are unaffected."""
    op = odo_params()
    eng = engine_factory(handle_params())
    odo = E.DeviceLidarOdometry(eng, op, 65536)
    ref = OracleOdometry(op)
    hp = handle_params(); hp.icp = op.scanMatcher.icp; hp.scanProcessing = op.scanProcessing; hp.seed = op.seed
    host = E.LidarOdometry(engine_factory(hp), op)
    lp = W.ClosedLoop()
    for k in range(32):
        raw = lp.scan(k, seed=40 + k)
        t = (k + 1) * TICK // 10
        odo.addRangeScan(eng.cloud(raw), t, slot=k)
        outcome, reg, n_pre = ref.step(raw, t)
        g = odo.fetchResult(k)
        check_odometry_step(g, outcome, reg, n_pre, ref.cum)
        assert host.addRangeScan(host.eng.cloud(raw), t)
        if k > 0:
            h = host.lastResult
            assert g.registration.iters == h.iters and g.registration.n_corr == h.n_corr
            assert rel_rot(g.registration.transformation_, h.transformation_) < 1e-8
        assert outcome == (L.ODOM_INIT if k == 0 else L.ODOM_OK)
    assert np.abs(host.getOdomToRangeSensor() - ref.cum).max() < 1e-7
    for (t, T) in ref.buf.entries:                       # every buffer entry
        assert np.abs(odo.getOdomToRangeSensor(t) - T).max() < 1e-7
    px, _ = odo.getPreProcessedCloud().download()
    assert len(px) == len(ref.prev[0]) and np.abs(canon(px) - canon(ref.prev[0])).max() < 1e-9
    # the handle's registration path is untouched by the odometry object's parameters and buffers
    other = engine_factory(handle_params())
    raw0, raw1 = lp.scan(0, seed=1), lp.scan(1, seed=2)
    results = []
    for e in (eng, other):
        icp = E.ScanToMapIcp(e)
        a = icp.processForScanMatchingAndMerging(e.cloud(raw0)).merge_
        b = icp.processForScanMatchingAndMerging(e.cloud(raw1)).merge_
        results.append(E.RegistrationIcpPointToPlane(e).registerClouds(a, b, np.eye(4)))
    assert results[0].iters == results[1].iters and results[0].n_corr == results[1].n_corr
    assert np.abs(results[0].transformation_ - results[1].transformation_).max() < 1e-12
    # ... and so is its mapper chain (b2s_mapper_step_async)
    chains = []
    for e in (eng, other):
        m = E.Mapper(e, 700_000)
        m.addRangeMeasurement(e.cloud(lp.scan(0, seed=0)), None)
        m.submap.setPose(np.eye(4))
        rs = []
        for k in range(1, 5):
            slot = m.addRangeMeasurementAsync(e.cloud(lp.scan(k, seed=k)), lp.delta(k), slot=k)
            rs.append(m.fetchResult(slot))
        chains.append(rs)
        m.submap.free()
    for a, b in zip(*chains):
        assert a.iters == b.iters and a.n_corr == b.n_corr and a.iters > 0
        assert np.abs(a.transformation_ - b.transformation_).max() < 1e-12
    odo.free()


def test_odometry_branches(engine_factory):
    """FAILED replaces cloudPrev_, FAILED_KEPT_PREV keeps it, an empty first scan leaves the next one to initialise,
    setInitialTransform replaces the pose at the next success only, the order and ownership checks"""
    op = odo_params()
    eng = engine_factory(handle_params())
    odo = E.DeviceLidarOdometry(eng, op, 65536)
    ref = OracleOdometry(op)
    lp = W.ClosedLoop()
    far = np.array([[100.0, 0.0, 0.0], [0.0, 200.0, 0.0]], dtype=np.float32)    # crops to nothing
    T0 = np.eye(4); T0[:3, 3] = (5.0, -2.0, 0.5)
    seq = [("far", far), ("scan", 0), ("scan", 1), ("sky", sky_scan()), ("scan", 2), ("scan", 3), ("far", far), ("scan", 4),
           ("init", T0), ("scan", 5), ("scan", 6)]
    expect = [L.ODOM_INIT, L.ODOM_INIT, L.ODOM_OK, L.ODOM_FAILED, L.ODOM_FAILED, L.ODOM_OK, L.ODOM_FAILED_KEPT_PREV, L.ODOM_OK, None, L.ODOM_OK,
              L.ODOM_OK]
    t = 0
    slot = 0
    for (kind, what), ex in zip(seq, expect):
        if kind == "init":
            odo.setInitialTransform(what); ref.setInitialTransform(what)
            continue
        raw = what if kind in ("far", "sky") else lp.scan(what, seed=what)
        t += TICK // 10
        odo.addRangeScan(eng.cloud(raw), t, slot=slot)
        outcome, reg, n_pre = ref.step(raw, t)
        assert outcome == ex
        check_odometry_step(odo.fetchResult(slot), outcome, reg, n_pre, ref.cum)
        slot += 1
    assert np.abs(ref.buf.entries[-2][1] - T0).max() == 0.0       # the step after setInitialTransform pushed T0 itself
    # the buffer's entries and lookups
    for tt, T in ref.buf.entries:
        assert np.abs(odo.getOdomToRangeSensor(tt) - T).max() < 1e-7
    assert not odo.getBuffer().has(0) and odo.getBuffer().has(ref.buf.entries[0][0])
    # order and ownership
    with pytest.raises(L.B2SError) as e:
        odo.addRangeScan(eng.cloud(lp.scan(7, seed=7)), t)
    assert e.value.code == L.E_INVALID
    other = engine_factory(handle_params())
    with pytest.raises(L.B2SError) as e:
        L.check(L.lib().b2s_odometry_step_async(other._h, odo._o, other.cloud(lp.scan(7, seed=7))._c, L.C.c_int64(t + 1), L.C.c_int32(0)))
    assert e.value.code == L.E_INVALID
    odo.free()


@pytest.mark.parametrize("buffer_size", [2000, 8])
def test_odometry_lookup_matches_numpy_buffer(engine_factory, buffer_size):
    """b2s_odometry_lookup on jittered, non-uniform timestamps with holes (failed steps push nothing), at entries, between them,
    before the earliest and after the latest; with buffer_size 8 after eviction"""
    op = odo_params(buffer_size=buffer_size)
    eng = engine_factory(handle_params())
    odo = E.DeviceLidarOdometry(eng, op, 65536)
    buf = TransformInterpolationBuffer(buffer_size)
    lp = W.ClosedLoop()
    rng = np.random.default_rng(5)
    t = 12345
    for k in range(20):
        t += int(rng.integers(200_000, 1_500_000))
        raw = sky_scan(seed=k) if k in (6, 7, 13) else lp.scan(k, seed=k)
        odo.addRangeScan(eng.cloud(raw), t, slot=k)
        g = odo.fetchResult(k)
        if g.outcome in (L.ODOM_INIT, L.ODOM_OK):
            buf.push(t, g.odomToRangeSensor)
    assert len(buf.entries) == 8 if buffer_size == 8 else len(buf.entries) >= 12
    times = [tt for tt, _ in buf.entries]
    queries = times + [times[0] - 1, times[0] - 10_000_000, times[-1] + 1, times[-1] + 10_000_000]
    queries += [int(v) for v in rng.integers(times[0], times[-1], 40)]
    queries += [(a + b) // 2 for a, b in zip(times[:-1], times[1:])]
    for q in queries:
        T, has = odo._lookup(q)
        assert has == buf.has(q)
        assert np.abs(T - buf.get_transform(q)).max() < 1e-12, q
    odo.free()


# ----------------------------------------------------------------------------------------------------------------------
# odometry + mapper in one step
# ----------------------------------------------------------------------------------------------------------------------
def _combined_inputs(lp, n):
    """scan 20 keeps only returns beyond 13 m (the odometry's 12 m cropper leaves nothing: a hole in its buffer, while the mapper
    still registers it without a prediction), scan 40 is the sky scan (odometry and mapper both fail)"""
    scans = []
    for k in range(n):
        raw = lp.scan(k, seed=k)
        if k == 20:
            raw = raw[np.linalg.norm(raw.astype(np.float64), axis=1) > 13.0]
        if k == 40:
            raw = sky_scan(seed=40)
        scans.append(raw)
    rng = np.random.default_rng(9)
    times = np.cumsum(rng.integers(800_000, 1_200_000, n)).tolist()
    return scans, times


def _oracle_combined(p, op, scans, times):
    """the odometry composition, then OracleBackend.step with motion = getTransform(t_last)^-1 getTransform(t) from the numpy buffer"""
    be = OracleBackend(copy.deepcopy(p), carving=False, dense=False)
    sm = be.new_submap()
    ref = OracleOdometry(op)
    be.first_scan(sm, scans[0])
    ref.step(scans[0], times[0])
    t_last = 0
    out = []
    for k in range(1, len(scans)):
        outcome, reg, n_pre = ref.step(scans[k], times[k])
        used = ref.buf.has(times[k])
        motion = np.linalg.inv(ref.buf.get_transform(t_last)) @ ref.buf.get_transform(times[k]) if used else np.eye(4)
        interpolated = used and t_last not in [tt for tt, _ in ref.buf.entries] and ref.buf.entries[0][0] < t_last
        res, acc = be.step(sm, scans[k], motion)
        if acc:
            t_last = times[k]
        out.append(dict(outcome=outcome, reg=reg, n_pre=n_pre, cum=ref.cum.copy(), used=used, res=res, acc=acc, interpolated=interpolated))
    return be, sm, out


@pytest.mark.parametrize("graph", [False, True])
def test_combined_chain_matches_oracle(engine_factory, graph):
    """>= 60 scans through b2s_slam_step_async: a step without odometry prediction, a mapper rejection (t_last lags behind) and a
    prediction interpolated across an odometry hole all occur; everything matches the oracle, and b2s_mapper_processed_scan
    returns the mapper's clouds of the step."""
    n = 62
    p = handle_params()
    op = odo_params(rmax=12.0)
    eng = engine_factory(p)
    lp = W.ClosedLoop()
    scans, times = _combined_inputs(lp, n)
    mapper = E.Mapper(eng, 700_000)
    odo = E.DeviceLidarOdometry(eng, op, 65536)
    mapper.addRangeMeasurement(eng.cloud(scans[0]), None)
    mapper.submap.setPose(np.eye(4))
    odo.addRangeScan(eng.cloud(scans[0]), times[0])
    staging = odo.enableGraph(65536) if graph else None
    got = []
    for k in range(1, n):
        c = eng.cloud(scans[k])
        if graph:
            L.check(L.lib().b2s_cloud_copy(eng._h, c._c, staging._c))
            slot = mapper.addRangeMeasurementWithOdometry(odo, staging, times[k], slot=k % 256)
        else:
            slot = mapper.addRangeMeasurementWithOdometry(odo, c, times[k], slot=k % 256)
        got.append(odo.fetchSlamResult(slot))
        if k == n - 1:
            last = mapper.lastProcessedScan(merge=True, match=True)
    be, sm, ref = _oracle_combined(p, op, scans, times)
    for k, (g, r) in enumerate(zip(got, ref), start=1):
        check_odometry_step(g.odometry, r["outcome"], r["reg"], r["n_pre"], r["cum"])
        assert g.odomUsed == r["used"] and g.mapperAccepted == r["acc"], k
        assert g.mapper.iters == r["res"].iters and g.mapper.n_corr == r["res"].n_corr, k
        assert np.abs(g.mapper.transformation_ - r["res"].T).max() < 1e-8, k
    assert any(not r["used"] for r in ref)                           # no prediction
    assert any(not r["acc"] for r in ref)                            # a rejection: t_last lags
    assert any(r["interpolated"] for r in ref)                       # getTransform(t_last) across a hole
    assert ref[19]["outcome"] == L.ODOM_FAILED_KEPT_PREV and not ref[19]["used"] and ref[19]["acc"] and ref[20]["interpolated"]
    gx, _ = mapper.submap.getMapPointCloud()
    assert len(gx) == len(sm.xyz) and np.abs(canon(gx) - canon(sm.xyz)).max() < 1e-8
    (mx, _), (ax, _) = be._process(scans[-1])
    lx, _ = last.merge_.download(); lm, _ = last.match_.download()
    assert len(lx) == len(mx) and len(lm) == len(ax) and np.abs(canon(lx) - canon(mx)).max() < 1e-9
    if graph:
        launches = eng.launches
        c = eng.cloud(lp.scan(n, seed=n))
        L.check(L.lib().b2s_cloud_copy(eng._h, c._c, staging._c))
        mapper.addRangeMeasurementWithOdometry(odo, staging, times[-1] + TICK // 10)
        eng.synchronize()
        assert eng.launches - launches > 40        # a replay counts the captured kernels
        assert eng.graphCaptures == 1              # captured once (third step), every later step replayed
    odo.free()
    mapper.submap.free()


class OracleOdometryBackend(OracleBackend):
    """OracleBackend + the odometry composition: the oracle side of SegmentMapper.addRangeScan"""

    def __init__(self, params, op, **kw):
        super().__init__(params, **kw)
        self.odo = OracleOdometry(op)
        self.t_last = 0

    def first_scan_with_odometry(self, sm, raw, t):
        merge = self.first_scan(sm, raw)
        self.odo.step(raw, t)
        return merge

    def step_with_odometry(self, sm, raw, t):
        self.odo.step(raw, t)
        b = self.odo.buf
        motion = np.linalg.inv(b.get_transform(self.t_last)) @ b.get_transform(t) if b.has(t) else np.eye(4)
        res, acc = self.step(sm, raw, motion)
        if acc:
            self.t_last = t
        return res, acc


def test_segment_mapper_from_raw_scans_and_timestamps():
    """SegmentMapper.addRangeScan over a radius-10 m segment with hand-overs (each new submap captures its own combined graph) --
    against the same control flow over the oracle"""
    N = 208
    p = E.MapperParameters(seed=3)
    op = odo_params()
    lp = W.ClosedLoop()
    sp = S.SubmapParameters(radius=10.0)
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=False, graph=True, odometry=op)
    ora = OracleOdometryBackend(copy.deepcopy(p), op, carving=True, dense=False)
    md, mo = S.SegmentMapper(dev, sp), S.SegmentMapper(ora, sp)
    for k in range(N):
        raw = lp.scan(k, seed=k)
        t = (k + 1) * TICK // 10
        rd = md.addRangeScan(raw, t)
        ro = mo.addRangeScan(raw, t)
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
    assert np.linalg.norm(md.mapToRangeSensor[:3, 3] - lp.map_frame_pose(N - 1)[:3, 3]) < 0.3
    dev.close()


def test_graphs_are_kept_per_submap_across_hand_overs(engine_factory):
    """one odometry, two submaps, the active one switching back and forth: one graph is captured per submap and replayed after every
    return without a new capture (b2s_graph_capture_count), and the replayed steps give exactly what the same sequence gives eagerly"""
    p = handle_params()
    lp = W.ClosedLoop()
    scans = [lp.scan(k, seed=k) for k in range(14)]
    runs = []
    for graph in (False, True):
        eng = engine_factory(p)
        odo = E.DeviceLidarOdometry(eng, odo_params(), 65536)
        mapper = E.Mapper(eng, 700_000)
        subs = [mapper.submap, E.Submap(eng, 700_000)]
        c0 = eng.cloud(scans[0])
        merge = E.ScanToMapIcp(eng).processForScanMatchingAndMerging(c0).merge_
        for sm in subs:                                         # Mapper.cpp:105-114 on each
            sm.insertScan(c0, merge, np.eye(4))
            sm.setPose(np.eye(4))
        odo.addRangeScan(eng.cloud(scans[0]), 1)
        staging = odo.enableGraph(65536) if graph else None
        out = []
        captures = {}
        for k in range(1, len(scans)):
            mapper.submap = subs[(k // 2) % 2]                  # A A B B A A ...: every submap is left and returned to
            c = eng.cloud(scans[k])
            if graph:
                L.check(L.lib().b2s_cloud_copy(eng._h, c._c, staging._c))
                c = staging
            mapper.addRangeMeasurementWithOdometry(odo, c, 1 + k * TICK // 10, slot=k)
            out.append(odo.fetchSlamResult(k))
            captures[k] = eng.graphCaptures
        runs.append(out)
        if graph:
            # A: eager at k = 1, 4, captured at 5; B: eager at 2, 3, captured at 6.  Every later step -- the returns to A at k = 8
            # and 12 and to B at k = 10 among them -- replays its submap's graph: no further capture
            assert captures[4] == 0 and captures[5] == 1 and captures[6] == 2 and captures[len(scans) - 1] == 2, captures
        else:
            assert captures[len(scans) - 1] == 0
        odo.free()
        for sm in subs:
            sm.free()
    for a, b in zip(*runs):
        assert a.odometry.outcome == b.odometry.outcome and a.odomUsed == b.odomUsed and a.mapperAccepted == b.mapperAccepted
        assert a.mapper.iters == b.mapper.iters and a.mapper.n_corr == b.mapper.n_corr
        assert np.abs(a.mapper.transformation_ - b.mapper.transformation_).max() < 1e-12


def test_captured_graph_follows_parameter_changes(engine_factory):
    """after the capture, b2s_odometry_set_params, b2s_set_config and b2s_submap_set_mapper_options each drop the combined graph:
    the graph-mode run re-captures after every change and gives, step for step, what an eager run with the same changes gives"""
    lp = W.ClosedLoop()
    n = 16
    scans = [lp.scan(k, seed=k) for k in range(n)]
    changes = {6: "odometry", 9: "config", 12: "options"}   # applied before the step of that scan
    runs, caps = [], []
    for graph in (False, True):
        p = handle_params()
        eng = engine_factory(p)
        odo = E.DeviceLidarOdometry(eng, odo_params(), 65536)
        mapper = E.Mapper(eng, 700_000)
        mapper.addRangeMeasurement(eng.cloud(scans[0]), None)
        mapper.submap.setPose(np.eye(4))
        odo.addRangeScan(eng.cloud(scans[0]), 1)
        staging = odo.enableGraph(65536) if graph else None
        out = []
        for k in range(1, n):
            what = changes.get(k)
            if what == "odometry":
                odo.setParameters(odo_params(seed=11))           # another RandomDownSample selection: other pre-processed clouds
            elif what == "config":
                p2 = handle_params(); p2.seed = 4                # another selection on the mapper side
                mapper.params_ = p2
                eng.set_parameters(p2)
            elif what == "options":
                mapper.submap.setMapperOptions(minMovement=100.0)   # nothing is fused any more
            c = eng.cloud(scans[k])
            if graph:
                L.check(L.lib().b2s_cloud_copy(eng._h, c._c, staging._c))
                c = staging
            mapper.addRangeMeasurementWithOdometry(odo, c, 1 + k * TICK // 10, slot=k)
            out.append(odo.fetchSlamResult(k))
        runs.append((out, mapper.submap.mapperCounters()))
        caps.append(eng.graphCaptures)
        odo.free()
        mapper.submap.free()
    (ea, ca), (ga, cg) = runs
    for k, (a, b) in enumerate(zip(ea, ga), start=1):
        assert a.odometry.outcome == b.odometry.outcome and a.odometry.nPreprocessed == b.odometry.nPreprocessed, k
        assert a.odometry.registration.n_corr == b.odometry.registration.n_corr, k
        assert np.abs(a.odometry.registration.transformation_ - b.odometry.registration.transformation_).max() < 1e-12, k
        assert a.mapper.iters == b.mapper.iters and a.mapper.n_corr == b.mapper.n_corr, k
        assert np.abs(a.mapper.transformation_ - b.mapper.transformation_).max() < 1e-12, k
    assert ca == cg and cg["inserted_map"] <= cg["accepted"] - 3        # the last option took effect in both: scans 12-15 not fused
    # captured at 3, dropped and re-captured after each change (one eager step in between): 4 captures in all
    assert caps == [0, 4], caps


def test_scan_above_the_staging_capacity_is_refused(engine_factory):
    """b2s_slam_step_host_async in graph mode: a scan that fits the odometry (200 000 points) but not its staging cloud (65 536)
    is refused with B2S_E_CAPACITY before anything is uploaded"""
    eng = engine_factory(handle_params())
    odo = E.DeviceLidarOdometry(eng, odo_params(), 200_000)
    odo.enableGraph(65536)
    mapper = E.Mapper(eng, 100_000)
    big = np.zeros((100_000, 3), dtype=np.float32)
    out = L.SlamResult()
    with pytest.raises(L.B2SError) as e:
        mapper.addRangeMeasurementWithOdometryHostAsync(odo, big.ctypes.data, len(big), 1, L.C.addressof(out))
    assert e.value.code == L.E_CAPACITY
    eng.synchronize()
    odo.free()
    mapper.submap.free()


# ----------------------------------------------------------------------------------------------------------------------
# lifetime
# ----------------------------------------------------------------------------------------------------------------------
def test_destroying_odometry_or_submap_with_captured_graphs_leaves_handle_usable(engine_factory):
    p = handle_params()
    eng = engine_factory(p)
    lp = W.ClosedLoop()
    scans = [lp.scan(k, seed=k) for k in range(8)]
    for victim in ("odometry", "submap"):
        mapper = E.Mapper(eng, 700_000)
        odo = E.DeviceLidarOdometry(eng, odo_params(), 65536)
        mapper.addRangeMeasurement(eng.cloud(scans[0]), None)
        mapper.submap.setPose(np.eye(4))
        odo.addRangeScan(eng.cloud(scans[0]), 1)
        staging = odo.enableGraph(65536)
        for k in range(1, 6):                                    # two eager steps, a capture, replays
            c = eng.cloud(scans[k])
            L.check(L.lib().b2s_cloud_copy(eng._h, c._c, staging._c))
            mapper.addRangeMeasurementWithOdometry(odo, staging, 1 + k * TICK // 10)
        eng.synchronize()
        if victim == "odometry":
            odo.free()
            r = mapper.addRangeMeasurementAsync(eng.cloud(scans[6]), lp.delta(6), slot=0)
            assert mapper.fetchResult(r).fitness_ > 0.5
        else:
            mapper.submap.free()
            mapper.submap = E.Submap(eng, 700_000)               # may reuse the address: the cached graph must not be replayed
            mapper.submap.insertScan(eng.cloud(scans[5]), E.ScanToMapIcp(eng).processForScanMatchingAndMerging(eng.cloud(scans[5])).merge_,
                                     np.eye(4))
            mapper.submap.setPose(np.eye(4))
            c = eng.cloud(scans[6])
            L.check(L.lib().b2s_cloud_copy(eng._h, c._c, staging._c))
            slot = mapper.addRangeMeasurementWithOdometry(odo, staging, 1 + 6 * TICK // 10, slot=3)
            assert odo.fetchSlamResult(slot).mapper.fitness_ > 0.5
            odo.free()
        eng.synchronize()
        mapper.submap.free()
