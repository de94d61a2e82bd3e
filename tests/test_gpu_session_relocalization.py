"""-m gpu: global localisation over every submap of a session (b2s_submaps_global_localization, DESIGN.md row M4) and
SegmentMapper.relocalize.  The session is 100 scans of the closed lap mapped in 2 m submaps on the device, saved and loaded into a new
DeviceBackend (a new handle); the localised scans are lap-2 scans (another noise seed) at positions inside different submaps, none of them
the last saved pose.

Tolerances as tests/test_gpu_global_localization.py: hits and candidates exact (integers), against the restatement in
tests/oracle_global_localization.{c,py} on the concatenated live points; each candidate's ICP within 1e-8 (T, rmse) of
b2s_register_to_submap in its assigned submap, same iterations and correspondences; found poses within 0.05 m / 0.5 degrees of the
truth; tracking after relocalize within 0.1 m."""
import copy
import ctypes as C
import math

import numpy as np
import pytest

import oracle_global_localization as G
from oracle_backend_relocalization import closest
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W

pytestmark = pytest.mark.gpu

N_MAPPED = 100
POSITIONS = (10, 33, 57, 80)


def box(truth, half=4.0, n_yaw=72):
    return E.GlobalLocalizationParameters(xMin=truth[0, 3] - half, xMax=truth[0, 3] + half, yMin=truth[1, 3] - half, yMax=truth[1, 3] + half,
                                          nYaw=n_yaw, yawStep=2 * math.pi / n_yaw)


def _yaw(T):
    return math.atan2(T[1][0], T[0][0])


@pytest.fixture(scope="module")
def saved_session(tmp_path_factory):
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    a = S.SegmentMapper(S.DeviceBackend(copy.deepcopy(p), carving=True, dense=False, graph=True), S.SubmapParameters(radius=2.0))
    for k in range(N_MAPPED):
        a.addRangeScan(lp.scan(k, seed=k), k * 1_000_000)
    assert len(a.submaps.submaps) >= 8
    path = str(tmp_path_factory.mktemp("relocalization") / "session.npz")
    a.saveSession(path)
    a.backend.close()
    return lp, p, path


def load(saved_session):
    lp, p, path = saved_session
    be = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=False, graph=True)
    return lp, be, S.SegmentMapper.loadSession(path, be)


def test_union_equals_the_concatenation_and_each_candidate_its_single_registration(saved_session):
    lp, be, m = load(saved_session)
    eng = be.eng
    sms = [s.handle for s in m.submaps.submaps]
    centers = np.array([s.mapToSubmapCenter() for s in m.submaps.submaps])
    cat = np.concatenate([sm.getMapPointCloud()[0] for sm in sms])
    reg = be.mapper.scan2MapReg_
    winners = []
    for k in POSITIONS:
        truth = lp.map_frame_pose(k)
        c = eng.cloud(lp.scan(k + lp.L, seed=700 + k))
        gp = box(truth)
        op = G.Params.of(gp)
        hits, q = E.debugGlobalLocalizationScoresInSubmaps(eng, sms, c, gp)
        g = G.grid(op, cat)
        want = G.scores(q, cat, op, g)
        assert len(hits) == g.n and np.array_equal(hits, want), k
        r = E.globalLocalizationInSubmaps(eng, sms, centers, c, gp, 0.7)
        cands = G.candidates(want, op, g)
        assert [x.hypothesis for x in r.candidates] == cands and [x.hits for x in r.candidates] == [int(want[h]) for h in cands]
        assert r.candidate_submaps == [closest(x.T_hypothesis[:3, 3], centers) for x in r.candidates]
        match = reg.processForScanMatchingAndMerging(c).match_
        for x, s in zip(r.candidates, r.candidate_submaps):
            single = reg.scanToMapRegistration(match, sms[s], x.T_hypothesis, x.T_hypothesis)
            assert np.abs(single.transformation_ - x.icp.transformation_).max() <= 1e-8 and abs(single.inlier_rmse_ - x.icp.inlier_rmse_) <= 1e-8
            assert single.iters == x.icp.iters and single.n_corr == x.icp.n_corr and abs(single.fitness_ - x.icp.fitness_) <= 1e-12
        w, found, ru = G.decide([x.icp.transformation_ for x in r.candidates], [x.icp.fitness_ for x in r.candidates], op, 0.7)
        assert (r.winner_rank, r.found, r.runner_up_fitness) == (w, found, ru)
        assert r.winner_submap == r.candidate_submaps[w] and np.array_equal(r.T, r.candidates[w].icp.transformation_)
        dt = np.linalg.norm(r.T[:3, 3] - truth[:3, 3])
        dyaw = abs(math.remainder(_yaw(r.T) - _yaw(truth), 2 * math.pi))
        assert found and dt < 0.05 and math.degrees(dyaw) < 0.5, (k, dt, dyaw)
        d = np.sort(np.linalg.norm(centers - truth[:3, 3], axis=1))
        if d[1] - d[0] > 0.5:                                           # the truth is clearly nearest to one centre: that submap wins
            assert r.winner_submap == closest(truth[:3, 3], centers), (k, r.winner_submap)
        winners.append(r.winner_submap)
        c.free()
    print("winner submaps:", winners)
    assert len(set(winners)) == len(POSITIONS)                          # every position lies in another submap
    be.close()


@pytest.fixture(scope="module")
def lap_map():
    lp = W.ClosedLoop()
    p = E.MapperParameters(seed=3, isUseInitialMap=True, isMergeScansIntoMap=False)
    parts = []
    for k in range(lp.L):
        T = lp.map_frame_pose(k)
        parts.append(lp.scan(k, seed=k).astype(np.float64) @ T[:3, :3].T + T[:3, 3])
    xyz = np.concatenate(parts)
    kk = np.floor(xyz / p.mapBuilder.mapVoxelSize).astype(np.int64)
    _u, inv, cnt = np.unique(kk, axis=0, return_inverse=True, return_counts=True)
    means = np.zeros((len(cnt), 3))
    np.add.at(means, inv.reshape(-1), xyz)
    return lp, p, means / cnt[:, None]


def test_one_submap_is_the_one_submap_call(lap_map):
    """n_submaps = 1 on the map of tests/test_gpu_global_localization.py: hits, candidates, their order and the decision of
    b2s_submap_global_localization"""
    lp, p, xyz = lap_map
    dev = S.DeviceBackend(p, carving=False, dense=False, graph=False, submap_capacity=600_000)
    m = S.SegmentMapper(dev, S.SubmapParameters(radius=1e4))
    m.setInitialMap(xyz)
    sm = m.submaps.getActiveSubmap().handle
    for k, gp in ((30, E.GlobalLocalizationParameters()), (75, box(lp.map_frame_pose(75), 6.0, 36))):
        c = dev.eng.cloud(lp.scan(k + lp.L, seed=530 + k))
        a, qa = E.debugGlobalLocalizationScores(dev.eng, sm, c, gp)
        b, qb = E.debugGlobalLocalizationScoresInSubmaps(dev.eng, [sm], c, gp)
        assert np.array_equal(a, b) and np.array_equal(qa, qb)
        one = sm.globalLocalization(c, gp, 0.7)
        many = E.globalLocalizationInSubmaps(dev.eng, [sm], np.zeros((1, 3)), c, gp, 0.7)
        assert (one.n_hypotheses, one.n_query, one.winner_rank, one.found) == (many.n_hypotheses, many.n_query, many.winner_rank, many.found)
        assert [(x.hypothesis, x.hits) for x in one.candidates] == [(x.hypothesis, x.hits) for x in many.candidates]
        for x, y in zip(one.candidates, many.candidates):
            assert np.array_equal(x.T_hypothesis, y.T_hypothesis)
            assert np.abs(x.icp.transformation_ - y.icp.transformation_).max() <= 1e-8 and x.icp.iters == y.icp.iters
            assert x.icp.n_corr == y.icp.n_corr and abs(x.icp.inlier_rmse_ - y.icp.inlier_rmse_) <= 1e-8
        assert many.candidate_submaps == [0] * len(many.candidates) and many.winner_submap == 0
        assert np.abs(one.T - many.T).max() <= 1e-8 and abs(one.runner_up_fitness - many.runner_up_fitness) <= 1e-12
        c.free()
    dev.close()


def test_mixed_batch_reads_several_submaps(saved_session):
    """the whole union as the box: the 16 candidates of the one ICP launch are refined in at least 3 different submaps, each as its
    single registration"""
    lp, be, m = load(saved_session)
    sms = [s.handle for s in m.submaps.submaps]
    centers = np.array([s.mapToSubmapCenter() for s in m.submaps.submaps])
    k = 45
    c = be.eng.cloud(lp.scan(k + lp.L, seed=745))
    r = E.globalLocalizationInSubmaps(be.eng, sms, centers, c, E.GlobalLocalizationParameters(), 0.7)
    print("candidate submaps:", r.candidate_submaps)
    assert len(r.candidates) == 16 and len(set(r.candidate_submaps)) >= 3
    reg = be.mapper.scan2MapReg_
    match = reg.processForScanMatchingAndMerging(c).match_
    for x, s in zip(r.candidates, r.candidate_submaps):
        assert s == closest(x.T_hypothesis[:3, 3], centers)
        single = reg.scanToMapRegistration(match, sms[s], x.T_hypothesis, x.T_hypothesis)
        assert np.abs(single.transformation_ - x.icp.transformation_).max() <= 1e-8 and single.iters == x.icp.iters
        assert single.n_corr == x.icp.n_corr
    assert r.found and np.linalg.norm(r.T[:3, 3] - lp.map_frame_pose(k)[:3, 3]) < 0.05
    be.close()


def test_relocalize_then_map_with_loop_closures(saved_session):
    lp, be, m = load(saved_session)
    sc = m.submaps
    m.isAttemptLoopClosures = True
    assert len(sc.overlapScansBuffer) > 0
    n0 = len(sc.submaps)
    sizes = [s.handle.size() for s in sc.submaps]
    k0 = 50                                                              # mid-lap, far from the last saved pose (scan 99)
    r = m.relocalize(lp.scan(k0 + lp.L, seed=950), t=2_000_000_000)
    w = r.winner_submap
    assert r.found and np.linalg.norm(r.T[:3, 3] - lp.map_frame_pose(k0)[:3, 3]) < 0.05
    assert sc.events[-1][0] == "relocalization" and sc.events[-1][6] == w
    assert len(sc.overlapScansBuffer) == 0 and np.array_equal(m.mapToRangeSensor, r.T)
    active = sc.activeSubmapIdx
    assert active == w or (active == n0 and sc.submaps[active].parent == w)
    assert [s.handle.size() for s in sc.submaps[:n0]] == sizes          # no saved scan was replayed into any submap
    n_ev = len(sc.events)
    for i in range(20):
        k = k0 + 1 + i
        m.addRangeScan(lp.scan(k + lp.L, seed=950 + k), 2_000_000_000 + (i + 1) * 1_000_000)
        if i == 0:
            assert be.last_slam_result.odometry.outcome == L.ODOM_INIT            # the odometry starts over at T
            assert np.array_equal(m.poses[-1], r.T)                                # rule 3: T kept ...
            assert [s.handle.size() for s in sc.submaps[:n0]] == sizes             # ... nothing inserted
    print("relocalized into", w, "active", active, "of", n0, "tracking errors:",
          [round(float(np.linalg.norm(P[:3, 3] - lp.map_frame_pose(k0 + 2 + i)[:3, 3])), 4) for i, P in enumerate(m.poses[-19:])])
    print("events after relocalize:", [e[:2] if e[0] != "loop_closure_correction" else (e[0], e[1], e[2], np.round(e[3][:3, 3], 4))
                                       for e in sc.events[n_ev:] if e[0] != "transform"])
    for i, P in enumerate(m.poses[-19:]):                              # from the second scan on, tracked from T
        assert np.linalg.norm(P[:3, 3] - lp.map_frame_pose(k0 + 2 + i)[:3, 3]) < 0.1, i
    grown = {j for j in range(n0) if sc.submaps[j].handle.size() != sizes[j]}
    entered = {e[3] for e in sc.events[n_ev:] if e[0] == "active_submap_changed"}
    assert grown <= ({active} | entered), (grown, active, entered)
    for e in sc.events[n_ev:]:                                           # only older submaps are loop-closure candidates now
        if e[0] == "loop_closure_candidates":
            assert all(i < e[2] for i in e[3]), e
    be.close()


def test_refusals(saved_session):
    lp, be, m = load(saved_session)
    eng = be.eng
    sms = [s.handle for s in m.submaps.submaps]
    centers = np.array([s.mapToSubmapCenter() for s in m.submaps.submaps])
    c = eng.cloud(lp.scan(20 + lp.L, seed=720))
    gp = E.GlobalLocalizationParameters().to_c()

    def code(handles, ctr, cloud=c, params=gp):
        n = len(handles)
        arr = (C.c_void_p * max(n, 1))(*[h._s if h is not None else None for h in handles])
        cc = np.ascontiguousarray(np.asarray(ctr, dtype=np.float64).reshape(-1, 3)) if len(handles) else np.zeros((1, 3))
        out, win = L.GlobalLocalizationResult(), C.c_int32(7)
        rc = L.lib().b2s_submaps_global_localization(eng._h, arr, C.c_int32(n), cc.ctypes.data_as(C.POINTER(C.c_double)), cloud._c,
                                                     C.byref(params), C.c_double(0.7), None, C.c_int32(0), None, C.byref(out), C.byref(win))
        return rc
    assert code([], []) == L.E_INVALID
    assert code(sms[:2] + [None], centers[:3]) == L.E_INVALID
    bad = centers.copy(); bad[1, 2] = float("nan")
    assert code(sms, bad) == L.E_INVALID
    bad[1, 2] = float("inf")
    assert code(sms, bad) == L.E_INVALID
    other = E.Engine(E.MapperParameters(seed=3))
    foreign = E.Submap(other, 1000)
    assert code(sms[:2] + [foreign], centers[:3]) == L.E_INVALID
    assert code(sms, centers, params=E.GlobalLocalizationParameters(step=0.0).to_c()) == L.E_INVALID
    empties = [E.Submap(eng, 1000), E.Submap(eng, 1000)]
    assert code(empties, np.zeros((2, 3))) == L.E_EMPTY
    empty_scan = eng.cloud(np.zeros((0, 3), dtype=np.float32))
    assert code(sms, centers, cloud=empty_scan) == L.E_EMPTY

    # the byte cap of the union's occupancy grid: two one-point submaps whose bounding boxes span 2^17 x 2^16 x 1 voxels of 1 m
    # (2^33 bits = 2^30 bytes, the cap) -- one voxel more in y is over it, while each submap alone is one voxel
    def one_point(x, y):
        s = E.Submap(eng, 16)
        s.setMapPointCloud(eng.cloud(np.array([[x, y, 0.5]]), np.array([[0.0, 0.0, 1.0]])))
        return s
    a = one_point(0.5, 0.5)
    tiny = E.GlobalLocalizationParameters(xMin=0.0, xMax=0.0, yMin=0.0, yMax=0.0, nYaw=1, yawStep=0.0)
    at_cap = [a, one_point(131071.5, 65535.5)]
    over = [a, one_point(131071.5, 65536.5)]
    hits, _q = E.debugGlobalLocalizationScoresInSubmaps(eng, at_cap, c, tiny)
    assert len(hits) == 1
    with pytest.raises(L.B2SError) as e:
        E.debugGlobalLocalizationScoresInSubmaps(eng, over, c, tiny)
    assert e.value.code == L.E_CAPACITY
    assert code(over, np.zeros((2, 3)), params=tiny.to_c()) == L.E_CAPACITY
    for s in over[1:]:
        assert code([s], np.zeros((1, 3)), params=tiny.to_c()) == L.OK   # alone, each is one voxel
    be.close()
