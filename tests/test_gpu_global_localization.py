"""-m gpu: global localisation in a prior map (b2s_submap_global_localization, DESIGN.md row M3) against its restatement in
tests/oracle_global_localization.{c,py}.  The prior map is one lap of the closed loop: every scan moved by map_frame_pose(k) and
voxelized at mapVoxelSize, loaded with SegmentMapper.setInitialMap.  The localised scans are lap-2 scans (another noise seed).

Tolerances: hits and candidates exact (integers); each candidate's ICP equal to b2s_register_to_submap from the same pose within 1e-8
(T, rmse) with the same iterations and correspondences;
found poses within 0.05 m and 0.5 degrees of the truth; tracking after it within 0.1 m like tests/test_gpu_localization.py."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import oracle as O
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import synth
from open3d_slam_b200 import workloads as W

import oracle_global_localization as G

pytestmark = pytest.mark.gpu

POSITIONS = 8


def _voxel_means(xyz, voxel):
    k = np.floor(xyz / voxel).astype(np.int64)
    _u, inv, cnt = np.unique(k, axis=0, return_inverse=True, return_counts=True)
    out = np.zeros((len(cnt), 3))
    np.add.at(out, inv.reshape(-1), xyz)
    return out / cnt[:, None]


@pytest.fixture(scope="module")
def lap_map():
    lp = W.ClosedLoop()
    p = E.MapperParameters(seed=3, isUseInitialMap=True, isMergeScansIntoMap=False)
    parts = []
    for k in range(lp.L):
        raw = lp.scan(k, seed=k).astype(np.float64)
        T = lp.map_frame_pose(k)
        parts.append(raw @ T[:3, :3].T + T[:3, 3])
    return lp, p, _voxel_means(np.concatenate(parts), p.mapBuilder.mapVoxelSize)


def _mapper(lap_map, graph=False):
    lp, p, xyz = lap_map
    dev = S.DeviceBackend(p, carving=False, dense=False, graph=graph, submap_capacity=600_000)
    m = S.SegmentMapper(dev, S.SubmapParameters(radius=1e4))
    m.setInitialMap(xyz)
    return dev, m, m.submaps.getActiveSubmap().handle


def _yaw(T):
    return math.atan2(T[1][0], T[0][0])


def _err(T, truth):
    return np.linalg.norm(np.asarray(T)[:3, 3] - truth[:3, 3]), abs(math.remainder(_yaw(T) - _yaw(truth), 2 * math.pi))


def test_scores_equal_the_oracle(lap_map):
    lp, p, _xyz = lap_map
    dev, m, sm = _mapper(lap_map)
    mx = dev.map_cloud(sm)[0]
    truth = lp.map_frame_pose(10)
    raw = lp.scan(10 + lp.L, seed=500)
    face = raw.copy()
    face[:64] = np.round(face[:64])                                          # query points on faces of both voxel grids
    for voxel in (1.0, 0.5):
        gp = E.GlobalLocalizationParameters(xMin=truth[0, 3] - 5, xMax=truth[0, 3] + 5, yMin=truth[1, 3] - 5, yMax=truth[1, 3] + 5, nYaw=36,
                                            yawStep=2 * math.pi / 36, scoreVoxel=voxel)
        for scan in (raw, face):
            c = dev.eng.cloud(scan)
            hits, q = E.debugGlobalLocalizationScores(dev.eng, sm, c, gp)
            cr = p.scanProcessing.cropper
            oc = O.cropper(cr.cropperName, cr.croppingMinRadius, cr.croppingMaxRadius, cr.croppingMinZ, cr.croppingMaxZ)
            want_q = O.voxel_down_sample(O.crop(oc, scan.astype(np.float64))[0], voxel)
            want_q = want_q[0] if isinstance(want_q, tuple) else want_q
            assert np.array_equal(np.sort(q, axis=0), np.sort(want_q, axis=0))
            want = G.scores(q, mx, G.Params.of(gp))
            assert len(hits) == 41 * 41 * 36 and np.array_equal(hits, want), voxel
            c.free()
    # tombstones: a carve of the map (force: outside the reference's schedule) leaves NaN slots behind
    carve = E.SpaceCarvingParameters()
    rawc = dev.eng.cloud(raw)
    removed = sm.carve(rawc, truth, carve, force=True)
    assert removed > 0
    gp = E.GlobalLocalizationParameters(xMin=truth[0, 3] - 5, xMax=truth[0, 3] + 5, yMin=truth[1, 3] - 5, yMax=truth[1, 3] + 5, nYaw=36,
                                        yawStep=2 * math.pi / 36)
    hits, q = E.debugGlobalLocalizationScores(dev.eng, sm, rawc, gp)
    assert np.array_equal(hits, G.scores(q, sm.getMapPointCloud()[0], G.Params.of(gp)))
    dev.close()


def test_candidates_and_refinement_equal_the_oracle_and_the_single_registration(lap_map):
    lp, p, _xyz = lap_map
    dev, m, sm = _mapper(lap_map)
    mx = dev.map_cloud(sm)[0]
    raw = lp.scan(30 + lp.L, seed=530)
    c = dev.eng.cloud(raw)
    gp = E.GlobalLocalizationParameters()
    r = sm.globalLocalization(c, gp, 0.7)
    hits, q = E.debugGlobalLocalizationScores(dev.eng, sm, c, gp)
    op = G.Params.of(gp)
    g = G.grid(op, mx)
    want = G.scores(q, mx, op, g)
    assert r.n_hypotheses == g.n == len(hits) and np.array_equal(hits, want)
    cands = G.candidates(want, op, g)
    assert [k.hypothesis for k in r.candidates] == cands
    assert [k.hits for k in r.candidates] == [int(want[h]) for h in cands]
    rot = G.rotations(op)
    reg = dev.mapper.scan2MapReg_
    match = reg.processForScanMatchingAndMerging(c).match_
    same = []
    for k in r.candidates:
        assert np.array_equal(k.T_hypothesis, G.pose(op, g, rot, k.hypothesis))
        single = reg.scanToMapRegistration(match, sm, k.T_hypothesis, k.T_hypothesis)
        again = reg.scanToMapRegistration(match, sm, k.T_hypothesis, k.T_hypothesis)
        same.append((np.array_equal(single.transformation_, k.icp.transformation_), np.array_equal(single.transformation_, again.transformation_)))
        assert np.abs(single.transformation_ - k.icp.transformation_).max() <= 1e-8 and abs(single.fitness_ - k.icp.fitness_) <= 1e-12
        assert abs(single.inlier_rmse_ - k.icp.inlier_rmse_) <= 1e-8 and single.iters == k.icp.iters and single.n_corr == k.icp.n_corr
    print("bitwise (batch == single, single == single):", same)
    w, found, ru = G.decide([k.icp.transformation_ for k in r.candidates], [k.icp.fitness_ for k in r.candidates], op, 0.7)
    assert (r.winner_rank, r.found, r.runner_up_fitness) == (w, found, ru)
    assert np.array_equal(r.T, r.candidates[w].icp.transformation_)
    dev.close()


def test_localises_lap_two_scans_without_a_pose(lap_map):
    lp, _p, _xyz = lap_map
    dev, m, sm = _mapper(lap_map)
    pose0 = sm.getPose()
    log = []
    for i in range(POSITIONS):
        k = (i * lp.L) // POSITIONS + 3
        c = dev.eng.cloud(lp.scan(k + lp.L, seed=700 + k))
        r = sm.globalLocalization(c, None, 0.7)
        dt, dyaw = _err(r.T, lp.map_frame_pose(k))
        log.append((k, r.found, round(r.fitness, 3), round(r.runner_up_fitness, 3), round(dt, 4), round(math.degrees(dyaw), 3)))
        c.free()
    print(log)
    for k, found, fit, _ru, dt, dyaw in log:
        assert found and fit >= 0.7 and dt < 0.05 and dyaw < 0.5, (k, log)
    assert np.array_equal(sm.getPose(), pose0)
    dev.close()


def test_segment_mapper_localises_then_tracks(lap_map):
    lp, _p, _xyz = lap_map
    dev, m, sm = _mapper(lap_map, graph=True)
    k0 = 20
    r = m.globalLocalization(lp.scan(k0 + lp.L, seed=900))
    assert r.found and m.submaps.events[-1][0] == "global_localization" and m.submaps.events[-1][2]
    assert np.array_equal(m.mapToRangeSensor, r.T)
    for i in range(10):
        k = k0 + 1 + i
        m.addRangeMeasurement(lp.scan(k + lp.L, seed=900 + k), lp.delta(k))
    for i, P in enumerate(m.poses[1:]):
        assert np.linalg.norm(P[:3, 3] - lp.map_frame_pose(k0 + 2 + i)[:3, 3]) < 0.1, i
    assert dev.eng.graphCaptures >= 1
    dev.close()


def test_not_found_leaves_the_submap_alone(lap_map):
    lp, p, _xyz = lap_map
    dev, m, sm = _mapper(lap_map)
    map0, pose0 = dev.map_cloud(sm), sm.getPose()
    # other cylinders, walls beyond the cropper, and the ground 6 m lower: on a flat site the ground plane alone registers anywhere with
    # a fitness near the mapper's minimum refinement fitness, so the scan of another place differs from the map in its ground as well
    scene = synth.Scene(cylinders=np.array([[3.0, -9.0], [-12.0, 4.0], [8.0, 8.0], [-5.0, -14.0], [10.0, -3.0], [-7.0, 9.0]]), half_x=60.0,
                        half_y=60.0, ground_z=-8.0)
    other = synth.lidar_scan(scene, np.eye(4), seed=5)
    c = dev.eng.cloud(other)
    r = sm.globalLocalization(c, None, 0.7)
    print("other scene:", r.found, r.fitness, r.runner_up_fitness)
    assert not r.found and r.fitness < 0.7
    k = 12
    truth = lp.map_frame_pose(k)
    c2 = dev.eng.cloud(lp.scan(k + lp.L, seed=1200))
    far = E.GlobalLocalizationParameters(xMin=truth[0, 3] + 8, xMax=truth[0, 3] + 12, yMin=truth[1, 3] + 8, yMax=truth[1, 3] + 12)
    r2 = sm.globalLocalization(c2, far, 0.7)
    print("box without the truth:", r2.found, r2.fitness, _err(r2.T, truth))
    assert not r2.found
    map1 = dev.map_cloud(sm)
    assert np.array_equal(map0[0], map1[0]) and np.array_equal(map0[1], map1[1], equal_nan=True)
    assert np.array_equal(sm.getPose(), pose0)
    dev.close()


def test_z_levels_and_errors(lap_map):
    lp, p, _xyz = lap_map
    dev, m, sm = _mapper(lap_map)
    k = 40
    truth = lp.map_frame_pose(k)
    raw = lp.scan(k + lp.L, seed=1400).astype(np.float64)
    c = dev.eng.cloud((raw - [0.0, 0.0, 0.5]).astype(np.float32))          # the sensor 0.5 m higher than when the map was made
    gp = E.GlobalLocalizationParameters(xMin=truth[0, 3] - 3, xMax=truth[0, 3] + 3, yMin=truth[1, 3] - 3, yMax=truth[1, 3] + 3, nZ=3,
                                        z0=-0.5, zStep=0.5)
    r = sm.globalLocalization(c, gp, 0.7)
    best = r.candidates[r.winner_rank]
    assert r.found and best.hypothesis // (r.n_hypotheses // 3) == 2       # iz = 2: z = +0.5
    assert np.linalg.norm(r.T[:3, 3] - (truth[:3, 3] + [0, 0, 0.5])) < 0.05

    def code(**kw):
        q = E.GlobalLocalizationParameters(**kw).to_c()
        out = L.GlobalLocalizationResult()
        return L.lib().b2s_submap_global_localization(dev.eng._h, sm._s, c._c, C.byref(q), C.c_double(0.7), None, C.c_int32(0), C.byref(out))
    assert code(step=0.0) == L.E_INVALID
    assert code(scoreVoxel=-1.0) == L.E_INVALID
    assert code(nYaw=0) == L.E_INVALID and code(nZ=0) == L.E_INVALID and code(nCandidates=0) == L.E_INVALID
    assert code(nCandidates=257) == L.E_INVALID
    assert code(xMin=float("nan")) == L.E_INVALID and code(yMax=float("inf")) == L.E_INVALID
    assert code(xMin=0.0, xMax=2e5, yMin=0.0, yMax=2e5, step=1.0) == L.E_INVALID            # > 2^31 - 1 hypotheses
    assert code(xMin=0.0, xMax=1e4, yMin=0.0, yMax=1e4, step=1.0, nYaw=4) == L.E_CAPACITY    # 4e8 scores: 1.6 GB
    assert code(scoreVoxel=0.002) == L.E_CAPACITY                                             # occupancy grid over the cap
    empty = dev.eng.cloud(np.zeros((0, 3), dtype=np.float32))
    assert L.lib().b2s_submap_global_localization(dev.eng._h, sm._s, empty._c, C.byref(E.GlobalLocalizationParameters().to_c()), C.c_double(0.7),
                                                  None, C.c_int32(0), C.byref(L.GlobalLocalizationResult())) == L.E_EMPTY
    sm2 = E.Submap(dev.eng, 1024)
    assert L.lib().b2s_submap_global_localization(dev.eng._h, sm2._s, c._c, C.byref(E.GlobalLocalizationParameters().to_c()), C.c_double(0.7),
                                                  None, C.c_int32(0), C.byref(L.GlobalLocalizationResult())) == L.E_EMPTY
    dev.close()
