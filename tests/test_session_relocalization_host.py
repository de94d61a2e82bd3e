"""CPU: global localisation over a set of submaps (b2s_submaps_global_localization, DESIGN.md row M4) and SegmentMapper.relocalize on the
oracle backend (tests/oracle_backend_relocalization.py).  The session is the first 30 scans of the closed lap mapped in 4 m submaps, which
overlap; an empty submap is added where the union is checked.  Boxes are cut to +-3 m around the truth and 36 yaws to keep the oracle fast."""
import copy
import math

import numpy as np
import pytest

import oracle_global_localization as G
from oracle_backend_relocalization import RelocalizationOracleBackend, closest, union_points
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import synth
from open3d_slam_b200 import workloads as W

K = 30


def box(truth, half=3.0):
    return E.GlobalLocalizationParameters(xMin=truth[0, 3] - half, xMax=truth[0, 3] + half, yMin=truth[1, 3] - half, yMax=truth[1, 3] + half,
                                          nYaw=36, yawStep=2 * math.pi / 36)


def session(p=None, radius=4.0):
    p = p or E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    m = S.SegmentMapper(RelocalizationOracleBackend(copy.deepcopy(p), carving=False, dense=False), S.SubmapParameters(radius=radius))
    for k in range(K):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    assert len(m.submaps.submaps) >= 3
    return lp, m


@pytest.fixture(scope="module")
def lap():
    return session()


def saved(m, path):
    m.saveSession(path)
    with np.load(path, allow_pickle=False) as z:
        return {k: z[k].copy() for k in z.files}


def test_union_scores_equal_the_restatement_on_the_concatenation(lap):
    """rules 1-4 over the union: the hits equal the one-map restatement on the concatenated live points and on one point per voxel of
    the union of the submaps' own voxel sets; an empty submap changes nothing; the default box is the union's live xy extent"""
    lp, m = lap
    be = m.backend
    sms = [s.handle for s in m.submaps.submaps] + [be.new_submap()]
    sms[1].xyz = sms[1].xyz.copy(); sms[1].xyz[::17] = np.nan            # tombstones
    for k in (6, 22):
        truth = lp.map_frame_pose(k)
        raw = lp.scan(k + lp.L, seed=400 + k)
        gp = box(truth)
        p = G.Params.of(gp)
        hits, q, g = be.union_scores(sms, raw, gp)
        cat = union_points(sms)
        assert np.array_equal(hits, G.scores(q, cat, p, g))
        inv = 1.0 / p.score_voxel
        keys = set()
        for sm in sms:                                                   # each submap's own occupied voxels, then their union
            lv = G.live(sm.xyz)
            f = np.floor(lv * inv)
            keys |= set(map(tuple, f[(np.abs(f) < G.KEY_LIMIT).all(axis=1)].astype(np.int64)))
        reps = (np.array(sorted(keys), dtype=np.float64) + 0.5) * p.score_voxel
        assert np.array_equal(hits, G.scores(q, reps, p, g))
        assert np.array_equal(hits, be.union_scores(sms[:-1], raw, gp)[0])
        assert hits.max() > 0.5 * len(q)
    lv = union_points(sms)
    g = G.grid(G.Params(), lv)
    assert (g.x_min, g.y_min) == (lv[:, 0].min(), lv[:, 1].min())
    assert g.nx == math.floor((lv[:, 0].max() - lv[:, 0].min()) / 0.25) + 1
    with pytest.raises(ValueError):
        be.union_scores([be.new_submap()], lp.scan(3, seed=3))


def test_candidates_are_refined_in_the_closest_submap(lap):
    lp, m = lap
    be = m.backend
    sms = [s.handle for s in m.submaps.submaps]
    centers = [s.mapToSubmapCenter() for s in m.submaps.submaps]
    k = 8
    r = be.global_localization_submaps(sms, centers, lp.scan(k + lp.L, seed=908), box(lp.map_frame_pose(k)))
    assert r.found and np.linalg.norm(r.T[:3, 3] - lp.map_frame_pose(k)[:3, 3]) < 0.05
    assert r.candidate_submaps == [closest(c.T_hypothesis[:3, 3], centers) for c in r.candidates]
    assert r.winner_submap == r.candidate_submaps[r.winner_rank]
    assert len(set(r.candidate_submaps)) >= 2                           # one search, refined in more than one submap


def test_assignment_ties_and_far_candidates():
    c = np.array([[1.0, 0.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    assert closest([0.0, 0.0, 0.0], c) == 0                              # three exact ties: the first
    assert closest([0.0, 0.0, 0.0], c[::-1]) == 0
    assert closest([0.0, 0.5, 0.0], c) == 2
    far = np.array([[0.0, 0.0, 0.0], [10.0, 0.0, 0.0], [5.0, 5.0, 0.0]])
    assert closest([100.0, 0.0, 0.0], far) == 1                          # outside every radius: still the nearest
    sc = S.SubmapCollection(None, S.SubmapParameters(radius=1.0))       # the host rule the device restates
    sc.submaps = [S.SubmapRecord(None, i, 0, x) for i, x in enumerate(far)]
    assert sc.findClosestSubmap(np.array([[1, 0, 0, 100.0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])) == 1


def test_relocalize_switches_to_an_existing_submap():
    lp, m = session()
    sc, be = m.submaps, m.backend
    prev, n0 = sc.activeSubmapIdx, len(sc.submaps)
    assert len(sc.overlapScansBuffer) > 0
    sc.params.radius = 50.0                                              # the found pose lies within the radius of its submap
    k = 5
    r = m.relocalize(lp.scan(k + lp.L, seed=905), params=box(lp.map_frame_pose(k)))
    T = r.T
    assert r.found and np.linalg.norm(T[:3, 3] - lp.map_frame_pose(k)[:3, 3]) < 0.05
    assert r.winner_submap != prev and sc.activeSubmapIdx == r.winner_submap and len(sc.submaps) == n0
    assert len(sc.overlapScansBuffer) == 0 and sc.numScansMergedInActiveSubmap == 0
    assert prev in sc.finishedSubmapsIdxs and sc.pendingFinishedSubmapIds[-1] == (prev, K)
    assert np.array_equal(m.mapToRangeSensor, T) and np.array_equal(be.pose, T) and be.isNewInitialValueSet and m.isNewInitialValueSet
    ev = sc.events[-1]
    assert ev[0] == "relocalization" and ev[1] == K and ev[2] and np.array_equal(ev[3], T) and ev[6] == r.winner_submap
    size = len(sc.getActiveSubmap().handle.xyz)
    m.addRangeMeasurement(lp.scan(k + 1 + lp.L, seed=906), lp.delta(k + 1))
    assert np.array_equal(m.poses[-1], T) and len(sc.getActiveSubmap().handle.xyz) == size   # rule 3: T kept, nothing inserted
    for j in range(k + 2, k + 6):
        m.addRangeMeasurement(lp.scan(j + lp.L, seed=900 + j), lp.delta(j))
        assert np.linalg.norm(m.poses[-1][:3, 3] - lp.map_frame_pose(j)[:3, 3]) < 0.1
    assert len(sc.getActiveSubmap().handle.xyz) > size


def test_relocalize_creates_a_child_of_the_winner_outside_its_radius():
    lp, m = session()
    sc, be = m.submaps, m.backend
    prev, n0 = sc.activeSubmapIdx, len(sc.submaps)
    sc.params.radius = 0.01
    k = 14
    r = m.relocalize(lp.scan(k + lp.L, seed=914), t=123, params=box(lp.map_frame_pose(k)))
    assert r.found and len(sc.submaps) == n0 + 1 and sc.activeSubmapIdx == n0
    new = sc.getActiveSubmap()
    assert new.parent == r.winner_submap and np.array_equal(new.origin, r.T[:3, 3])
    assert sc.isAdjacent(r.winner_submap, n0) and n0 in sc.adjacencyMatrix.adjacency_[r.winner_submap]
    assert len(new.handle.xyz) > 0 and sc.numScansMergedInActiveSubmap == 1   # the relocalisation scan is the new submap's first
    assert len(sc.overlapScansBuffer) == 0
    assert (prev, 123) in sc.pendingFinishedSubmapIds
    assert np.array_equal(m.mapToRangeSensor, r.T) and np.array_equal(be.pose, r.T)
    for j in range(k + 1, k + 5):
        m.addRangeMeasurement(lp.scan(j + lp.L, seed=900 + j), lp.delta(j))
    assert np.linalg.norm(m.poses[-1][:3, 3] - lp.map_frame_pose(k + 4)[:3, 3]) < 0.1


def test_failed_gate_changes_nothing(tmp_path):
    lp, m = session()
    before = saved(m, str(tmp_path / "a.npz"))
    n_events = len(m.submaps.events)
    scene = synth.Scene(cylinders=np.array([[3.0, -9.0], [-12.0, 4.0], [8.0, 8.0], [-5.0, -14.0], [10.0, -3.0], [-7.0, 9.0]]), half_x=60.0,
                        half_y=60.0, ground_z=-8.0)
    m.backend.p.minRefinementFitness = 1.01                              # no fitness reaches the gate
    r = m.relocalize(synth.lidar_scan(scene, np.eye(4), seed=5), params=box(lp.map_frame_pose(10)))
    m.backend.p.minRefinementFitness = E.MapperParameters().minRefinementFitness
    assert not r.found and len(m.submaps.events) == n_events + 1 and m.submaps.events[-1][0] == "relocalization"
    after = saved(m, str(tmp_path / "b.npz"))
    assert before.keys() == after.keys()
    for key in before:
        assert np.array_equal(before[key], after[key]), key
    assert not m.backend.isNewInitialValueSet


def test_localisation_mode_never_creates_a_submap():
    lp = W.ClosedLoop()
    p = E.MapperParameters(seed=3, isUseInitialMap=True, isMergeScansIntoMap=False)
    parts = []
    for k in range(0, 40, 2):
        T = lp.map_frame_pose(k)
        parts.append(lp.scan(k, seed=k).astype(np.float64) @ T[:3, :3].T + T[:3, 3])
    m = S.SegmentMapper(RelocalizationOracleBackend(copy.deepcopy(p), carving=False, dense=False), S.SubmapParameters(radius=0.01))
    m.setInitialMap(np.concatenate(parts)[::3])
    k = 20
    r = m.relocalize(lp.scan(k + lp.L, seed=920), params=box(lp.map_frame_pose(k)))
    assert r.found and r.winner_submap == 0 and len(m.submaps.submaps) == 1 and m.submaps.activeSubmapIdx == 0
    assert m.submaps.finishedSubmapsIdxs == [] and len(m.submaps.overlapScansBuffer) == 0
    assert np.array_equal(m.backend.pose, r.T) and m.backend.isNewInitialValueSet
    for j in range(k + 1, k + 4):
        m.addRangeMeasurement(lp.scan(j + lp.L, seed=900 + j), lp.delta(j))
    assert np.linalg.norm(m.poses[-1][:3, 3] - lp.map_frame_pose(k + 3)[:3, 3]) < 0.1
    assert len(m.submaps.submaps) == 1


def test_relocalize_needs_a_submap():
    m = S.SegmentMapper(RelocalizationOracleBackend(E.MapperParameters(seed=3), carving=False, dense=False))
    with pytest.raises(RuntimeError):
        m.relocalize(np.zeros((10, 3), dtype=np.float32))
