"""CPU tests of the loop-closing schedule in slam.py: AdjacencyMatrix (src/AdjacencyMatrix.cpp:16-71) on hand-built graphs with each of
its quirks, getLoopClosureCandidatesIdxs (src/PlaceRecognition.cpp:231-284) one rule at a time, and SegmentMapper with
isAttemptLoopClosures over an oracle backend that has every loop-closure step (LoopClosingOracleBackend, below) on a short lap with
10 m submaps: a loop closes without being named, and with the flag off nothing changes."""
import copy

import numpy as np
import pytest

from oracle_backend_pose_graph import PoseGraphOracleBackend
from oracle_backend_ransac import RansacOracleBackend
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W


class LoopClosingOracleBackend(PoseGraphOracleBackend, RansacOracleBackend):
    """The oracle backend with every step of the schedule: features and RANSAC (RansacOracleBackend), odometry constraints, the solve
    and the correction (PoseGraphOracleBackend), the refinement of OracleBackend."""


# ----------------------------------------------------------------------------------------------------------------------
# AdjacencyMatrix
# ----------------------------------------------------------------------------------------------------------------------
def chain(n):
    a = S.AdjacencyMatrix()
    for i in range(n - 1):
        a.addEdge(i, i + 1)
    return a


def test_int_max_until_an_edge_is_added():
    a = S.AdjacencyMatrix()
    assert a.getDistanceToNearestLoopClosureSubmap(0) == S.INT_MAX == 2**31 - 1
    assert a.getDistanceToNearestLoopClosureSubmap(7) == S.INT_MAX       # no lookup happens before the emptiness test
    a.addEdge(0, 1)
    assert a.getDistanceToNearestLoopClosureSubmap(0) == 0               # nothing marked: path to the last dequeued node (1), minus 1
    with pytest.raises(KeyError):
        a.getDistanceToNearestLoopClosureSubmap(5)                       # isLoopClosureSubmap_.at(5)


def test_self_adjacency_and_symmetry():
    a = S.AdjacencyMatrix()
    assert a.isAdjacent(3, 3) and not a.isAdjacent(3, 4)
    a.addEdge(3, 4)
    assert a.isAdjacent(3, 4) and a.isAdjacent(4, 3) and not a.isAdjacent(3, 5)


def test_mark_throws_for_an_id_without_an_edge():
    a = chain(3)
    with pytest.raises(KeyError):
        a.markAsLoopClosureSubmap(3)
    a.markAsLoopClosureSubmap(2)
    assert a.isLoopClosureSubmap_ == {0: False, 1: False, 2: True}


def test_distance_to_a_marked_node():
    a = chain(8)                       # 0 - 1 - ... - 7
    a.markAsLoopClosureSubmap(2)
    assert [a.getDistanceToNearestLoopClosureSubmap(i) for i in range(8)] == [1, 0, 0, 0, 1, 2, 3, 4]
    a.markAsLoopClosureSubmap(6)
    assert [a.getDistanceToNearestLoopClosureSubmap(i) for i in range(8)] == [1, 0, 0, 0, 1, 0, 0, 0]


def test_unreachable_mark_measures_the_path_to_the_last_dequeued_node():
    """two components: 0-1-2-3 and 10-11 with 11 marked; from 1 the BFS never reaches a mark and stops at the last node it dequeued
    (3, at distance 2), so the distance is 1 -- not INT_MAX"""
    a = chain(4)
    a.addEdge(10, 11)
    a.markAsLoopClosureSubmap(11)
    assert a.getDistanceToNearestLoopClosureSubmap(1) == 1
    assert a.getDistanceToNearestLoopClosureSubmap(0) == 2
    assert a.getDistanceToNearestLoopClosureSubmap(10) == 0
    # a star: from the centre every leaf is at distance 1; the last one dequeued is the largest id (std::set order) -> 0
    s = S.AdjacencyMatrix()
    for leaf in (5, 3, 9):
        s.addEdge(0, leaf)
    assert s.getDistanceToNearestLoopClosureSubmap(0) == 0
    assert s.getDistanceToNearestLoopClosureSubmap(3) == 1      # 3 -> 0 -> {5, 9}: the last dequeued (9) is 2 away


def test_add_edge_unmarks_both_ends():
    """a hand-over edge after a loop closure resets the loop-closure mark of both of its ends"""
    a = chain(6)
    a.addEdge(5, 0)
    a.markAsLoopClosureSubmap(5)
    a.markAsLoopClosureSubmap(0)
    assert a.getDistanceToNearestLoopClosureSubmap(3) == 1
    a.addEdge(5, 6)                     # hand-over 5 -> 6
    assert a.isLoopClosureSubmap_[5] is False and a.isLoopClosureSubmap_[0] is True
    assert a.getDistanceToNearestLoopClosureSubmap(5) == 0      # 5 -> 0 (marked), one edge
    assert a.getDistanceToNearestLoopClosureSubmap(4) == 1      # 4 -> 5 -> 0
    a.addEdge(0, 1)                     # an edge that already exists still unmarks
    assert a.isLoopClosureSubmap_[0] is False
    assert a.getDistanceToNearestLoopClosureSubmap(3) == 2      # nothing marked: last dequeued from 3 is 6 (3-4-5-6), 3 edges


def test_collection_feeds_the_matrix_from_hand_overs_and_loop_closures():
    sc = S.SubmapCollection(None, S.SubmapParameters())
    sc.updateAdjacencyMatrix([S.Constraint(np.eye(4), 4, 0, np.eye(6))])
    assert sc.adjacencyMatrix.isLoopClosureSubmap_ == {4: True, 0: True}
    assert sc.isAdjacent(0, 4) and sc.adjacencyMatrix.isAdjacent(0, 4) and sc.loopClosureSubmaps == {0, 4}


# ----------------------------------------------------------------------------------------------------------------------
# getLoopClosureCandidatesIdxs: one collection per rule, built so that only that rule excludes submap 0
# ----------------------------------------------------------------------------------------------------------------------
def line(n, spacing=4.0, radius=10.0, centers=None):
    """n submap records, centres every `spacing` m on x (or as given), the chain of hand-over edges in the matrix"""
    sc = S.SubmapCollection(None, S.SubmapParameters(radius=radius))
    for i in range(n):
        c = np.array([spacing * i, 0.0, 0.0]) if centers is None else np.asarray(centers[i], dtype=np.float64)
        sc.submaps.append(S.SubmapRecord(f"sm{i}", i, max(i - 1, 0), np.zeros(3), center=c))
    for i in range(n - 1):
        sc.adjacencyMatrix.addEdge(i, i + 1)
    sc.activeSubmapIdx = n - 1
    return sc


def candidates(sc, last, params=None):
    return S.getLoopClosureCandidatesIdxs(sc, sc.adjacencyMatrix, last, sc.activeSubmapIdx, params)


def test_baseline_candidate():
    sc = line(7)                        # last = 5, active = 6: 0, 1 and 2 are candidates (|i - 5| > ceil(20 / 10) = 2)
    assert candidates(sc, 5) == [0, 1, 2]


def test_rule_active_submap():
    sc = line(7)
    sc.activeSubmapIdx = 0
    assert candidates(sc, 5) == [2]     # 0 is active, 1 adjacent to it; 6 is adjacent to 5


def test_rule_adjacent_to_active():
    sc = line(7)
    sc.adjacencyMatrix.addEdge(0, 6)    # 0 adjacent to the active submap 6, and nothing else changes for it
    assert candidates(sc, 5) == [1, 2]


def test_rule_neighbour_index_or_adjacent_to_last():
    # a search radius of 0 with every centre in one place: the distance rule passes every submap and the consecutive threshold is 0
    p = S.LoopClosureCandidateParameters(loopClosureSearchRadius=0.0, minSubmapsBetweenLoopClosures=0)
    sc = line(6, spacing=0.0)
    sc.adjacencyMatrix = S.AdjacencyMatrix()
    assert candidates(sc, 2, p) == [0, 4]     # 1 and 3 by |i - 2| == 1, 2 by self-adjacency, 5 active
    sc.adjacencyMatrix.addEdge(0, 2)
    assert candidates(sc, 2, p) == [4]        # 0 is adjacent to the last finished submap


def test_rule_search_radius():
    sc = line(7, centers=[[-30, 0, 0], [4, 0, 0], [8, 0, 0], [12, 0, 0], [16, 0, 0], [20, 0, 0], [24, 0, 0]])
    assert candidates(sc, 5) == [1, 2]  # 0 is 50 m from 5 (and 20 m, at the radius, is kept: the rule is distance > radius)


def test_rule_consecutive_threshold():
    sc = line(7, radius=6.0)            # ceil(20 / 6) = 4: |0 - 5| = 5 stays, |1 - 5| = 4 goes
    assert candidates(sc, 5) == [0]
    sc = line(7, radius=4.0)            # ceil(20 / 4) = 5: |0 - 5| = 5 goes as well
    assert candidates(sc, 5) == []


def test_rule_min_submaps_between_loop_closures():
    sc = line(7)
    sc.adjacencyMatrix.addEdge(5, 3)    # a loop closure 5 -> 3 marks both ends...
    sc.adjacencyMatrix.markAsLoopClosureSubmap(5)
    sc.adjacencyMatrix.markAsLoopClosureSubmap(3)
    assert sc.adjacencyMatrix.getDistanceToNearestLoopClosureSubmap(5) == 0
    assert candidates(sc, 5) == []
    assert candidates(sc, 5, S.LoopClosureCandidateParameters(minSubmapsBetweenLoopClosures=0)) == [0, 1, 2]
    sc.adjacencyMatrix.addEdge(5, 6)    # ...and the next hand-over unmarks 5: 5 -> 3 is still one edge to a mark
    assert sc.adjacencyMatrix.getDistanceToNearestLoopClosureSubmap(5) == 0 and candidates(sc, 5) == []
    sc = line(9)
    sc.adjacencyMatrix.markAsLoopClosureSubmap(4)        # 7 -> 6 -> 5 -> 4: distance 2 >= 2
    assert candidates(sc, 7) == [2, 3, 4]                # 0 and 1 are farther than 20 m
    sc.adjacencyMatrix.markAsLoopClosureSubmap(5)        # 7 -> 6 -> 5: distance 1 < 2
    assert candidates(sc, 7) == []


def test_centres_fall_back_to_the_origin_before_the_submap_is_finished():
    sc = line(7)
    sc.submaps[0].center = None
    sc.submaps[0].origin = np.array([-25.0, 0.0, 0.0])   # getMapToSubmapCenter: mapToSubmap_ until computeSubmapCenter ran
    assert candidates(sc, 5) == [1, 2]


# ----------------------------------------------------------------------------------------------------------------------
# the schedule over the oracle backend
# ----------------------------------------------------------------------------------------------------------------------
def test_constraint_timestamps_choose_the_correction():
    """updateSubmapsAndTrajectory: the greatest timestamp wins, the first of equal ones (std::max_element); a constraint without a
    timestamp leaves the last one in the list"""
    import oracle_pose_graph as PG
    from test_pose_graph_host import collection
    for stamps, want in (((30, 70, 70, 40), 6), ((None, 70, 70, 40), 4)):
        b, sc = collection([0, 0, 1, 2, 3, 4, 5, 6])
        sc.activeSubmapIdx = 7
        m = S.SegmentMapper.__new__(S.SegmentMapper)
        m.backend, m.submaps, m.mapToRangeSensor = b, sc, np.eye(4)
        prob = S.OptimizationProblem(b)
        lcs = [S.Constraint(PG.rigid([0, 0, 0.01 * s], [0.1 * s, 0, 0]), s, 0, np.eye(6) * 50.0, timestamp=t)
               for s, t in zip((5, 6, 3, 4), stamps)]
        dT = S.loopClosureCycle(b, m, prob, lcs)
        inc = prob.getOptimizedTransformIncrements()
        assert np.abs(inc[6].dT_ - inc[4].dT_).max() > 1e-6
        assert np.array_equal(dT, inc[want].dT_)


# On the closed lap (a 16 m courtyard loop) a 20 m search reaches submaps across the courtyard, whose maps alias: with the default
# radius the oracle accepts 3 -> 0, 12 m apart, with a 1.6 m error.  A 10 m search keeps the candidates to the places the lap
# revisits.
SEARCH_RADIUS = 10.0


def lap_mapper(n_scans, **kw):
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    be = LoopClosingOracleBackend(copy.deepcopy(p), carving=True, dense=False)
    if kw.get("isAttemptLoopClosures"):
        kw["loopClosing"] = S.LoopClosingParameters.fromMapperParameters(p)
        kw["loopClosing"].candidates.loopClosureSearchRadius = SEARCH_RADIUS
    m = S.SegmentMapper(be, S.SubmapParameters(radius=10.0), **kw)
    for k in range(n_scans):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    return m


N_LAP = 145


def test_the_schedule_closes_a_loop_on_its_own():
    """145 scans of the closed lap (1.2 laps) with 10 m submaps: every finished submap gets its features in the scan that finished
    it, candidate selection finds an earlier submap on its own, the constraint is accepted and the cycle solves and corrects in that
    same scan; finishProcessing finishes the active submap and attempts it."""
    m = lap_mapper(N_LAP, isAttemptLoopClosures=True)
    sc, ev = m.submaps, m.submaps.events
    hand_overs = [e for e in ev if e[0] == "active_submap_changed"]
    assert len(hand_overs) >= 4
    assert [e[1:] for e in ev if e[0] == "features"] == [(k, [prev]) for _, k, prev, _new in hand_overs]
    assert [e[1:3] for e in ev if e[0] == "loop_closure_candidates"] == [(k, prev) for _, k, prev, _new in hand_overs]
    closing = [e for e in ev if e[0] == "loop_closure_decisions" and any(d == "accepted" for _i, d, _n in e[3])]
    assert closing
    k, src = closing[0][1], closing[0][2]
    (tgt,) = [i for i, d, _n in closing[0][3] if d == "accepted"]
    assert src - tgt > 2 and ("loop_closure_candidates", k, src, [i for i, _d, _n in closing[0][3]]) in ev
    solves = [e for e in ev if e[0] == "pose_graph_solve"]
    corrections = [e for e in ev if e[0] == "loop_closure_correction"]
    assert solves[0][1] == k and solves[0][2][0][0] and corrections[0][1:3] == (k, src)
    dT = corrections[0][3]
    assert 0.0 < np.linalg.norm(dT[:3, 3]) < 0.05    # the lap's own drift is about a centimetre: the right place was closed
    # the pose graph: one odometry constraint per finished submap but the first, and the loop closure marked in the matrix
    assert [(c.sourceSubmapIdx, c.targetSubmapIdx) for c in sc.odometryConstraints][:len(hand_overs) - 1] == \
           [(sc.submaps[prev].parent, prev) for _, _k, prev, _new in hand_overs[1:]]
    assert sc.adjacencyMatrix.isAdjacent(src, tgt) and sc.adjacencyMatrix.isLoopClosureSubmap_[tgt]
    assert m.optimizationProblem.getLoopClosureConstraints()[0].timestamp == k   # the finishing scan of the source submap
    n_before = len(sc.submaps)
    m.finishProcessing()
    forced = [e for e in ev if e[0] == "active_submap_changed"][-1]
    assert forced[1] == N_LAP and forced[3] == n_before == sc.activeSubmapIdx and len(sc.submaps) == n_before + 1
    assert [e for e in ev if e[0] == "features"][-1] == ("features", N_LAP, [forced[2]])
    assert sc.submaps[forced[2]].feature is not None and sc.pendingFinishedSubmapIds == []


def test_flag_off_is_the_mapper_of_before():
    """30 scans (one hand-over): the default mapper and one with the flag given as False log the same events and poses, and none of
    the schedule's"""
    a, b = lap_mapper(30), lap_mapper(30, isAttemptLoopClosures=False)
    assert a.submaps.events == b.submaps.events and any(e[0] == "active_submap_changed" for e in a.submaps.events)
    assert all(np.array_equal(x, y) for x, y in zip(a.poses, b.poses)) and len(a.poses) == 30
    assert not any(e[0] in ("features", "loop_closure_candidates", "loop_closure_decisions") for e in a.submaps.events)
    assert all(r.feature is None for r in a.submaps.submaps) and a.submaps.odometryConstraints == []
