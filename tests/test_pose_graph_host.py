"""CPU tests of the loop-closure host flow in slam.py against hand-worked cases: OptimizationProblem's node initialisation (first and
incremental call), its loop-closure dedupe and asserts, SubmapCollection.transform's parent-chain rule, and the order of
SegmentMapper.loopClosureUpdate against the device's pose slot.  The backend is a recorder; the solve is the numpy restatement."""
import numpy as np
import pytest

import oracle_pose_graph as PG
from oracle_backend_pose_graph import global_optimization
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S


class Recorder:
    """the backend calls the host flow makes, recorded; pose slots as the device keeps them (one per submap)"""

    def __init__(self):
        self.calls = []
        self.slots = {}

    def global_optimization(self, poseGraph, criteria, option):
        self.calls.append(("solve", len(poseGraph.nodes_), len(poseGraph.edges_)))
        return global_optimization(poseGraph, criteria, option)

    def transform_submap(self, sm, sparse, T):
        self.calls.append(("transform", sm, np.array(T)))
        self.slots[sm] = self.slots.get(sm, np.eye(4)) @ T     # b2s_submap_transform right-multiplies the slot

    def loop_closure_update(self, sm, T):
        self.calls.append(("pose", sm, np.array(T)))
        self.slots[sm] = np.array(T)

    def odometry_constraints(self, pairs, params):
        self.calls.append(("odometry_constraints", list(pairs)))
        return [E.OdometryConstraintResult(np.eye(4), np.eye(6) * 100.0, 1, 1) for _ in pairs]


def odo(s, t, T):
    return S.Constraint(np.asarray(T, dtype=np.float64), s, t, np.eye(6) * 50.0, isOdometryConstraint=True)


def lc(s, t, T=None):
    return S.Constraint(np.eye(4) if T is None else np.asarray(T, dtype=np.float64), s, t, np.eye(6) * 50.0)


def test_node_initialisation_and_incremental_second_call():
    b = Recorder()
    prob = S.OptimizationProblem(b)
    X = [PG.rigid([0, 0, 0.1 * k], [1.0 + k, 0, 0]) for k in range(4)]
    prob.insertOdometryConstraints([odo(1, 2, X[1]), odo(0, 1, X[0])])   # sorted by source before use
    prob.insertLoopClosureConstraints([lc(2, 0, np.linalg.inv(X[1] @ X[0]))])
    prob.buildOptimizationProblem()
    n = prob.poseGraph_.nodes_
    assert [(e.source_node_id_, e.target_node_id_, e.uncertain_) for e in prob.poseGraph_.edges_] == [(0, 1, False), (1, 2, False), (2, 0, True)]
    assert len(n) == 3 and np.array_equal(n[0].pose_, np.eye(4))   # nodes: the inverse of the chained odometry
    assert np.allclose(n[1].pose_, np.linalg.inv(X[0])) and np.allclose(n[2].pose_, np.linalg.inv(X[1] @ X[0]))
    prob.solve()
    last = np.array(prob.poseGraphOptimized_.nodes_[-1].pose_)
    # second call: one more odometry edge; the new node chains from the LAST OPTIMISED node, not from the identity
    prob.clearOdometryConstraints()
    prob.insertOdometryConstraints([odo(0, 1, X[0]), odo(1, 2, X[1]), odo(2, 3, X[2])])
    prob.buildOptimizationProblem()
    n = prob.poseGraph_.nodes_
    assert len(n) == 4
    assert np.allclose(n[3].pose_, np.linalg.inv(X[2] @ np.linalg.inv(last)))


def test_loop_closure_dedupe_and_asserts():
    prob = S.OptimizationProblem(Recorder())
    prob.insertLoopClosureConstraints([lc(5, 1), lc(5, 1, PG.rigid([0, 0, 1], [1, 0, 0])), lc(5, 2)])
    prob.insertLoopClosureConstraints([lc(5, 2), lc(6, 1)])
    assert [(c.sourceSubmapIdx, c.targetSubmapIdx) for c in prob.getLoopClosureConstraints()] == [(5, 1), (5, 2), (6, 1)]
    assert np.array_equal(prob.getLoopClosureConstraints()[0].sourceToTarget, np.eye(4))   # the first one stays
    bad = S.OptimizationProblem(Recorder())
    bad.insertLoopClosureConstraints([lc(1, 5)])   # source must be the later submap
    with pytest.raises(RuntimeError):
        bad.buildOptimizationProblem()
    bad = S.OptimizationProblem(Recorder())
    bad.insertOdometryConstraints([odo(2, 1, np.eye(4))])
    with pytest.raises(RuntimeError):
        bad.buildOptimizationProblem()


def collection(parents):
    b = Recorder()
    sc = S.SubmapCollection(b, S.SubmapParameters())
    for i, p in enumerate(parents):
        sc.submaps.append(S.SubmapRecord(f"sm{i}", i, p, np.zeros(3), center=np.array([float(i), 0.0, 0.0])))
    return b, sc


def test_transform_parent_chain_rule():
    """submaps 0..2 are in the graph; 3 (parent 1) takes 1's increment; 4 (parent 3, itself outside) climbs to 1 as well; 5 (parent 2)
    takes 2's.  The overlap buffer is flushed; centers move by T."""
    b, sc = collection([0, 0, 1, 1, 3, 2])
    sc.overlapScansBuffer.append(("scan", np.eye(4)))
    inc = [S.OptimizedTransform(PG.rigid([0, 0, 0.1 * i], [i, 2.0 * i, 0]), i) for i in range(3)]
    sc.transform(inc)
    got = [(c[1], c[2]) for c in b.calls if c[0] == "transform"]
    assert [g[0] for g in got] == ["sm0", "sm1", "sm2", "sm3", "sm4", "sm5"]
    for (name, T), want in zip(got, [0, 1, 2, 1, 1, 2]):
        assert np.array_equal(T, inc[want].dT_), name
    assert len(sc.overlapScansBuffer) == 0
    assert np.allclose(sc.submaps[3].center, inc[1].dT_[:3, :3] @ [3.0, 0, 0] + inc[1].dT_[:3, 3])
    b, sc = collection([0, 1])   # 1 is its own parent and not in the graph: the reference's "Stuck in a loop"
    with pytest.raises(RuntimeError):
        sc.transform([S.OptimizedTransform(np.eye(4), 0)])
    b, sc = collection([0, 0])
    sc.transform([])   # no increments: nothing moves
    assert not [c for c in b.calls if c[0] == "transform"]


def test_loop_closure_update_leaves_the_active_slot_at_dT_times_the_mapper_pose():
    b, sc = collection([0, 0, 1])
    m = S.SegmentMapper.__new__(S.SegmentMapper)
    m.backend, m.submaps = b, sc
    sc.activeSubmapIdx = 2
    pose = PG.rigid([0.1, 0.2, 0.3], [4.0, 5.0, 6.0])
    m.mapToRangeSensor = pose.copy()
    b.slots["sm2"] = pose.copy()
    inc = [S.OptimizedTransform(PG.rigid([0, 0, 0.05 * i], [0.1 * i, 0, 0]), i) for i in range(3)]
    sc.transform(inc)   # the slot is right-multiplied: pose * dT (Submap::mapToRangeSensor_ of the reference)
    assert np.allclose(b.slots["sm2"], pose @ inc[2].dT_)
    m.loopClosureUpdate(inc[2].dT_)   # then the mapper: dT * pose, and that is what the next step predicts from
    assert np.allclose(m.mapToRangeSensor, inc[2].dT_ @ pose)
    assert np.array_equal(b.slots["sm2"], m.mapToRangeSensor)


def test_loop_closure_cycle_composes_the_reference_steps():
    b, sc = collection([0, 0, 1, 2])
    sc.activeSubmapIdx = 3
    m = S.SegmentMapper.__new__(S.SegmentMapper)
    m.backend, m.submaps, m.mapToRangeSensor = b, sc, np.eye(4)
    prob = S.OptimizationProblem(b)
    c = lc(2, 0, PG.rigid([0, 0, 0.02], [0.05, 0, 0]))
    dT = S.loopClosureCycle(b, m, prob, [c])
    kinds = [k[0] for k in b.calls]
    # odometry constraints of every pair not touching the active submap (3), one batched call; then the solve; then the transforms
    assert kinds[0] == "odometry_constraints" and b.calls[0][1] == [("sm0", "sm1"), ("sm1", "sm2")]
    assert kinds[1] == "solve" and b.calls[1][1:] == (3, 3)
    assert kinds[2:6] == ["transform"] * 4 and kinds[6] == "pose"
    inc = prob.getOptimizedTransformIncrements()
    assert np.array_equal(dT, inc[2].dT_)                                   # the latest loop closure's SOURCE submap
    assert np.array_equal(prob.getLoopClosureConstraints()[0].sourceToTarget, np.eye(4))   # reset to identity
    assert sc.isAdjacent(0, 2) and sc.loopClosureSubmaps == {0, 2}
