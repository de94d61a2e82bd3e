"""CPU: slam.buildLoopClosureConstraints through slam.refineLoopClosuresOfSubmaps, on the constructed pairs of test_loop_closure_host,
over the oracle backend.  Three ways to refine the survivors give the same decision log and the same constraints -- accepted,
rejected by the correspondence gate, by the consistency check, by the refinement's fitness gate, after an empty overlap:
    old       the composition buildLoopClosureConstraints ran before it refined submaps: two map copies, then refineLoopClosures
    composed  the oracle backend as it is (no refine_loop_closures of its own): refineLoopClosuresOfSubmaps composes its operations
    batched   a backend with refine_loop_closures shaped like DeviceBackend's: one call for all survivors, the information matrix
              filled for every pair, rejected ones included
Also: the survivors reach a batched backend in one call; getMapVoxelSize (PlaceRecognition.cpp:98)."""
import copy

import numpy as np
import pytest

from oracle_backend_ransac import RansacOracleBackend
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from test_loop_closure_host import P, collection
from test_ransac_oracle import rigid


class OldBackend(RansacOracleBackend):
    """the refinement buildLoopClosureConstraints composed before: the raw map voxel, no getMapVoxelSize"""

    def refine_loop_closures(self, source_sm, target_sms, inits, mapVoxelSize, lc=None):
        return S.refineLoopClosures(self, self.submap_as_cloud(source_sm), [self.submap_as_cloud(t) for t in target_sms], inits, mapVoxelSize, lc)


class BatchedBackend(RansacOracleBackend):
    """the records of DeviceBackend.refine_loop_closures from the oracle's operations: one call per source, every pair's information"""
    calls: list

    def refine_loop_closures(self, source_sm, target_sms, inits, mapVoxelSize, lc=None):
        self.calls.append((source_sm, list(target_sms), [np.array(T) for T in inits], mapVoxelSize))
        lc = lc or S.LoopClosureParameters()
        v = lc.voxelExpansionFactorOverlapComputation * E.getMapVoxelSize(mapVoxelSize, 0.04)
        src = self.submap_as_cloud(source_sm)
        out = []
        for t, T0 in zip(target_sms, inits):
            so, to = self.overlap(src, self.submap_as_cloud(t), T0, v, lc.minNumPointsPerVoxel)
            (r,) = self.register_batch([so], [to], [T0], lc.maxIcpCorrespondenceDistance, lc.maxNumIter)
            out.append({"n_source_overlap": len(so), "n_target_overlap": len(to), "result": r, "accepted": not (r.fitness_ < lc.minRefinementFitness),
                        "information": self.information_matrix(so, to, lc.maxIcpCorrespondenceDistance, r.transformation_)})
        return out


def run(backend_cls, T, mutate=None, candidates=(1,), mapVoxelSize=0.1, params=P):
    be, sc = collection(T)
    be.__class__ = backend_cls   # the collection keeps this object: swap how it refines, keep its maps
    be.calls = []
    if mutate:
        mutate(sc)
    cons, log = S.buildLoopClosureConstraints(be, sc, 0, list(candidates), params, mapVoxelSize)
    return be, cons, log


def same_constraints(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert (x.sourceSubmapIdx, x.targetSubmapIdx, x.isInformationMatrixValid, x.isOdometryConstraint) == \
               (y.sourceSubmapIdx, y.targetSubmapIdx, y.isInformationMatrixValid, y.isOdometryConstraint)
        assert np.array_equal(x.sourceToTarget, y.sourceToTarget) and np.array_equal(x.informationMatrix, y.informationMatrix)


def drop_box(sc):
    """the target keeps the floor and the two walls only: the source's box points find no partner, the fitness falls below 0.7"""
    t = sc.submaps[1].handle
    k = len(t.xyz) // 5
    t.xyz, t.nrm = t.xyz[:3 * k], t.nrm[:3 * k]


def far_away(sc):
    t = sc.submaps[1].handle
    t.xyz = t.xyz + [0.0, 0.0, 100.0]      # the proposal (from the shared sparse clouds) no longer fits the map: no overlap


@pytest.mark.parametrize("case,T,mutate,decision", [
    ("accepted", rigid(0.4, [3.0, -1.5, 0.2], 0.02, -0.01), None, "accepted"),
    ("identity", np.eye(4), None, "accepted"),
    ("fitness", rigid(0.4, [3.0, -1.5, 0.2]), drop_box, "rejected_refinement_fitness"),
    ("empty_overlap", rigid(0.1, [2.0, 1.0, 0.0]), far_away, "rejected_refinement_fitness"),
    ("ransac_inconsistent", rigid(0.1, [100.0, 0.0, 0.0]), None, "rejected_ransac_inconsistent"),
])
def test_same_decisions_and_constraints(case, T, mutate, decision):
    _, old_c, old_log = run(OldBackend, T, mutate)
    for cls in (RansacOracleBackend, BatchedBackend):
        _, c, log = run(cls, T, mutate)
        assert log == old_log and log[0][1] == decision, (case, cls, log)
        same_constraints(c, old_c)
    if decision == "accepted":
        assert len(old_c) == 1 and np.abs(old_c[0].sourceToTarget - T).max() < 1e-6


def test_correspondence_gate_never_reaches_the_refinement():
    p = copy.deepcopy(P)
    p.ransacMinCorrespondenceSetSize = 10 ** 9
    be, cons, log = run(BatchedBackend, rigid(0.4, [3.0, -1.5, 0.2]), params=p)
    assert cons == [] and log[0][1] == "rejected_correspondences" and be.calls == []


def test_survivors_in_one_call():
    """the same candidate listed three times: every survivor and its RANSAC T reach the backend in one refine_loop_closures call,
    and the three records are the same"""
    T = rigid(0.4, [3.0, -1.5, 0.2])
    be, cons, log = run(BatchedBackend, T, candidates=(1, 1, 1))
    assert len(be.calls) == 1
    _src, tgts, inits, v = be.calls[0]
    assert len(tgts) == 3 and all(t is tgts[0] for t in tgts) and v == 0.1
    assert all(np.abs(Ti - T).max() < 1e-6 for Ti in inits)
    assert [d for _, d, _ in log] == ["accepted"] * 3 and len(cons) == 3
    for c in cons[1:]:
        assert np.array_equal(c.sourceToTarget, cons[0].sourceToTarget) and np.array_equal(c.informationMatrix, cons[0].informationMatrix)


@pytest.mark.parametrize("v", [0.0, 1e-3, -1e-3])
def test_map_voxel_size_rule(v):
    """getMapVoxelSize(mapBuilder_, 0.04) (PlaceRecognition.cpp:98): |v| <= 1e-3 refines as an explicit 0.04 does, on both paths"""
    T = rigid(0.4, [3.0, -1.5, 0.2])
    for cls in (RansacOracleBackend, BatchedBackend):
        _, c0, l0 = run(cls, T, mapVoxelSize=v)
        _, c1, l1 = run(cls, T, mapVoxelSize=0.04)
        assert l0 == l1 and l0[0][1] == "accepted"
        same_constraints(c0, c1)
