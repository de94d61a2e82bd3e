"""CPU: the odometry constraints between consecutive submaps (computeOdometryConstraints / buildOdometryConstraint,
core/src/constraint_builders.cpp:23-118) over the oracle backend (tests/oracle_backend_constraints.py): the reference's control flow
(submap 0 skipped, the parent lookup, no rebuild of an existing pair, the active submap left out by the all-submaps overload, one
batched backend call), getMapVoxelSize, the oracle's constraint on two overlapping patches with a known offset, and the ctypes mirror
of the new structs against the C compiler's layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from oracle_backend import OracleSubmap
from oracle_backend_constraints import ConstraintOracleBackend
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from test_loop_closure_host import room
from test_ransac_oracle import rigid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class RecordingBackend(ConstraintOracleBackend):
    def __init__(self):
        super().__init__(E.MapperParameters())
        self.calls = []

    def odometry_constraints(self, pairs, params):
        self.calls.append([(self.ids[id(s)], self.ids[id(t)]) for s, t in pairs])
        return super().odometry_constraints(pairs, params)


def chain(parents, active):
    """a SubmapCollection whose submap k has parent parents[k]: small overlapping patches along x"""
    be = RecordingBackend()
    sc = S.SubmapCollection(be, S.SubmapParameters())
    xyz, nrm = room(0, 2000)
    be.ids = {}
    for k, p in enumerate(parents):
        sm = OracleSubmap(None)
        sm.xyz, sm.nrm = xyz + [0.5 * k, 0, 0], nrm
        be.ids[id(sm)] = k
        sc.submaps.append(S.SubmapRecord(sm, k, p, np.zeros(3)))
    sc.activeSubmapIdx = active
    return be, sc


def test_finished_ids_overload_skips_submap_zero_and_uses_the_parent():
    be, sc = chain([0, 0, 1, 1], active=3)
    cons = []
    added = S.computeOdometryConstraints(be, sc, cons, finishedIds=[0, 1, 2, 3])
    assert be.calls == [[(0, 1), (1, 2), (1, 3)]]          # one batched call; (parent, child); the active submap is NOT left out here
    assert [(c.sourceSubmapIdx, c.targetSubmapIdx) for c in cons] == [(0, 1), (1, 2), (1, 3)] and added == cons
    assert all(c.isOdometryConstraint and c.isInformationMatrixValid for c in cons)


def test_existing_pairs_are_not_rebuilt():
    be, sc = chain([0, 0, 1, 2], active=3)
    cons = []
    S.computeOdometryConstraints(be, sc, cons, finishedIds=[1])
    S.computeOdometryConstraints(be, sc, cons, finishedIds=[1, 2, 2])
    assert be.calls == [[(0, 1)], [(1, 2)]]
    assert S.computeOdometryConstraints(be, sc, cons, finishedIds=[1, 2]) == [] and len(be.calls) == 2
    assert S.hasConstraint(0, 1, cons) and not S.hasConstraint(1, 0, cons)


def test_all_submaps_overload_leaves_out_the_active_submap():
    be, sc = chain([0, 0, 1, 2, 2], active=2)
    cons = []
    S.computeOdometryConstraints(be, sc, cons)
    assert be.calls == [[(0, 1)]]                            # (1, 2) and (2, 3), (2, 4) touch the active submap 2
    sc.activeSubmapIdx = 4
    S.computeOdometryConstraints(be, sc, cons)
    assert be.calls[-1] == [(1, 2), (2, 3)]


def test_get_map_voxel_size():
    assert E.getMapVoxelSize(0.0, 0.04) == 0.04 and E.getMapVoxelSize(1e-3, 0.04) == 0.04 and E.getMapVoxelSize(-1e-3, 0.04) == 0.04
    assert E.getMapVoxelSize(0.1, 0.04) == 0.1 and E.getMapVoxelSize(-0.2, 0.04) == -0.2   # a negative size passes through
    assert E.getMapVoxelSize(1.0001e-3, 0.04) == 1.0001e-3


def patches(T):
    xyz, nrm = room(3, 6000)
    return (xyz, nrm), (xyz @ T[:3, :3].T + T[:3, 3], nrm @ T[:3, :3].T)


def test_refined_constraint_recovers_the_offset():
    T = rigid(0.01, [0.05, -0.03, 0.02])
    be = ConstraintOracleBackend(E.MapperParameters())
    sc = S.SubmapCollection(be, S.SubmapParameters())
    for k, (x, n) in enumerate(patches(T)):
        sm = OracleSubmap(None); sm.xyz, sm.nrm = x, n
        sc.submaps.append(S.SubmapRecord(sm, k, 0, np.zeros(3)))
    c = S.buildOdometryConstraint(be, sc, 0, 1, E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=True))
    assert np.abs(c.sourceToTarget - T).max() < 2e-3          # from 5 cm and 0.6 deg off at the identity; stops at rel. change 1e-6
    assert c.isOdometryConstraint and c.isInformationMatrixValid
    assert np.allclose(c.informationMatrix, c.informationMatrix.T) and c.informationMatrix[3, 3] > 0.8 * 6000


def test_unrefined_constraint_keeps_the_identity():
    T = rigid(0.01, [0.05, -0.03, 0.02])
    (sx, sn), (tx, tn) = patches(T)
    p = E.OdometryConstraintParameters()
    from oracle_backend_constraints import odometry_constraint
    r, (so, _), (to, _) = odometry_constraint(sx, sn, tx, tn, p)
    assert np.array_equal(r.sourceToTarget_, np.eye(4)) and r.icp is None
    assert (r.nSourceOverlap, r.nTargetOverlap) == (len(so), len(to)) and len(so) > 0.9 * len(sx)
    assert np.array_equal(r.informationMatrix_, O.information_matrix(so, to, 0.15, np.eye(4)))
    with pytest.raises(ValueError):   # refinement without the child's normals
        odometry_constraint(sx, sn, tx, np.full_like(tn, np.nan), E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=True))


def test_ctypes_mirror_matches_the_header(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b2s.h"\nint main(void) {\n'
                    '  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(b2s_odometry_constraint_params), offsetof(b2s_odometry_constraint_params, rel_fitness),\n'
                    '         sizeof(b2s_odometry_constraint), offsetof(b2s_odometry_constraint, n_source_overlap), offsetof(b2s_odometry_constraint, refined),\n'
                    '         offsetof(b2s_odometry_constraint, icp));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    P, R = L.OdometryConstraintParams, L.OdometryConstraint
    assert got == [C.sizeof(P), P.rel_fitness.offset, C.sizeof(R), R.n_source_overlap.offset, R.refined.offset, R.icp.offset]
    p = P()
    L.lib().b2s_default_odometry_constraint_params(C.byref(p))
    d = E.OdometryConstraintParameters()
    assert (p.map_voxel_size, p.voxel_if_zero, p.overlap_factor, p.icp_factor, p.min_points_per_voxel, p.refine, p.max_iter, p.rel_fitness,
            p.rel_rmse) == (d.mapVoxelSize, d.voxelSizeIfMapVoxelSizeIsZero, d.voxelExpansionFactorOverlapComputation,
                            d.voxelExpansionFactorIcpCorrespondenceDistance, d.minNumPointsPerVoxel, 0, d.maxNumIter, d.relativeFitness,
                            d.relativeRmse)
