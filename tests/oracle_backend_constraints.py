"""The oracle backend with the odometry constraints (TEST INFRASTRUCTURE): odometry_constraints = buildOdometryConstraint
(core/src/constraint_builders.cpp:33-90) restated over the oracle, one pair after the other -- the counterpart of
slam.DeviceBackend.odometry_constraints under slam.computeOdometryConstraints."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O
from oracle_backend import OracleBackend
from open3d_slam_b200 import engine as E


def odometry_constraint(source_xyz, source_nrm, target_xyz, target_nrm, params: E.OdometryConstraintParameters):
    """(OdometryConstraintResult, source overlap, target overlap) of one (parent, child) pair of whole maps"""
    v = E.getMapVoxelSize(params.mapVoxelSize, params.voxelSizeIfMapVoxelSizeIsZero)
    if not v > 0.0:
        raise ValueError("map voxel size must be > 0")
    r = params.voxelExpansionFactorIcpCorrespondenceDistance * v
    fs, ft = O.overlap_flags(source_xyz, target_xyz, np.eye(4), params.voxelExpansionFactorOverlapComputation * v, params.minNumPointsPerVoxel)
    sx, tx = source_xyz[fs], target_xyz[ft]
    T, icp = np.eye(4), None
    if params.isRefineOdometryConstraintsBetweenSubmaps:
        tn = None if target_nrm is None else target_nrm[ft]
        if tn is None or np.isnan(tn).any():
            raise ValueError("TransformationEstimationPointToPlane requires target normals")
        res = O.registration_icp_p2plane(sx, tx, tn, r, np.eye(4), max_iter=params.maxNumIter, rel_fitness=params.relativeFitness,
                                         rel_rmse=params.relativeRmse)
        T = np.array(res.T)
        icp = E.RegistrationResult(T, res.fitness, res.inlier_rmse, res.n_corr, res.iters)
    info = O.information_matrix(sx, tx, r, T)
    res = E.OdometryConstraintResult(T, info, len(sx), len(tx), icp)
    return res, (sx, None if source_nrm is None else source_nrm[fs]), (tx, None if target_nrm is None else target_nrm[ft])


class ConstraintOracleBackend(OracleBackend):
    def odometry_constraints(self, pairs, params: E.OdometryConstraintParameters):
        return [odometry_constraint(s.xyz, s.nrm, t.xyz, t.nrm, params)[0] for s, t in pairs]
