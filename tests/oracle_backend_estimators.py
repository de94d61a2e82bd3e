"""The oracle backend with the loop-closure refinement's estimator (TEST INFRASTRUCTURE): register_batch dispatches on the registration
type like cloudRegistrationFactory (src/CloudRegistration.cpp:85-100), the counterpart of slam.DeviceBackend.register_batch, and the
overlap accepts maps without normals (a point-to-point mapper's), which only the point-to-point estimator can register."""
from __future__ import annotations

from oracle import oracle as O
from oracle_backend import OracleCloud
from oracle_backend_ransac import RansacOracleBackend


class EstimatorOracleBackend(RansacOracleBackend):
    def overlap(self, source, target, T0, voxel, min_pts):
        fs, ft = O.overlap_flags(source.xyz, target.xyz, T0, voxel, min_pts)
        sel = lambda nrm, f: None if nrm is None else nrm[f]
        return OracleCloud(source.xyz[fs], sel(source.nrm, fs)), OracleCloud(target.xyz[ft], sel(target.nrm, ft))

    def register_batch(self, sources, targets, inits, max_corr, max_iter, regType="PointToPlaneIcp"):
        """cloudRegistrationFactory(regType)->registerClouds for every pair; generalized ICP takes both clouds' covariances from their
        normals"""
        reg = {"PointToPlaneIcp": lambda s, t, T0: O.registration_icp_p2plane(s.xyz, t.xyz, t.nrm, max_corr, T0, max_iter=max_iter),
               "PointToPointIcp": lambda s, t, T0: O.registration_icp_p2point(s.xyz, t.xyz, max_corr, T0, max_iter=max_iter),
               "GeneralizedIcp": lambda s, t, T0: O.registration_gicp(s.xyz, s.nrm, t.xyz, t.nrm, max_corr, T0, max_iter=max_iter)}
        if regType not in reg:
            raise RuntimeError("cloud: unknown type of cloud registration")
        out = []
        for s, t, T0 in zip(sources, targets, inits):
            r = reg[regType](s, t, T0)
            r.transformation_ = r.T; r.fitness_ = r.fitness; r.inlier_rmse_ = r.inlier_rmse
            out.append(r)
        return out
