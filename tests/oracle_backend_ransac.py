"""The oracle backend with the loop-closure proposal (TEST INFRASTRUCTURE): ransac = the C restatement of tests/oracle_ransac.c, one
candidate after the other, the counterpart of slam.DeviceBackend.ransac under slam.buildLoopClosureConstraints.  Features are
(n, 33) arrays, sparse clouds OracleClouds, as FeatureOracleBackend.compute_features returns them."""
from __future__ import annotations

import numpy as np

import oracle_ransac as OR
from oracle_backend_features import FeatureOracleBackend
from open3d_slam_b200 import engine as E


class RansacOracleBackend(FeatureOracleBackend):
    def ransac(self, source_sparse, source_feature, target_sparses, target_features, params: E.PlaceRecognitionParameters):
        out = []
        for ts, tf in zip(target_sparses, target_features):
            r = OR.ransac(source_sparse.xyz, np.asarray(source_feature), ts.xyz, np.asarray(tf), OR.Params.of(params))
            out.append(E.RansacResult(r.T, r.fitness, r.rmse, r.inliers, 0, r.hypotheses, r.validations, r.best_h, r.n_feature_corr,
                                      r.used_mutual))
        return out
