"""The oracle backend with every loop-closure step (features, RANSAC, odometry constraints, the solve and the correction) and the session
methods of slam.DeviceBackend (TEST INFRASTRUCTURE): a submap's and the mapper's state are deep copies of the oracle's numpy state, and
clouds and features travel as the arrays they are, so SegmentMapper.saveSession / loadSession run on the CPU."""
from __future__ import annotations

import copy

import numpy as np

from oracle_backend import OracleCloud
from oracle_backend_pose_graph import PoseGraphOracleBackend
from oracle_backend_ransac import RansacOracleBackend


class SessionOracleBackend(PoseGraphOracleBackend, RansacOracleBackend):
    def export_submaps(self, sms):
        if any(sm.dense is not None for sm in sms):   # oracle.DenseMap is a C table without a copy: run the session without it
            raise NotImplementedError("the oracle's dense map cannot be copied")
        return [copy.deepcopy(sm) for sm in sms]

    def import_submap(self, blob):
        return copy.deepcopy(blob)

    def export_odometry(self):
        """the oracle mapper's state outside the submaps: Mapper::mapToRangeSensorPrev_"""
        return {"pose": np.array(self.pose)}

    def import_odometry(self, blob):
        self.pose = np.array(blob["pose"])

    def cloud_arrays(self, c):
        return c.xyz.copy(), None if c.nrm is None else c.nrm.copy()

    def make_cloud(self, xyz, nrm=None):
        return OracleCloud(xyz, nrm)

    def feature_arrays(self, sparse, feature):
        return sparse.xyz.copy(), sparse.nrm.copy(), np.array(feature)

    def restore_features(self, sm, xyz, nrm, data):
        return OracleCloud(xyz, nrm), np.array(data)
