"""The oracle backend with the pose-graph optimisation and the loop-closure correction (TEST INFRASTRUCTURE): global_optimization =
[O3D] GlobalOptimization restated in numpy (tests/oracle_pose_graph.py), transform_submap = Submap::transform (src/Submap.cpp:94-107)
on the oracle's arrays, loop_closure_update = the mapper pose the next step predicts from -- the counterparts of
slam.DeviceBackend's methods under slam.loopClosureCycle."""
from __future__ import annotations

import numpy as np

import oracle_pose_graph as PG
from oracle_backend_constraints import ConstraintOracleBackend


def global_optimization(poseGraph, criteria, option, use_cholesky=False):
    """engine.globalOptimization's contract over the restatement: poseGraph updated in place, the two passes' stats returned"""
    p = PG.Params(option.max_correspondence_distance_, option.edge_prune_threshold_, option.preference_loop_closure_, option.reference_node_,
                  criteria.max_iteration_, criteria.min_relative_increment_, criteria.min_relative_residual_increment_, criteria.min_right_term_,
                  criteria.min_residual_, criteria.max_iteration_lm_, criteria.upper_scale_factor_, criteria.lower_scale_factor_)
    edges = [PG.Edge(e.source_node_id_, e.target_node_id_, np.asarray(e.transformation_), np.asarray(e.information_), bool(e.uncertain_))
             for e in poseGraph.edges_]
    poses, kept, conf, stats = PG.global_optimization([np.asarray(n.pose_) for n in poseGraph.nodes_], edges, p, use_cholesky)
    if edges and stats[0].valid:
        for n, T in zip(poseGraph.nodes_, poses):
            n.pose_ = np.array(T)
        for e, c in zip(poseGraph.edges_, conf):
            e.confidence_ = float(c)
        poseGraph.edges_ = [e for e, k in zip(poseGraph.edges_, kept) if k]
    return stats


def o3d_transform(T, xyz, nrm=None):
    """[O3D] PointCloud::Transform: points by T (homogeneous), normals by R; no duplication quirk"""
    T = np.asarray(T, dtype=np.float64)
    x = xyz @ T[:3, :3].T + T[:3, 3]
    return x, (None if nrm is None else nrm @ T[:3, :3].T)


class PoseGraphOracleBackend(ConstraintOracleBackend):
    def global_optimization(self, poseGraph, criteria, option):
        return global_optimization(poseGraph, criteria, option)

    def transform_submap(self, sm, sparse, T):
        sm.xyz, sm.nrm = o3d_transform(T, sm.xyz, sm.nrm)
        if sm.dense is not None:
            sm.dense.transform(T)
        if sparse is not None:
            sparse.xyz, sparse.nrm = o3d_transform(T, sparse.xyz, sparse.nrm)

    def loop_closure_update(self, sm, mapToRangeSensor):
        self.pose = np.array(mapToRangeSensor)
