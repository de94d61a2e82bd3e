// STAND-IN for open3d::pipelines::registration::PoseGraph / PoseGraphNode / PoseGraphEdge: the fields GlobalOptimization reads and writes.
#pragma once
#include <Eigen/Dense>
#include <vector>
namespace open3d { namespace pipelines { namespace registration {
class PoseGraphNode {
 public:
  Eigen::Matrix4d pose_ = Eigen::Matrix4d::Identity();
};
class PoseGraphEdge {
 public:
  int source_node_id_ = -1, target_node_id_ = -1;
  Eigen::Matrix4d transformation_ = Eigen::Matrix4d::Identity();
  Eigen::Matrix6d information_ = Eigen::Matrix6d::Identity();
  bool uncertain_ = false;
  double confidence_ = 1.0;
};
class PoseGraph {
 public:
  std::vector<PoseGraphNode> nodes_;
  std::vector<PoseGraphEdge> edges_;
};
}}}  // namespace
