// STAND-IN for open3d::pipelines::registration::Feature: the data_ matrix (Dimension() x Num(), column-major) and its accessors.
#pragma once
#include <Eigen/Dense>
#include <cstddef>
namespace open3d { namespace pipelines { namespace registration {
class Feature {
 public:
  void Resize(int dim, int n) { data_.resize(dim, n); }
  size_t Dimension() const { return (size_t)data_.rows(); }
  size_t Num() const { return (size_t)data_.cols(); }
  Eigen::MatrixXd data_;
};
}}}  // namespace
