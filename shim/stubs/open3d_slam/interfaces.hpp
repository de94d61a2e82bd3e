// STAND-IN declarations of the reference seam -- NOT copies of the reference headers.  They restate only the virtual
// signatures the shim overrides so that it can be type-checked without Open3D / Eigen / the reference tree:
//   CloudRegistration          include/open3d_slam/CloudRegistration.hpp:19-27
//   ScanToMapRegistration      include/open3d_slam/ScanToMapRegistration.hpp:24-38
//   parameter structs          include/open3d_slam/Parameters.hpp:51-98,118-122,148-153,172
//   Constraint                 include/open3d_slam/Constraint.hpp:14-20
// In a real build, include the reference's own headers instead (INTEGRATION.md).
#pragma once
#include <Eigen/Dense>
#include <memory>
#include <string>
#include <vector>
#include "open3d/geometry/PointCloud.h"
#include "open3d/pipelines/registration/Registration.h"
namespace o3d_slam {
using PointCloud = open3d::geometry::PointCloud;
using PointCloudPtr = std::shared_ptr<PointCloud>;
using Transform = Eigen::Isometry3d;
using RegistrationResult = open3d::pipelines::registration::RegistrationResult;
struct ScanCroppingParameters { double croppingMinZ_ = -10, croppingMaxZ_ = 10, croppingMinRadius_ = 0, croppingMaxRadius_ = 20; std::string cropperName_ = "MaxRadius"; };
struct ScanProcessingParameters { double downSamplingRatio_ = 1.0, voxelSize_ = 0.03; ScanCroppingParameters cropper_; };
struct IcpParameters { int maxNumIter_ = 50; double maxCorrespondenceDistance_ = 0.2; int knn_ = 5; double maxDistanceKnn_ = 10.0; };
struct CloudRegistrationParameters { IcpParameters icp_; };
struct SpaceCarvingParameters { double voxelSize_ = 0.1, maxRaytracingLength_ = 20.0, truncationDistance_ = 0.1; int carveSpaceEveryNscans_ = 10; double minDotProductWithNormal_ = 0.5, neighborhoodRadiusDenseMap_ = 0.1; };
struct MapBuilderParameters { double mapVoxelSize_ = 0.03; ScanCroppingParameters cropper_; SpaceCarvingParameters carving_; };
enum class ScanToMapRegistrationType : int { PointToPlaneIcp, PointToPointIcp, GeneralizedIcp };   // Parameters.hpp:44-49
struct ScanToMapRegistrationParameters { double minRefinementFitness_ = 0.7; IcpParameters icp_; ScanToMapRegistrationType scanToMapRegType_ = ScanToMapRegistrationType::PointToPlaneIcp; };
struct PlaceRecognitionParameters { double normalEstimationRadius_ = 1.0, featureVoxelSize_ = 0.5, featureRadius_ = 2.5; int featureKnn_ = 100, normalKnn_ = 10;
  int ransacNumIter_ = 1000000; double ransacProbability_ = 0.99; int ransacModelSize_ = 3; double ransacMaxCorrespondenceDistance_ = 0.75,
  correspondenceCheckerDistance_ = 0.75, correspondenceCheckerEdgeLength_ = 0.5; int ransacMinCorrespondenceSetSize_ = 25; };   // Parameters.hpp:118-129
struct MapperParameters { ScanToMapRegistrationParameters scanMatcher_; ScanProcessingParameters scanProcessing_; MapBuilderParameters mapBuilder_; MapBuilderParameters denseMapBuilder_;
  bool isRefineOdometryConstraintsBetweenSubmaps_ = false; };
struct Constraint { Transform sourceToTarget_ = Transform::Identity(); size_t sourceSubmapIdx_ = 0, targetSubmapIdx_ = 0;
  Eigen::Matrix6d informationMatrix_ = Eigen::Matrix6d::Identity(); bool isInformationMatrixValid_ = false, isOdometryConstraint_ = false; };
using Constraints = std::vector<Constraint>;
class Submap;  // the shim only needs getMapPointCloud(); see b2s_open3d_slam.cpp
class CloudRegistration {
 public:
  virtual ~CloudRegistration() = default;
  virtual RegistrationResult registerClouds(const PointCloud& source, const PointCloud& target, const Transform& init) const = 0;
  virtual void estimateNormalsOrCovariancesIfNeeded(PointCloud* cloud) const {}
};
struct ProcessedScans { PointCloudPtr merge_; PointCloudPtr match_; };
class ScanToMapRegistration {
 public:
  virtual ~ScanToMapRegistration() = default;
  virtual ProcessedScans processForScanMatchingAndMerging(const PointCloud& in, const Transform& mapToRangeSensor) const = 0;
  virtual RegistrationResult scanToMapRegistration(const PointCloud& scan, const Submap& activeSubmap, const Transform& mapToRangeSensor,
                                                   const Transform& initialGuess) const = 0;
  virtual bool isMergeScanValid(const PointCloud& in) const = 0;
  virtual void prepareInitialMap(PointCloud* map) const = 0;
};
const PointCloud& getMapPointCloudOf(const Submap& submap);  // = submap.getMapPointCloud() (Submap.hpp:45)
}  // namespace o3d_slam
