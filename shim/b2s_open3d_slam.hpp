// b2s_open3d_slam.hpp -- the C++ subclasses a maintainer adds to open3d_slam to run the hot path on an H100 through the
// C ABI of include/b2s.h.  They implement the reference's own abstract interfaces
//     o3d_slam::CloudRegistration        (include/open3d_slam/CloudRegistration.hpp:19-27)
//     o3d_slam::ScanToMapRegistration    (include/open3d_slam/ScanToMapRegistration.hpp:29-38)
// and are selected from the reference's factories (src/CloudRegistration.cpp:85-100, src/ScanToMapRegistration.cpp:91-103)
// by one extra enum value each (INTEGRATION.md).  Host data stays in the reference's own layout
// (std::vector<Eigen::Vector3d>, 24-byte stride), which is exactly what the ABI takes.
#pragma once
#ifdef B2S_SHIM_STANDALONE_CHECK
#include "open3d_slam/interfaces.hpp"   // stand-in declarations (shim/stubs), type-check only
#else
#include "open3d_slam/CloudRegistration.hpp"
#include "open3d_slam/ScanToMapRegistration.hpp"
#include "open3d_slam/Submap.hpp"
#endif
#include <memory>
#include <mutex>
#include "b2s.h"
#include "open3d/pipelines/registration/Feature.h"

namespace o3d_slam {

// one engine handle per host thread (the reference calls registerClouds from up to three threads, SlamWrapper.cpp:228-231)
b2s_handle* b2sThreadHandle(const b2s_config& cfg);
b2s_config b2sConfigFrom(const IcpParameters& icp, const ScanProcessingParameters* scan, const MapBuilderParameters* mapBuilder);
[[noreturn]] void b2sThrow(int32_t code);   // status -> std::runtime_error, the reference's failure mode (assert.hpp:12-63)

class RegistrationIcpPointToPlaneB200 : public CloudRegistration {
 public:
  explicit RegistrationIcpPointToPlaneB200(const CloudRegistrationParameters& p);
  RegistrationResult registerClouds(const PointCloud& source, const PointCloud& target, const Transform& init) const final;
  void estimateNormalsOrCovariancesIfNeeded(PointCloud* cloud) const final;

 private:
  b2s_config cfg_;
};

// RegistrationIcpPointToPoint (src/CloudRegistration.cpp:69-82) on the device: same ICP loop, Eigen::umeyama updates
class RegistrationIcpPointToPointB200 : public CloudRegistration {
 public:
  explicit RegistrationIcpPointToPointB200(const CloudRegistrationParameters& p);
  RegistrationResult registerClouds(const PointCloud& source, const PointCloud& target, const Transform& init) const final;

 private:
  b2s_config cfg_;
};

// RegistrationIcpGeneralized (src/CloudRegistration.cpp:15-38) on the device: covariances from the normals the reference's own
// estimateNormalsOrCovariancesIfNeeded leaves on the clouds ([O3D] InitializePointCloudForGeneralizedICP, normals branch)
class RegistrationIcpGeneralizedB200 : public CloudRegistration {
 public:
  explicit RegistrationIcpGeneralizedB200(const CloudRegistrationParameters& p);
  RegistrationResult registerClouds(const PointCloud& source, const PointCloud& target, const Transform& init) const final;
  void estimateNormalsOrCovariancesIfNeeded(PointCloud* cloud) const final;

 private:
  b2s_config cfg_;
};

// Submap::carve for the sparse map (src/Submap.cpp:109-123): removes the carved points from *map in place.  cropperPose is
// the pose mapBuilderCropper_ currently holds (the previous insertion); the caller keeps the every-N-scans schedule.
void carveB200(const PointCloud& rawScan, const Transform& mapToRangeSensor, const Transform& cropperPose, const MapBuilderParameters& p,
               PointCloud* map);

// The map side of o3d_slam::Submap, device-resident: what a maintainer puts behind Submap's own methods (one member,
// `std::unique_ptr<SubmapB200> device_`, INTEGRATION.md section 4).  Same method names and argument meaning as the methods it replaces:
//     Submap::insertScan            src/Submap.cpp:39-75     (transform, carve every N insertions, append, voxelize within the cropper)
//     Submap::insertScanDenseMap    src/Submap.cpp:77-92
//     Submap::transform             src/Submap.cpp:94-107
//     Submap::getMapPointCloud      src/Submap.cpp:184-186   (download on demand, cached until the next change)
//     Submap::isEmpty               src/Submap.cpp:221-223
//     Submap::computeFeatures       src/Submap.cpp:239-244   (the feature half: sparse cloud, its normals, FPFH; the voxel map of
//                                                            the revisit check and the minSecondsBetweenFeatureComputation_
//                                                            timer stay with the caller)
//     Submap::getFeatures / getSparseMapPointCloud          (download on demand, cached until the next computeFeatures)
// The b2s_submap lives on the handle of the thread that created the SubmapB200 (the mapping thread); computeFeatures must run on
// that handle too (the reference runs it on a worker thread: hand the call to the mapping thread, or build the SubmapB200 there).
class SubmapB200 {
 public:
  using Feature = open3d::pipelines::registration::Feature;
  SubmapB200(const MapperParameters& p, size_t capacityPoints = 2000000);
  ~SubmapB200();
  SubmapB200(const SubmapB200&) = delete;
  SubmapB200& operator=(const SubmapB200&) = delete;
  bool insertScan(const PointCloud& rawScan, const PointCloud& preProcessedScan, const Transform& mapToRangeSensor, bool isPerformCarving);
  bool insertScanDenseMap(const PointCloud& rawScan, const Transform& mapToRangeSensor, bool isPerformCarving);
  void transform(const Transform& T);
  const PointCloud& getMapPointCloud() const;
  bool isEmpty() const;
  void setMapPointCloud(const PointCloud& cloud);           // initial map (SlamWrapper::setInitialMap)
  void setMergeScans(bool on);                              // isMergeScansIntoMap_ for the device chain: false = pure localisation
  void computeFeatures(const PlaceRecognitionParameters& p);
  const PointCloud& getSparseMapPointCloud() const;
  const Feature& getFeatures() const;                       // throws before the first computeFeatures, like the reference
  b2s_submap* handle() const { return sm_; }
  b2s_handle* engine() const { return h_; }
  b2s_cloud* sparseCloud() const { return sparse_; }        // device-resident sparse cloud / feature (null before computeFeatures)
  b2s_feature* feature() const { return feature_; }

 private:
  b2s_config cfg_;
  MapBuilderParameters mapBuilder_;
  MapBuilderParameters denseMapBuilder_;
  b2s_handle* h_ = nullptr;
  b2s_submap* sm_ = nullptr;
  size_t nScansInsertedMap_ = 0, nScansInsertedDenseMap_ = 0;
  Transform cropperPose_ = Transform::Identity();           // mapBuilderCropper_'s pose: set after every insertion (Submap.cpp:71)
  mutable PointCloud cache_;
  mutable bool cacheValid_ = false;
  b2s_cloud* sparse_ = nullptr;                             // sparseMapCloud_, device-resident
  b2s_feature* feature_ = nullptr;                          // feature_, device-resident
  mutable PointCloud sparseCache_;
  mutable Feature featureCache_;
  mutable bool sparseValid_ = false, featureValid_ = false;
};

// PlaceRecognition::buildLoopClosureConstraints, src/PlaceRecognition.cpp:81-84: RegistrationRANSACBasedOnFeatureMatching(
// sourceSparse, targetSparse, sourceFeature, targetFeature, true, cfg.ransacMaxCorrespondenceDistance_, PointToPoint(false),
// cfg.ransacModelSize_, {distance, edge length checkers}, RANSACConvergenceCriteria(cfg.ransacNumIter_, cfg.ransacProbability_))
// on the device, reading both SubmapB200s' device-resident sparse cloud and feature (computeFeatures must have run on both, on
// the source's handle).  The proposal is deterministic for a given seed (DESIGN.md row K-ransac).  The device keeps the inlier
// count, not the pairs: the gate at :86 reads numCorrespondences instead of correspondence_set_.size().
struct RansacResultB200 {
  RegistrationResult result;
  size_t numCorrespondences = 0;
};
RansacResultB200 registrationRansacBasedOnFeatureMatchingB200(const SubmapB200& source, const SubmapB200& target,
                                                              const PlaceRecognitionParameters& cfg, uint64_t seed = 1);

// computeOdometryConstraints (src/constraint_builders.cpp:92-118) over device-resident submaps: submaps[i] is the SubmapB200 of submap
// id i and parentIds[i] its getParentId().  candidates = the finished submap ids (the overload of SubmapCollection::computeFeatures,
// :92-106), or nullptr for every submap (the overload of SlamWrapper::loopClosureWorker, :108-118, which leaves out the pairs that touch
// activeSubmapIdx).  Submap 0 and the pairs constraints already holds are skipped; every missing (parent, child) pair is built by
// buildOdometryConstraint (:33-90) in ONE b2s_submap_odometry_constraints call on the resident maps (all SubmapB200s on one handle),
// with p.mapBuilder_.mapVoxelSize_ and p.isRefineOdometryConstraintsBetweenSubmaps_, and appended in the reference's order.
void computeOdometryConstraintsB200(const std::vector<const SubmapB200*>& submaps, const std::vector<size_t>& parentIds, size_t activeSubmapIdx,
                                    const std::vector<size_t>* candidates, const MapperParameters& p, Constraints* constraints);

class ScanToMapIcpB200 : public ScanToMapRegistration {
 public:
  explicit ScanToMapIcpB200(const MapperParameters& p);
  // device-resident variant: no upload of the map, the patch crop and the index build run on the resident cloud
  RegistrationResult scanToMapRegistration(const PointCloud& scan, const SubmapB200& activeSubmap, const Transform& mapToRangeSensor,
                                           const Transform& initialGuess) const;
  ProcessedScans processForScanMatchingAndMerging(const PointCloud& in, const Transform& mapToRangeSensor) const final;
  RegistrationResult scanToMapRegistration(const PointCloud& scan, const Submap& activeSubmap, const Transform& mapToRangeSensor,
                                           const Transform& initialGuess) const final;
  bool isMergeScanValid(const PointCloud& in) const final { return in.HasNormals(); }
  void prepareInitialMap(PointCloud* map) const final;

 private:
  b2s_config cfg_;
};

}  // namespace o3d_slam
