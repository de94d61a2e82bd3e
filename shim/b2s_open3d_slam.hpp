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
#include "open3d/pipelines/registration/PoseGraph.h"

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
  // getDenseMapCopy().toPointCloud() (src/Voxel.cpp:90-115) as SlamWrapperRos::publishDenseMap publishes it for the active submap: the
  // dense map's voxel means, no normals, no colours.  One b2s_assemble_dense_maps call and one download (DESIGN.md row A2).
  PointCloud getDenseMapPointCloud() const;
  bool isEmpty() const;
  void setMapPointCloud(const PointCloud& cloud);           // initial map (SlamWrapper::setInitialMap)
  void setMergeScans(bool on);                              // isMergeScansIntoMap_ for the device chain: false = pure localisation
  // stands in for SlamMapInitializer's marker pose: the raw scan's mapToRangeSensor in this submap's map without an initial pose
  // (b2s_submap_global_localization); the submap is left as it was.  If result.found, pass result.T to SlamWrapper::setInitialTransform.
  b2s_global_localization_result globalLocalization(const PointCloud& rawScan, const b2s_global_localization_params& params,
                                                    double minRefinementFitness) const;
  void computeFeatures(const PlaceRecognitionParameters& p);
  const PointCloud& getSparseMapPointCloud() const;
  const Feature& getFeatures() const;                       // throws before the first computeFeatures, like the reference
  // a submap whose device state is a blob of exportSubmapStatesB200 (b2s_submap_import_state, DESIGN.md row A3), on h (any handle whose
  // map voxel size is the exporter's; the blob's own capacities).  The insertion counters and the map-builder cropper's pose come from
  // the blob; a blob the library refuses throws.
  static std::unique_ptr<SubmapB200> importState(b2s_handle* h, const std::vector<uint8_t>& blob, const MapperParameters& p);
  b2s_submap* handle() const { return sm_; }
  b2s_handle* engine() const { return h_; }
  b2s_cloud* sparseCloud() const { return sparse_; }        // device-resident sparse cloud / feature (null before computeFeatures)
  b2s_feature* feature() const { return feature_; }

 private:
  SubmapB200(const MapperParameters& p, b2s_handle* h, b2s_submap* sm);   // adopts sm (importState)
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

// PlaceRecognition::buildLoopClosureConstraints, src/PlaceRecognition.cpp:96-149, for every candidate whose proposal passed the gates
// at :86 and :92: overlap of the two whole maps at the proposal (20 x getMapVoxelSize(mapBuilder_, 0.04)), ICP of the overlaps from
// the proposal with r = placeRecognition_.maxIcpCorrespondenceDistance_ and 100 iterations, the fitness gate of :118 and the
// information matrix at the ICP's T (:148-149), all candidates in ONE b2s_submap_loop_closure_refinement call on the resident maps (all
// SubmapB200s on one handle).  regType is the refinement's estimator, point-to-plane unless given; the reference uses the scan matcher's
// type (:47), so pass toCloudRegistrationType(cfg.scanMatcher_).regType_ for its behaviour (GeneralizedIcp in the shipped Lua presets).
// Point-to-plane needs normals on every target map, GeneralizedIcp on the source and every target, PointToPointIcp none; a missing
// one throws (B2S_E_NO_NORMALS).  The consistency check of the ICP's T (:124) and the Constraint record (:140-150) stay with the caller.
struct LoopClosureRefinementB200 {
  RegistrationResult icpResult;                 // :110
  Eigen::Matrix6d informationMatrix;            // :148-149, at icpResult.transformation_ (computed for every candidate)
  bool isAccepted = false;                      // !(icpResult.fitness_ < minRefinementFitness_), :118
  size_t numSourceOverlap = 0, numTargetOverlap = 0;
};
std::vector<LoopClosureRefinementB200> refineLoopClosuresB200(const SubmapB200& source, const std::vector<const SubmapB200*>& targets,
                                                              const std::vector<Transform>& initialGuesses, const MapperParameters& cfg,
                                                              CloudRegistrationType regType = CloudRegistrationType::PointToPlaneIcp);

// computeOdometryConstraints (src/constraint_builders.cpp:92-118) over device-resident submaps: submaps[i] is the SubmapB200 of submap
// id i and parentIds[i] its getParentId().  candidates = the finished submap ids (the overload of SubmapCollection::computeFeatures,
// :92-106), or nullptr for every submap (the overload of SlamWrapper::loopClosureWorker, :108-118, which leaves out the pairs that touch
// activeSubmapIdx).  Submap 0 and the pairs constraints already holds are skipped; every missing (parent, child) pair is built by
// buildOdometryConstraint (:33-90) in ONE b2s_submap_odometry_constraints call on the resident maps (all SubmapB200s on one handle),
// with p.mapBuilder_.mapVoxelSize_ and p.isRefineOdometryConstraintsBetweenSubmaps_, and appended in the reference's order.
void computeOdometryConstraintsB200(const std::vector<const SubmapB200*>& submaps, const std::vector<size_t>& parentIds, size_t activeSubmapIdx,
                                    const std::vector<size_t>* candidates, const MapperParameters& p, Constraints* constraints);

// Mapper::getAssembledMapPointCloud (src/Mapper.cpp:183-208) over device-resident submaps (all on one handle), in the order given, then
// o3d_slam::voxelize(voxelSize) (a no-op for voxelSize <= 0): SlamWrapper::saveMap passes 0, SlamWrapperRos::publishMaps
// assembledMapVoxelSize_.  One b2s_assemble_map call; points_ and normals_ (normals only when every submap that contributes a point has
// them, DESIGN.md row A1).
PointCloud getAssembledMapPointCloudB200(const std::vector<const SubmapB200*>& submaps, double voxelSize);
// assembleColoredPointCloud (ros/open3d_slam_ros/src/helpers_ros.cpp:51-70) + voxelize(voxelSize) as publishMaps runs it with
// submapVoxelSize_: points_ and colors_ (submap j in Color::getColor(j % 11 + 2)), no normals.  One b2s_assemble_colored_map call.
PointCloud assembleColoredPointCloudB200(const std::vector<const SubmapB200*>& submaps, double voxelSize);
// SubmapCollection::dumpToFile(dir, "denseSubmap", true) (src/SubmapCollection.cpp:269-283), which SlamWrapper::saveDenseSubmaps calls:
// getDenseMapCopy().toPointCloud() of every submap (all on one handle), one PointCloud per submap in the order given (empty for a submap
// whose dense map was never fed).  One b2s_assemble_dense_maps call, one download, split by its offsets; writing the PCDs stays with the
// caller, as for saveMap.
std::vector<PointCloud> getDenseSubmapPointCloudsB200(const std::vector<const SubmapB200*>& submaps);
// Session state (DESIGN.md row A3): every submap's device state as one self-contained blob, in the order given (all on one handle), for
// saving a mission next to saveMap / saveDenseSubmaps and restoring it with SubmapB200::importState.  One b2s_submaps_export_state size
// call and one fill call; writing the files stays with the caller.
std::vector<std::vector<uint8_t>> exportSubmapStatesB200(const std::vector<const SubmapB200*>& submaps);
// Relocalisation in a restored session (DESIGN.md row M4), in place of SlamMapInitializer's marker pose: the raw scan's mapToRangeSensor
// in the union of every submap (all on h) without an initial pose, each candidate refined in the submap findClosestSubmap picks for it
// from centers (Submap::getMapToSubmapCenter of each, in the same order).  One b2s_submaps_global_localization call; the submaps are
// left as they were.  If result.found, make `submap` the active one (or open a new submap there), then SlamWrapper::setInitialTransform.
struct GlobalLocalizationB200 {
  b2s_global_localization_result result;
  int submap;                                               // the winner's submap (index into the list), -1 without a candidate
};
GlobalLocalizationB200 globalLocalizationB200(b2s_handle* h, const std::vector<const SubmapB200*>& submaps,
                                              const std::vector<Eigen::Vector3d>& centers, const PointCloud& rawScan,
                                              const b2s_global_localization_params& params, double minRefinementFitness);

// OptimizationProblem::solve (src/OptimizationProblem.cpp:25-44): in place of GlobalOptimization(poseGraph_, LevenbergMarquardt, criteria,
// option) at :40, with option from params_.globalOptimization_ and [O3D]'s default GlobalOptimizationConvergenceCriteria.  One
// b2s_global_optimization call on h (any handle: the solve touches no submap; the mapping thread's, or b2sThreadHandle on the
// loop-closure worker).  Like [O3D]: the node poses are optimised in place and edges_ becomes the kept edges with the confidences the
// solve ended with; a graph that fails validation (not connected over all edges or over the certain ones) is left as it is.
void globalOptimizationB200(b2s_handle* h, open3d::pipelines::registration::PoseGraph* poseGraph, const GlobalOptimizationParameters& p);

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
