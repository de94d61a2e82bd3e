// b2s_open3d_slam.cpp -- see b2s_open3d_slam.hpp.  Everything here is marshalling: AoS fp64 host vectors <-> the C ABI.
#include "b2s_open3d_slam.hpp"

#include <cstring>
#include <stdexcept>
#include <string>

namespace o3d_slam {

namespace {
void toRowMajor(const Eigen::Matrix4d& m, double out[16]) {
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) out[4 * r + c] = m(r, c);   // Eigen is column-major: copy element-wise
}
RegistrationResult toResult(const b2s_result& r) {
  RegistrationResult out;
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) out.transformation_(i, j) = r.T[4 * i + j];
  out.fitness_ = r.fitness;
  out.inlier_rmse_ = r.inlier_rmse;
  return out;
}
int32_t cropperKind(const std::string& name) {   // croppers.hpp cropperNames
  if (name == "Cylinder") return B2S_CROP_CYLINDER;
  if (name == "MinRadius") return B2S_CROP_MIN_RADIUS;
  if (name == "MaxRadius") return B2S_CROP_MAX_RADIUS;
  if (name == "MinMaxRadius") return B2S_CROP_MINMAX_RADIUS;
  throw std::runtime_error("Unknown cropper type");
}
b2s_cropper toCropper(const ScanCroppingParameters& p) {
  b2s_cropper c;
  std::memset(&c, 0, sizeof(c));
  c.kind = cropperKind(p.cropperName_);
  c.rmin = p.croppingMinRadius_; c.rmax = p.croppingMaxRadius_; c.zmin = p.croppingMinZ_; c.zmax = p.croppingMaxZ_;
  return c;
}
struct DeviceCloud {   // RAII wrapper of a b2s_cloud uploaded from a reference PointCloud
  b2s_handle* h; b2s_cloud* c = nullptr;
  DeviceCloud(b2s_handle* h_, const PointCloud& pc, bool withNormals) : h(h_) {
    int32_t rc = b2s_cloud_create(h, &c);
    if (rc != B2S_OK) b2sThrow(rc);
    const double* xyz = pc.points_.empty() ? nullptr : pc.points_.front().data();
    const double* nrm = (withNormals && pc.HasNormals()) ? pc.normals_.front().data() : nullptr;
    rc = b2s_cloud_upload_f64(h, c, xyz, nrm, pc.points_.size());
    if (rc != B2S_OK) { b2s_cloud_destroy(c); b2sThrow(rc); }
  }
  explicit DeviceCloud(b2s_handle* h_) : h(h_) { int32_t rc = b2s_cloud_create(h, &c); if (rc != B2S_OK) b2sThrow(rc); }
  ~DeviceCloud() { b2s_cloud_destroy(c); }
  PointCloudPtr download() const {
    size_t n = 0; int32_t hasN = 0;
    int32_t rc = b2s_cloud_size(h, c, &n, &hasN);
    if (rc != B2S_OK) b2sThrow(rc);
    auto out = std::make_shared<PointCloud>();
    out->points_.resize(n);
    if (hasN) out->normals_.resize(n);
    rc = b2s_cloud_download(h, c, n ? out->points_.front().data() : nullptr, (hasN && n) ? out->normals_.front().data() : nullptr, n, &n);
    if (rc != B2S_OK) b2sThrow(rc);
    return out;
  }
};
}  // namespace

void b2sThrow(int32_t code) { throw std::runtime_error(std::string("b2s error ") + std::to_string(code) + ": " + b2s_last_error()); }

b2s_config b2sConfigFrom(const IcpParameters& icp, const ScanProcessingParameters* scan, const MapBuilderParameters* mapBuilder) {
  b2s_config cfg;
  b2s_default_config(&cfg);
  cfg.icp.reg_type = B2S_REG_POINT_TO_PLANE;
  cfg.icp.max_iter = icp.maxNumIter_;                       // src/CloudRegistration.cpp:63
  cfg.icp.max_corr_dist = icp.maxCorrespondenceDistance_;   // :60
  cfg.icp.knn = icp.knn_;                                   // :61
  cfg.icp.knn_radius = icp.maxDistanceKnn_;                 // :62
  if (scan) {
    cfg.scan.voxel_size = scan->voxelSize_;
    cfg.scan.downsampling_ratio = scan->downSamplingRatio_;
    cfg.scan.scan_matcher_cropper = toCropper(scan->cropper_);   // src/ScanToMapRegistration.cpp:31
  }
  if (mapBuilder) {
    cfg.map_voxel_size = mapBuilder->mapVoxelSize_;
    cfg.scan.map_builder_cropper = toCropper(mapBuilder->cropper_);   // src/ScanToMapRegistration.cpp:30
  }
  return cfg;
}

b2s_handle* b2sThreadHandle(const b2s_config& cfg) {
  struct Holder { b2s_handle* h = nullptr; ~Holder() { b2s_destroy(h); } };
  thread_local Holder holder;
  if (!holder.h) {
    int32_t rc = b2s_create(&cfg, 0, nullptr, &holder.h);
    if (rc != B2S_OK) b2sThrow(rc);
  } else {
    int32_t rc = b2s_set_config(holder.h, &cfg);
    if (rc != B2S_OK) b2sThrow(rc);
  }
  return holder.h;
}

RegistrationIcpPointToPlaneB200::RegistrationIcpPointToPlaneB200(const CloudRegistrationParameters& p) : cfg_(b2sConfigFrom(p.icp_, nullptr, nullptr)) {}

RegistrationResult RegistrationIcpPointToPlaneB200::registerClouds(const PointCloud& source, const PointCloud& target, const Transform& init) const {
  b2s_handle* h = b2sThreadHandle(cfg_);
  double T0[16];
  toRowMajor(init.matrix(), T0);
  b2s_result r;
  const double* tn = target.HasNormals() ? target.normals_.front().data() : nullptr;   // nullptr -> B2S_E_NO_NORMALS, like [O3D] LogError
  int32_t rc = b2s_register_host(h, source.points_.empty() ? nullptr : source.points_.front().data(), source.points_.size(),
                                 target.points_.empty() ? nullptr : target.points_.front().data(), tn, target.points_.size(), T0, &r);
  if (rc != B2S_OK) b2sThrow(rc);
  return toResult(r);
}

void RegistrationIcpPointToPlaneB200::estimateNormalsOrCovariancesIfNeeded(PointCloud* cloud) const {
  b2s_handle* h = b2sThreadHandle(cfg_);
  DeviceCloud d(h, *cloud, false);
  int32_t rc = b2s_estimate_normals(h, d.c, cfg_.icp.knn, cfg_.icp.knn_radius);   // asserts radius > 0, knn > 0 like :50-51
  if (rc != B2S_OK) b2sThrow(rc);
  cloud->normals_ = d.download()->normals_;
}

RegistrationIcpPointToPointB200::RegistrationIcpPointToPointB200(const CloudRegistrationParameters& p) : cfg_(b2sConfigFrom(p.icp_, nullptr, nullptr)) {
  cfg_.icp.reg_type = B2S_REG_POINT_TO_POINT;
}

RegistrationResult RegistrationIcpPointToPointB200::registerClouds(const PointCloud& source, const PointCloud& target, const Transform& init) const {
  b2s_handle* h = b2sThreadHandle(cfg_);
  double T0[16];
  toRowMajor(init.matrix(), T0);
  b2s_result r;
  int32_t rc = b2s_register_host(h, source.points_.empty() ? nullptr : source.points_.front().data(), source.points_.size(),
                                 target.points_.empty() ? nullptr : target.points_.front().data(), nullptr, target.points_.size(), T0, &r);
  if (rc != B2S_OK) b2sThrow(rc);
  return toResult(r);
}

RegistrationIcpGeneralizedB200::RegistrationIcpGeneralizedB200(const CloudRegistrationParameters& p) : cfg_(b2sConfigFrom(p.icp_, nullptr, nullptr)) {
  cfg_.icp.reg_type = B2S_REG_GENERALIZED;
}

RegistrationResult RegistrationIcpGeneralizedB200::registerClouds(const PointCloud& source, const PointCloud& target, const Transform& init) const {
  b2s_handle* h = b2sThreadHandle(cfg_);
  DeviceCloud ds(h, source, true), dt(h, target, true);   // both with normals: the covariances are derived from them on the device
  double T0[16];
  toRowMajor(init.matrix(), T0);
  b2s_result r;
  int32_t rc = b2s_register(h, ds.c, dt.c, T0, &r);
  if (rc != B2S_OK) b2sThrow(rc);
  return toResult(r);
}

void RegistrationIcpGeneralizedB200::estimateNormalsOrCovariancesIfNeeded(PointCloud* cloud) const {
  b2s_handle* h = b2sThreadHandle(cfg_);
  DeviceCloud d(h, *cloud, false);
  int32_t rc = b2s_estimate_normals(h, d.c, cfg_.icp.knn, cfg_.icp.knn_radius);   // src/CloudRegistration.cpp:21-30
  if (rc != B2S_OK) b2sThrow(rc);
  cloud->normals_ = d.download()->normals_;
}

void carveB200(const PointCloud& rawScan, const Transform& mapToRangeSensor, const Transform& cropperPose, const MapBuilderParameters& p,
               PointCloud* map) {
  if (map->points_.empty()) return;   // Submap.cpp:111
  IcpParameters unused;
  b2s_config cfg = b2sConfigFrom(unused, nullptr, &p);
  b2s_handle* h = b2sThreadHandle(cfg);
  DeviceCloud raw(h, rawScan, false), dmap(h, *map, true);
  b2s_submap* sm = nullptr;
  int32_t rc = b2s_submap_create(h, map->points_.size() + 1, &sm);
  if (rc != B2S_OK) b2sThrow(rc);
  rc = b2s_submap_set_cloud(h, sm, dmap.c);
  double Ts[16], Tc[16];
  toRowMajor(mapToRangeSensor.matrix(), Ts);
  toRowMajor(cropperPose.matrix(), Tc);
  const b2s_carving_params prm = {p.carving_.voxelSize_, p.carving_.maxRaytracingLength_, p.carving_.truncationDistance_,
                                  p.carving_.minDotProductWithNormal_, p.carving_.neighborhoodRadiusDenseMap_};
  size_t removed = 0;
  if (rc == B2S_OK) rc = b2s_submap_carve(h, sm, raw.c, Ts, Tc, &prm, &removed);
  size_t n = 0;
  if (rc == B2S_OK) rc = b2s_submap_size(h, sm, &n);
  if (rc == B2S_OK) {
    map->points_.resize(n);
    if (map->HasNormals() || n == 0) map->normals_.resize(n);
    rc = b2s_submap_download(h, sm, n ? map->points_.front().data() : nullptr, (n && !map->normals_.empty()) ? map->normals_.front().data() : nullptr, n, &n);
  }
  b2s_submap_destroy(sm);
  if (rc != B2S_OK) b2sThrow(rc);
}

ScanToMapIcpB200::ScanToMapIcpB200(const MapperParameters& p) : cfg_(b2sConfigFrom(p.scanMatcher_.icp_, &p.scanProcessing_, &p.mapBuilder_)) {
  switch (p.scanMatcher_.scanToMapRegType_) {   // toCloudRegistrationType, src/ScanToMapRegistration.cpp:105-129
    case ScanToMapRegistrationType::PointToPointIcp: cfg_.icp.reg_type = B2S_REG_POINT_TO_POINT; break;
    case ScanToMapRegistrationType::GeneralizedIcp: cfg_.icp.reg_type = B2S_REG_GENERALIZED; break;
    default: cfg_.icp.reg_type = B2S_REG_POINT_TO_PLANE; break;
  }
}

ProcessedScans ScanToMapIcpB200::processForScanMatchingAndMerging(const PointCloud& in, const Transform&) const {
  b2s_handle* h = b2sThreadHandle(cfg_);
  DeviceCloud raw(h, in, false), merge(h), match(h);
  int32_t rc = b2s_process_scan(h, raw.c, merge.c, match.c);
  if (rc == B2S_OK) rc = b2s_synchronize(h);     // B2S_E_EMPTY here == the reference's assert_gt on the cropped sizes (:51-52)
  if (rc != B2S_OK) b2sThrow(rc);
  ProcessedScans out;
  out.merge_ = merge.download();
  out.match_ = match.download();
  return out;
}

RegistrationResult ScanToMapIcpB200::scanToMapRegistration(const PointCloud& scan, const Submap& activeSubmap, const Transform& mapToRangeSensor,
                                                           const Transform& initialGuess) const {
  // Host-resident submap variant: the map cloud is uploaded per call.  With the device-resident b2s_submap
  // (b2s_submap_insert / b2s_register_to_submap) the upload disappears; that needs Submap to own a b2s_submap* (INTEGRATION.md).
  b2s_handle* h = b2sThreadHandle(cfg_);
#ifdef B2S_SHIM_STANDALONE_CHECK
  const PointCloud& map = getMapPointCloudOf(activeSubmap);
#else
  const PointCloud& map = activeSubmap.getMapPointCloud();
#endif
  // the scan goes up WITH its normals when it has them: the generalized estimator derives the source covariances from them
  // ([O3D] InitializePointCloudForGeneralizedICP), exactly the match_ normals the reference's own preprocess left on the cloud
  DeviceCloud dscan(h, scan, true), dmap(h, map, true);
  b2s_submap* sm = nullptr;
  int32_t rc = b2s_submap_create(h, map.points_.size() + 1, &sm);
  if (rc != B2S_OK) b2sThrow(rc);
  rc = b2s_submap_set_cloud(h, sm, dmap.c);   // a map without normals is accepted for PointToPointIcp only (like the reference)
  double Ts[16], Tg[16];
  toRowMajor(mapToRangeSensor.matrix(), Ts);
  toRowMajor(initialGuess.matrix(), Tg);
  b2s_result r;
  if (rc == B2S_OK) rc = b2s_register_to_submap(h, dscan.c, sm, Ts, Tg, &r);   // B2S_E_EMPTY == "map patch size is zero" (:60)
  b2s_submap_destroy(sm);
  if (rc != B2S_OK) b2sThrow(rc);
  return toResult(r);
}

RegistrationResult ScanToMapIcpB200::scanToMapRegistration(const PointCloud& scan, const SubmapB200& activeSubmap, const Transform& mapToRangeSensor,
                                                           const Transform& initialGuess) const {
  b2s_handle* h = activeSubmap.engine();   // the submap's own handle: the map never leaves the device
  int32_t rc = b2s_set_config(h, &cfg_);
  if (rc != B2S_OK) b2sThrow(rc);
  DeviceCloud dscan(h, scan, true);
  double Ts[16], Tg[16];
  toRowMajor(mapToRangeSensor.matrix(), Ts);
  toRowMajor(initialGuess.matrix(), Tg);
  b2s_result r;
  rc = b2s_register_to_submap(h, dscan.c, activeSubmap.handle(), Ts, Tg, &r);   // B2S_E_EMPTY == "map patch size is zero" (:60)
  if (rc != B2S_OK) b2sThrow(rc);
  return toResult(r);
}

// ---- SubmapB200 -----------------------------------------------------------------------------------------------------------
SubmapB200::SubmapB200(const MapperParameters& p, size_t capacityPoints)
    : cfg_(b2sConfigFrom(p.scanMatcher_.icp_, &p.scanProcessing_, &p.mapBuilder_)), mapBuilder_(p.mapBuilder_), denseMapBuilder_(p.denseMapBuilder_) {
  cfg_.dense_voxel_size = p.denseMapBuilder_.mapVoxelSize_;
  switch (p.scanMatcher_.scanToMapRegType_) {
    case ScanToMapRegistrationType::PointToPointIcp: cfg_.icp.reg_type = B2S_REG_POINT_TO_POINT; break;
    case ScanToMapRegistrationType::GeneralizedIcp: cfg_.icp.reg_type = B2S_REG_GENERALIZED; break;
    default: cfg_.icp.reg_type = B2S_REG_POINT_TO_PLANE; break;
  }
  h_ = b2sThreadHandle(cfg_);
  const int32_t rc = b2s_submap_create(h_, capacityPoints, &sm_);
  if (rc != B2S_OK) b2sThrow(rc);
}

SubmapB200::~SubmapB200() {
  b2s_feature_destroy(feature_);
  b2s_cloud_destroy(sparse_);
  b2s_submap_destroy(sm_);
}

bool SubmapB200::insertScan(const PointCloud& rawScan, const PointCloud& preProcessedScan, const Transform& mapToRangeSensor, bool isPerformCarving) {
  if (preProcessedScan.IsEmpty()) return true;   // Submap.cpp:41-43
  double Ts[16], Tc[16];
  toRowMajor(mapToRangeSensor.matrix(), Ts);
  int32_t rc = B2S_OK;
  if (isPerformCarving && nScansInsertedMap_ % static_cast<size_t>(mapBuilder_.carving_.carveSpaceEveryNscans_) == 1 && !isEmpty()) {   // Submap.cpp:111
    DeviceCloud raw(h_, rawScan, false);
    toRowMajor(cropperPose_.matrix(), Tc);
    const b2s_carving_params prm = {mapBuilder_.carving_.voxelSize_, mapBuilder_.carving_.maxRaytracingLength_, mapBuilder_.carving_.truncationDistance_,
                                    mapBuilder_.carving_.minDotProductWithNormal_, mapBuilder_.carving_.neighborhoodRadiusDenseMap_};
    rc = b2s_submap_carve(h_, sm_, raw.c, Ts, Tc, &prm, nullptr);
    if (rc != B2S_OK) b2sThrow(rc);
  }
  DeviceCloud scan(h_, preProcessedScan, true);
  rc = b2s_submap_insert(h_, sm_, scan.c, Ts);   // transform (duplication quirk kept), append, voxelizeWithinCroppingVolume
  if (rc != B2S_OK) b2sThrow(rc);
  cropperPose_ = mapToRangeSensor;
  ++nScansInsertedMap_;
  cacheValid_ = false;
  return true;
}

bool SubmapB200::insertScanDenseMap(const PointCloud& rawScan, const Transform& mapToRangeSensor, bool isPerformCarving) {
  DeviceCloud raw(h_, rawScan, false);
  double Ts[16];
  toRowMajor(mapToRangeSensor.matrix(), Ts);
  const b2s_cropper crop = toCropper(denseMapBuilder_.cropper_);
  int32_t rc = b2s_submap_insert_dense(h_, sm_, raw.c, Ts, &crop);
  if (rc != B2S_OK) b2sThrow(rc);
  if (isPerformCarving && nScansInsertedDenseMap_ % static_cast<size_t>(denseMapBuilder_.carving_.carveSpaceEveryNscans_) == 1) {   // Submap.cpp:127
    const double sensor[3] = {mapToRangeSensor.matrix()(0, 3), mapToRangeSensor.matrix()(1, 3), mapToRangeSensor.matrix()(2, 3)};   // .translation()
    const b2s_carving_params prm = {denseMapBuilder_.carving_.voxelSize_, denseMapBuilder_.carving_.maxRaytracingLength_,
                                    denseMapBuilder_.carving_.truncationDistance_, denseMapBuilder_.carving_.minDotProductWithNormal_,
                                    denseMapBuilder_.carving_.neighborhoodRadiusDenseMap_};
    rc = b2s_dense_carve(h_, sm_, raw.c, sensor, &prm, nullptr);   // the reference hands over the RAW scan with the map-frame position (:88)
    if (rc != B2S_OK) b2sThrow(rc);
  }
  ++nScansInsertedDenseMap_;
  return true;
}

void SubmapB200::transform(const Transform& T) {
  double Tm[16];
  toRowMajor(T.matrix(), Tm);
  const int32_t rc = b2s_submap_transform(h_, sm_, Tm);
  if (rc != B2S_OK) b2sThrow(rc);
  cacheValid_ = false;
}

bool SubmapB200::isEmpty() const {
  size_t n = 0;
  const int32_t rc = b2s_submap_size(h_, sm_, &n);
  if (rc != B2S_OK) b2sThrow(rc);
  return n == 0;
}

const PointCloud& SubmapB200::getMapPointCloud() const {
  if (!cacheValid_) {   // ROS publishers, saving and place recognition read the map a few times per second at most
    size_t n = 0;
    int32_t rc = b2s_submap_size(h_, sm_, &n);
    if (rc != B2S_OK) b2sThrow(rc);
    cache_.points_.resize(n);
    cache_.normals_.resize(n);
    rc = b2s_submap_download(h_, sm_, n ? cache_.points_.front().data() : nullptr, n ? cache_.normals_.front().data() : nullptr, n, &n);
    if (rc != B2S_OK) b2sThrow(rc);
    cacheValid_ = true;
  }
  return cache_;
}

void SubmapB200::setMapPointCloud(const PointCloud& cloud) {
  DeviceCloud d(h_, cloud, true);
  const int32_t rc = b2s_submap_set_cloud(h_, sm_, d.c);
  if (rc != B2S_OK) b2sThrow(rc);
  cacheValid_ = false;
}

void SubmapB200::setMergeScans(bool on) {   // Mapper.cpp:163-167; off also keeps the static patch table (b2s.h)
  const int32_t rc = b2s_submap_set_merge_scans(h_, sm_, on ? 1 : 0);
  if (rc != B2S_OK) b2sThrow(rc);
}

void SubmapB200::computeFeatures(const PlaceRecognitionParameters& p) {
  int32_t rc = B2S_OK;
  if (!sparse_ && (rc = b2s_cloud_create(h_, &sparse_)) != B2S_OK) b2sThrow(rc);
  if (!feature_ && (rc = b2s_feature_create(h_, &feature_)) != B2S_OK) b2sThrow(rc);
  b2s_feature_params fp;
  b2s_default_feature_params(&fp);
  fp.feature_voxel_size = p.featureVoxelSize_;              // src/Submap.cpp:241
  fp.normal_estimation_radius = p.normalEstimationRadius_;  // :242
  fp.normal_knn = p.normalKnn_;
  fp.feature_radius = p.featureRadius_;                     // :245
  fp.feature_knn = p.featureKnn_;
  rc = b2s_submap_compute_features(h_, sm_, &fp, sparse_, feature_);
  if (rc != B2S_OK) b2sThrow(rc);
  sparseValid_ = featureValid_ = false;
}

const PointCloud& SubmapB200::getSparseMapPointCloud() const {
  if (sparse_ && !sparseValid_) {   // before the first computeFeatures: the empty default cloud, like the reference's member
    size_t n = 0;
    int32_t hasN = 0;
    int32_t rc = b2s_cloud_size(h_, sparse_, &n, &hasN);
    if (rc != B2S_OK) b2sThrow(rc);
    sparseCache_.points_.resize(n);
    sparseCache_.normals_.resize(hasN ? n : 0);
    rc = b2s_cloud_download(h_, sparse_, n ? sparseCache_.points_.front().data() : nullptr, (hasN && n) ? sparseCache_.normals_.front().data() : nullptr,
                            n, &n);
    if (rc != B2S_OK) b2sThrow(rc);
    sparseValid_ = true;
  }
  return sparseCache_;
}

const SubmapB200::Feature& SubmapB200::getFeatures() const {
  if (!feature_) throw std::runtime_error("Feature ptr is nullptr");   // src/Submap.cpp:250 assert_nonNullptr
  if (!featureValid_) {
    size_t n = 0;
    int32_t rc = b2s_feature_size(h_, feature_, &n);
    if (rc != B2S_OK) b2sThrow(rc);
    featureCache_.Resize(B2S_FEATURE_DIM, (int)n);   // data_ is column-major: point after point, the ABI's layout
    rc = b2s_feature_download(h_, feature_, n ? featureCache_.data_.data() : nullptr, n, &n);
    if (rc != B2S_OK) b2sThrow(rc);
    featureValid_ = true;
  }
  return featureCache_;
}

void ScanToMapIcpB200::prepareInitialMap(PointCloud* map) const {
  b2s_handle* h = b2sThreadHandle(cfg_);
  DeviceCloud d(h, *map, false);
  int32_t rc = b2s_estimate_normals(h, d.c, cfg_.icp.knn, cfg_.icp.knn_radius);
  if (rc != B2S_OK) b2sThrow(rc);
  map->normals_ = d.download()->normals_;
}

RansacResultB200 registrationRansacBasedOnFeatureMatchingB200(const SubmapB200& source, const SubmapB200& target,
                                                              const PlaceRecognitionParameters& cfg, uint64_t seed) {
  if (!source.feature() || !target.feature()) throw std::runtime_error("Feature ptr is nullptr");   // Submap.cpp:250
  b2s_ransac_params rp;
  b2s_default_ransac_params(&rp);
  rp.mutual_filter = 1;                                                   // PlaceRecognition.cpp:82
  rp.ransac_n = cfg.ransacModelSize_;
  rp.max_correspondence_distance = cfg.ransacMaxCorrespondenceDistance_;
  rp.checker_distance = cfg.correspondenceCheckerDistance_;               // :56-57
  rp.checker_edge_length = cfg.correspondenceCheckerEdgeLength_;
  rp.max_iteration = cfg.ransacNumIter_;
  rp.confidence = cfg.ransacProbability_;
  rp.seed = seed;
  const b2s_cloud* tc = target.sparseCloud();
  const b2s_feature* tf = target.feature();
  b2s_ransac_result r;
  const int32_t rc = b2s_ransac_feature_matching(source.engine(), source.sparseCloud(), source.feature(), 1, &tc, &tf, &rp, &r);
  if (rc != B2S_OK) b2sThrow(rc);
  RansacResultB200 out;
  out.result = toResult(r.result);
  out.numCorrespondences = (size_t)r.result.n_corr;
  return out;
}

void computeOdometryConstraintsB200(const std::vector<const SubmapB200*>& submaps, const std::vector<size_t>& parentIds, size_t activeSubmapIdx,
                                    const std::vector<size_t>* candidates, const MapperParameters& p, Constraints* constraints) {
  auto has = [&](size_t s, size_t t) {   // hasConstraint (:23-30), the pairs of this call included
    for (const Constraint& c : *constraints) if (c.sourceSubmapIdx_ == s && c.targetSubmapIdx_ == t) return true;
    return false;
  };
  std::vector<std::pair<size_t, size_t>> pairs;
  auto consider = [&](size_t t, bool skipActive) {
    if (t < 1) return;
    const size_t s = parentIds.at(t);
    if (skipActive && (s == activeSubmapIdx || t == activeSubmapIdx)) return;
    for (const auto& q : pairs) if (q.first == s && q.second == t) return;
    if (!has(s, t)) pairs.emplace_back(s, t);
  };
  if (candidates) { for (size_t t : *candidates) consider(t, false); }
  else { for (size_t t = 1; t < submaps.size(); ++t) consider(t, true); }
  if (pairs.empty()) return;
  std::vector<const b2s_submap*> src, tgt;
  for (const auto& q : pairs) { src.push_back(submaps.at(q.first)->handle()); tgt.push_back(submaps.at(q.second)->handle()); }
  b2s_odometry_constraint_params prm;
  b2s_default_odometry_constraint_params(&prm);
  prm.map_voxel_size = p.mapBuilder_.mapVoxelSize_;                        // getMapVoxelSize is applied by the call
  prm.refine = p.isRefineOdometryConstraintsBetweenSubmaps_ ? 1 : 0;
  std::vector<b2s_odometry_constraint> out(pairs.size());
  const int32_t rc = b2s_submap_odometry_constraints(submaps.at(pairs.front().second)->engine(), (int32_t)pairs.size(), src.data(), tgt.data(), &prm,
                                                     nullptr, nullptr, out.data());
  if (rc != B2S_OK) b2sThrow(rc);
  for (size_t k = 0; k < pairs.size(); ++k) {
    Constraint c;
    c.sourceSubmapIdx_ = pairs[k].first;
    c.targetSubmapIdx_ = pairs[k].second;
    for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) c.sourceToTarget_.matrix()(i, j) = out[k].T[4 * i + j];
    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) c.informationMatrix_(i, j) = out[k].information[6 * i + j];
    c.isInformationMatrixValid_ = true;
    c.isOdometryConstraint_ = true;
    constraints->push_back(c);
  }
}

}  // namespace o3d_slam
