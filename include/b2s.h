/*
 * b2s.h -- C ABI of the H100-native scan-to-map registration and voxel-map fusion engine.
 *
 * This is the drop-in boundary behind open3d_slam's CloudRegistration / ScanToMapRegistration /
 * Submap interfaces.  The reference has NO C/FFI boundary today: its seam is a pair of abstract C++
 * classes plus factories (paths relative to /root/reference/open3d_slam/open3d_slam/):
 *     include/open3d_slam/CloudRegistration.hpp:19-27      CloudRegistration::registerClouds,
 *                                                          estimateNormalsOrCovariancesIfNeeded
 *     include/open3d_slam/ScanToMapRegistration.hpp:29-38  ScanToMapRegistration::processForScanMatchingAndMerging,
 *                                                          scanToMapRegistration, prepareInitialMap
 *     include/open3d_slam/Submap.hpp:38-45                 Submap::insertScan / insertScanDenseMap / getMapPointCloud
 * Each entry point below names the reference interface (file:line) it replaces.  The C++ subclasses a
 * maintainer adds on the reference side live in shim/ and are described in INTEGRATION.md.
 *
 * Conventions
 *   - plain C99, no torch / CUDA types in any signature (a CUDA stream crosses as void*).
 *   - every function returns int32_t status: B2S_OK (0) or a negative B2S_E_* code; the message of the
 *     last failure on the calling thread is available from b2s_last_error().  No exception crosses.
 *   - host point data is the reference's own memory layout: array-of-xyz doubles, 24-byte stride
 *     (std::vector<Eigen::Vector3d>, include/open3d_slam/typedefs.hpp:23), or float32 xyz with an arbitrary
 *     stride (sensor_msgs/PointCloud2 wire format, open3d_conversions.cpp:61-67).
 *   - 4x4 transforms are 16 doubles in ROW-MAJOR order (Eigen::Matrix4d is column-major: copy element-wise).
 *   - all arithmetic on the device is fp64 like the reference (ScanToMap ICP parity target 1e-4, achieved ~1e-12).
 *   - a handle owns one CUDA stream; calls on one handle are serialised by an internal mutex and are
 *     asynchronous with respect to the host unless they return data to host memory.  Use one handle per
 *     host thread for concurrency (the reference calls registerClouds from 3 threads, SlamWrapper.cpp:228-231).
 *   - the CUDA extension is the only implementation: there is no CPU fallback.
 */
#ifndef B2S_H_
#define B2S_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)   /* the library itself is built with -fvisibility=hidden */
#endif

#define B2S_OK 0
#define B2S_E_INVALID (-1)      /* bad argument (reference: assert_* / LogError -> std::runtime_error) */
#define B2S_E_CUDA (-2)         /* CUDA runtime failure */
#define B2S_E_EMPTY (-3)        /* empty cloud where the reference asserts non-empty (ScanToMapRegistration.cpp:51-52,60) */
#define B2S_E_NO_NORMALS (-4)   /* point-to-plane target without normals ([O3D] RegistrationICP LogError) */
#define B2S_E_CAPACITY (-5)     /* a fixed-capacity device structure would overflow */
#define B2S_E_UNSUPPORTED (-6)

typedef struct b2s_handle b2s_handle;
typedef struct b2s_cloud b2s_cloud;     /* device-resident point cloud: xyz (+ normals) fp64 */
typedef struct b2s_submap b2s_submap;   /* device-resident sparse map cloud (+ optional dense voxel map) */

/* CroppingVolumeEnum / croppingVolumeFactory  (src/croppers.cpp:27-51, include/open3d_slam/croppers.hpp) */
enum { B2S_CROP_NONE = 0, B2S_CROP_MAX_RADIUS = 1, B2S_CROP_MIN_RADIUS = 2, B2S_CROP_MINMAX_RADIUS = 3, B2S_CROP_CYLINDER = 4 };

/* ScanCroppingParameters (include/open3d_slam/Parameters.hpp:51-57) + the CroppingVolume state
 * (isInvertVolume_, pose_ translation; src/croppers.cpp:57-67).  Only the translation of the pose is used. */
typedef struct b2s_cropper {
  int32_t kind;
  int32_t invert;
  double rmin, rmax, zmin, zmax;
  double center[3];
} b2s_cropper;

/* CloudRegistrationType (Parameters.hpp:37).  All three estimators run on the device; GeneralizedIcp derives the per-point
 * covariances from the clouds' normals like [O3D] does when no covariances are present. */
enum { B2S_REG_POINT_TO_PLANE = 0, B2S_REG_POINT_TO_POINT = 1, B2S_REG_GENERALIZED = 2 };

/* IcpParameters + ICPConvergenceCriteria (Parameters.hpp:66-71; src/CloudRegistration.cpp:58-66; [O3D] defaults
 * relative_fitness = relative_rmse = 1e-6) */
typedef struct b2s_icp_params {
  int32_t reg_type;
  int32_t max_iter;            /* icp.max_n_iter */
  double max_corr_dist;        /* icp.max_correspondence_dist */
  int32_t knn;                 /* icp.knn            (normal estimation) */
  double knn_radius;           /* icp.max_distance_knn */
  double rel_fitness, rel_rmse;
} b2s_icp_params;

/* ScanProcessingParameters + the two croppers ScanToMapIcp holds (Parameters.hpp:59-64, ScanToMapRegistration.cpp:29-33) */
typedef struct b2s_scan_params {
  double voxel_size;           /* scan_processing.voxel_size */
  double downsampling_ratio;   /* scan_processing.downsampling_ratio */
  uint32_t seed;               /* replaces std::random_device in [O3D] RandomDownSample */
  b2s_cropper map_builder_cropper;   /* params_.mapBuilder_.cropper_  : applied to the raw scan (preprocess) */
  b2s_cropper scan_matcher_cropper;  /* params_.scanProcessing_.cropper_ : narrow crop / map patch crop */
} b2s_scan_params;

typedef struct b2s_config {
  b2s_icp_params icp;
  b2s_scan_params scan;
  double map_voxel_size;       /* map_builder.map_voxel_size (Parameters.hpp:94) */
  double dense_voxel_size;     /* dense_map_builder.map_voxel_size */
  double nn_cell_size;         /* 0 = automatic (max_corr_dist / 4) : cell edge of the nearest-neighbour grid */
  int32_t icp_cluster_ctas;    /* 0 = automatic: CTAs (= SMs) one registration may spread over: 8 suits many concurrent registrations
                                * (throughput), 16 a single stream of scans (latency); rounded down to a power of two, at most 16 */
  int32_t reserved_;
} b2s_config;

/* open3d::pipelines::registration::RegistrationResult as read by the callers
 * (src/Mapper.cpp:151-159, src/Odometry.cpp:51-72, src/PlaceRecognition.cpp:118-149) */
typedef struct b2s_result {
  double T[16];                /* transformation_ (row-major) */
  double fitness;              /* fitness_ */
  double inlier_rmse;          /* inlier_rmse_ */
  int32_t n_corr;              /* correspondence_set_.size() */
  int32_t iters;               /* ICP updates applied */
} b2s_result;

void b2s_default_config(b2s_config* cfg);   /* Lua defaults, parameter_structure_definitions.lua:52-72,102, PointToPlaneIcp */

/* ---- engine life cycle : cloudRegistrationFactory / scanToMapRegistrationFactory
 *      (src/CloudRegistration.cpp:85-100, src/ScanToMapRegistration.cpp:91-103) ------------------------------- */
int32_t b2s_create(const b2s_config* cfg, int32_t device, void* cuda_stream_or_null, b2s_handle** out);
void b2s_destroy(b2s_handle* h);
int32_t b2s_set_config(b2s_handle* h, const b2s_config* cfg);    /* ScanToMapIcp::setParameters (ScanToMapRegistration.cpp:24-27) */
int32_t b2s_synchronize(b2s_handle* h);
const char* b2s_last_error(void);
const char* b2s_version(void);
int32_t b2s_device_count(void);
/* number of kernels launched by this handle since creation ("gpu_launches" evidence for bench.py) */
int64_t b2s_launch_count(const b2s_handle* h);
/* number of CUDA graphs the per-scan chains of this handle captured since creation (b2s_mapper_graph_enable, b2s_slam_graph_enable),
 * and the LM tries of b2s_global_optimization (one capture per padded size and edge capacity): in steady state a replay adds
 * launches but no capture */
int64_t b2s_graph_capture_count(const b2s_handle* h);

/* per-kernel-group device time, CUDA events on the handle's stream (the reference prints per-stage wall times with
 * o3d_slam::Timer, src/time.cpp:35-78).  kinds: 0 icp, 1 normals, 2 radix sort, 3 NN-grid build, 4 voxel keys+means,
 * 5 fusion, 6 select, 7 crop.  b2s_profile_read synchronises, returns the sums since the last read and resets them. */
#define B2S_PROFILE_KINDS 8
int32_t b2s_profile_enable(b2s_handle* h, int32_t on);
int32_t b2s_profile_read(b2s_handle* h, double* ms_by_kind, int64_t* count_by_kind, int32_t n_kinds);
/* debug aid (1024 words): [0..255] clock64 stamps {start, search end, reduce end, solve end} x 64 evaluations of the ICP kernel (CTA 0),
 * [256..511] per-CTA phase times, [512 + 8 e + 0..3] search statistics of evaluation e < 32 (candidates scanned in phase 1, point
 * evaluations, points queued for phase 2, candidates scanned in phase 2) */
int32_t b2s_debug_icp_clocks(b2s_handle* h, int32_t enable, long long* out_1024);

/* ---- clouds (open3d::geometry::PointCloud points_/normals_) ------------------------------------------------ */
int32_t b2s_cloud_create(b2s_handle* h, b2s_cloud** out);
void b2s_cloud_destroy(b2s_cloud* c);
int32_t b2s_cloud_upload_f64(b2s_handle* h, b2s_cloud* c, const double* xyz, const double* normals_or_null, size_t n);
int32_t b2s_cloud_upload_f32(b2s_handle* h, b2s_cloud* c, const void* xyz, size_t n, size_t stride_bytes);
int32_t b2s_cloud_size(b2s_handle* h, const b2s_cloud* c, size_t* n, int32_t* has_normals);   /* synchronises */
int32_t b2s_cloud_download(b2s_handle* h, const b2s_cloud* c, double* xyz, double* normals_or_null, size_t capacity, size_t* n);
int32_t b2s_cloud_copy(b2s_handle* h, const b2s_cloud* src, b2s_cloud* dst);

/* ---- stages of the hot path (SURVEY.md section 8a row ids) ---------------------------------------------- */
/* P1  CroppingVolume::crop                                   src/croppers.cpp:76-106 */
int32_t b2s_crop(b2s_handle* h, const b2s_cloud* in, const b2s_cropper* cropper, b2s_cloud* out);
/* P2  o3d_slam::voxelize -> [O3D] VoxelDownSample             src/helpers.cpp:107-113 */
int32_t b2s_voxel_down_sample(b2s_handle* h, const b2s_cloud* in, double voxel_size, b2s_cloud* out);
/* P3  estimateNormalsOrCovariancesIfNeeded                    src/CloudRegistration.cpp:49-56 */
int32_t b2s_estimate_normals(b2s_handle* h, b2s_cloud* cloud, int32_t knn, double radius);
/* P4  [O3D] RandomDownSample (seeded)                         src/ScanToMapRegistration.cpp:39 */
int32_t b2s_random_down_sample(b2s_handle* h, const b2s_cloud* in, double ratio, uint32_t seed, b2s_cloud* out);
/* F0  o3d_slam::transform (keeps the near-identity duplication quirk)   src/helpers.cpp:273-305 */
int32_t b2s_transform(b2s_handle* h, const b2s_cloud* in, const double T[16], b2s_cloud* out);
/* S1  ScanToMapIcp::processForScanMatchingAndMerging          src/ScanToMapRegistration.cpp:42-54
 *     raw scan -> merge_ (wide) and match_ (narrow); B2S_E_EMPTY when either is empty (checked lazily, see DESIGN.md) */
int32_t b2s_process_scan(b2s_handle* h, const b2s_cloud* raw, b2s_cloud* merge, b2s_cloud* match);
/* R1  CloudRegistration::registerClouds (point-to-plane)      src/CloudRegistration.cpp:44-48 */
int32_t b2s_register(b2s_handle* h, const b2s_cloud* source, const b2s_cloud* target, const double init[16], b2s_result* out);
/* config 4: n independent registrations in one launch (PlaceRecognition.cpp:71,111 iterates them serially) */
int32_t b2s_register_batch(b2s_handle* h, int32_t n, const b2s_cloud* const* sources, const b2s_cloud* const* targets,
                           const double* inits /* n x 16 */, b2s_result* out /* n */);
/* R3  the correspondence search of [O3D] GetRegistrationResultAndCorrespondences (KDTreeFlann::SearchHybrid(q, r, 1)) on its own:
 *     for every point of `queries`, moved by T first when T is given, the index of its nearest point of `target` with d^2 < r^2
 *     (-1 = none; exact, ties -> lower index) and the squared distance (-1 when none).  The correspondence_set_ of a
 *     RegistrationResult is this call at the result's transformation.  Host arrays hold `capacity` >= query count entries. */
int32_t b2s_nearest_neighbors(b2s_handle* h, const b2s_cloud* queries, const b2s_cloud* target, double max_correspondence_distance,
                              const double T_or_null[16], int32_t* index_out, double* d2_out_or_null, size_t capacity, size_t* n_queries);
/* host-pointer convenience form of R1 used by the C++ shim: uploads, registers, returns. */
int32_t b2s_register_host(b2s_handle* h, const double* src_xyz, size_t n_src, const double* tgt_xyz, const double* tgt_normals,
                          size_t n_tgt, const double init[16], b2s_result* out);

/* ---- submap (Submap::mapCloud_ / denseMap_)   include/open3d_slam/Submap.hpp:38-45 ----------------------- */
int32_t b2s_submap_create(b2s_handle* h, size_t capacity_points, b2s_submap** out);
void b2s_submap_destroy(b2s_submap* sm);
/* Key limit of the map side.  The fusion hash, the dense map, sparse carving (map points), the overlap and the voxel map key a
 * point by k = floor(p * (1/voxel)) on the global-origin grid, packed as three 21-bit fields: |k| <= 2^20 - 2 per axis.  A point
 * with |k| >= 2^20 - 1 (about 52 km at a 0.05 m voxel, 105 km at 0.1 m) is refused: the insertion reports B2S_E_INVALID at the
 * next synchronising call, and a query reports its voxel as absent.  The ray set of dense carving (b2s_dense_carve) keys with
 * the full int32 range instead, like the reference, so a far return still casts its ray.
 *
 * F1  Submap::insertScan without carving: transform, append, voxelizeWithinCroppingVolume around the sensor
 *     src/Submap.cpp:39-75, src/helpers.cpp:115-183 */
int32_t b2s_submap_insert(b2s_handle* h, b2s_submap* sm, const b2s_cloud* preprocessed_scan, const double map_to_sensor[16]);
/* C1  Submap::carve of the sparse map (space carving)   src/Submap.cpp:55-60,109-123, src/helpers.cpp:235-271,
 *     src/Voxel.cpp:123-149.  The caller keeps the reference's schedule (nScansInsertedMap_ % carveSpaceEveryNscans_ == 1,
 *     before the scan is appended) and passes the pose the map-builder cropper was LAST set to (the previous insertion:
 *     src/Submap.cpp:59 runs before :71).  raw_scan is in the sensor frame.  n_removed may be NULL (no synchronisation). */
typedef struct b2s_carving_params {     /* SpaceCarvingParameters, include/open3d_slam/Parameters.hpp:85-92 */
  double voxel_size;                    /* voxelSize_ = 0.1 */
  double max_raytracing_length;         /* maxRaytracingLength_ = 20.0 */
  double truncation_distance;           /* truncationDistance_ = 0.1 */
  double min_dot_product_with_normal;   /* minDotProductWithNormal_ = 0.5 */
  double neighborhood_radius_dense_map; /* neighborhoodRadiusDenseMap_ = 0.1 (dense map only) */
} b2s_carving_params;
int32_t b2s_submap_carve(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const double map_to_sensor[16],
                         const double cropper_pose[16], const b2s_carving_params* params, size_t* n_removed);
/* D1  ConstantVelocityMotionCompensation::undistortInputPointCloud (src/MotionCompensation.cpp:64-139): per-point motion
 *     compensation by azimuth phase (computePhase), for the linear / angular (roll-pitch-yaw) velocity the host estimated from
 *     its pose buffer (estimateLinearAndAngularVelocity, :33-57).  in != out; the output carries no normals. */
int32_t b2s_undistort(b2s_handle* h, const b2s_cloud* in, const double linear_velocity[3], const double angular_velocity_rpy[3],
                      double scan_duration, int32_t is_spinning_clockwise, b2s_cloud* out);
/* L1  the two steps either side of the loop-closure ICP (src/PlaceRecognition.cpp:103-111,148; src/constraint_builders.cpp:54,71)
 *     computeIndicesOfOverlappingPoints + SelectByIndex   src/helpers.cpp:307-332 : the points of source / target whose
 *     voxel (edge voxel_size, source moved by source_to_target) holds >= min_points_per_voxel points of BOTH clouds, in
 *     their original order (the reference's index lists come in hash-map order; only the sets matter to its callers).
 *     [O3D] GetInformationMatrixFromPointClouds(source, target, max_correspondence_distance, transformation): 6x6, row-major. */
int32_t b2s_overlap(b2s_handle* h, const b2s_cloud* source, const b2s_cloud* target, const double source_to_target[16], double voxel_size,
                    int32_t min_points_per_voxel, b2s_cloud* source_overlap, b2s_cloud* target_overlap);
int32_t b2s_information_matrix(b2s_handle* h, const b2s_cloud* source, const b2s_cloud* target, double max_correspondence_distance,
                               const double transformation[16], double info_out[36]);
/* C2  Submap::carve of the DENSE map   src/Submap.cpp:86-89,125-136, src/helpers.cpp:347-377, src/VoxelHashMap.cpp:13-45,
 *     src/Voxel.cpp:162-192.  `scan` is used in the frame the caller hands over (the reference passes the raw scan together with
 *     the map-frame sensor position); the every-N-scans schedule stays with the caller.  Uses voxel = dense_voxel_size,
 *     neighborhood_radius_dense_map, truncation_distance, max_raytracing_length.  n_removed may be NULL (no synchronisation). */
int32_t b2s_dense_carve(b2s_handle* h, b2s_submap* sm, const b2s_cloud* scan, const double sensor_position[3],
                        const b2s_carving_params* params, size_t* n_removed);
/* F3  Submap::insertScanDenseMap -> VoxelizedPointCloud::insert           src/Submap.cpp:77-92, src/Voxel.cpp:66-88 */
int32_t b2s_submap_insert_dense(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const double map_to_sensor[16],
                                const b2s_cropper* dense_cropper);
/* F2  VoxelHashMap<Voxel> query interface (include/open3d_slam/VoxelHashMap.hpp:104-158) on the dense map, batched over
 *     the points of a device cloud:  hasVoxelContainingPoint / getVoxelContainingPointPtr -> counts[i] (0 = no voxel) and,
 *     optionally, the aggregated position (AggregatedVoxel::getAggregatedPosition, src/Voxel.cpp:35-40) in means_xyz[3i..];
 *     removeKey(getKey(p)) for every point; size(); clear().  Host arrays must hold `capacity` >= cloud size entries. */
int32_t b2s_dense_query(b2s_handle* h, const b2s_submap* sm, const b2s_cloud* points, int32_t* counts, double* means_xyz, size_t capacity);
int32_t b2s_dense_remove(b2s_handle* h, b2s_submap* sm, const b2s_cloud* points);
int32_t b2s_dense_size(b2s_handle* h, const b2s_submap* sm, size_t* n_voxels);
int32_t b2s_dense_clear(b2s_handle* h, b2s_submap* sm);
/* Submap::transform (loop-closure correction of a whole submap)              src/Submap.cpp:94-107
 *     mapCloud_.Transform(T) ([O3D] PointCloud::Transform: points T p / w, normals R n; no duplication quirk),
 *     denseMap_.transform(T) (src/Voxel.cpp:49-64: applied to the voxel SUMS, keys unchanged -- kept as it is),
 *     mapToRangeSensor_ = mapToRangeSensor_ * T (the pose state of b2s_submap_set_pose / b2s_submap_get_pose). */
int32_t b2s_submap_transform(b2s_handle* h, b2s_submap* sm, const double T[16]);
/* [O3D] PointCloud::Transform of a cloud in place, points and normals (no duplication quirk): Submap::transform applies it to the
 * submap's sparse feature cloud, sparseMapCloud_ (src/Submap.cpp:96), with the same kernel as the map */
int32_t b2s_cloud_transform_inplace(b2s_handle* h, b2s_cloud* c, const double T[16]);
/* Submap::getMapPointCloud (copy-out)                                       src/Submap.cpp:184-191 */
int32_t b2s_submap_size(b2s_handle* h, const b2s_submap* sm, size_t* n);
int32_t b2s_submap_download(b2s_handle* h, const b2s_submap* sm, double* xyz, double* normals, size_t capacity, size_t* n);
/* Submap::getMapPointCloudCopy (src/Submap.cpp:187-191) without leaving the device: the map cloud as a b2s_cloud (what place
 * recognition, the overlap selection and the voxel map of the revisit check read, src/PlaceRecognition.cpp:69,96, src/Submap.cpp:236) */
int32_t b2s_submap_to_cloud(b2s_handle* h, const b2s_submap* sm, b2s_cloud* out);
int32_t b2s_submap_dense_download(b2s_handle* h, const b2s_submap* sm, double* xyz, double* normals, int32_t* keys, size_t capacity,
                                  size_t* n);
int32_t b2s_submap_set_cloud(b2s_handle* h, b2s_submap* sm, const b2s_cloud* cloud);   /* load / initial map */
/* S2  ScanToMapIcp::scanToMapRegistration: crop the map patch around the sensor, then R1
 *     src/ScanToMapRegistration.cpp:55-62 */
int32_t b2s_register_to_submap(b2s_handle* h, const b2s_cloud* scan, const b2s_submap* sm, const double map_to_sensor[16],
                               const double init[16], b2s_result* out);

/* ---- fused device-side chain for throughput runs: S1 -> S2 -> fitness gate -> F1, no host round trip.
 *      Restates the steady-state branch of Mapper::addRangeMeasurement (src/Mapper.cpp:139-177) with the pose
 *      prediction supplied by the caller.  The result is written to device memory and fetched with
 *      b2s_scan_result_fetch after b2s_synchronize. ------------------------------------------------------------ */
/* the pose state mapToRangeSensor_ lives on the device next to the map (Mapper.hpp mapToRangeSensor_/mapToRangeSensorPrev_) */
int32_t b2s_submap_set_pose(b2s_handle* h, b2s_submap* sm, const double map_to_sensor[16]);
int32_t b2s_submap_get_pose(b2s_handle* h, const b2s_submap* sm, double map_to_sensor[16]);
/* one scan: guess = pose * odometry_motion (Mapper.cpp:130-137); S1; S2 around the pose state; gate
 * (fitness < min_refinement_fitness rejects unless ignore_min_fitness, Mapper.cpp:151); accepted -> pose = result, F1. */
int32_t b2s_mapper_step_async(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const double odometry_motion[16],
                              double min_refinement_fitness, int32_t ignore_min_fitness, int32_t slot /* 0..255 */);
int32_t b2s_scan_result_fetch(b2s_handle* h, int32_t slot, b2s_result* out);   /* synchronises */
/* the same chain end to end with HOST buffers: float32 xyz (wire format; pinned memory keeps the copy asynchronous) in,
 * RegistrationResult out -- upload + S1 + S2 + gate + F1 + read-back in one call (Mapper::addRangeMeasurement as the
 * ROS callback sees it, rospkg/src/OnlineRangeDataProcessorRos.cpp:38-43 -> core/src/Mapper.cpp:101-181) */
int32_t b2s_mapper_step_host(b2s_handle* h, b2s_submap* sm, const void* xyz_f32, size_t n, size_t stride_bytes,
                             const double odometry_motion[16], double min_refinement_fitness, int32_t ignore_min_fitness,
                             b2s_result* out);
/* the same without waiting: the upload, the chain and the copy of the result into *out_pinned (page-locked host memory,
 * valid after the next b2s_synchronize) are only enqueued -- one host thread can keep many mappers (handles) busy */
int32_t b2s_mapper_step_host_async(b2s_handle* h, b2s_submap* sm, const void* xyz_f32, size_t n, size_t stride_bytes,
                                   const double odometry_motion[16], double min_refinement_fitness, int32_t ignore_min_fitness,
                                   b2s_result* out_pinned);
/* CUDA-graph replay of b2s_mapper_step_async for this submap: after two eager steps the ~45 launches of one scan are
 * captured once and replayed with a single cudaGraphLaunch.  Every scan must be uploaded (b2s_cloud_upload_f32/_f64) or
 * copied (b2s_cloud_copy) into the returned fixed-capacity staging cloud, which is then passed as raw_scan; the slot
 * argument must equal (number of graph steps so far) % 256.  Falls back to eager launches when the chain cannot be
 * captured (e.g. a cropper without a maximum radius needs a host round trip). */
int32_t b2s_mapper_graph_enable(b2s_handle* h, b2s_submap* sm, size_t raw_capacity_points, double min_refinement_fitness,
                                int32_t ignore_min_fitness, b2s_cloud** staging_out);

/* ---- options of the device-resident Mapper chain (b2s_mapper_step_async / _host / _host_async) -----------------------
 * What Mapper::addRangeMeasurement and SubmapCollection::insertScan do around S1/S2/F1 with their default wiring:
 *   - the minimum-motion gate in front of the map insertion                       src/Mapper.cpp:170-176
 *   - Submap::insertScan(..., isPerformCarving = true): space carving of the sparse map every carveSpaceEveryNscans_
 *     insertions (nScansInsertedMap_ % N == 1, map not empty), with the cropper at the pose of the LAST insertion
 *                                                                                 src/SubmapCollection.cpp:178,205, src/Submap.cpp:55-60,109-123
 *   - insertScanDenseMap(raw scan, mapToRangeSensor, carving = true) for every scan addRangeMeasurement accepted
 *                                                                                 src/SlamWrapper.cpp:318-327,363-376, src/Submap.cpp:77-92,125-136
 * All decisions are taken ON THE DEVICE from device-resident counters (the host never learns whether a scan passed
 * the fitness gate before it reads the result), so the chain stays free of host round trips and graph-replayable.
 * Options are per submap; changing them drops a captured graph (it is re-captured on the next step). */
typedef struct b2s_mapper_options {
  double min_movement_between_mapping_steps;   /* MapperParameters::minMovementBetweenMappingSteps_ (Parameters.hpp:161), default 0 */
  int32_t carve_enabled;                       /* isPerformCarving of Submap::insertScan */
  int32_t carve_every_n_scans;                 /* SpaceCarvingParameters::carveSpaceEveryNscans_ (Parameters.hpp:89), default 10 */
  b2s_carving_params carving;                  /* mapBuilder_.carving_ */
  int32_t dense_enabled;                       /* feed the dense map with every accepted raw scan */
  int32_t dense_carve_every_n_scans;           /* denseMapBuilder_.carving_.carveSpaceEveryNscans_; 0 = no dense carving */
  b2s_carving_params dense_carving;            /* denseMapBuilder_.carving_ */
  b2s_cropper dense_cropper;                   /* denseMapBuilder_.cropper_ (applied in the sensor frame, Submap.cpp:78-79) */
} b2s_mapper_options;
void b2s_default_mapper_options(b2s_mapper_options* o);
int32_t b2s_submap_set_mapper_options(b2s_handle* h, b2s_submap* sm, const b2s_mapper_options* o);
/* device-side bookkeeping of the chain, read back (synchronises): what the reference keeps in Mapper / Submap members */
typedef struct b2s_mapper_counters {
  int64_t steps;                 /* scans that went through S1 + S2 on this submap */
  int64_t accepted;              /* passed the fitness gate (addRangeMeasurement returned true) */
  int64_t inserted_map;          /* Submap::nScansInsertedMap_ */
  int64_t inserted_dense;        /* Submap::nScansInsertedDenseMap_ */
  int64_t carve_runs;            /* how often the sparse carving actually ran */
  int64_t carved_points_total;   /* map points removed by it */
  int64_t dense_carve_runs;
  int64_t carved_voxels_total;   /* dense voxels emptied */
} b2s_mapper_counters;
int32_t b2s_submap_get_mapper_counters(b2s_handle* h, const b2s_submap* sm, b2s_mapper_counters* out);

/* ---- localisation against a prior map (MapperParameters::isUseInitialMap_ / isMergeScansIntoMap_, Parameters.hpp:173-174) --------
 * The reference's rules, with paths relative to open3d_slam/open3d_slam/:
 *   1. initial map (SlamWrapper::setInitialMap, src/SlamWrapper.cpp:209-220): normals on the full map (prepareInitialMap: the caller runs
 *      b2s_estimate_normals), then Submap::insertScan's initial branch, mapCloud_ = map; voxelize(mapVoxelSize) ([O3D] VoxelDownSample,
 *      normals averaged, no carving, no fusion, src/Submap.cpp:47-52): b2s_submap_set_initial_map.
 *   2. initial pose (SlamWrapper::setInitialTransform, :222-225): Mapper::setMapToRangeSensorInitial, mapToRangeSensor_ =
 *      mapToRangeSensorPrev_ = T and isNewInitialValueSet_ = true (src/Mapper.cpp:87-91): b2s_submap_set_initial_transform.  The
 *      odometry half is b2s_odometry_set_initial_transform.
 *   3. the next step of b2s_mapper_step_* / b2s_slam_step_* (src/Mapper.cpp:130-149): the guess is the pose without odometry, the ICP
 *      runs and its result is discarded, the pose stays T (the slam step pushes it into the map-pose buffer), no fitness gate, no
 *      insertion, the step counts as accepted (the dense map is fed at T), lastMeasurementTimestamp_ is kept, and the step after it
 *      predicts without odometry as well.
 *   4. pure localisation (merge off, :163-167): an accepted scan moves the pose only -- no carving, no insertion, the pose of the last
 *      insertion is kept.  The dense map is still fed.  b2s_submap_set_merge_scans(sm, 0); on is the default (mapping).
 *   5. localisation with map building (merge on) merges as in mapping; the submap hand-over is host policy (SubmapCollection).
 * Eager steps and graph replay follow the same rules; switching the merge flag drops a captured graph. */
int32_t b2s_submap_set_initial_map(b2s_handle* h, b2s_submap* sm, const b2s_cloud* cloud, double map_voxel_size);
int32_t b2s_submap_set_initial_transform(b2s_handle* h, b2s_submap* sm, const double map_to_sensor[16]);
int32_t b2s_submap_set_merge_scans(b2s_handle* h, b2s_submap* sm, int32_t on);
/* Static map patch.  While a submap's merge is off its map cannot change, so its slots are kept counting-sorted by a 2 m tile (built by
 * the first registration after merge goes off), and every registration against it (the device chains and b2s_register_to_submap)
 * gathers its patch from the tiles the cropper's box touches: the same indexed points, grid header and original indices as the full
 * path, at O(points in the touched tiles) instead of O(map).  A cropper without a bounded extent (MIN_RADIUS, invert) uses the full
 * path; b2s_submap_set_cloud / _set_initial_map / _insert / _carve / _transform and switching merge on drop the table (and a captured
 * chain that reads it).  B2S_PATCH_FULL=1 in the environment forces the full path (read once per process).
 * Debug aid: header {origin, cell}, {dims, ncell, n}, cell starts and original indices of the NN index the last registration built. */
int32_t b2s_debug_nn_index(b2s_handle* h, double origin_cell[4], int32_t dims_n[5], int32_t* cell_start, size_t cap_cells, int32_t* orig,
                           size_t cap_pts);

/* ---- device-resident LidarOdometry (src/Odometry.cpp:19-110) and the combined per-scan step of SlamWrapper: odometry, then
 *      Mapper::addRangeMeasurement with the prediction read from the odometry's TransformInterpolationBuffer on the device.
 *      Every decision (initialise / ok / failed, the buffer, the prediction, the mapper gates) is taken on the device.
 *      Timestamps are UniversalTimeScaleClock ticks (100 ns, include/open3d_slam/time.hpp:43-55).  They are host values, so the
 *      order check stays on the host: a step whose t is not greater than the previous step's t on that odometry object returns
 *      B2S_E_INVALID.  (Deliberate difference: the reference prints a warning and returns false, Odometry.cpp:41-44, Mapper.cpp:117-120.)
 *      An odometry object belongs to the handle that created it: passing it with another handle -> B2S_E_INVALID. */
/* OdometryParameters (Parameters.hpp:78-83): scanMatcher_ + scanProcessing_, plus the two constants the reference hard-codes */
typedef struct b2s_odometry_params {
  b2s_icp_params icp;            /* scanMatcher_ (reg_type, max_iter, max_corr_dist, knn, knn_radius, rel_*) */
  double voxel_size;             /* scanProcessing_.voxelSize_ */
  double downsampling_ratio;     /* scanProcessing_.downSamplingRatio_ */
  uint32_t seed;                 /* replaces std::random_device in [O3D] RandomDownSample */
  b2s_cropper cropper;           /* scanProcessing_.cropper_, applied in the sensor frame (Odometry.cpp:21,26) */
  double min_fitness;            /* the "todo magic" 0.1 of Odometry.cpp:51: the registration succeeds iff fitness > min_fitness */
  int32_t buffer_size;           /* size limit of odomToRangeSensorBuffer_: TransformInterpolationBuffer() = 2000; fixed at creation */
} b2s_odometry_params;
/* the Lua odometry block: the same scan-processing / ICP values as b2s_default_config, min_fitness 0.1, buffer_size 2000 */
void b2s_default_odometry_params(b2s_odometry_params* p);
enum { B2S_ODOM_INIT = 0, B2S_ODOM_OK = 1, B2S_ODOM_FAILED = 2, B2S_ODOM_FAILED_KEPT_PREV = 3 };
typedef struct b2s_odometry b2s_odometry;
/* capacity_points: the largest raw scan a step accepts (B2S_E_CAPACITY above it) */
int32_t b2s_odometry_create(b2s_handle* h, const b2s_odometry_params* p, size_t capacity_points, b2s_odometry** out);
void b2s_odometry_destroy(b2s_odometry* od);
/* LidarOdometry::setParameters (Odometry.cpp:96-100); buffer_size must stay what the object was created with */
int32_t b2s_odometry_set_params(b2s_handle* h, b2s_odometry* od, const b2s_odometry_params* p);
/* LidarOdometry::setInitialTransform (Odometry.cpp:102-110): the cumulative pose becomes T now, and again (instead of the
 * composition) at the next successful registration */
int32_t b2s_odometry_set_initial_transform(b2s_handle* h, b2s_odometry* od, const double T[16]);
/* LidarOdometry::addRangeScan(raw, t) (Odometry.cpp:32-79), enqueue only:
 *   pre = RandomDownSample(normals(voxelize(crop(raw))))                        :25-30 (one crop, sensor frame)
 *   cloudPrev_ empty          -> cloudPrev_ = pre, push (t, cumulative)         :33-39  outcome INIT
 *   registerClouds(cloudPrev_, pre, I) with the object's own icp parameters    :48
 *   fitness > min_fitness     -> cumulative = pending initial transform or cumulative * T^-1, cloudPrev_ = pre, push   outcome OK
 *   otherwise                 -> cloudPrev_ = pre when pre is not empty, no push          outcome FAILED / FAILED_KEPT_PREV
 * slot 0..255: where b2s_odometry_result_fetch finds the result.  The host may run at most 32 steps ahead of the device. */
int32_t b2s_odometry_step_async(b2s_handle* h, b2s_odometry* od, const b2s_cloud* raw, int64_t t, int32_t slot);
typedef struct b2s_odometry_result {
  b2s_result registration;           /* registerClouds(cloudPrev_, pre, I); zeros on an initialising step */
  double odom_to_range_sensor[16];   /* odomToRangeSensorCumulative_ after the step */
  int32_t outcome;                   /* B2S_ODOM_* */
  int32_t n_preprocessed;            /* points of pre */
} b2s_odometry_result;
int32_t b2s_odometry_result_fetch(b2s_handle* h, b2s_odometry* od, int32_t slot, b2s_odometry_result* out);   /* synchronises */
/* getTransform(t, odomToRangeSensorBuffer_) and buffer.has(t) (TransformInterpolationBuffer.cpp:76-157, Transform.cpp:16-41):
 * clamped to the earliest / latest entry, exact on an equal timestamp, else translation interpolated linearly and rotation by
 * Eigen's slerp between the neighbours, factor = dt(t, start) / (dt(end, start) + 1e-6 s).  An empty buffer: has = 0, T = I.
 * Synchronises. */
int32_t b2s_odometry_lookup(b2s_handle* h, const b2s_odometry* od, int64_t t, double T[16], int32_t* has);
/* LidarOdometry::getPreProcessedCloud (Odometry.cpp:84-86) = cloudPrev_, copied into out */
int32_t b2s_odometry_preprocessed(b2s_handle* h, const b2s_odometry* od, b2s_cloud* out);

/* One scan through SlamWrapper's two workers (odometryWorker + mappingWorker): b2s_odometry_step_async(raw, t), then
 * Mapper::addRangeMeasurement(raw, t) on the submap (the steady-state branch of b2s_mapper_step_async) with
 *   odom_used = buffer.has(t);  guess = pose * getTransform(t_last)^-1 * getTransform(t) if odom_used, else pose   Mapper.cpp:122-137
 * t_last = lastMeasurementTimestamp_ of that mapper: Time() = 0 at first, set to t by every scan the fitness gate accepts (:164,178).
 * It lives on the device with the odometry object (one robot's stream of scans), so a submap hand-over keeps it, as the
 * reference's Mapper member does.  The submap must not be empty: the caller inserts the first scan (Mapper.cpp:105-114) and
 * runs b2s_odometry_step_async on that scan and timestamp.  The mapper options, gates, carving, F1 and dense map follow
 * unchanged; b2s_mapper_processed_scan returns this step's merge_ / match_. */
typedef struct b2s_slam_result {
  b2s_odometry_result odometry;
  b2s_result mapper;
  int32_t odom_used;                 /* the buffer had t (the prediction came from the odometry) */
  int32_t mapper_accepted;           /* addRangeMeasurement returned true */
} b2s_slam_result;
int32_t b2s_slam_step_async(b2s_handle* h, b2s_submap* sm, b2s_odometry* od, const b2s_cloud* raw, int64_t t, double min_refinement_fitness,
                            int32_t ignore_min_fitness, int32_t slot);
int32_t b2s_slam_result_fetch(b2s_handle* h, b2s_odometry* od, int32_t slot, b2s_slam_result* out);   /* synchronises */
/* the same with a float32 host scan (pinned memory keeps the copy asynchronous): upload, both chains and the copy of the result
 * into *out_pinned (page-locked host memory, valid after the next b2s_synchronize) are only enqueued */
int32_t b2s_slam_step_host_async(b2s_handle* h, b2s_submap* sm, b2s_odometry* od, const void* xyz_f32, size_t n, size_t stride_bytes, int64_t t,
                                 double min_refinement_fitness, int32_t ignore_min_fitness, b2s_slam_result* out_pinned);
/* CUDA-graph replay of b2s_slam_step_async: after two eager steps per submap the launches of one scan (odometry + mapper) are
 * captured once and replayed with one cudaGraphLaunch.  The graphs are kept per submap on the odometry object, so a hand-over
 * back to a submap seen before replays without a new capture (the graphs of destroyed submaps are released when the object next
 * meets a submap it has no graph for); b2s_odometry_set_params, b2s_set_config and
 * b2s_submap_set_mapper_options on that submap invalidate them.  Every scan must be uploaded or copied into the returned
 * fixed-capacity staging cloud (one input stream per odometry object), which is then passed as raw. */
int32_t b2s_slam_graph_enable(b2s_handle* h, b2s_odometry* od, size_t raw_capacity_points, b2s_cloud** staging_out);

/* D2  motion compensation (de-skew) inside the device step, SlamWrapper::loadParametersAndInitialize (src/SlamWrapper.cpp:195-200):
 *     with enabled set, every step of b2s_odometry_step_async / b2s_slam_step_async / _host_async de-skews the raw scan twice, as
 *     odometryWorker (:266-268) and mappingWorker (:298-304) do, each with ConstantVelocityMotionCompensation::undistortInputPointCloud
 *     (src/MotionCompensation.cpp:64-139, the per-point arithmetic of b2s_undistort):
 *       - the odometry's input: velocities from the odometry buffer as it is before this scan's odometry step;
 *       - the mapper's input:   velocities from the mapper's buffer (mapToRangeSensorBuffer_) as it is before this scan's mapper
 *                               step.  That cloud is the raw scan of everything downstream: pre-processing, ICP, carving, F1 and
 *                               the dense map (Mapper.cpp:139,174, SlamWrapper.cpp:322).
 *     The velocity estimate, at the step's timestamp t with offset = num_poses_velocity_estimation (:32-57):
 *       size <= offset -> v = w = 0;   latest_time < t -> dT = start^-1 * finish with finish = the latest entry and start the entry
 *       `offset` before it, dt = toSeconds(finish.t - start.t), v = dT.translation / (dt + 1e-6),
 *       w = toRPY(Quaterniond(dT.rotation).normalized()) / (dt + 1e-6) (src/math.cpp:39-46);   otherwise v = w = 0.
 *     The mapper's buffer lives on the odometry object (one robot's Mapper), so a submap hand-over keeps it.  Its size limit is the
 *     object's buffer_size.  Every step the mapper's fitness gate accepts pushes (t, mapToRangeSensor) into it, before the minimum-
 *     motion gate (Mapper.cpp:160), whether or not de-skew is enabled; loop-closure corrections never touch it.  A push earlier than
 *     the earliest or the latest entry is ignored, an equal time is accepted (TransformInterpolationBuffer.cpp:21-43).
 *     Disabled (the default), the steps issue exactly the launches they issue without this feature. */
typedef struct b2s_motion_compensation_params {
  int32_t enabled;                        /* motion_compensation.is_undistort_scan (isUndistortInputCloud_), default 0 */
  int32_t spinning_clockwise;             /* isSpinningClockwise_, default 1 */
  double scan_duration;                   /* scanDuration_ [s], default 0.1; must be > 0 (assert_gt, MotionCompensation.cpp:61) */
  int32_t num_poses_velocity_estimation;  /* numPosesVelocityEstimation_, default 3; must be >= 1 */
} b2s_motion_compensation_params;
/* the Lua defaults of parameter_structure_definitions.lua:33-36 (Parameters.hpp:192-197) */
void b2s_default_motion_compensation_params(b2s_motion_compensation_params* p);
/* SlamWrapper.cpp:195-200 (both ConstantVelocityMotionCompensation objects).  scan_duration <= 0 or num_poses_velocity_estimation < 1
 * -> B2S_E_INVALID and nothing changes.  The first call with enabled set allocates the two de-skewed clouds (the object's capacity).
 * Drops the captured combined graphs of this object (they bake the parameters in). */
int32_t b2s_odometry_set_motion_compensation(b2s_handle* h, b2s_odometry* od, const b2s_motion_compensation_params* p);
/* mapToRangeSensorBuffer_.push(t, T) for the pushes the caller's host code makes: the first scan (Mapper.cpp:112) and a new initial
 * value (:145).  Enqueued on the handle's stream. */
int32_t b2s_slam_map_pose_push(b2s_handle* h, b2s_odometry* od, int64_t t, const double T[16]);
/* Mapper::getMapToRangeSensor(t) = getTransform(t, mapToRangeSensorBuffer_) with the semantics of b2s_odometry_lookup (has = 0,
 * T = I on an empty buffer).  Synchronises. */
int32_t b2s_slam_map_lookup(b2s_handle* h, const b2s_odometry* od, int64_t t, double T[16], int32_t* has);
/* the velocities each de-skew of the step written to `slot` used, and whether they were not all zero.  Written by the de-skew
 * kernels only: a half whose de-skew did not run in that step keeps what it held.  Synchronises. */
typedef struct b2s_motion_compensation_result {
  double odometry_linear_velocity[3];
  double odometry_angular_velocity_rpy[3];
  double map_linear_velocity[3];
  double map_angular_velocity_rpy[3];
  int32_t odometry_applied;               /* the odometry's de-skew moved the points (a velocity was non-zero) */
  int32_t map_applied;                    /* the mapper's de-skew did */
} b2s_motion_compensation_result;
int32_t b2s_slam_motion_fetch(b2s_handle* h, b2s_odometry* od, int32_t slot, b2s_motion_compensation_result* out);
/* device copies of the last de-skewed clouds: the odometry's input (odo_out) and the mapper's (map_out); either may be NULL.
 * B2S_E_INVALID when de-skew was never enabled on this object. */
int32_t b2s_slam_undistorted(b2s_handle* h, const b2s_odometry* od, b2s_cloud* odo_out, b2s_cloud* map_out);

/* ---- F4  o3d_slam::VoxelMap (include/open3d_slam/Voxel.hpp:19-36, src/Voxel.cpp:123-160): voxel -> per-layer lists of point indices.
 *      Keys are getVoxelIdx(p, 1 / voxelSize) = floor(p * inv) per axis (VoxelHashMap.hpp:43-50).  Layers are integers
 *      0..B2S_VOXEL_MAP_LAYERS-1 (the shim maps the reference's layer names, e.g. Submap::voxelMapLayer).  The users on this path:
 *      the revisit check of SubmapCollection::isSwitchingSubmapsConsistant (src/SubmapCollection.cpp:352-364) =
 *      b2s_voxel_map_has_voxel over the scan moved by mapToRangeSensor; Submap::computeFeatures fills it with
 *      voxelMap_.clear(); voxelMap_.insertCloud(voxelMapLayer, mapCloud_) (src/Submap.cpp:235-236). ------------------------------ */
#define B2S_VOXEL_MAP_LAYERS 4
typedef struct b2s_voxel_map b2s_voxel_map;
int32_t b2s_voxel_map_create(b2s_handle* h, const double voxel_size[3], size_t capacity_voxels, b2s_voxel_map** out);   /* VoxelMap(voxelSize) */
void b2s_voxel_map_destroy(b2s_voxel_map* vm);
int32_t b2s_voxel_map_clear(b2s_handle* h, b2s_voxel_map* vm);                                                        /* clear() */
int32_t b2s_voxel_map_insert_cloud(b2s_handle* h, b2s_voxel_map* vm, int32_t layer, const b2s_cloud* cloud);          /* insertCloud(layer, cloud) */
int32_t b2s_voxel_map_size(b2s_handle* h, const b2s_voxel_map* vm, size_t* n_voxels);                                 /* size() */
/* hasVoxelContainingPoint for every point of `points` (moved by the isometry T first when T is given): flags (optional, one per
 * point, `capacity` entries) and the number of hits */
int32_t b2s_voxel_map_has_voxel(b2s_handle* h, const b2s_voxel_map* vm, const b2s_cloud* points, const double T_or_null[16],
                                int32_t* flags_or_null, size_t capacity, size_t* n_hits);
/* getIndicesInVoxel(layer, p) for every point: CSR answer, offsets[n + 1] and the concatenated index lists (each sorted ascending =
 * insertion order of insertCloud(layer, cloud)).  indices may be NULL to query the sizes only. */
int32_t b2s_voxel_map_indices_in_voxel(b2s_handle* h, const b2s_voxel_map* vm, int32_t layer, const b2s_cloud* points, int32_t* offsets,
                                       size_t offsets_capacity, int32_t* indices, size_t indices_capacity, size_t* n_indices);
/* copies of the clouds the last mapper step produced on this handle (ProcessedScans of Mapper.cpp:139; SubmapCollection keeps
 * the merge_ cloud in its overlap buffer, src/SubmapCollection.cpp:83-92,180).  Either output may be NULL. */
int32_t b2s_mapper_processed_scan(b2s_handle* h, b2s_cloud* merge_out, b2s_cloud* match_out);

/* ---- loop-closure features: Submap::computeFeatures -> [O3D] ComputeFPFHFeature (src/Submap.cpp:244) ----------------------
 *      A b2s_feature is the device-resident [O3D] pipelines::registration::Feature: B2S_FEATURE_DIM x n fp64, stored point after
 *      point (the memory order of the reference's column-major data_ matrix), so host arrays hold n * B2S_FEATURE_DIM doubles.
 *      b2s_compute_fpfh(cloud, radius, knn): FPFH over the exact hybrid neighbourhood (the knn nearest points with d^2 < radius^2,
 *      ascending (d^2, index)).  Errors: radius <= 0 or knn <= 0 -> B2S_E_INVALID; knn > B2S_FEATURE_MAX_KNN -> B2S_E_UNSUPPORTED;
 *      a non-empty cloud without normals -> B2S_E_NO_NORMALS ([O3D] LogError); an empty cloud gives a feature of zero points.
 *      A feature belongs to the handle that created it: passing it with another handle -> B2S_E_INVALID.
 *      Synchronises once (point count).  Semantics and deterministic choices: DESIGN.md, row K-fpfh. */
#define B2S_FEATURE_DIM 33
#define B2S_FEATURE_MAX_KNN 128
typedef struct b2s_feature b2s_feature;
int32_t b2s_feature_create(b2s_handle* h, b2s_feature** out);
void b2s_feature_destroy(b2s_feature* f);
int32_t b2s_feature_size(b2s_handle* h, const b2s_feature* f, size_t* n);
int32_t b2s_feature_download(b2s_handle* h, const b2s_feature* f, double* data, size_t capacity_points, size_t* n);
int32_t b2s_feature_upload(b2s_handle* h, b2s_feature* f, const double* data, size_t n);
int32_t b2s_compute_fpfh(b2s_handle* h, const b2s_cloud* cloud, double radius, int32_t knn, b2s_feature* feature);

/* The feature-cloud front end of Submap::computeFeatures (src/Submap.cpp:239-244) on the submap's map cloud, read in place:
 *     sparse = VoxelDownSample(map, feature_voxel_size)              normals averaged per voxel, like b2s_voxel_down_sample
 *     sparse.EstimateNormals(Hybrid(normal_estimation_radius, normal_knn)), NormalizeNormals,
 *     OrientNormalsTowardsCameraLocation(0)                          the sparse cloud HAS normals (the voxel means): [O3D] keeps
 *                                                                    the prior where the solver returns a zero vector and flips a
 *                                                                    normal that points against it (DESIGN.md, row K-features)
 *     feature = ComputeFPFHFeature(sparse, Hybrid(feature_radius, feature_knn))
 * b2s_default_feature_params gives the Lua defaults (parameter_structure_definitions.lua:155-159): 0.5 / 2.0 / 20 / 2.5 / 100.
 * The C++ struct PlaceRecognitionParameters (Parameters.hpp:118-122) defaults differ: normalEstimationRadius_ 1.0, normalKnn_ 10.
 * Errors: a size <= 0 or a knn <= 0 -> B2S_E_INVALID; normal_knn > 32 or feature_knn > B2S_FEATURE_MAX_KNN -> B2S_E_UNSUPPORTED;
 * a submap or an output of another handle -> B2S_E_INVALID.  An empty map gives an empty sparse cloud and a feature of zero points.
 * A map loaded without normals (point-to-point, stored as NaN) gives zero prior normals, which change nothing.
 * Synchronises once (the sparse cloud's point count, as b2s_compute_fpfh does). */
typedef struct b2s_feature_params {     /* PlaceRecognitionParameters, the fields computeFeatures reads */
  double feature_voxel_size;            /* featureVoxelSize_ */
  double normal_estimation_radius;      /* normalEstimationRadius_ */
  int32_t normal_knn;                   /* normalKnn_ (<= 32) */
  double feature_radius;                /* featureRadius_ */
  int32_t feature_knn;                  /* featureKnn_ (<= B2S_FEATURE_MAX_KNN) */
} b2s_feature_params;
void b2s_default_feature_params(b2s_feature_params* p);
int32_t b2s_submap_compute_features(b2s_handle* h, b2s_submap* sm, const b2s_feature_params* params, b2s_cloud* sparse_out,
                                    b2s_feature* feature_out);

/* ---- loop-closure proposal: [O3D] RegistrationRANSACBasedOnFeatureMatching as PlaceRecognition::buildLoopClosureConstraints
 *      calls it (src/PlaceRecognition.cpp:81-86): mutual filter, TransformationEstimationPointToPoint(false), the distance and
 *      edge-length checkers, RANSACConvergenceCriteria(max_iteration, confidence).  The exact semantics, including the
 *      counter-based hypothesis stream that replaces std::random_device and the sequential best / stop rule that makes a run
 *      independent of how the device batches it, are DESIGN.md row K-ransac.
 * b2s_default_ransac_params gives the Lua values (parameter_structure_definitions.lua:156-161): mutual 1, ransac_n 3,
 * max_correspondence_distance 0.75, checker_distance 0.8, checker_edge_length 0.6, max_iteration 10 000 000, confidence 0.999.
 * The C++ struct PlaceRecognitionParameters (Parameters.hpp:123-129) defaults differ: ransacNumIter_ 1 000 000, ransacProbability_
 * 0.99, correspondenceCheckerDistance_ 0.75, correspondenceCheckerEdgeLength_ 0.5. */
#define B2S_RANSAC_MAX_N 8
typedef struct b2s_ransac_params {
  int32_t mutual_filter;                /* mutual_filter (true at PlaceRecognition.cpp:82) */
  int32_t ransac_n;                     /* ransacModelSize_ (3 <= n <= B2S_RANSAC_MAX_N; n < 3 gives the empty result) */
  double max_correspondence_distance;   /* ransacMaxCorrespondenceDistance_ (validation radius) */
  double checker_distance;              /* correspondenceCheckerDistance_ */
  double checker_edge_length;           /* correspondenceCheckerEdgeLength_ */
  int64_t max_iteration;                /* ransacNumIter_ */
  double confidence;                    /* ransacProbability_, in (0, 1) */
  uint64_t seed;                        /* replaces std::random_device: the hypothesis stream of DESIGN.md row K-ransac */
} b2s_ransac_params;
void b2s_default_ransac_params(b2s_ransac_params* p);
typedef struct b2s_ransac_result {
  b2s_result result;                    /* T, fitness, inlier_rmse, n_corr = inliers (correspondence_set_.size(), :86); iters = 0 */
  int64_t hypotheses;                   /* the h the sequential loop stopped at */
  int64_t validations;                  /* hypotheses that passed both checkers and were validated by that loop */
  int64_t best_hypothesis;              /* the h of the result (-1 = the empty result) */
  int32_t n_feature_corr;               /* size of the feature correspondence set RANSAC drew from */
  int32_t used_mutual;                  /* 1 when that set is the mutual one */
} b2s_ransac_result;
/* One source (its sparse cloud and FPFH) against n_targets candidates, the loop of PlaceRecognition.cpp:71 in one call; out[k]
 * belongs to target k and does not depend on the other targets.  Errors: a feature whose size differs from its cloud's, an object
 * of another handle, n_targets < 0, confidence outside (0, 1) or max_iteration < 0 -> B2S_E_INVALID; ransac_n > B2S_RANSAC_MAX_N ->
 * B2S_E_UNSUPPORTED.  ransac_n < 3, max_correspondence_distance <= 0, an empty cloud or a correspondence set smaller than ransac_n
 * give the empty result (T = I, zeros) with B2S_OK.  Synchronises once per batch of hypotheses (B2S_RANSAC_BATCH, DESIGN.md 5). */
int32_t b2s_ransac_feature_matching(b2s_handle* h, const b2s_cloud* source_sparse, const b2s_feature* source_feature, int32_t n_targets,
                                    const b2s_cloud* const* target_sparses, const b2s_feature* const* target_features,
                                    const b2s_ransac_params* params, b2s_ransac_result* out);
/* The two exact nearest-feature arrays RANSAC's correspondence set is built from: src_to_tgt[i] = argmin_j d2(i, j),
 * tgt_to_src[j] = argmin_i d2(i, j), d2 summed over the 33 bins in ascending order, ties to the lower index; -1 when the other
 * feature is empty.  Host arrays hold the capacities given (>= the feature sizes, else B2S_E_CAPACITY).  Synchronises. */
int32_t b2s_feature_correspondences(b2s_handle* h, const b2s_feature* source_feature, const b2s_feature* target_feature, int32_t* src_to_tgt,
                                    size_t src_capacity, int32_t* tgt_to_src, size_t tgt_capacity);

/* ---- odometry constraints between consecutive submaps: buildOdometryConstraint -> buildConstraint (src/constraint_builders.cpp:33-90),
 *      as SubmapCollection::computeFeatures (src/SubmapCollection.cpp:238) and SlamWrapper::loopClosureWorker (src/SlamWrapper.cpp:427-428)
 *      reach it through computeOdometryConstraints (src/constraint_builders.cpp:92-118).  For every pair k, on the maps where they live:
 *   - source = sources[k] is the PARENT, target = targets[k] the CHILD: buildOdometryConstraint(parent, child)            :33, :100-102
 *   - both clouds are the WHOLE map, getMapPointCloudCopy (the live map slots in map order), no cropper                   :46-47
 *   - voxel = getMapVoxelSize(map_voxel_size, voxel_if_zero): |v| <= 1e-3 -> voxel_if_zero, else v (a negative v passes
 *     through, as it does in the reference)                                                                              helpers.cpp:343-345
 *   - overlap at the IDENTITY with edge overlap_factor x voxel and minNumPointsPerVoxel = min_points_per_voxel: the points of
 *     either map whose voxel holds points of both, each map's survivors in map order (b2s_overlap's rule)               :51-58
 *   - refine != 0 only: RegistrationICP(sourceOverlap, targetOverlap, r = icp_factor x voxel, Identity,
 *     TransformationEstimationPointToPlane, max_iter / rel_fitness / rel_rmse) -- ALWAYS point-to-plane, whatever
 *     b2s_config.icp.reg_type is: the reference calls raw [O3D] RegistrationICP here, not the mapper's cloudRegistration    :62-68
 *   - the information matrix is always estimated: GetInformationMatrixFromPointClouds(sourceOverlap, targetOverlap, r, T) with
 *     T = the ICP result, or the identity without refinement ([O3D]'s no-transform branch, as b2s_information_matrix)    :69-73
 *   - sourceToTarget_ = T (identity unless refined); isOdometryConstraint_ = isInformationMatrixValid_ = true            :75-82
 * Errors: a submap or an overlap cloud of another handle, a voxel <= 0 after the getMapVoxelSize rule, overlap_factor or icp_factor
 * <= 0, min_points_per_voxel < 1, max_iter < 0, n_pairs < 0 -> B2S_E_INVALID; refine != 0 and a child map without normals (a
 * point-to-point map, stored as NaN) -> B2S_E_NO_NORMALS.  n_pairs = 0 -> B2S_OK.  One call runs every pair in one set of launches
 * and synchronises once.  source_overlaps_or_null / target_overlaps_or_null (each an array of n_pairs clouds, or NULL) receive the
 * selected points, in map order.  Semantics and kernels: DESIGN.md row L2. */
typedef struct b2s_odometry_constraint_params {   /* constraint_builders.cpp:33-41, magic.hpp, helpers.cpp:343-345 */
  double map_voxel_size;          /* map_builder.map_voxel_size (0.1) */
  double voxel_if_zero;           /* magic::voxelSizeCorrespondenceSearchIfMapVoxelSizeIsZero = 0.04 */
  double overlap_factor;          /* magic::voxelExpansionFactorOverlapComputation = 20 */
  double icp_factor;              /* magic::voxelExpansionFactorIcpCorrespondenceDistance = 1.5 */
  int32_t min_points_per_voxel;   /* 1 */
  int32_t refine;                 /* is_refine_odometry_constraints_between_submaps (false) */
  int32_t max_iter;               /* magic::icpRunUntilConvergenceNumberOfIterations = 100 */
  double rel_fitness, rel_rmse;   /* [O3D] ICPConvergenceCriteria defaults, 1e-6 */
} b2s_odometry_constraint_params;
typedef struct b2s_odometry_constraint {
  double T[16];                   /* sourceToTarget_ (identity unless refined), row-major */
  double information[36];         /* informationMatrix_, row-major */
  int64_t n_source_overlap, n_target_overlap;
  int32_t refined;                /* the ICP ran */
  b2s_result icp;                 /* its RegistrationResult when refined, zeros otherwise */
} b2s_odometry_constraint;
void b2s_default_odometry_constraint_params(b2s_odometry_constraint_params* p);
int32_t b2s_submap_odometry_constraints(b2s_handle* h, int32_t n_pairs, const b2s_submap* const* sources /* parent */,
                                        const b2s_submap* const* targets /* child */, const b2s_odometry_constraint_params* p,
                                        b2s_cloud* const* source_overlaps_or_null, b2s_cloud* const* target_overlaps_or_null,
                                        b2s_odometry_constraint* out);

/* ---- submap pose-graph optimisation: [O3D] GlobalOptimization with GlobalOptimizationLevenbergMarquardt, as
 *      OptimizationProblem::solve (src/OptimizationProblem.cpp:25-44) calls it.  Restated semantics (DESIGN.md row G1):
 *   - validation: every edge id in [0, n_nodes) (else B2S_E_INVALID); the graph connected from node 0 over all edges and over the
 *     certain edges alone (BFS), else B2S_OK with the poses unchanged and stats[0].valid = stats[1].valid = 0
 *   - lpw = preference_loop_closure * max_correspondence_distance^2 * mean_e information_e(5,5) (0 without edges)
 *   - zeta_e = lin(X^-1 Tt^-1 Ts), lin(M) = ((M21-M12)/2, (M02-M20)/2, (M10-M01)/2, M03, M13, M23); inverses are the rigid ones
 *   - uncertain edges: conf = (lpw / (lpw + zeta' Info zeta))^2; certain edges keep 1
 *   - residual = sum_e conf zeta' Info zeta + lpw (sqrt(conf) - 1)^2; H, b: conf-weighted J' Info J, -conf J' Info zeta
 *   - LM: lambda = 1e-5 max diag H, nu = 2; delta = (H + lambda I)^-1 b by an UNPIVOTED LDL' (|d| <= 1/DBL_MAX zeroes the
 *     component); trial T_i <- V2M(delta_i) T_i; rho = (cur - new) / (delta.(lambda delta + b) + 1e-3); criteria of [O3D]
 *   - two passes (all edges; then the certain edges and the uncertain edges with conf > edge_prune_threshold), then every pose is
 *     left-multiplied by T_ref(input) T_ref(new)^-1 when reference_node is in range.
 * The LM control flow runs on the host; every try runs one CUDA graph (H + lambda I, blocked LDL' on fp64 mma.sync, substitution,
 * trial poses, trial residual) and reads back one record.  Results repeat bit for bit. */
typedef struct b2s_pose_graph_edge {   /* [O3D] PoseGraphEdge */
  int32_t source, target;              /* node ids */
  int32_t uncertain;                   /* uncertain_: a loop closure (line process); odometry edges are certain */
  int32_t reserved_;
  double T[16];                        /* transformation_, row-major (the source-to-target measurement X) */
  double information[36];              /* information_, row-major */
} b2s_pose_graph_edge;
typedef struct b2s_global_optimization_params {   /* GlobalOptimizationOption + GlobalOptimizationConvergenceCriteria */
  double max_correspondence_distance;  /* 1000 (Lua, parameter_structure_definitions.lua:45-50; the C++ struct has 10) */
  double edge_prune_threshold;         /* 0.2 */
  double preference_loop_closure;      /* loop_closure_preference, 2.0 */
  int32_t reference_node;              /* 0; out of range = no compensation */
  int32_t max_iteration;               /* 100 */
  double min_relative_increment;       /* 1e-6 */
  double min_relative_residual_increment; /* 1e-6 */
  double min_right_term;               /* 1e-6 */
  double min_residual;                 /* 1e-6 */
  int32_t max_iteration_lm;            /* 20 */
  int32_t reserved_;
  double upper_scale_factor;           /* 2/3 */
  double lower_scale_factor;           /* 1/3 */
} b2s_global_optimization_params;
enum {   /* b2s_global_optimization_stats.stop_reason: the first criterion that stopped the pass */
  B2S_LM_STOP_NONE = 0, B2S_LM_STOP_RIGHT_TERM = 1, B2S_LM_STOP_RELATIVE_INCREMENT = 2, B2S_LM_STOP_RELATIVE_RESIDUAL_INCREMENT = 3,
  B2S_LM_STOP_MAX_ITERATION_LM = 4, B2S_LM_STOP_RESIDUAL = 5, B2S_LM_STOP_MAX_ITERATION = 6
};
typedef struct b2s_global_optimization_stats {   /* one per pass: [0] all edges, [1] the pruned graph */
  int32_t valid;                       /* the graph passed validation (the pass ran) */
  int32_t n_edges;                     /* edges of the pass */
  int32_t outer_iterations;
  int32_t lm_tries;                    /* solves of (H + lambda I) delta = b */
  int32_t accepted_steps;              /* tries with rho > 0 */
  int32_t stop_reason;                 /* B2S_LM_STOP_* */
  double initial_residual, final_residual;   /* the pass's residual at its start, and of its last accepted poses */
  double final_lambda;
} b2s_global_optimization_stats;
void b2s_default_global_optimization_params(b2s_global_optimization_params* p);
/* node_poses: n_nodes row-major 4x4, optimised in place.  edge_kept_out (n_edges int32, optional): 1 = the edge survived the pruning.
 * edge_confidence_out (n_edges, optional): the edge's confidence at the end (the second pass's for kept edges, the first pass's
 * for pruned ones).  stats_out (2, optional).  Errors: n_nodes < 1, n_edges < 0, an id out of range, a non-positive tolerance or
 * iteration limit -> B2S_E_INVALID.  n_edges = 0 -> B2S_OK, poses unchanged (valid = 1 for a single node, as the BFS finds). */
int32_t b2s_global_optimization(b2s_handle* h, int32_t n_nodes, double* node_poses, int32_t n_edges, const b2s_pose_graph_edge* edges,
                                const b2s_global_optimization_params* p, int32_t* edge_kept_out, double* edge_confidence_out,
                                b2s_global_optimization_stats* stats_out);

/* ---- device-to-device hand-over of a cloud's arrays (SURVEY.md section 8e: a submap that is the registration target on
 *      several GPUs is built once by its owner and broadcast over NVLink by the host side -- torch.distributed / NCCL own
 *      the transfer, this library only copies between its cloud and the caller's device buffers on the handle's stream).
 *      xyz / normals are 3 x f64 per point, like every cloud.  export: synchronises (the count is returned). -------------- */
int32_t b2s_cloud_export_device(b2s_handle* h, const b2s_cloud* c, void* xyz_dev, void* normals_dev_or_null, size_t capacity_points, size_t* n);
int32_t b2s_cloud_import_device(b2s_handle* h, b2s_cloud* c, const void* xyz_dev, const void* normals_dev_or_null, size_t n);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* B2S_H_ */
