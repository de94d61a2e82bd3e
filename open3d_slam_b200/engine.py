"""Host-side mirror of the reference's operator interface for the hot path, on top of the C ABI (include/b2s.h).

Names, argument meaning and error behaviour follow open3d_slam (paths relative to
/root/reference/open3d_slam/open3d_slam/):
    CloudRegistration / RegistrationIcpPointToPlane / cloudRegistrationFactory   include/open3d_slam/CloudRegistration.hpp:19-73
    ScanToMapRegistration / ScanToMapIcp / scanToMapRegistrationFactory          include/open3d_slam/ScanToMapRegistration.hpp:24-61
    Submap.insertScan / getMapPointCloud                                         include/open3d_slam/Submap.hpp:38-45
    Mapper.addRangeMeasurement (host control flow only)                          src/Mapper.cpp:101-181
The reference itself is C++; its C++ subclasses live in shim/.  This Python mirror exists so that tests/ and
bench.py read like tests of the reference interface.  All arithmetic happens in libb2s.so on the GPU.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field

import numpy as np

from . import _lib as L

# --------------------------------------------------------------------------------------------------------------------
# parameters (include/open3d_slam/Parameters.hpp:51-98); defaults = the Lua defaults
# (ros/open3d_slam_ros/param/default/parameter_structure_definitions.lua:52-72,102) with PointToPlaneIcp
# --------------------------------------------------------------------------------------------------------------------


def regTypeOf(name: str) -> int:
    """CloudRegistrationType by its Lua name (Parameters.hpp:37-49) -> B2S_REG_*; an unknown name is what the factories throw on"""
    types = {"PointToPlaneIcp": L.REG_POINT_TO_PLANE, "PointToPointIcp": L.REG_POINT_TO_POINT, "GeneralizedIcp": L.REG_GENERALIZED}
    if name not in types:
        raise L.B2SError(L.E_UNSUPPORTED, f"unknown registration type {name}")
    return types[name]


@dataclass
class ScanCroppingParameters:
    cropperName: str = "MinMaxRadius"
    croppingMinRadius: float = 2.0
    croppingMaxRadius: float = 30.0
    croppingMinZ: float = -50.0
    croppingMaxZ: float = 50.0

    def to_c(self, center=(0.0, 0.0, 0.0), invert=False) -> L.Cropper:
        c = L.Cropper()
        c.kind = L.CROPPER_NAMES[self.cropperName]
        c.invert = int(invert)
        c.rmin, c.rmax, c.zmin, c.zmax = self.croppingMinRadius, self.croppingMaxRadius, self.croppingMinZ, self.croppingMaxZ
        c.center[0], c.center[1], c.center[2] = (float(v) for v in center)
        return c


@dataclass
class IcpParameters:
    maxNumIter: int = 50
    maxCorrespondenceDistance: float = 1.0
    knn: int = 20
    maxDistanceKnn: float = 3.0


@dataclass
class ScanProcessingParameters:
    voxelSize: float = 0.1
    downSamplingRatio: float = 0.3
    cropper: ScanCroppingParameters = field(default_factory=ScanCroppingParameters)


@dataclass
class SpaceCarvingParameters:
    """include/open3d_slam/Parameters.hpp:85-92"""
    voxelSize: float = 0.1
    maxRaytracingLength: float = 20.0
    truncationDistance: float = 0.1
    carveSpaceEveryNscans: int = 10
    minDotProductWithNormal: float = 0.5
    neighborhoodRadiusDenseMap: float = 0.1

    def to_c(self) -> L.CarvingParams:
        return L.CarvingParams(self.voxelSize, self.maxRaytracingLength, self.truncationDistance, self.minDotProductWithNormal,
                               self.neighborhoodRadiusDenseMap)


@dataclass
class MapBuilderParameters:
    mapVoxelSize: float = 0.1
    cropper: ScanCroppingParameters = field(default_factory=ScanCroppingParameters)
    carving: SpaceCarvingParameters = field(default_factory=SpaceCarvingParameters)


@dataclass
class CloudRegistrationParameters:
    regType: str = "PointToPlaneIcp"
    icp: IcpParameters = field(default_factory=IcpParameters)


@dataclass
class PlaceRecognitionParameters:
    """The fields of include/open3d_slam/Parameters.hpp:118-129 that Submap::computeFeatures and the RANSAC proposal of
    PlaceRecognition::buildLoopClosureConstraints read.  Defaults = the Lua values (parameter_structure_definitions.lua:151-162); the
    C++ struct's own defaults differ (normalEstimationRadius_ 1.0, normalKnn_ 10, ransacNumIter_ 1e6, ransacProbability_ 0.99,
    correspondenceCheckerDistance_ 0.75, correspondenceCheckerEdgeLength_ 0.5)."""
    featureVoxelSize: float = 0.5
    normalEstimationRadius: float = 2.0
    normalKnn: int = 20
    featureRadius: float = 2.5
    featureKnn: int = 100
    ransacNumIter: int = 10_000_000
    ransacProbability: float = 0.999
    ransacModelSize: int = 3
    ransacMaxCorrespondenceDistance: float = 0.75
    correspondenceCheckerDistance: float = 0.8
    correspondenceCheckerEdgeLength: float = 0.6
    ransacMinCorrespondenceSetSize: int = 25
    ransacSeed: int = 1            # replaces std::random_device of [O3D] RANSAC (DESIGN.md row K-ransac)

    def ransac_c(self, mutual_filter: bool = True) -> L.RansacParams:
        return L.RansacParams(int(mutual_filter), int(self.ransacModelSize), float(self.ransacMaxCorrespondenceDistance),
                              float(self.correspondenceCheckerDistance), float(self.correspondenceCheckerEdgeLength), int(self.ransacNumIter),
                              float(self.ransacProbability), int(self.ransacSeed))

    def to_c(self) -> L.FeatureParams:
        return L.FeatureParams(float(self.featureVoxelSize), float(self.normalEstimationRadius), int(self.normalKnn), float(self.featureRadius),
                               int(self.featureKnn))


@dataclass
class MapperParameters:
    scanToMapRegType: str = "PointToPlaneIcp"
    minRefinementFitness: float = 0.7
    icp: IcpParameters = field(default_factory=IcpParameters)
    scanProcessing: ScanProcessingParameters = field(default_factory=ScanProcessingParameters)
    mapBuilder: MapBuilderParameters = field(default_factory=MapBuilderParameters)
    denseMapVoxelSize: float = 0.05
    denseMapCropper: ScanCroppingParameters = field(default_factory=ScanCroppingParameters)       # denseMapBuilder_.cropper_
    denseMapCarving: SpaceCarvingParameters = field(default_factory=SpaceCarvingParameters)       # denseMapBuilder_.carving_
    isIgnoreMinRefinementFitness: bool = False
    minMovementBetweenMappingSteps: float = 0.0
    # localisation against a prior map (Parameters.hpp:173-174), both false as in Lua (is_use_map_initialization /
    # is_merge_scans_into_map); the C++ struct defaults the merge flag to true.  The merge flag only matters with isUseInitialMap.
    isUseInitialMap: bool = False
    isMergeScansIntoMap: bool = False
    seed: int = 0            # replaces std::random_device of [O3D] RandomDownSample
    nnCellSize: float = 0.0  # engine knob: NN grid cell (0 = maxCorrespondenceDistance / 4)
    icpClusterCtas: int = 0  # engine knob: SMs one registration spreads over (0 = automatic; 8 = throughput, 16 = latency)

    def to_config(self) -> L.Config:
        reg_type = regTypeOf(self.scanToMapRegType)
        cfg = L.Config()
        L.lib().b2s_default_config(C.byref(cfg))
        cfg.icp.reg_type = reg_type
        cfg.icp.max_iter = int(self.icp.maxNumIter)
        cfg.icp.max_corr_dist = float(self.icp.maxCorrespondenceDistance)
        cfg.icp.knn = int(self.icp.knn)
        cfg.icp.knn_radius = float(self.icp.maxDistanceKnn)
        cfg.icp.rel_fitness = 1e-6
        cfg.icp.rel_rmse = 1e-6
        cfg.scan.voxel_size = float(self.scanProcessing.voxelSize)
        cfg.scan.downsampling_ratio = float(self.scanProcessing.downSamplingRatio)
        cfg.scan.seed = int(self.seed)
        cfg.scan.map_builder_cropper = self.mapBuilder.cropper.to_c()
        cfg.scan.scan_matcher_cropper = self.scanProcessing.cropper.to_c()
        cfg.map_voxel_size = float(self.mapBuilder.mapVoxelSize)
        cfg.dense_voxel_size = float(self.denseMapVoxelSize)
        cfg.nn_cell_size = float(self.nnCellSize)
        cfg.icp_cluster_ctas = int(self.icpClusterCtas)
        return cfg


@dataclass
class RegistrationResult:
    """open3d::pipelines::registration::RegistrationResult as read by the callers."""
    transformation_: np.ndarray
    fitness_: float
    inlier_rmse_: float
    n_corr: int = 0
    iters: int = 0


def _res(r: L.Result) -> RegistrationResult:
    return RegistrationResult(np.array(r.T, dtype=np.float64).reshape(4, 4), float(r.fitness), float(r.inlier_rmse), int(r.n_corr),
                              int(r.iters))


def _mat(T) -> np.ndarray:
    T = np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(4, 4))
    return T


def _pd(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


# --------------------------------------------------------------------------------------------------------------------
# engine handle and device clouds
# --------------------------------------------------------------------------------------------------------------------


class Engine:
    """One b2s_handle (one CUDA stream).  Use one per host thread."""

    def __init__(self, params: MapperParameters | None = None, device: int = 0, cuda_stream: int | None = None):
        self.params = params or MapperParameters()
        self._h = C.c_void_p()
        cfg = self.params.to_config()
        L.check(L.lib().b2s_create(C.byref(cfg), C.c_int32(device), C.c_void_p(cuda_stream or 0), C.byref(self._h)))
        self.device = device

    def set_parameters(self, params: MapperParameters):
        self.params = params
        cfg = params.to_config()
        L.check(L.lib().b2s_set_config(self._h, C.byref(cfg)))

    def synchronize(self):
        L.check(L.lib().b2s_synchronize(self._h))

    @property
    def launches(self) -> int:
        return int(L.lib().b2s_launch_count(self._h))

    @property
    def graphCaptures(self) -> int:
        """CUDA graphs the per-scan chains of this handle have captured (a replay adds launches, not captures)"""
        return int(L.lib().b2s_graph_capture_count(self._h))

    def profile_enable(self, on: bool = True):
        L.check(L.lib().b2s_profile_enable(self._h, C.c_int32(int(on))))

    def profile_read(self) -> dict:
        """{kind: (total_ms, count)} of the kernel groups launched since the last read (CUDA events, this stream)."""
        n = len(L.PROFILE_KINDS)
        ms = (C.c_double * n)(); cnt = (C.c_int64 * n)()
        L.check(L.lib().b2s_profile_read(self._h, ms, cnt, C.c_int32(n)))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(L.PROFILE_KINDS)}

    def close(self):
        if self._h:
            L.lib().b2s_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- clouds
    def cloud(self, xyz=None, normals=None) -> "Cloud":
        c = Cloud(self)
        if xyz is not None:
            c.upload(xyz, normals)
        return c


class Cloud:
    """Device-resident open3d::geometry::PointCloud (points_ + normals_)."""

    def __init__(self, eng: Engine):
        self.eng = eng
        self._c = C.c_void_p()
        L.check(L.lib().b2s_cloud_create(eng._h, C.byref(self._c)))

    def upload(self, xyz, normals=None):
        xyz = np.asarray(xyz)
        if xyz.dtype == np.float32 and normals is None:
            xyz = np.ascontiguousarray(xyz.reshape(-1, 3))
            L.check(L.lib().b2s_cloud_upload_f32(self.eng._h, self._c, xyz.ctypes.data_as(C.c_void_p), C.c_size_t(len(xyz)),
                                                 C.c_size_t(12)))
            return self
        xyz = np.ascontiguousarray(xyz, dtype=np.float64).reshape(-1, 3)
        n = len(xyz)
        nptr = None
        if normals is not None:
            normals = np.ascontiguousarray(normals, dtype=np.float64).reshape(-1, 3)
            assert len(normals) == n
            nptr = _pd(normals)
        L.check(L.lib().b2s_cloud_upload_f64(self.eng._h, self._c, _pd(xyz), nptr, C.c_size_t(n)))
        return self

    def upload_pinned_f32(self, ptr: int, n: int, stride: int = 12):
        L.check(L.lib().b2s_cloud_upload_f32(self.eng._h, self._c, C.c_void_p(ptr), C.c_size_t(n), C.c_size_t(stride)))
        return self

    def size(self):
        n = C.c_size_t(); hn = C.c_int32()
        L.check(L.lib().b2s_cloud_size(self.eng._h, self._c, C.byref(n), C.byref(hn)))
        return int(n.value), bool(hn.value)

    def __len__(self):
        return self.size()[0]

    def HasNormals(self):
        return self.size()[1]

    def download(self):
        n, hn = self.size()
        xyz = np.empty((n, 3)); nrm = np.empty((n, 3)) if hn else None
        m = C.c_size_t()
        L.check(L.lib().b2s_cloud_download(self.eng._h, self._c, _pd(xyz), _pd(nrm) if hn else None, C.c_size_t(n), C.byref(m)))
        return xyz, nrm

    def export_device(self, xyz_ptr: int, nrm_ptr: int | None, capacity_points: int) -> int:
        """device-to-device copy of the arrays into caller-owned device buffers (3 x f64 per point); returns the point count"""
        n = C.c_size_t()
        L.check(L.lib().b2s_cloud_export_device(self.eng._h, self._c, C.c_void_p(xyz_ptr), C.c_void_p(nrm_ptr) if nrm_ptr else None,
                                                C.c_size_t(capacity_points), C.byref(n)))
        return int(n.value)

    def import_device(self, xyz_ptr: int, nrm_ptr: int | None, n: int):
        L.check(L.lib().b2s_cloud_import_device(self.eng._h, self._c, C.c_void_p(xyz_ptr), C.c_void_p(nrm_ptr) if nrm_ptr else None, C.c_size_t(n)))
        return self

    def free(self):
        if self._c and not getattr(self, "_borrowed", False):
            L.lib().b2s_cloud_destroy(self._c)
        self._c = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


# --------------------------------------------------------------------------------------------------------------------
# stage-level operators (SURVEY.md section 8a rows P1-P4, F0)
# --------------------------------------------------------------------------------------------------------------------


def crop(eng: Engine, cloud: Cloud, cropper: L.Cropper) -> Cloud:
    out = Cloud(eng)
    L.check(L.lib().b2s_crop(eng._h, cloud._c, C.byref(cropper), out._c))
    return out


def voxelize(eng: Engine, cloud: Cloud, voxel_size: float) -> Cloud:
    """o3d_slam::voxelize (src/helpers.cpp:107-113)."""
    out = Cloud(eng)
    L.check(L.lib().b2s_voxel_down_sample(eng._h, cloud._c, C.c_double(voxel_size), out._c))
    return out


def random_down_sample(eng: Engine, cloud: Cloud, ratio: float, seed: int) -> Cloud:
    out = Cloud(eng)
    L.check(L.lib().b2s_random_down_sample(eng._h, cloud._c, C.c_double(ratio), C.c_uint32(seed), out._c))
    return out


def transform(eng: Engine, T, cloud: Cloud) -> Cloud:
    """o3d_slam::transform (src/helpers.cpp:273-305)."""
    out = Cloud(eng)
    T = _mat(T)
    L.check(L.lib().b2s_transform(eng._h, cloud._c, _pd(T), out._c))
    return out


# --------------------------------------------------------------------------------------------------------------------
# CloudRegistration (include/open3d_slam/CloudRegistration.hpp)
# --------------------------------------------------------------------------------------------------------------------


class ConstantVelocityMotionCompensation:
    """src/MotionCompensation.cpp:31-139.  The velocity estimate (two poses of the caller's buffer, :33-57) is host logic;
    the per-point correction runs on the device (b2s_undistort)."""

    def __init__(self, eng: Engine, isSpinningClockwise: bool = True, scanDuration: float = 0.1, numPosesVelocityEstimation: int = 3):
        if not scanDuration > 0.0:
            raise RuntimeError("lidar scanDuration_: must be > 0")   # assert_gt, :61
        self.eng = eng
        self.isSpinningClockwise_ = isSpinningClockwise
        self.scanDuration_ = scanDuration
        self.numPosesVelocityEstimation_ = numPosesVelocityEstimation

    @staticmethod
    def estimateLinearAndAngularVelocity(startPose, finishPose, dt: float):
        """:41-52 -- dT = start^-1 * finish; v = dT.translation / (dt + 1e-6); w = toRPY(dT.rotation) / (dt + 1e-6)."""
        dT = np.linalg.inv(_mat(startPose)) @ _mat(finishPose)
        R = dT[:3, :3]
        roll = np.arctan2(R[2, 1], R[2, 2]); pitch = np.arcsin(-R[2, 0]); yaw = np.arctan2(R[1, 0], R[0, 0])
        return dT[:3, 3] / (dt + 1e-6), np.array([roll, pitch, yaw]) / (dt + 1e-6)

    def undistortInputPointCloud(self, cloud: Cloud, linearVelocity, angularVelocityRpy) -> Cloud:
        out = Cloud(self.eng)
        lv = np.ascontiguousarray(np.asarray(linearVelocity, dtype=np.float64).reshape(3))
        av = np.ascontiguousarray(np.asarray(angularVelocityRpy, dtype=np.float64).reshape(3))
        L.check(L.lib().b2s_undistort(self.eng._h, cloud._c, _pd(lv), _pd(av), C.c_double(self.scanDuration_), C.c_int32(int(self.isSpinningClockwise_)),
                                      out._c))
        return out


def computeOverlappingClouds(eng: Engine, source: Cloud, target: Cloud, sourceToTarget, voxelSize: float, minNumPointsPerVoxel: int = 1):
    """computeIndicesOfOverlappingPoints + SelectByIndex (src/helpers.cpp:307-332, src/PlaceRecognition.cpp:103-106):
    returns (sourceOverlap, targetOverlap), the selected points in their original order."""
    so, to = Cloud(eng), Cloud(eng)
    L.check(L.lib().b2s_overlap(eng._h, source._c, target._c, _pd(_mat(sourceToTarget)), C.c_double(voxelSize), C.c_int32(minNumPointsPerVoxel),
                                so._c, to._c))
    return so, to


def getInformationMatrixFromPointClouds(eng: Engine, source: Cloud, target: Cloud, maxCorrespondenceDistance: float, transformation) -> np.ndarray:
    """[O3D] GetInformationMatrixFromPointClouds as called at src/PlaceRecognition.cpp:148 and src/constraint_builders.cpp:71."""
    G = np.zeros((6, 6))
    L.check(L.lib().b2s_information_matrix(eng._h, source._c, target._c, C.c_double(maxCorrespondenceDistance), _pd(_mat(transformation)), _pd(G)))
    return G


@dataclass
class OdometryConstraintParameters:
    """What buildOdometryConstraint reads (src/constraint_builders.cpp:33-41): the map voxel and the magic constants (magic.hpp:12-15),
    isRefineOdometryConstraintsBetweenSubmaps_ (default false) and the [O3D] ICPConvergenceCriteria of the refinement."""
    mapVoxelSize: float = 0.1
    voxelSizeIfMapVoxelSizeIsZero: float = 0.04                  # magic::voxelSizeCorrespondenceSearchIfMapVoxelSizeIsZero
    voxelExpansionFactorOverlapComputation: float = 20.0
    voxelExpansionFactorIcpCorrespondenceDistance: float = 1.5
    minNumPointsPerVoxel: int = 1
    isRefineOdometryConstraintsBetweenSubmaps: bool = False
    maxNumIter: int = 100                                        # magic::icpRunUntilConvergenceNumberOfIterations
    relativeFitness: float = 1e-6
    relativeRmse: float = 1e-6

    def to_c(self) -> L.OdometryConstraintParams:
        return L.OdometryConstraintParams(float(self.mapVoxelSize), float(self.voxelSizeIfMapVoxelSizeIsZero), float(self.voxelExpansionFactorOverlapComputation),
                                          float(self.voxelExpansionFactorIcpCorrespondenceDistance), int(self.minNumPointsPerVoxel),
                                          int(self.isRefineOdometryConstraintsBetweenSubmaps), int(self.maxNumIter), float(self.relativeFitness),
                                          float(self.relativeRmse))


def getMapVoxelSize(mapVoxelSize: float, valueIfZero: float) -> float:
    """src/helpers.cpp:343-345: |v| <= 1e-3 -> valueIfZero, else v (a negative v passes through)."""
    return valueIfZero if abs(mapVoxelSize) <= 1e-3 else mapVoxelSize


@dataclass
class OdometryConstraintResult:
    """buildOdometryConstraint's Constraint (sourceToTarget_, informationMatrix_) and the overlap sizes; icp is the refinement's
    RegistrationResult (None when it did not run)."""
    sourceToTarget_: np.ndarray
    informationMatrix_: np.ndarray
    nSourceOverlap: int
    nTargetOverlap: int
    icp: RegistrationResult | None = None


def buildOdometryConstraintsBatch(eng: Engine, sources, targets, params: OdometryConstraintParameters | None = None, sourceOverlaps=None,
                                  targetOverlaps=None) -> list[OdometryConstraintResult]:
    """buildOdometryConstraint(parent, child) (src/constraint_builders.cpp:33-90) for every pair (sources[k] = parent Submap, targets[k]
    = child Submap) in one device call on the resident maps.  sourceOverlaps / targetOverlaps (lists of Cloud, optional) receive the
    overlap selections in map order."""
    p = (params or OdometryConstraintParameters()).to_c()
    n = len(sources)
    assert len(targets) == n
    arr = lambda objs: (C.c_void_p * max(n, 1))(*objs)
    so = arr([c._c for c in sourceOverlaps]) if sourceOverlaps is not None else None
    to = arr([c._c for c in targetOverlaps]) if targetOverlaps is not None else None
    out = (L.OdometryConstraint * max(n, 1))()
    L.check(L.lib().b2s_submap_odometry_constraints(eng._h, C.c_int32(n), arr([s._s for s in sources]), arr([t._s for t in targets]), C.byref(p),
                                                    so, to, out))
    return [OdometryConstraintResult(np.array(o.T, dtype=np.float64).reshape(4, 4), np.array(o.information, dtype=np.float64).reshape(6, 6),
                                     int(o.n_source_overlap), int(o.n_target_overlap), _res(o.icp) if o.refined else None) for o in out[:n]]


def buildOdometryConstraint(eng: Engine, source, target, params: OdometryConstraintParameters | None = None) -> OdometryConstraintResult:
    """src/constraint_builders.cpp:33-41 for one (parent, child) pair of Submaps."""
    return buildOdometryConstraintsBatch(eng, [source], [target], params)[0]


@dataclass
class LoopClosureRefinementParameters:
    """What the refinement half of PlaceRecognition::buildLoopClosureConstraints reads (src/PlaceRecognition.cpp:96-149): the map
    voxel (getMapVoxelSize, :98), the magic constants (magic.hpp), placeRecognition.maxIcpCorrespondenceDistance_ /
    minRefinementFitness_ (Parameters.hpp:130-131) and the [O3D] ICPConvergenceCriteria of the refinement."""
    mapVoxelSize: float = 0.1
    voxelSizeIfMapVoxelSizeIsZero: float = 0.04                  # magic::voxelSizeCorrespondenceSearchIfMapVoxelSizeIsZero
    voxelExpansionFactorOverlapComputation: float = 20.0
    minNumPointsPerVoxel: int = 1
    maxNumIter: int = 100                                        # magic::icpRunUntilConvergenceNumberOfIterations
    maxIcpCorrespondenceDistance: float = 0.3
    relativeFitness: float = 1e-6
    relativeRmse: float = 1e-6
    minRefinementFitness: float = 0.7
    regType: str = "PointToPlaneIcp"                             # the refinement's estimator; the reference's: the scan matcher's (:47)

    def to_c(self) -> L.LoopClosureRefinementParams:
        return L.LoopClosureRefinementParams(float(self.mapVoxelSize), float(self.voxelSizeIfMapVoxelSizeIsZero),
                                             float(self.voxelExpansionFactorOverlapComputation), int(self.minNumPointsPerVoxel), int(self.maxNumIter),
                                             float(self.maxIcpCorrespondenceDistance), float(self.relativeFitness), float(self.relativeRmse),
                                             float(self.minRefinementFitness), regTypeOf(self.regType))


@dataclass
class LoopClosureRefinementResult:
    """One candidate's refinement: the ICP's RegistrationResult, the information matrix at its T (computed for every candidate),
    the fitness gate (:118) and the overlap sizes."""
    result: RegistrationResult
    information: np.ndarray
    accepted: bool
    nSourceOverlap: int
    nTargetOverlap: int


def refineLoopClosuresBatch(eng: Engine, sourceSubmap, targetSubmaps, inits, params: LoopClosureRefinementParameters | None = None,
                            sourceOverlaps=None, targetOverlaps=None) -> list[LoopClosureRefinementResult]:
    """src/PlaceRecognition.cpp:96-149 for one source Submap against every target Submap in one device call on the resident maps:
    overlap at inits[k], ICP with params.regType from inits[k], fitness gate, information matrix.  sourceOverlaps / targetOverlaps (lists
    of Cloud, optional) receive the overlap selections in map order."""
    p = (params or LoopClosureRefinementParameters()).to_c()
    n = len(targetSubmaps)
    T = np.ascontiguousarray(np.asarray(inits, dtype=np.float64).reshape(n, 16) if n else np.zeros((1, 16)))
    arr = lambda objs: (C.c_void_p * max(n, 1))(*objs)
    so = arr([c._c for c in sourceOverlaps]) if sourceOverlaps is not None else None
    to = arr([c._c for c in targetOverlaps]) if targetOverlaps is not None else None
    out = (L.LoopClosureRefinement * max(n, 1))()
    L.check(L.lib().b2s_submap_loop_closure_refinement(eng._h, sourceSubmap._s, C.c_int32(n), arr([t._s for t in targetSubmaps]), _pd(T), C.byref(p),
                                                       so, to, out))
    return [LoopClosureRefinementResult(_res(o.icp), np.array(o.information, dtype=np.float64).reshape(6, 6), bool(o.accepted), int(o.n_source_overlap),
                                        int(o.n_target_overlap)) for o in out[:n]]


@dataclass
class VisualizationParameters:
    """include/open3d_slam/Parameters.hpp:179-183: the voxel sizes SlamWrapperRos::publishMaps applies to the assembled map and to the
    coloured submap cloud, and how often it publishes them"""
    assembledMapVoxelSize: float = 0.1
    submapVoxelSize: float = 0.1
    visualizeEveryNmsec: float = 250.0


def _submap_array(submaps):
    n = len(submaps)
    return n, (C.c_void_p * max(n, 1))(*[s._s for s in submaps])


def getAssembledMapPointCloud(eng: Engine, submaps, voxelSize: float = 0.0) -> Cloud:
    """Mapper::getAssembledMapPointCloud (src/Mapper.cpp:183-208) over the given Submaps in list order, then o3d_slam::voxelize(voxelSize)
    (a no-op for voxelSize <= 0), in one device call (b2s_assemble_map; rules in include/b2s.h)."""
    n, arr = _submap_array(submaps)
    out = Cloud(eng)
    L.check(L.lib().b2s_assemble_map(eng._h, C.c_int32(n), arr, C.c_double(voxelSize), out._c))
    return out


def assembleColoredPointCloud(eng: Engine, submaps, voxelSize: float = 0.0):
    """assembleColoredPointCloud (ros/open3d_slam_ros/src/helpers_ros.cpp:51-70), then voxelize(voxelSize): (Cloud without normals,
    colours as an n x 3 float64 array in the cloud's order)."""
    n, arr = _submap_array(submaps)
    out = Cloud(eng)
    cap = sum(int(s.capacity) for s in submaps)   # an upper bound of the live points; np.empty only commits the pages written
    rgb = np.empty((max(cap, 1), 3)); m = C.c_size_t()
    L.check(L.lib().b2s_assemble_colored_map(eng._h, C.c_int32(n), arr, C.c_double(voxelSize), out._c, _pd(rgb), C.c_size_t(cap), C.byref(m)))
    return out, rgb[:m.value].copy()


def assembleDenseMaps(eng: Engine, submaps, out: "Cloud | None" = None):
    """VoxelizedPointCloud::toPointCloud (src/Voxel.cpp:90-115) of every Submap's dense map in list order, in one device call
    (b2s_assemble_dense_maps; rules in include/b2s.h): (Cloud without normals, int64 offsets of n + 1 entries -- submap k's points are
    rows offsets[k]:offsets[k + 1]).  A submap without a dense map gives an empty range."""
    n, arr = _submap_array(submaps)
    out = out if out is not None else Cloud(eng)
    offsets = np.zeros(n + 1, dtype=np.int64)
    L.check(L.lib().b2s_assemble_dense_maps(eng._h, C.c_int32(n), arr, out._c, offsets.ctypes.data_as(C.POINTER(C.c_int64))))
    return out, offsets


# ---- session state: a submap's / an odometry object's device state as self-contained blobs (include/b2s.h "session state",
#      DESIGN.md row A3).  Writing them to files is the caller's business.

_VOXEL_REC = np.dtype([("key", "<u8"), ("slot", "<i4"), ("head", "<i4"), ("stamp", "<i4"), ("reserved_", "<i4")])
_DENSE_REC = np.dtype([("key", "<u8"), ("sum", "<f8", (6,)), ("slot", "<i4"), ("count", "<i4")])


@dataclass
class StateHeader:
    """The parsed header of a session-state blob: kind ("submap" / "odometry"), the words of include/b2s.h, and every section's
    (offset, length) in bytes by name."""
    kind: str
    version: int
    total_bytes: int
    map_voxel_size: float
    sections: dict
    params: dict

    def section(self, blob, name: str, dtype=np.uint8) -> np.ndarray:
        """the bytes of one section, viewed as dtype (the records as structured arrays: dtype "voxels" / "dense")"""
        dt = {"voxels": _VOXEL_REC, "dense": _DENSE_REC}.get(dtype, dtype) if isinstance(dtype, str) else dtype
        o, n = self.sections[name]
        return np.frombuffer(blob, dtype=np.uint8, count=n, offset=o).view(dt)


def parseStateHeader(blob) -> StateHeader:
    """Reads the header of a blob of exportSubmapStates / DeviceLidarOdometry.exportState (no checks beyond the magic: the import
    validates)."""
    w = np.frombuffer(blob, dtype="<u8", count=L.STATE_HEADER_BYTES // 8)
    magic = int(w[L.STATE_W_MAGIC])
    if magic == L.STATE_MAGIC_SUBMAP:
        kind, names, pnames = "submap", L.STATE_SUBMAP_SECTIONS, L.STATE_SUBMAP_PARAMS
    elif magic == L.STATE_MAGIC_ODOMETRY:
        kind, names, pnames = "odometry", L.STATE_ODOMETRY_SECTIONS, L.STATE_ODOMETRY_PARAMS
    else:
        raise ValueError(f"not a session-state blob (magic {magic:#x})")
    sections, off = {}, L.STATE_HEADER_BYTES
    for k, name in enumerate(names):
        n = int(w[L.STATE_W_SECTIONS + k])
        sections[name] = (off, n)
        off += n
    params = {name: int(w[L.STATE_W_PARAMS + k]) for k, name in enumerate(pnames)}
    if kind == "submap":
        params["dense_voxel"] = float(w[L.STATE_W_PARAMS + 4:L.STATE_W_PARAMS + 5].view("<f8")[0])
    return StateHeader(kind, int(w[L.STATE_W_VERSION]), int(w[L.STATE_W_TOTAL_BYTES]), float(w[L.STATE_W_MAP_VOXEL:L.STATE_W_MAP_VOXEL + 1].view("<f8")[0]),
                       sections, params)


def exportSubmapStates(eng: Engine, submaps) -> list:
    """Every Submap's device state as one self-contained blob (bytes), in list order, in one batched device call
    (b2s_submaps_export_state: one synchronisation for the sizes, one for the data).  The submaps are only read."""
    n, arr = _submap_array(submaps)
    offs = (C.c_size_t * (n + 1))()
    L.check(L.lib().b2s_submaps_export_state(eng._h, C.c_int32(n), arr, None, C.c_size_t(0), offs))
    buf = np.empty(max(int(offs[n]), 1), dtype=np.uint8)
    L.check(L.lib().b2s_submaps_export_state(eng._h, C.c_int32(n), arr, buf.ctypes.data_as(C.c_void_p), C.c_size_t(int(offs[n])), offs))
    return [buf[offs[k]:offs[k + 1]].tobytes() for k in range(n)]


def importSubmapState(eng: Engine, blob: bytes) -> "Submap":
    """A new Submap on eng holding exactly the exported state (b2s_submap_import_state); a blob the library refuses raises B2SError
    with B2S_E_INVALID and creates nothing.  The host-side schedule counters and the map-builder cropper pose are taken from the
    device words the blob restores (nScansInsertedMap_, nScansInsertedDenseMap_, the pose of the last insertion)."""
    blob = bytes(blob)
    s = C.c_void_p()
    L.check(L.lib().b2s_submap_import_state(eng._h, blob, C.c_size_t(len(blob)), C.byref(s)))
    hdr = parseStateHeader(blob)
    sm = Submap.__new__(Submap)
    sm.eng, sm._s, sm.capacity = eng, s, hdr.params["capacity"]
    ms = hdr.section(blob, "mstate", "<i4")
    sm.nScansInsertedMap_, sm.nScansInsertedDenseMap_ = int(ms[5]), int(ms[6])   # MS_NINS, MS_NDENSE
    sm._cropperPose = hdr.section(blob, "pose", "<f8").reshape(L.STATE_POSE_SLOTS, 4, 4)[5].copy()
    sm.lastCarvedCount = 0
    sm.sparseMapCloud_ = None
    sm.feature_ = None
    return sm


@dataclass
class PoseGraphNode:
    """[O3D] PoseGraphNode: pose_ (4x4)"""
    pose_: np.ndarray = field(default_factory=lambda: np.eye(4))


@dataclass
class PoseGraphEdge:
    """[O3D] PoseGraphEdge: the measurement transformation_ (source to target), information_, uncertain_, and confidence_ (1 until
    globalOptimization writes the value it ended with)"""
    source_node_id_: int
    target_node_id_: int
    transformation_: np.ndarray = field(default_factory=lambda: np.eye(4))
    information_: np.ndarray = field(default_factory=lambda: np.eye(6))
    uncertain_: bool = False
    confidence_: float = 1.0


@dataclass
class PoseGraph:
    """[O3D] PoseGraph: nodes_ and edges_"""
    nodes_: list = field(default_factory=list)
    edges_: list = field(default_factory=list)


@dataclass
class GlobalOptimizationOption:
    """[O3D] GlobalOptimizationOption with the project's values (parameter_structure_definitions.lua:45-50): max_correspondence_distance
    1000 (the C++ struct, Parameters.hpp:138-143, has 10), edge_prune_threshold 0.2, loop_closure_preference 2.0, reference_node 0"""
    max_correspondence_distance_: float = 1000.0
    edge_prune_threshold_: float = 0.2
    preference_loop_closure_: float = 2.0
    reference_node_: int = 0


@dataclass
class GlobalOptimizationConvergenceCriteria:
    """[O3D] GlobalOptimizationConvergenceCriteria defaults"""
    max_iteration_: int = 100
    min_relative_increment_: float = 1e-6
    min_relative_residual_increment_: float = 1e-6
    min_right_term_: float = 1e-6
    min_residual_: float = 1e-6
    max_iteration_lm_: int = 20
    upper_scale_factor_: float = 2.0 / 3.0
    lower_scale_factor_: float = 1.0 / 3.0


@dataclass
class GlobalOptimizationPassStats:
    """b2s_global_optimization_stats of one pass (0: all edges, 1: the pruned graph)"""
    valid: bool
    n_edges: int
    outer_iterations: int
    lm_tries: int
    accepted_steps: int
    stop_reason: str
    initial_residual: float
    final_residual: float
    final_lambda: float


def _go_params(criteria: GlobalOptimizationConvergenceCriteria, option: GlobalOptimizationOption) -> L.GlobalOptimizationParams:
    p = L.GlobalOptimizationParams()
    L.lib().b2s_default_global_optimization_params(C.byref(p))
    p.max_correspondence_distance = float(option.max_correspondence_distance_); p.edge_prune_threshold = float(option.edge_prune_threshold_)
    p.preference_loop_closure = float(option.preference_loop_closure_); p.reference_node = int(option.reference_node_)
    p.max_iteration = int(criteria.max_iteration_); p.min_relative_increment = float(criteria.min_relative_increment_)
    p.min_relative_residual_increment = float(criteria.min_relative_residual_increment_); p.min_right_term = float(criteria.min_right_term_)
    p.min_residual = float(criteria.min_residual_); p.max_iteration_lm = int(criteria.max_iteration_lm_)
    p.upper_scale_factor = float(criteria.upper_scale_factor_); p.lower_scale_factor = float(criteria.lower_scale_factor_)
    return p


def globalOptimization(eng: Engine, poseGraph: PoseGraph, criteria: GlobalOptimizationConvergenceCriteria | None = None,
                       option: GlobalOptimizationOption | None = None) -> list[GlobalOptimizationPassStats]:
    """[O3D] GlobalOptimization(pose_graph, GlobalOptimizationLevenbergMarquardt, criteria, option) on the device (one
    b2s_global_optimization call).  Like [O3D], poseGraph is updated in place: the node poses, and edges_ becomes the surviving edge set
    (with the confidences the optimisation ended with).  A graph that fails validation is left as it is.  Returns the two passes' stats."""
    criteria = criteria or GlobalOptimizationConvergenceCriteria()
    option = option or GlobalOptimizationOption()
    p = _go_params(criteria, option)
    n, ne = len(poseGraph.nodes_), len(poseGraph.edges_)
    poses = np.ascontiguousarray(np.stack([np.asarray(nd.pose_, dtype=np.float64) for nd in poseGraph.nodes_]) if n else np.zeros((0, 4, 4)))
    edges = (L.PoseGraphEdge * max(ne, 1))()
    for k, e in enumerate(poseGraph.edges_):
        edges[k].source, edges[k].target, edges[k].uncertain = int(e.source_node_id_), int(e.target_node_id_), int(bool(e.uncertain_))
        edges[k].T[:] = np.asarray(e.transformation_, dtype=np.float64).ravel().tolist()
        edges[k].information[:] = np.asarray(e.information_, dtype=np.float64).ravel().tolist()
    kept = np.zeros(max(ne, 1), dtype=np.int32)
    conf = np.zeros(max(ne, 1), dtype=np.float64)
    stats = (L.GlobalOptimizationStats * 2)()
    L.check(L.lib().b2s_global_optimization(eng._h, C.c_int32(n), _pd(poses), C.c_int32(ne), edges, C.byref(p), kept.ctypes.data_as(C.POINTER(C.c_int32)), _pd(conf), stats))
    out = [GlobalOptimizationPassStats(bool(s.valid), int(s.n_edges), int(s.outer_iterations), int(s.lm_tries), int(s.accepted_steps),
                                       L.LM_STOP_REASONS[s.stop_reason], float(s.initial_residual), float(s.final_residual), float(s.final_lambda))
           for s in stats]
    if ne > 0 and out[0].valid:
        for nd, T in zip(poseGraph.nodes_, poses):
            nd.pose_ = np.array(T)
        for e, c in zip(poseGraph.edges_, conf):
            e.confidence_ = float(c)
        poseGraph.edges_ = [e for e, k in zip(poseGraph.edges_, kept) if k]
    return out


def nearestNeighbors(eng: Engine, queries: Cloud, target: Cloud, maxCorrespondenceDistance: float, T=None):
    """The correspondence search of [O3D] RegistrationICP on its own (KDTreeFlann::SearchHybrid(q, r, 1) per query): index of the
    nearest target point with d^2 < r^2 (-1 = none), squared distance.  correspondence_set_ = this at the result's transformation."""
    n = len(queries)
    idx = np.full(max(n, 1), -1, dtype=np.int32); d2 = np.full(max(n, 1), -1.0)
    m = C.c_size_t()
    Tm = _mat(T) if T is not None else None
    L.check(L.lib().b2s_nearest_neighbors(eng._h, queries._c, target._c, C.c_double(maxCorrespondenceDistance), _pd(Tm) if Tm is not None else None,
                                          idx.ctypes.data_as(C.POINTER(C.c_int32)), _pd(d2), C.c_size_t(len(idx)), C.byref(m)))
    return idx[:n], d2[:n]


class Feature:
    """Device-resident [O3D] pipelines::registration::Feature (33 x n fp64), what Submap::computeFeatures keeps in feature_."""

    def __init__(self, eng: Engine, data=None):
        self.eng = eng
        self._f = C.c_void_p()
        L.check(L.lib().b2s_feature_create(eng._h, C.byref(self._f)))
        if data is not None:
            self.upload(data)

    def upload(self, data):
        """data_ as [O3D] holds it: a Dimension() x Num() matrix."""
        d = np.ascontiguousarray(np.asarray(data, dtype=np.float64).reshape(L.FEATURE_DIM, -1).T)
        L.check(L.lib().b2s_feature_upload(self.eng._h, self._f, _pd(d), C.c_size_t(len(d))))
        return self

    def Num(self) -> int:
        n = C.c_size_t()
        L.check(L.lib().b2s_feature_size(self.eng._h, self._f, C.byref(n)))
        return int(n.value)

    def Dimension(self) -> int:
        return L.FEATURE_DIM

    @property
    def data_(self) -> np.ndarray:
        n = self.Num()
        buf = np.empty((max(n, 1), L.FEATURE_DIM))
        m = C.c_size_t()
        L.check(L.lib().b2s_feature_download(self.eng._h, self._f, _pd(buf), C.c_size_t(len(buf)), C.byref(m)))
        return buf[:n].T.copy()

    def free(self):
        if self._f:
            L.lib().b2s_feature_destroy(self._f)
        self._f = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def computeFPFHFeature(eng: Engine, cloud: Cloud, radius: float, max_nn: int) -> Feature:
    """[O3D] ComputeFPFHFeature(cloud, KDTreeSearchParamHybrid(radius, max_nn)) as called at src/Submap.cpp:244 (max_nn <= 128)."""
    f = Feature(eng)
    L.check(L.lib().b2s_compute_fpfh(eng._h, cloud._c, C.c_double(radius), C.c_int32(max_nn), f._f))
    return f


@dataclass
class RansacResult(RegistrationResult):
    """RegistrationResult of RegistrationRANSACBasedOnFeatureMatching (n_corr = correspondence_set_.size() = inliers) plus how the
    run went: the h the loop stopped at, the validated hypotheses, the size of the feature correspondence set and whether it is the
    mutual one, and the h of the hypothesis the result comes from (-1 = none)."""
    hypotheses: int = 0
    validations: int = 0
    best_hypothesis: int = -1
    n_feature_corr: int = 0
    used_mutual: bool = False


def _ransac_res(r: L.RansacResult) -> RansacResult:
    b = _res(r.result)
    return RansacResult(b.transformation_, b.fitness_, b.inlier_rmse_, b.n_corr, b.iters, int(r.hypotheses), int(r.validations),
                        int(r.best_hypothesis), int(r.n_feature_corr), bool(r.used_mutual))


def registrationRANSACBasedOnFeatureMatchingBatch(eng: Engine, source: Cloud, targets, sourceFeature: Feature, targetFeatures,
                                                  params: PlaceRecognitionParameters | None = None, mutual_filter: bool = True):
    """[O3D] RegistrationRANSACBasedOnFeatureMatching of one source sparse cloud against every candidate, as
    src/PlaceRecognition.cpp:71-84 loops over them, in one device call.  Returns one RansacResult per target."""
    p = (params or PlaceRecognitionParameters()).ransac_c(mutual_filter)
    n = len(targets)
    assert len(targetFeatures) == n
    tc = (C.c_void_p * max(n, 1))(*[t._c for t in targets])
    tf = (C.c_void_p * max(n, 1))(*[f._f for f in targetFeatures])
    out = (L.RansacResult * max(n, 1))()
    L.check(L.lib().b2s_ransac_feature_matching(eng._h, source._c, sourceFeature._f, C.c_int32(n), tc, tf, C.byref(p), out))
    return [_ransac_res(out[k]) for k in range(n)]


def registrationRANSACBasedOnFeatureMatching(eng: Engine, source: Cloud, target: Cloud, sourceFeature: Feature, targetFeature: Feature,
                                             params: PlaceRecognitionParameters | None = None, mutual_filter: bool = True) -> RansacResult:
    """src/PlaceRecognition.cpp:81-84 for one candidate (mutual_filter = true there)."""
    return registrationRANSACBasedOnFeatureMatchingBatch(eng, source, [target], sourceFeature, [targetFeature], params, mutual_filter)[0]


def featureCorrespondences(eng: Engine, sourceFeature: Feature, targetFeature: Feature):
    """The exact nearest-feature indices both ways (src_to_tgt, tgt_to_src) that the RANSAC correspondence set is built from;
    -1 where the other feature is empty."""
    ns, nt = sourceFeature.Num(), targetFeature.Num()
    s2t = np.full(max(ns, 1), -1, dtype=np.int32); t2s = np.full(max(nt, 1), -1, dtype=np.int32)
    L.check(L.lib().b2s_feature_correspondences(eng._h, sourceFeature._f, targetFeature._f, s2t.ctypes.data_as(C.POINTER(C.c_int32)),
                                                C.c_size_t(len(s2t)), t2s.ctypes.data_as(C.POINTER(C.c_int32)), C.c_size_t(len(t2s))))
    return s2t[:ns], t2s[:nt]


class CloudRegistration:
    def registerClouds(self, source: Cloud, target: Cloud, init) -> RegistrationResult:  # pragma: no cover - abstract
        raise NotImplementedError

    def estimateNormalsOrCovariancesIfNeeded(self, cloud: Cloud) -> None:
        return None


class RegistrationIcpPointToPlane(CloudRegistration):
    """src/CloudRegistration.cpp:44-66"""

    def __init__(self, eng: Engine, p: CloudRegistrationParameters | None = None):
        self.eng = eng
        p = p or CloudRegistrationParameters(icp=eng.params.icp)
        self.maxCorrespondenceDistance_ = p.icp.maxCorrespondenceDistance
        self.knnNormalEstimation_ = p.icp.knn
        self.maxRadiusNormalEstimation_ = p.icp.maxDistanceKnn
        self.max_iteration_ = p.icp.maxNumIter

    _regType = "PointToPlaneIcp"

    def _apply(self):
        mp = self.eng.params
        if (mp.icp.maxCorrespondenceDistance, mp.icp.maxNumIter, mp.scanToMapRegType) != (self.maxCorrespondenceDistance_, self.max_iteration_,
                                                                                         self._regType):
            import copy
            mp = copy.deepcopy(mp)
            mp.icp.maxCorrespondenceDistance = self.maxCorrespondenceDistance_
            mp.icp.maxNumIter = self.max_iteration_
            mp.scanToMapRegType = self._regType
            self.eng.set_parameters(mp)

    def registerClouds(self, source: Cloud, target: Cloud, init) -> RegistrationResult:
        self._apply()
        T = _mat(init)
        r = L.Result()
        L.check(L.lib().b2s_register(self.eng._h, source._c, target._c, _pd(T), C.byref(r)))
        return _res(r)

    def registerCloudsBatch(self, sources, targets, inits):
        """n independent registrations in one launch (the loop of src/PlaceRecognition.cpp:71,111)."""
        self._apply()
        n = len(sources)
        S = (C.c_void_p * n)(*[s._c for s in sources]); Tg = (C.c_void_p * n)(*[t._c for t in targets])
        I = np.ascontiguousarray(np.asarray(inits, dtype=np.float64).reshape(n, 16))
        R = (L.Result * n)()
        L.check(L.lib().b2s_register_batch(self.eng._h, C.c_int32(n), S, Tg, _pd(I), R))
        return [_res(r) for r in R]

    def estimateNormalsOrCovariancesIfNeeded(self, cloud: Cloud) -> None:
        L.check(L.lib().b2s_estimate_normals(self.eng._h, cloud._c, C.c_int32(self.knnNormalEstimation_),
                                             C.c_double(self.maxRadiusNormalEstimation_)))


class RegistrationIcpPointToPoint(RegistrationIcpPointToPlane):
    """src/CloudRegistration.cpp:69-82: RegistrationICP with TransformationEstimationPointToPoint (Eigen::umeyama updates).
    The target needs no normals and estimateNormalsOrCovariancesIfNeeded is the base-class no-op."""
    _regType = "PointToPointIcp"

    def estimateNormalsOrCovariancesIfNeeded(self, cloud: Cloud) -> None:
        return None


class RegistrationIcpGeneralized(RegistrationIcpPointToPlane):
    """src/CloudRegistration.cpp:15-38: [O3D] RegistrationGeneralizedICP.  estimateNormalsOrCovariancesIfNeeded estimates
    NORMALS exactly like the point-to-plane class (the reference's EstimateCovariances call is commented out, :29), and [O3D]
    derives the per-point covariances from them -- so both clouds must carry normals."""
    _regType = "GeneralizedIcp"


def cloudRegistrationFactory(eng: Engine, p: CloudRegistrationParameters) -> CloudRegistration:
    """src/CloudRegistration.cpp:85-100"""
    if p.regType == "PointToPlaneIcp":
        return RegistrationIcpPointToPlane(eng, p)
    if p.regType == "PointToPointIcp":
        return RegistrationIcpPointToPoint(eng, p)
    if p.regType == "GeneralizedIcp":
        return RegistrationIcpGeneralized(eng, p)
    raise RuntimeError("cloud: unknown type of cloud registration")


# --------------------------------------------------------------------------------------------------------------------
# Submap (map side) and ScanToMapIcp
# --------------------------------------------------------------------------------------------------------------------


class Submap:
    """Device-resident Submap::mapCloud_ (+ dense map).  src/Submap.cpp:39-92,184-191"""

    def __init__(self, eng: Engine, capacity_points: int = 2_000_000):
        self.eng = eng
        self._s = C.c_void_p()
        L.check(L.lib().b2s_submap_create(eng._h, C.c_size_t(capacity_points), C.byref(self._s)))
        self.capacity = capacity_points
        self.nScansInsertedMap_ = 0
        self.nScansInsertedDenseMap_ = 0
        self._cropperPose = np.eye(4)   # mapBuilderCropper_'s pose: set AFTER each insertion (Submap.cpp:71), Identity before the first
        self.lastCarvedCount = 0
        self.sparseMapCloud_: Cloud | None = None
        self.feature_: Feature | None = None

    def setMapperOptions(self, *, minMovement: float = 0.0, carving: "SpaceCarvingParameters | None" = None, dense: bool = False,
                         denseCarving: "SpaceCarvingParameters | None" = None, denseCropper: "ScanCroppingParameters | None" = None) -> None:
        """What Mapper / SubmapCollection / SlamWrapper wire around S1-S2-F1 for this submap, decided on the device by the chain:
        minimum-motion gate (Mapper.cpp:170-176), carving every N insertions (Submap.cpp:55-60,109-123), dense-map feed with
        every accepted scan and its carving (SlamWrapper.cpp:318-327,363-376; Submap.cpp:77-92,125-136)."""
        o = L.MapperOptions()
        L.lib().b2s_default_mapper_options(C.byref(o))
        o.min_movement_between_mapping_steps = float(minMovement)
        if carving is not None:
            o.carve_enabled = 1; o.carve_every_n_scans = int(carving.carveSpaceEveryNscans); o.carving = carving.to_c()
        if dense:
            o.dense_enabled = 1
            if denseCarving is not None:
                o.dense_carve_every_n_scans = int(denseCarving.carveSpaceEveryNscans); o.dense_carving = denseCarving.to_c()
            if denseCropper is not None:
                o.dense_cropper = denseCropper.to_c()
        L.check(L.lib().b2s_submap_set_mapper_options(self.eng._h, self._s, C.byref(o)))

    def mapperCounters(self) -> dict:
        c = L.MapperCounters()
        L.check(L.lib().b2s_submap_get_mapper_counters(self.eng._h, self._s, C.byref(c)))
        return {n: int(getattr(c, n)) for n, _ in L.MapperCounters._fields_}

    def isEmpty(self) -> bool:
        return self.size() == 0

    def size(self) -> int:
        n = C.c_size_t()
        L.check(L.lib().b2s_submap_size(self.eng._h, self._s, C.byref(n)))
        return int(n.value)

    def insertScan(self, rawScan, preProcessedScan: Cloud, mapToRangeSensor, time=None, isPerformCarving=False) -> bool:
        T = _mat(mapToRangeSensor)
        if isPerformCarving:
            self.carve(rawScan, T, self.eng.params.mapBuilder.carving)
        L.check(L.lib().b2s_submap_insert(self.eng._h, self._s, preProcessedScan._c, _pd(T)))
        self._cropperPose = T.copy()
        self.nScansInsertedMap_ += 1
        return True

    def carve(self, rawScan: Cloud, mapToRangeSensor, params: "SpaceCarvingParameters", force: bool = False) -> int:
        """Submap::carve (src/Submap.cpp:109-123): only when nScansInsertedMap_ % carveSpaceEveryNscans_ == 1 and the map is
        not empty; the candidates are the map points inside the map-builder cropper at its LAST pose."""
        if not force and not (self.nScansInsertedMap_ % params.carveSpaceEveryNscans == 1):
            return 0
        if self.size() == 0:
            return 0
        T = _mat(mapToRangeSensor); P = np.ascontiguousarray(self._cropperPose, dtype=np.float64)
        prm = params.to_c(); n = C.c_size_t()
        L.check(L.lib().b2s_submap_carve(self.eng._h, self._s, rawScan._c, _pd(T), _pd(P), C.byref(prm), C.byref(n)))
        self.lastCarvedCount = int(n.value)
        return self.lastCarvedCount

    def insertScanDenseMap(self, rawScan: Cloud, mapToRangeSensor, denseCropper: L.Cropper | None = None, isPerformCarving: bool = False,
                           carving: "SpaceCarvingParameters | None" = None) -> bool:
        T = _mat(mapToRangeSensor)
        L.check(L.lib().b2s_submap_insert_dense(self.eng._h, self._s, rawScan._c, _pd(T), C.byref(denseCropper) if denseCropper else None))
        if isPerformCarving:   # Submap.cpp:86-89: after the insertion, with the raw scan and the map-frame sensor position
            prm = carving or self.eng.params.mapBuilder.carving
            if self.nScansInsertedDenseMap_ % prm.carveSpaceEveryNscans == 1:
                self.carveDenseMap(rawScan, T[:3, 3], prm)
        self.nScansInsertedDenseMap_ += 1
        return True

    def carveDenseMap(self, scan: Cloud, sensorPosition, params: "SpaceCarvingParameters") -> int:
        """Submap::carve(scan, sensorPosition, param, &denseMap_) (src/Submap.cpp:125-136), unconditionally."""
        s = np.ascontiguousarray(np.asarray(sensorPosition, dtype=np.float64).reshape(3)); prm = params.to_c(); n = C.c_size_t()
        L.check(L.lib().b2s_dense_carve(self.eng._h, self._s, scan._c, _pd(s), C.byref(prm), C.byref(n)))
        return int(n.value)

    def getMapPointCloud(self):
        n = self.size()
        xyz = np.empty((n, 3)); nrm = np.empty((n, 3)); m = C.c_size_t()
        L.check(L.lib().b2s_submap_download(self.eng._h, self._s, _pd(xyz), _pd(nrm), C.c_size_t(n), C.byref(m)))
        return xyz[:m.value], nrm[:m.value]

    def toCloud(self, out: "Cloud | None" = None) -> "Cloud":
        """getMapPointCloudCopy without leaving the device"""
        out = out if out is not None else Cloud(self.eng)
        L.check(L.lib().b2s_submap_to_cloud(self.eng._h, self._s, out._c))
        return out

    def getDenseMap(self, capacity=1 << 22):
        xyz = np.empty((capacity, 3)); keys = np.empty((capacity, 3), dtype=np.int32); m = C.c_size_t()
        L.check(L.lib().b2s_submap_dense_download(self.eng._h, self._s, _pd(xyz), None, keys.ctypes.data_as(C.POINTER(C.c_int32)),
                                                  C.c_size_t(capacity), C.byref(m)))
        return xyz[:m.value].copy(), keys[:m.value].copy()

    def getDenseMapPointCloud(self, out: "Cloud | None" = None) -> "Cloud":
        """getDenseMapCopy().toPointCloud() (src/Voxel.cpp:90-115) without leaving the device: the dense map's voxel means in slot
        order, no normals (b2s_assemble_dense_maps of this submap alone)"""
        return assembleDenseMaps(self.eng, [self], out)[0]

    # ---- VoxelHashMap query interface on the dense map (include/open3d_slam/VoxelHashMap.hpp:104-158), batched ----
    def denseQuery(self, points: Cloud, with_means: bool = True):
        """hasVoxelContainingPoint / getVoxelContainingPointPtr for every point: (counts, aggregated positions or None)."""
        n = len(points)
        counts = np.zeros(n, dtype=np.int32); means = np.zeros((n, 3)) if with_means else None
        L.check(L.lib().b2s_dense_query(self.eng._h, self._s, points._c, counts.ctypes.data_as(C.POINTER(C.c_int32)),
                                        _pd(means) if with_means else None, C.c_size_t(n)))
        return counts, means

    def denseRemove(self, points: Cloud) -> None:
        """removeKey(getKey(p)) for every point."""
        L.check(L.lib().b2s_dense_remove(self.eng._h, self._s, points._c))

    def denseSize(self) -> int:
        n = C.c_size_t()
        L.check(L.lib().b2s_dense_size(self.eng._h, self._s, C.byref(n)))
        return int(n.value)

    def denseClear(self) -> None:
        L.check(L.lib().b2s_dense_clear(self.eng._h, self._s))

    def transform(self, T) -> None:
        """Submap::transform (src/Submap.cpp:94-107): map cloud, dense map and mapToRangeSensor_ follow a loop-closure correction."""
        L.check(L.lib().b2s_submap_transform(self.eng._h, self._s, _pd(_mat(T))))
        self._cropperPose = self._cropperPose   # mapBuilderCropper_ keeps its pose in the reference as well

    def transformSparseMapCloud(self, T) -> None:
        """The sparseMapCloud_ line of Submap::transform (src/Submap.cpp:96): [O3D] PointCloud::Transform of the feature cloud in place
        (a no-op before computeFeatures)."""
        if self.sparseMapCloud_ is not None:
            L.check(L.lib().b2s_cloud_transform_inplace(self.eng._h, self.sparseMapCloud_._c, _pd(_mat(T))))

    def setMapPointCloud(self, cloud: Cloud):
        L.check(L.lib().b2s_submap_set_cloud(self.eng._h, self._s, cloud._c))

    def setInitialMap(self, cloud: Cloud, mapVoxelSize: float) -> None:
        """Submap::insertScan's initial-map branch (src/Submap.cpp:47-52): the map becomes VoxelDownSample(cloud, mapVoxelSize), normals
        averaged, without carving or fusion; nScansInsertedMap_ is not counted.  cloud carries the normals prepareInitialMap estimated."""
        L.check(L.lib().b2s_submap_set_initial_map(self.eng._h, self._s, cloud._c, C.c_double(float(mapVoxelSize))))

    def setInitialTransform(self, T) -> None:
        """Mapper::setMapToRangeSensorInitial (src/Mapper.cpp:87-91) on the device pose slot: the next step keeps T (see b2s.h)"""
        L.check(L.lib().b2s_submap_set_initial_transform(self.eng._h, self._s, _pd(_mat(T))))

    def globalLocalization(self, rawCloud: "Cloud", params: "GlobalLocalizationParameters | None" = None,
                           minRefinementFitness: float = 0.0) -> "GlobalLocalizationResult":
        """b2s_submap_global_localization (include/b2s.h): the map_to_sensor of rawCloud in this submap's map without an initial pose.
        Reads the submap and changes nothing; apply the pose with setInitialTransform."""
        return globalLocalization(self.eng, self, rawCloud, params, minRefinementFitness)

    def setMergeScans(self, on: bool) -> None:
        """isMergeScansIntoMap_ for the device chain on this submap: off = pure localisation (src/Mapper.cpp:163-167)"""
        L.check(L.lib().b2s_submap_set_merge_scans(self.eng._h, self._s, C.c_int32(1 if on else 0)))

    def computeFeatures(self, params: PlaceRecognitionParameters | None = None) -> None:
        """The feature half of Submap::computeFeatures (src/Submap.cpp:239-244): sparse cloud (voxel down-sample of the map), its
        normals, their FPFH -- on the device, kept on this object.  Repeated calls reuse the same cloud and feature."""
        prm = (params or PlaceRecognitionParameters()).to_c()
        if self.sparseMapCloud_ is None:
            self.sparseMapCloud_ = Cloud(self.eng)
            self.feature_ = Feature(self.eng)
        L.check(L.lib().b2s_submap_compute_features(self.eng._h, self._s, C.byref(prm), self.sparseMapCloud_._c, self.feature_._f))

    def getSparseMapPointCloud(self) -> Cloud:
        if self.sparseMapCloud_ is None:
            raise RuntimeError("Submap::getSparseMapPointCloud: computeFeatures has not run")
        return self.sparseMapCloud_

    def getFeatures(self) -> "Feature":
        if self.feature_ is None:
            raise RuntimeError("Feature ptr is nullptr")   # Submap.cpp:250 assert_nonNullptr
        return self.feature_

    def setPose(self, T):
        T = _mat(T)
        L.check(L.lib().b2s_submap_set_pose(self.eng._h, self._s, _pd(T)))

    def getPose(self):
        T = np.empty((4, 4))
        L.check(L.lib().b2s_submap_get_pose(self.eng._h, self._s, _pd(T)))
        return T

    def free(self):
        for o in (getattr(self, "sparseMapCloud_", None), getattr(self, "feature_", None)):
            if o is not None:
                o.free()
        self.sparseMapCloud_ = self.feature_ = None
        if self._s:
            L.lib().b2s_submap_destroy(self._s)
            self._s = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class VoxelMap:
    """o3d_slam::VoxelMap (include/open3d_slam/Voxel.hpp:19-36, src/Voxel.cpp:123-160) on the device; layers are named like
    the reference's and mapped to small integers."""

    def __init__(self, eng: Engine, voxelSize=0.25, capacity_voxels: int = 1 << 20):
        self.eng = eng
        v = np.ascontiguousarray(np.broadcast_to(np.asarray(voxelSize, dtype=np.float64), (3,)))
        self._v = C.c_void_p()
        L.check(L.lib().b2s_voxel_map_create(eng._h, _pd(v), C.c_size_t(capacity_voxels), C.byref(self._v)))
        self._layers = {}

    def _layer(self, name: str) -> int:
        if name not in self._layers:
            self._layers[name] = len(self._layers)
        return self._layers[name]

    def clear(self) -> None:
        L.check(L.lib().b2s_voxel_map_clear(self.eng._h, self._v))

    def insertCloud(self, layer: str, cloud: Cloud) -> None:
        L.check(L.lib().b2s_voxel_map_insert_cloud(self.eng._h, self._v, C.c_int32(self._layer(layer)), cloud._c))

    def size(self) -> int:
        n = C.c_size_t()
        L.check(L.lib().b2s_voxel_map_size(self.eng._h, self._v, C.byref(n)))
        return int(n.value)

    def hasVoxelContainingPoint(self, points: Cloud, T=None):
        """batched: (flags per point, number of hits); T (optional) moves the points first (isSwitchingSubmapsConsistant)."""
        n = len(points)
        flags = np.zeros(max(n, 1), dtype=np.int32); hits = C.c_size_t()
        Tm = _mat(T) if T is not None else None
        L.check(L.lib().b2s_voxel_map_has_voxel(self.eng._h, self._v, points._c, _pd(Tm) if Tm is not None else None,
                                                flags.ctypes.data_as(C.POINTER(C.c_int32)), C.c_size_t(len(flags)), C.byref(hits)))
        return flags[:n].astype(bool), int(hits.value)

    def getIndicesInVoxel(self, layer: str, points: Cloud):
        """batched getIndicesInVoxel(layer, p): list of index arrays, one per query point."""
        if layer not in self._layers:
            return [np.zeros(0, dtype=np.int64) for _ in range(len(points))]
        n = len(points)
        offs = np.zeros(n + 1, dtype=np.int32); tot = C.c_size_t()
        lay = C.c_int32(self._layers[layer])
        L.check(L.lib().b2s_voxel_map_indices_in_voxel(self.eng._h, self._v, lay, points._c, offs.ctypes.data_as(C.POINTER(C.c_int32)),
                                                       C.c_size_t(n + 1), None, C.c_size_t(0), C.byref(tot)))
        idx = np.zeros(max(int(tot.value), 1), dtype=np.int32)
        L.check(L.lib().b2s_voxel_map_indices_in_voxel(self.eng._h, self._v, lay, points._c, offs.ctypes.data_as(C.POINTER(C.c_int32)),
                                                       C.c_size_t(n + 1), idx.ctypes.data_as(C.POINTER(C.c_int32)), C.c_size_t(len(idx)),
                                                       C.byref(tot)))
        return [idx[offs[i]:offs[i + 1]].astype(np.int64) for i in range(n)]

    def free(self):
        if self._v:
            L.lib().b2s_voxel_map_destroy(self._v)
            self._v = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


@dataclass
class ProcessedScans:
    merge_: Cloud
    match_: Cloud


class ScanToMapRegistration:
    pass


class ScanToMapIcp(ScanToMapRegistration):
    """src/ScanToMapRegistration.cpp:19-89"""

    def __init__(self, eng: Engine):
        self.eng = eng
        self.params_ = eng.params

    def setParameters(self, p: MapperParameters):
        self.params_ = p
        self.eng.set_parameters(p)

    def processForScanMatchingAndMerging(self, rawScan: Cloud, mapToRangeSensor=None) -> ProcessedScans:
        merge, match = Cloud(self.eng), Cloud(self.eng)
        L.check(L.lib().b2s_process_scan(self.eng._h, rawScan._c, merge._c, match._c))
        # assert_gt(narrowCropped / wideCropped size, 0)   ScanToMapRegistration.cpp:51-52
        self.eng.synchronize()
        return ProcessedScans(merge, match)

    def scanToMapRegistration(self, scan: Cloud, activeSubmap: Submap, mapToRangeSensor, initialGuess) -> RegistrationResult:
        T0 = _mat(mapToRangeSensor); T1 = _mat(initialGuess)
        r = L.Result()
        L.check(L.lib().b2s_register_to_submap(self.eng._h, scan._c, activeSubmap._s, _pd(T0), _pd(T1), C.byref(r)))
        return _res(r)

    def isMergeScanValid(self, cloud: Cloud) -> bool:
        return cloud.HasNormals()

    def prepareInitialMap(self, mapCloud: Cloud) -> None:
        ic = self.params_.icp
        L.check(L.lib().b2s_estimate_normals(self.eng._h, mapCloud._c, C.c_int32(ic.knn), C.c_double(ic.maxDistanceKnn)))


def scanToMapRegistrationFactory(eng: Engine, p: MapperParameters) -> ScanToMapRegistration:
    """src/ScanToMapRegistration.cpp:91-103"""
    if p.scanToMapRegType in ("PointToPlaneIcp", "GeneralizedIcp", "PointToPointIcp"):
        # one ScanToMapIcp for all three, like the reference; its cloud registration follows toCloudRegistrationType (:105-129).
        # Note for PointToPointIcp: the reference's estimateNormalsOrCovariancesIfNeeded is a no-op there, so its merge_/match_
        # clouds and its map carry no normals; the device chain still estimates and carries them (the estimator ignores
        # them and the map positions are the same).
        s = ScanToMapIcp(eng)
        s.setParameters(p)
        return s
    raise RuntimeError("scanToMapRegistrationFactory: unknown type of registration scan to map")


@dataclass
class OdometryParameters:
    """include/open3d_slam/Parameters.hpp:155-159 (scanMatcher_ + scanProcessing_); defaults = the Lua odometry block"""
    scanMatcher: CloudRegistrationParameters = field(default_factory=CloudRegistrationParameters)
    scanProcessing: ScanProcessingParameters = field(default_factory=ScanProcessingParameters)
    seed: int = 0
    minFitness: float = 0.1        # the "todo magic" of Odometry.cpp:51
    bufferSize: int = 2000         # odomToRangeSensorBuffer_ size limit (TransformInterpolationBuffer())

    def to_c(self) -> L.OdometryParams:
        reg_type = regTypeOf(self.scanMatcher.regType)
        p = L.OdometryParams()
        L.lib().b2s_default_odometry_params(C.byref(p))
        ic = self.scanMatcher.icp
        p.icp.reg_type = reg_type
        p.icp.max_iter, p.icp.max_corr_dist, p.icp.knn, p.icp.knn_radius = int(ic.maxNumIter), float(ic.maxCorrespondenceDistance), int(ic.knn), float(ic.maxDistanceKnn)
        p.voxel_size = float(self.scanProcessing.voxelSize)
        p.downsampling_ratio = float(self.scanProcessing.downSamplingRatio)
        p.seed = int(self.seed)
        p.cropper = self.scanProcessing.cropper.to_c()
        p.min_fitness = float(self.minFitness)
        p.buffer_size = int(self.bufferSize)
        return p


@dataclass
class ConstantVelocityMotionCompensationParameters:
    """include/open3d_slam/Parameters.hpp:192-197; defaults = parameter_structure_definitions.lua:33-36 (de-skew off)"""
    isUndistortInputCloud: bool = False      # motion_compensation.is_undistort_scan
    isSpinningClockwise: bool = True
    scanDuration: float = 0.1                # seconds
    numPosesVelocityEstimation: int = 3

    def to_c(self) -> L.MotionCompensationParams:
        p = L.MotionCompensationParams()
        L.lib().b2s_default_motion_compensation_params(C.byref(p))
        p.enabled = int(bool(self.isUndistortInputCloud))
        p.spinning_clockwise = int(bool(self.isSpinningClockwise))
        p.scan_duration = float(self.scanDuration)
        p.num_poses_velocity_estimation = int(self.numPosesVelocityEstimation)
        return p


@dataclass
class MotionCompensationStepResult:
    """b2s_motion_compensation_result: the velocities each de-skew of a step used and whether they moved the points"""
    odometryLinearVelocity: np.ndarray
    odometryAngularVelocityRpy: np.ndarray
    mapLinearVelocity: np.ndarray
    mapAngularVelocityRpy: np.ndarray
    odometryApplied: bool
    mapApplied: bool


class LidarOdometry:
    """src/Odometry.cpp:19-79 -- scan-to-scan odometry: preprocess = crop -> voxelize -> estimateNormalsOrCovariancesIfNeeded ->
    RandomDownSample; addRangeScan registers the PREVIOUS pre-processed cloud (source) against the new one (target) from Identity
    and accumulates odomToRangeSensorCumulative_ *= result^-1.  Host control flow here, every stage on the device."""

    def __init__(self, eng: Engine, params: OdometryParameters | None = None):
        self.eng = eng
        self.params_ = params or OdometryParameters()
        self.cloudRegistration_ = cloudRegistrationFactory(eng, self.params_.scanMatcher)
        self.cloudPrev_: Cloud | None = None
        self.odomToRangeSensorCumulative_ = np.eye(4)
        self.buffer = []            # odomToRangeSensorBuffer_ (timestamp, transform)
        self.lastResult: RegistrationResult | None = None

    def preprocess(self, cloud: Cloud) -> Cloud:   # :25-30
        sp = self.params_.scanProcessing
        c = crop(self.eng, cloud, sp.cropper.to_c())
        v = voxelize(self.eng, c, sp.voxelSize)
        self.cloudRegistration_.estimateNormalsOrCovariancesIfNeeded(v)
        out = random_down_sample(self.eng, v, sp.downSamplingRatio, self.params_.seed)
        c.free(); v.free()
        return out

    def addRangeScan(self, cloud: Cloud, timestamp=None) -> bool:   # :32-79
        pre = self.preprocess(cloud)
        if self.cloudPrev_ is None or len(self.cloudPrev_) == 0:
            self.cloudPrev_ = pre
            self.buffer.append((timestamp, self.odomToRangeSensorCumulative_.copy()))
            return True
        result = self.cloudRegistration_.registerClouds(self.cloudPrev_, pre, np.eye(4))
        self.lastResult = result
        isOdomOkay = result.fitness_ > 0.1   # "todo magic" in the reference
        if not isOdomOkay:
            if len(pre) > 0:
                self.cloudPrev_.free(); self.cloudPrev_ = pre
            return False
        self.odomToRangeSensorCumulative_ = self.odomToRangeSensorCumulative_ @ np.linalg.inv(result.transformation_)
        self.cloudPrev_.free()
        self.cloudPrev_ = pre
        self.buffer.append((timestamp, self.odomToRangeSensorCumulative_.copy()))
        return True

    def getOdomToRangeSensor(self) -> np.ndarray:
        return self.odomToRangeSensorCumulative_.copy()


@dataclass
class OdometryStepResult:
    """b2s_odometry_result: the registration of the step (zeros when it initialised), the cumulative pose after it, the outcome"""
    registration: RegistrationResult
    odomToRangeSensor: np.ndarray
    outcome: int
    nPreprocessed: int


def _odo_res(r: L.OdometryResult) -> OdometryStepResult:
    return OdometryStepResult(_res(r.registration), np.array(r.odom_to_range_sensor, dtype=np.float64).reshape(4, 4), int(r.outcome),
                              int(r.n_preprocessed))


@dataclass
class SlamStepResult:
    """b2s_slam_result: the odometry step, the scan-to-map registration, whether the prediction came from the odometry buffer and
    whether the mapper accepted the scan"""
    odometry: OdometryStepResult
    mapper: RegistrationResult
    odomUsed: bool
    mapperAccepted: bool


def _slam_res(r: L.SlamResult) -> SlamStepResult:
    return SlamStepResult(_odo_res(r.odometry), _res(r.mapper), bool(r.odom_used), bool(r.mapper_accepted))


class _OdometryBuffer:
    """LidarOdometry::getBuffer() as far as callers read it: has(t)"""

    def __init__(self, odo: "DeviceLidarOdometry"):
        self.odo = odo

    def has(self, t: int) -> bool:
        return self.odo._lookup(t)[1]


class DeviceLidarOdometry:
    """src/Odometry.cpp:19-110 on the device (b2s_odometry): its own parameters, cloudPrev_, cumulative pose and
    TransformInterpolationBuffer.  addRangeScan only enqueues; fetchResult reads the outcome of a step.  Timestamps are
    UniversalTimeScaleClock ticks (100 ns) and must increase from call to call."""

    def __init__(self, eng: Engine, params: OdometryParameters | None = None, capacity_points: int = 200_000):
        self.eng = eng
        self.params_ = params or OdometryParameters()
        self._o = C.c_void_p()
        p = self.params_.to_c()
        L.check(L.lib().b2s_odometry_create(eng._h, C.byref(p), C.c_size_t(capacity_points), C.byref(self._o)))

    def setParameters(self, params: OdometryParameters):
        p = params.to_c()
        L.check(L.lib().b2s_odometry_set_params(self.eng._h, self._o, C.byref(p)))
        self.params_ = params

    def setInitialTransform(self, T):
        M = _mat(T)
        L.check(L.lib().b2s_odometry_set_initial_transform(self.eng._h, self._o, _pd(M)))

    def addRangeScan(self, cloud: Cloud, t: int, slot: int = 0) -> int:
        L.check(L.lib().b2s_odometry_step_async(self.eng._h, self._o, cloud._c, C.c_int64(int(t)), C.c_int32(slot)))
        return slot

    def fetchResult(self, slot: int = 0) -> OdometryStepResult:
        r = L.OdometryResult()
        L.check(L.lib().b2s_odometry_result_fetch(self.eng._h, self._o, C.c_int32(slot), C.byref(r)))
        return _odo_res(r)

    def _lookup(self, t: int):
        T = np.zeros(16, dtype=np.float64)
        has = C.c_int32()
        L.check(L.lib().b2s_odometry_lookup(self.eng._h, self._o, C.c_int64(int(t)), _pd(T), C.byref(has)))
        return T.reshape(4, 4), bool(has.value)

    def getOdomToRangeSensor(self, t: int) -> np.ndarray:
        """getTransform(t, odomToRangeSensorBuffer_)"""
        return self._lookup(t)[0]

    def getBuffer(self) -> _OdometryBuffer:
        return _OdometryBuffer(self)

    def getPreProcessedCloud(self) -> Cloud:
        c = Cloud(self.eng)
        L.check(L.lib().b2s_odometry_preprocessed(self.eng._h, self._o, c._c))
        return c

    def enableGraph(self, raw_capacity_points: int = 65536) -> Cloud:
        """Replay the combined odometry + mapper step as CUDA graphs (one per submap).  Returns the staging cloud every scan
        must be uploaded / copied into."""
        st = C.c_void_p()
        L.check(L.lib().b2s_slam_graph_enable(self.eng._h, self._o, C.c_size_t(raw_capacity_points), C.byref(st)))
        c = Cloud.__new__(Cloud)
        c.eng = self.eng; c._c = st; c._borrowed = True
        self._staging = c
        return c

    def exportState(self) -> bytes:
        """The object's device state as one self-contained blob (b2s_odometry_export_state)"""
        n = C.c_size_t()
        L.check(L.lib().b2s_odometry_export_state(self.eng._h, self._o, None, C.c_size_t(0), C.byref(n)))
        buf = np.empty(int(n.value), dtype=np.uint8)
        L.check(L.lib().b2s_odometry_export_state(self.eng._h, self._o, buf.ctypes.data_as(C.c_void_p), C.c_size_t(int(n.value)), C.byref(n)))
        return buf.tobytes()

    @classmethod
    def importState(cls, eng: Engine, blob: bytes, params: OdometryParameters | None = None) -> "DeviceLidarOdometry":
        """A new object on eng holding exactly the exported state (b2s_odometry_import_state).  The device parameters come from the
        blob; params (optional) is only the host-side copy setParameters would keep."""
        blob = bytes(blob)
        od = cls.__new__(cls)
        od.eng, od.params_, od._o = eng, params, C.c_void_p()
        L.check(L.lib().b2s_odometry_import_state(eng._h, blob, C.c_size_t(len(blob)), C.byref(od._o)))
        return od

    def fetchSlamResult(self, slot: int = 0) -> SlamStepResult:
        r = L.SlamResult()
        L.check(L.lib().b2s_slam_result_fetch(self.eng._h, self._o, C.c_int32(slot), C.byref(r)))
        return _slam_res(r)

    # -- motion compensation (de-skew) of both inputs of a step, SlamWrapper.cpp:195-200,266-268,298-304
    def setMotionCompensation(self, params: ConstantVelocityMotionCompensationParameters):
        p = params.to_c()
        L.check(L.lib().b2s_odometry_set_motion_compensation(self.eng._h, self._o, C.byref(p)))

    def pushMapToRangeSensor(self, t: int, T):
        """mapToRangeSensorBuffer_.push(t, T) (Mapper.cpp:112,145); the combined step pushes every accepted scan itself"""
        M = _mat(T)
        L.check(L.lib().b2s_slam_map_pose_push(self.eng._h, self._o, C.c_int64(int(t)), _pd(M)))

    def _map_lookup(self, t: int):
        T = np.zeros(16, dtype=np.float64)
        has = C.c_int32()
        L.check(L.lib().b2s_slam_map_lookup(self.eng._h, self._o, C.c_int64(int(t)), _pd(T), C.byref(has)))
        return T.reshape(4, 4), bool(has.value)

    def getMapToRangeSensor(self, t: int) -> np.ndarray:
        """Mapper::getMapToRangeSensor(t) = getTransform(t, mapToRangeSensorBuffer_)"""
        return self._map_lookup(t)[0]

    def fetchMotionCompensation(self, slot: int = 0) -> MotionCompensationStepResult:
        r = L.MotionCompensationResult()
        L.check(L.lib().b2s_slam_motion_fetch(self.eng._h, self._o, C.c_int32(slot), C.byref(r)))
        v = lambda a: np.array(a, dtype=np.float64)   # noqa: E731
        return MotionCompensationStepResult(v(r.odometry_linear_velocity), v(r.odometry_angular_velocity_rpy), v(r.map_linear_velocity),
                                            v(r.map_angular_velocity_rpy), bool(r.odometry_applied), bool(r.map_applied))

    def undistortedScans(self) -> tuple[Cloud, Cloud]:
        """device copies of the last step's de-skewed odometry input and mapper input"""
        a, b = Cloud(self.eng), Cloud(self.eng)
        L.check(L.lib().b2s_slam_undistorted(self.eng._h, self._o, a._c, b._c))
        return a, b

    def free(self):
        if getattr(self, "_o", None) and self._o.value:
            L.lib().b2s_odometry_destroy(self._o)
            self._o = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Mapper:
    """Host control flow of Mapper::addRangeMeasurement (src/Mapper.cpp:101-181), single active submap, no carving.
    The odometry prediction is supplied per call as `odometryMotion` (odomToRangeSensorPrev^-1 * odomToRangeSensor)."""

    def __init__(self, eng: Engine, submap_capacity: int = 2_000_000):
        self.eng = eng
        self.params_ = eng.params
        self.scan2MapReg_ = scanToMapRegistrationFactory(eng, eng.params)
        self.submap = Submap(eng, submap_capacity)
        self.mapToRangeSensor_ = np.eye(4)
        self.mapToRangeSensorPrev_ = np.eye(4)
        self.mapToRangeSensorLastScanInsertion_ = np.eye(4)
        self._first = True
        self.isNewInitialValueSet_ = False
        self.isIgnoreOdometryPrediction_ = False
        self.lastResult = None
        if self.params_.isUseInitialMap and not self.params_.isMergeScansIntoMap:
            self.submap.setMergeScans(False)

    def setInitialMap(self, mapCloud: Cloud) -> None:
        """SlamWrapper::setInitialMap (src/SlamWrapper.cpp:209-220) with isUseInitialMap_: prepareInitialMap (normals on the full map),
        then the first-scan branch of addRangeMeasurement (Mapper.cpp:106-108), which loads the map voxelized (Submap.cpp:47-52)."""
        if not self.params_.isUseInitialMap:
            raise RuntimeError("setInitialMap needs MapperParameters.isUseInitialMap")
        self.scan2MapReg_.prepareInitialMap(mapCloud)
        if not self.scan2MapReg_.isMergeScanValid(mapCloud):
            raise RuntimeError("Init map invalid!!!!")   # assert_true at Mapper.cpp:107
        self.submap.setInitialMap(mapCloud, self.params_.mapBuilder.mapVoxelSize)
        self._first = False

    def setMapToRangeSensorInitial(self, T) -> None:
        """src/Mapper.cpp:87-91, on the host state and on the device pose slot the device chain reads"""
        self.mapToRangeSensor_ = _mat(T).copy()
        self.mapToRangeSensorPrev_ = self.mapToRangeSensor_.copy()
        self.isNewInitialValueSet_ = True
        if self.submap is not None:
            self.submap.setInitialTransform(T)

    def _deviceStep(self) -> None:
        """a device step applied rules 3 / the ignore-once rule to the device words: the host copies follow, so that the host flow
        and the device chain can be mixed on one Mapper"""
        self.isIgnoreOdometryPrediction_ = self.isNewInitialValueSet_
        self.isNewInitialValueSet_ = False

    def addRangeMeasurement(self, rawScan: Cloud, odometryMotion=None) -> bool:
        if self._first:  # Mapper.cpp:105-114
            processed = self.scan2MapReg_.processForScanMatchingAndMerging(rawScan, self.mapToRangeSensor_)
            self.submap.insertScan(rawScan, processed.merge_, np.eye(4))
            self._first = False
            return True
        predict = odometryMotion is not None and not self.isNewInitialValueSet_ and not self.isIgnoreOdometryPrediction_   # :130-137
        estimate = self.mapToRangeSensorPrev_ @ _mat(odometryMotion) if predict else self.mapToRangeSensorPrev_
        self.isIgnoreOdometryPrediction_ = False
        processed = self.scan2MapReg_.processForScanMatchingAndMerging(rawScan, self.mapToRangeSensor_)
        result = self.scan2MapReg_.scanToMapRegistration(processed.match_, self.submap, self.mapToRangeSensor_, estimate)
        self.lastResult = result
        if self.isNewInitialValueSet_:   # :143-149: the result is discarded, the pose stays the initial value
            self.mapToRangeSensorPrev_ = self.mapToRangeSensor_.copy()
            self.isNewInitialValueSet_ = False
            self.isIgnoreOdometryPrediction_ = True
            return True
        if (not self.params_.isIgnoreMinRefinementFitness) and result.fitness_ < self.params_.minRefinementFitness:
            return False  # Mapper.cpp:151-156
        self.mapToRangeSensor_ = result.transformation_.copy()
        if self.params_.isUseInitialMap and not self.params_.isMergeScansIntoMap:   # :163-167 pure localisation
            self.mapToRangeSensorPrev_ = self.mapToRangeSensor_.copy()
            return True
        motion = np.linalg.inv(self.mapToRangeSensorLastScanInsertion_) @ self.mapToRangeSensor_
        if not (np.linalg.norm(motion[:3, 3]) < self.params_.minMovementBetweenMappingSteps):
            self.submap.insertScan(rawScan, processed.merge_, self.mapToRangeSensor_)
            self.mapToRangeSensorLastScanInsertion_ = self.mapToRangeSensor_.copy()
        self.mapToRangeSensorPrev_ = self.mapToRangeSensor_.copy()
        return True

    # ---- asynchronous device-resident chain (no host round trip per scan) ---------------------------------------------
    def enableGraph(self, raw_capacity_points: int = 65536) -> "Cloud":
        """Replay the per-scan chain as one CUDA graph.  Returns the staging cloud every scan must be uploaded / copied into;
        in graph mode addRangeMeasurementAsync ignores its `slot` argument and returns the slot it used."""
        st = C.c_void_p()
        L.check(L.lib().b2s_mapper_graph_enable(self.eng._h, self.submap._s, C.c_size_t(raw_capacity_points),
                                                C.c_double(self.params_.minRefinementFitness),
                                                C.c_int32(int(self.params_.isIgnoreMinRefinementFitness)), C.byref(st)))
        c = Cloud.__new__(Cloud)
        c.eng = self.eng; c._c = st; c._borrowed = True
        self._staging = c
        self._gstep = 0
        return c

    def stageCopy(self, src: Cloud):
        """device->device copy of a resident cloud into the graph staging cloud"""
        L.check(L.lib().b2s_cloud_copy(self.eng._h, src._c, self._staging._c))

    def addRangeMeasurementAsync(self, rawScan: Cloud, odometryMotion, slot: int = 0):
        if getattr(self, "_staging", None) is not None:
            slot = self._gstep % 256
            self._gstep += 1
        M = _mat(odometryMotion)
        self._deviceStep()
        L.check(L.lib().b2s_mapper_step_async(self.eng._h, self.submap._s, rawScan._c, _pd(M), C.c_double(self.params_.minRefinementFitness),
                                              C.c_int32(int(self.params_.isIgnoreMinRefinementFitness)), C.c_int32(slot)))
        return slot

    def addRangeMeasurementHost(self, xyz_f32_ptr: int, n: int, odometryMotion, stride: int = 12) -> RegistrationResult:
        """End to end with host buffers: float32 scan (pinned host pointer) in, RegistrationResult out, one C call."""
        M = _mat(odometryMotion)
        r = L.Result()
        self._deviceStep()
        L.check(L.lib().b2s_mapper_step_host(self.eng._h, self.submap._s, C.c_void_p(xyz_f32_ptr), C.c_size_t(n), C.c_size_t(stride), _pd(M),
                                             C.c_double(self.params_.minRefinementFitness),
                                             C.c_int32(int(self.params_.isIgnoreMinRefinementFitness)), C.byref(r)))
        if getattr(self, "_staging", None) is not None:
            self._gstep += 1
        return _res(r)

    def addRangeMeasurementHostAsync(self, xyz_f32_ptr: int, n: int, odometryMotion, out_pinned_ptr: int, stride: int = 12) -> None:
        """Like addRangeMeasurementHost but only enqueues: the b2s_result lands at out_pinned_ptr (page-locked host memory,
        ctypes layout _lib.Result) once the engine's stream has been synchronised."""
        M = _mat(odometryMotion)
        self._deviceStep()
        L.check(L.lib().b2s_mapper_step_host_async(self.eng._h, self.submap._s, C.c_void_p(xyz_f32_ptr), C.c_size_t(n), C.c_size_t(stride), _pd(M),
                                                   C.c_double(self.params_.minRefinementFitness),
                                                   C.c_int32(int(self.params_.isIgnoreMinRefinementFitness)), C.c_void_p(out_pinned_ptr)))
        if getattr(self, "_staging", None) is not None:
            self._gstep += 1

    def lastProcessedScan(self, merge: bool = True, match: bool = False, merge_into: "Cloud | None" = None) -> ProcessedScans:
        """Copies of the merge_ / match_ clouds the last device step produced (SubmapCollection buffers merge_ for the overlap
        between consecutive submaps, src/SubmapCollection.cpp:83-92,180).  merge_into: an existing cloud to overwrite."""
        m = merge_into if merge_into is not None else (Cloud(self.eng) if merge else None)
        a = Cloud(self.eng) if match else None
        # (Cloud has __len__: no truth tests on clouds)
        L.check(L.lib().b2s_mapper_processed_scan(self.eng._h, m._c if m is not None else None, a._c if a is not None else None))
        return ProcessedScans(m, a)

    def fetchResult(self, slot: int = 0) -> RegistrationResult:
        r = L.Result()
        L.check(L.lib().b2s_scan_result_fetch(self.eng._h, C.c_int32(slot), C.byref(r)))
        return _res(r)

    # ---- odometry + mapper for the same scan, the prediction read from the odometry's buffer on the device --------------------
    def addRangeMeasurementWithOdometry(self, odometry: DeviceLidarOdometry, rawScan: Cloud, t: int, slot: int = 0) -> int:
        """odometry.addRangeScan(rawScan, t), then addRangeMeasurement(rawScan, t) on the active submap (b2s_slam_step_async): only
        enqueues; odometry.fetchSlamResult(slot) reads the result.  After odometry.enableGraph() rawScan must be its staging cloud."""
        self._deviceStep()
        L.check(L.lib().b2s_slam_step_async(self.eng._h, self.submap._s, odometry._o, rawScan._c, C.c_int64(int(t)),
                                            C.c_double(self.params_.minRefinementFitness), C.c_int32(int(self.params_.isIgnoreMinRefinementFitness)),
                                            C.c_int32(slot)))
        return slot

    def addRangeMeasurementWithOdometryHostAsync(self, odometry: DeviceLidarOdometry, xyz_f32_ptr: int, n: int, t: int, out_pinned_ptr: int,
                                                 stride: int = 12) -> None:
        """The same from a float32 host scan: upload, both chains and the copy of the b2s_slam_result to out_pinned_ptr (page-locked
        host memory, ctypes layout _lib.SlamResult, valid once the engine's stream has been synchronised) are only enqueued."""
        self._deviceStep()
        L.check(L.lib().b2s_slam_step_host_async(self.eng._h, self.submap._s, odometry._o, C.c_void_p(xyz_f32_ptr), C.c_size_t(n), C.c_size_t(stride),
                                                 C.c_int64(int(t)), C.c_double(self.params_.minRefinementFitness),
                                                 C.c_int32(int(self.params_.isIgnoreMinRefinementFitness)), C.c_void_p(out_pinned_ptr)))


# --------------------------------------------------------------------------------------------------------------------
# global localisation in a prior map (b2s_submap_global_localization, DESIGN.md row M3)
# --------------------------------------------------------------------------------------------------------------------
@dataclass
class GlobalLocalizationParameters:
    """b2s_global_localization_params.  A box with xMin > xMax (the default) is the xy extent of the map's live points."""
    xMin: float = 1.0
    xMax: float = -1.0
    yMin: float = 1.0
    yMax: float = -1.0
    step: float = 0.25
    z0: float = 0.0
    zStep: float = 0.25
    nZ: int = 1
    nYaw: int = 144
    yaw0: float = -math.pi
    yawStep: float = 2.0 * math.pi / 144.0
    roll: float = 0.0
    pitch: float = 0.0
    scoreVoxel: float = 1.0
    nCandidates: int = 16
    nmsDistance: float = 1.0
    nmsYaw: float = math.radians(10.0)

    def to_c(self) -> L.GlobalLocalizationParams:
        return L.GlobalLocalizationParams(self.xMin, self.xMax, self.yMin, self.yMax, self.step, self.z0, self.zStep, int(self.nZ), int(self.nYaw),
                                          self.yaw0, self.yawStep, self.roll, self.pitch, self.scoreVoxel, int(self.nCandidates), 0,
                                          self.nmsDistance, self.nmsYaw)


@dataclass
class GlobalLocalizationCandidate:
    T_hypothesis: np.ndarray
    hypothesis: int
    hits: int
    icp: RegistrationResult


@dataclass
class GlobalLocalizationResult:
    found: bool
    T: np.ndarray
    fitness: float
    inlier_rmse: float
    runner_up_fitness: float     # -1: no candidate beyond the suppression distances of the winner
    winner_rank: int             # -1: no candidate
    n_hypotheses: int
    n_query: int
    candidates: list             # GlobalLocalizationCandidate in rank order


def globalLocalization(eng: Engine, submap: "Submap", rawCloud: "Cloud", params: GlobalLocalizationParameters | None = None,
                       minRefinementFitness: float = 0.0) -> GlobalLocalizationResult:
    """Localise rawCloud (sensor frame) in submap's map with no initial pose (b2s_submap_global_localization)."""
    p = (params or GlobalLocalizationParameters()).to_c()
    cap = max(int(p.n_candidates), 1)
    cands = (L.GlobalLocalizationCandidate * cap)()
    out = L.GlobalLocalizationResult()
    L.check(L.lib().b2s_submap_global_localization(eng._h, submap._s, rawCloud._c, C.byref(p), C.c_double(float(minRefinementFitness)), cands,
                                                   C.c_int32(cap), C.byref(out)))
    cl = [GlobalLocalizationCandidate(np.array(c.T_hypothesis, dtype=np.float64).reshape(4, 4), int(c.hypothesis), int(c.hits), _res(c.icp))
          for c in cands[:out.n_candidates]]
    return GlobalLocalizationResult(bool(out.found), np.array(out.T, dtype=np.float64).reshape(4, 4), float(out.fitness), float(out.inlier_rmse),
                                    float(out.runner_up_fitness), int(out.winner_rank), int(out.n_hypotheses), int(out.n_query), cl)


def debugGlobalLocalizationScores(eng: Engine, submap: "Submap", rawCloud: "Cloud", params: GlobalLocalizationParameters | None = None):
    """b2s_debug_global_localization_scores: (hits per hypothesis, query cloud)"""
    p = (params or GlobalLocalizationParameters()).to_c()
    nh, nq = C.c_size_t(0), C.c_size_t(0)
    one = np.zeros(1, dtype=np.int32)
    rc = L.lib().b2s_debug_global_localization_scores(eng._h, submap._s, rawCloud._c, C.byref(p), one.ctypes.data_as(C.c_void_p), C.c_size_t(0),
                                                      C.byref(nh), None, C.c_size_t(0), C.byref(nq))
    if rc != L.E_CAPACITY or nh.value == 0:
        L.check(rc)
    hits = np.zeros(nh.value, dtype=np.int32)
    q = np.zeros((nq.value, 3), dtype=np.float64)
    L.check(L.lib().b2s_debug_global_localization_scores(eng._h, submap._s, rawCloud._c, C.byref(p), hits.ctypes.data_as(C.c_void_p),
                                                         C.c_size_t(hits.size), C.byref(nh), q.ctypes.data_as(C.c_void_p), C.c_size_t(len(q)),
                                                         C.byref(nq)))
    return hits, q


# --------------------------------------------------------------------------------------------------------------------
# global localisation over every submap of a session (b2s_submaps_global_localization, DESIGN.md row M4)
# --------------------------------------------------------------------------------------------------------------------
@dataclass
class SubmapsGlobalLocalizationResult(GlobalLocalizationResult):
    """GlobalLocalizationResult over a list of submaps: the submap (list index) each candidate was refined in, and the winner's"""
    candidate_submaps: list = None   # int per entry of candidates
    winner_submap: int = -1          # -1: no candidate


def _centers(submaps, centers) -> np.ndarray:
    c = np.ascontiguousarray(np.asarray(centers, dtype=np.float64).reshape(-1, 3))
    if len(c) != len(submaps):
        raise ValueError(f"{len(c)} centres for {len(submaps)} submaps")
    return c


def globalLocalizationInSubmaps(eng: Engine, submaps, centers, rawCloud: "Cloud", params: GlobalLocalizationParameters | None = None,
                                minRefinementFitness: float = 0.0) -> SubmapsGlobalLocalizationResult:
    """Localise rawCloud (sensor frame) in the union of the Submaps' maps with no initial pose (b2s_submaps_global_localization, one
    device call).  centers (n x 3, map frame): Submap::getMapToSubmapCenter of each, which picks the submap a candidate is refined in."""
    n, arr = _submap_array(submaps)
    c = _centers(submaps, centers)
    p = (params or GlobalLocalizationParameters()).to_c()
    cap = max(int(p.n_candidates), 1)
    cands = (L.GlobalLocalizationCandidate * cap)()
    owners = (C.c_int32 * cap)()
    out = L.GlobalLocalizationResult()
    win = C.c_int32(-1)
    L.check(L.lib().b2s_submaps_global_localization(eng._h, arr, C.c_int32(n), _pd(c), rawCloud._c, C.byref(p), C.c_double(float(minRefinementFitness)),
                                                    cands, C.c_int32(cap), owners, C.byref(out), C.byref(win)))
    cl = [GlobalLocalizationCandidate(np.array(k.T_hypothesis, dtype=np.float64).reshape(4, 4), int(k.hypothesis), int(k.hits), _res(k.icp))
          for k in cands[:out.n_candidates]]
    return SubmapsGlobalLocalizationResult(bool(out.found), np.array(out.T, dtype=np.float64).reshape(4, 4), float(out.fitness),
                                           float(out.inlier_rmse), float(out.runner_up_fitness), int(out.winner_rank), int(out.n_hypotheses),
                                           int(out.n_query), cl, [int(owners[k]) for k in range(out.n_candidates)], int(win.value))


def debugGlobalLocalizationScoresInSubmaps(eng: Engine, submaps, rawCloud: "Cloud", params: GlobalLocalizationParameters | None = None):
    """b2s_debug_submaps_global_localization_scores: (hits per hypothesis over the union of the submaps, query cloud)"""
    n, arr = _submap_array(submaps)
    p = (params or GlobalLocalizationParameters()).to_c()
    nh, nq = C.c_size_t(0), C.c_size_t(0)
    one = np.zeros(1, dtype=np.int32)
    rc = L.lib().b2s_debug_submaps_global_localization_scores(eng._h, arr, C.c_int32(n), rawCloud._c, C.byref(p), one.ctypes.data_as(C.c_void_p),
                                                              C.c_size_t(0), C.byref(nh), None, C.c_size_t(0), C.byref(nq))
    if rc != L.E_CAPACITY or nh.value == 0:
        L.check(rc)
    hits = np.zeros(nh.value, dtype=np.int32)
    q = np.zeros((nq.value, 3), dtype=np.float64)
    L.check(L.lib().b2s_debug_submaps_global_localization_scores(eng._h, arr, C.c_int32(n), rawCloud._c, C.byref(p),
                                                                 hits.ctypes.data_as(C.c_void_p), C.c_size_t(hits.size), C.byref(nh),
                                                                 q.ctypes.data_as(C.c_void_p), C.c_size_t(len(q)), C.byref(nq)))
    return hits, q
