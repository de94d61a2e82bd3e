"""Host control flow of the full mapper (config 5 of BASELINE.json) around the device hot path.

What stays on the host in the reference and is restated here as plain control flow (paths relative to
/root/reference/open3d_slam/open3d_slam/):
    Mapper::addRangeMeasurement                                   src/Mapper.cpp:101-181
    SubmapCollection::insertScan / updateActiveSubmap / createNewSubmap / insertBufferedScans / findClosestSubmap /
    isSwitchingSubmapsConsistant                                  src/SubmapCollection.cpp:83-131,133-158,172-207,352-364
    Submap::computeSubmapCenter / computeFeatures (voxel map part) src/Submap.cpp:228-259
    PlaceRecognition::buildLoopClosureConstraints for given candidates: RANSAC proposal -> correspondence gate -> consistency
    check -> refinement (overlap -> ICP -> information matrix) -> consistency check      src/PlaceRecognition.cpp:50-229
    computeOdometryConstraints / buildOdometryConstraint: the constraints between consecutive submaps, all missing pairs in one
    batched device call                                           src/constraint_builders.cpp:23-118
Every arithmetic step is a call into a *backend*: `DeviceBackend` (below) drives libb2s.so; the parity tests run the very
same control flow over a CPU backend built on the oracle (tests/oracle_backend.py) -- the product never imports it.

The per-scan step of the device backend is ONE C call with host buffers (float32 scan in, RegistrationResult out) that
replays the captured CUDA graph of the chain S1 -> S2 -> gates -> [carving] -> F1 -> [dense map]; the host decisions
(submap hand-over, revisits) are taken from the returned result, like the reference's mapping thread does.
"""
from __future__ import annotations

import collections
import copy
import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _lib as L
from . import engine as E


@dataclass
class SubmapParameters:
    """include/open3d_slam/Parameters.hpp:100-106"""
    radius: float = 20.0
    minNumRangeData: int = 5
    adjacencyBasedRevisitingMinFitness: float = 0.4
    numScansOverlap: int = 3


@dataclass
class LoopClosureParameters:
    """the PlaceRecognitionParameters the refinement half reads (Parameters.hpp:132-135) + magic.hpp:14"""
    maxIcpCorrespondenceDistance: float = 0.3
    minRefinementFitness: float = 0.7
    maxNumIter: int = 100                       # magic::icpRunUntilConvergenceNumberOfIterations
    voxelExpansionFactorOverlapComputation: float = 20.0
    minNumPointsPerVoxel: int = 1


VOXEL_EXPANSION_ADJACENCY_REVISITING = 2.5     # magic::voxelExpansionFactorAdjacencyBasedRevisiting
VOXEL_MAP_LAYER = "map"                        # Submap::voxelMapLayer


@dataclass
class SubmapRecord:
    """What SubmapCollection knows about one Submap besides its clouds."""
    handle: object                      # backend submap object
    id: int
    parent: int
    origin: np.ndarray                  # mapToSubmap_ translation at creation
    center: np.ndarray | None = None    # computeSubmapCenter() once finished
    has_voxel_map: bool = False
    sparse: object = None               # computeFeatures(): sparseMapCloud_ (backend cloud) ...
    feature: object = None              # ... and feature_ (backend feature)

    def mapToSubmapCenter(self) -> np.ndarray:   # Submap::getMapToSubmapCenter
        return self.center if self.center is not None else self.origin


class SubmapCollection:
    """src/SubmapCollection.cpp, the parts Mapper::addRangeMeasurement reaches (no place recognition, no optimisation)."""

    def __init__(self, backend, params: SubmapParameters):
        self.backend = backend
        self.params = params
        self.submaps: list[SubmapRecord] = []
        self.activeSubmapIdx = 0
        self.numScansMergedInActiveSubmap = 0
        assert params.numScansOverlap <= 14   # DeviceBackend recycles merge_ clouds through a ring of 16
        self.overlapScansBuffer = collections.deque(maxlen=params.numScansOverlap)   # CircularBuffer, :216
        self.finishedSubmapsIdxs: list[int] = []
        self.adjacency: set[tuple[int, int]] = set()
        self.loopClosureSubmaps: set[int] = set()   # adjacencyMatrix_.markAsLoopClosureSubmap
        self.odometryConstraints: list = []          # odometryConstraints_ (SubmapCollection::computeFeatures appends to it)
        self.isUseInitialMap = False                 # MapperParameters::isUseInitialMap_: localisation mode never hands over (:105-107)
        self.events: list[tuple] = []   # (scan index, what, ...) -- compared between backends by the parity test

    # -- helpers
    def getActiveSubmap(self) -> SubmapRecord:
        return self.submaps[self.activeSubmapIdx]

    def isAdjacent(self, a: int, b: int) -> bool:
        return (min(a, b), max(a, b)) in self.adjacency

    def createNewSubmap(self, mapToSubmap: np.ndarray) -> None:   # :133-145
        rec = SubmapRecord(self.backend.new_submap(), len(self.submaps), self.activeSubmapIdx, np.array(mapToSubmap[:3, 3], dtype=np.float64))
        self.submaps.append(rec)
        self.activeSubmapIdx = len(self.submaps) - 1
        self.numScansMergedInActiveSubmap = 0

    def findClosestSubmap(self, mapToRangeSensor: np.ndarray) -> int:   # :147-158 (std::min_element: first minimum)
        p0 = mapToRangeSensor[:3, 3]
        d = [float(np.linalg.norm(p0 - s.mapToSubmapCenter())) for s in self.submaps]
        return int(np.argmin(d))

    def updateActiveSubmap(self, mapToRangeSensor: np.ndarray, scan) -> None:   # :94-131
        if self.numScansMergedInActiveSubmap < self.params.minNumRangeData:
            return
        if self.isUseInitialMap:   # "do not switch maps if we are doing in the localization mode"
            return
        closest = self.findClosestSubmap(mapToRangeSensor)
        closestSubmap, activeSubmap = self.submaps[closest], self.submaps[self.activeSubmapIdx]
        p = mapToRangeSensor[:3, 3]
        if np.linalg.norm(p - closestSubmap.mapToSubmapCenter()) < self.params.radius:
            if closest == self.activeSubmapIdx:
                return
            if self.isAdjacent(closestSubmap.id, activeSubmap.id) and self.isSwitchingSubmapsConsistant(scan, closest, mapToRangeSensor):
                self.activeSubmapIdx = closest
            elif np.linalg.norm(p - activeSubmap.mapToSubmapCenter()) > self.params.radius:
                self.createNewSubmap(mapToRangeSensor)
        else:
            self.createNewSubmap(mapToRangeSensor)

    def isSwitchingSubmapsConsistant(self, scan, candidate: int, mapToRangeSensor: np.ndarray) -> bool:   # :352-364
        rec = self.submaps[candidate]
        if not rec.has_voxel_map:          # a default-constructed VoxelMap is empty: no point hits a voxel
            fitness = 0.0
        else:
            fitness = self.backend.revisit_fitness(rec.handle, scan, mapToRangeSensor)
        self.events.append(("revisit_check", candidate, fitness))
        return fitness > self.params.adjacencyBasedRevisitingMinFitness

    def finishSubmap(self, idx: int) -> None:
        """computeSubmapCenter (:184) and the voxel-map half of Submap::computeFeatures (Submap.cpp:233-237), which the
        reference runs asynchronously once a submap is finished (SlamWrapper::computeFeaturesIfReady)."""
        rec = self.submaps[idx]
        rec.center = self.backend.map_center(rec.handle)
        self.backend.build_voxel_map(rec.handle)
        rec.has_voxel_map = True

    def computeFeatures(self, params: E.PlaceRecognitionParameters | None = None) -> list[int]:
        """SubmapCollection::computeFeatures (src/SubmapCollection.cpp:219-243): the loop-closure features of every finished submap
        (Submap::computeFeatures, src/Submap.cpp:239-244), kept on its record.  Returns the submaps it computed, in order -- the
        reference queues them as loop-closure candidates.  The reference's worker thread, its odometry constraints and the
        minSecondsBetweenFeatureComputation_ timer are host policy and stay with the caller; the mapper never calls this."""
        params = params or E.PlaceRecognitionParameters()
        for idx in self.finishedSubmapsIdxs:
            rec = self.submaps[idx]
            rec.sparse, rec.feature = self.backend.compute_features(rec.handle, params)
        return list(self.finishedSubmapsIdxs)

    def getOdometryConstraints(self) -> list:
        return list(self.odometryConstraints)

    def updateAdjacencyMatrix(self, loopClosureConstraints) -> None:   # :75-81
        for c in loopClosureConstraints:
            self.adjacency.add((min(c.sourceSubmapIdx, c.targetSubmapIdx), max(c.sourceSubmapIdx, c.targetSubmapIdx)))
            self.loopClosureSubmaps.update((c.sourceSubmapIdx, c.targetSubmapIdx))

    def transformSubmap(self, idx: int, T: np.ndarray) -> None:
        """Submap::transform (src/Submap.cpp:94-107): the map, the dense map and the sparse feature cloud ([O3D] PointCloud::Transform),
        mapToRangeSensor_ * T on the submap's pose, submapCenter_ = T * submapCenter_.  The revisit VoxelMap is not moved, as in the
        reference.  A submap whose center has not been computed yet keeps using its origin (mapToSubmap_, which Submap::transform
        leaves alone as well)."""
        rec = self.submaps[idx]
        T = np.asarray(T, dtype=np.float64)
        self.backend.transform_submap(rec.handle, rec.sparse, T)
        if rec.center is not None:
            rec.center = T[:3, :3] @ rec.center + T[:3, 3]
        self.events.append(("transform", idx))

    def transform(self, transformIncrements) -> None:
        """SubmapCollection::transform (src/SubmapCollection.cpp:284-335): every submap of the graph by its increment; every other
        submap by the increment of its first ancestor that is in the graph; then the overlap buffer is flushed."""
        optimized = []
        for u in transformIncrements:
            if u.submapId_ < len(self.submaps):
                self.transformSubmap(u.submapId_, u.dT_)
                optimized.append(u.submapId_)
            else:   # the reference prints "This should not happen!" and goes on
                self.events.append(("transform_out_of_range", u.submapId_))
        toUpdate = sorted(set(range(len(self.submaps))) - set(optimized))
        for idx in toUpdate:
            if not transformIncrements:
                break
            cur = idx
            while True:
                cur = self.submaps[cur].parent
                if cur not in toUpdate:   # the parent is in the pose graph
                    self.transformSubmap(idx, transformIncrements[cur].dT_)
                    break
                if cur == self.submaps[cur].parent:
                    raise RuntimeError("Stuck in a loop, this should not happen")
        self.overlapScansBuffer.clear()

    # -- the call the mapper makes after an accepted registration (:172-207).  The scan itself has ALREADY been fused into the
    # submap that was active during the registration (with carving), because the device chain does that without a host
    # round trip; in the reference that is either branch of :185-204 (prevActive.insertScan / active.insertScan, both on
    # the submap that was active during the registration).
    def afterInsertion(self, scan_index: int, preProcessedScan, mapToRangeSensor: np.ndarray) -> None:
        if len(self.submaps) == 0:
            raise RuntimeError("SubmapCollection: no submap")
        self.overlapScansBuffer.append((preProcessedScan, np.array(mapToRangeSensor)))   # addScanToBuffer :83-85
        prev = self.activeSubmapIdx
        self.updateActiveSubmap(mapToRangeSensor, preProcessedScan)
        if prev != self.activeSubmapIdx:
            self.finishSubmap(prev)
            self.finishedSubmapsIdxs.append(prev)
            self.numScansMergedInActiveSubmap = 0
            a, b = self.submaps[prev].id, self.submaps[self.activeSubmapIdx].id
            self.adjacency.add((min(a, b), max(a, b)))
            self.events.append(("active_submap_changed", scan_index, prev, self.activeSubmapIdx))
            while self.overlapScansBuffer:   # insertBufferedScans :87-92 (no carving)
                cloud, T = self.overlapScansBuffer.popleft()
                self.backend.insert_scan(self.submaps[self.activeSubmapIdx].handle, cloud, T)
            self.backend.set_pose(self.submaps[self.activeSubmapIdx].handle, mapToRangeSensor)
        self.numScansMergedInActiveSubmap += 1


class SegmentMapper:
    """Mapper::addRangeMeasurement over a SubmapCollection, one scan per call (src/Mapper.cpp:101-181)."""

    def __init__(self, backend, submapParams: SubmapParameters | None = None):
        self.backend = backend
        self.submaps = SubmapCollection(backend, submapParams or SubmapParameters())
        self.mapToRangeSensor = np.eye(4)
        self.results: list = []
        self.poses: list[np.ndarray] = []
        self._k = 0
        mp = getattr(backend, "params", None)   # MapperParameters (a backend without them maps)
        self.isUseInitialMap = bool(mp is not None and mp.isUseInitialMap)
        self.isMergeScansIntoMap = bool(mp is not None and mp.isMergeScansIntoMap)
        self.submaps.isUseInitialMap = self.isUseInitialMap
        self.isNewInitialValueSet = False   # Mapper::isNewInitialValueSet_ (the backend keeps the device's copy)

    def setInitialMap(self, mapXyz: np.ndarray) -> None:
        """SlamWrapper::setInitialMap (src/SlamWrapper.cpp:209-220) with isUseInitialMap_: the backend estimates the normals on the full
        map (prepareInitialMap) and loads it voxelized (Submap.cpp:47-52); SubmapCollection::insertScan buffers it for the overlap,
        keeps the active submap and counts one merged scan (SubmapCollection.cpp:172-207).  Nothing is pushed to the pose buffer."""
        sc = self.submaps
        if not self.isUseInitialMap:
            raise RuntimeError("setInitialMap needs MapperParameters.isUseInitialMap")
        if sc.submaps:
            raise RuntimeError("setInitialMap: the map already holds scans")
        sc.createNewSubmap(np.eye(4))
        prepared = self.backend.initial_map(sc.getActiveSubmap().handle, mapXyz)
        sc.overlapScansBuffer.append((prepared, np.eye(4)))
        sc.numScansMergedInActiveSubmap += 1

    def setInitialTransform(self, T: np.ndarray) -> None:
        """SlamWrapper::setInitialTransform (src/SlamWrapper.cpp:222-225): the odometry's initial transform and
        Mapper::setMapToRangeSensorInitial (Mapper.cpp:87-91).  The device pose slot lives in the submap: load the map first."""
        if not self.submaps.submaps:
            raise RuntimeError("setInitialTransform: no submap yet (call setInitialMap first)")
        self.mapToRangeSensor = np.array(T, dtype=np.float64)
        self.isNewInitialValueSet = True
        self.backend.set_initial_transform(self.submaps.getActiveSubmap().handle, self.mapToRangeSensor)

    def addRangeMeasurement(self, rawScanF32: np.ndarray, odometryMotion: np.ndarray):
        sc = self.submaps
        k = self._k
        self._k += 1
        if not sc.submaps:   # Mapper.cpp:105-114 / SubmapCollection.cpp:176-181
            sc.createNewSubmap(self.mapToRangeSensor)
            merge = self.backend.first_scan(sc.getActiveSubmap().handle, rawScanF32)
            sc.numScansMergedInActiveSubmap += 1
            self.poses.append(self.mapToRangeSensor.copy())
            self.results.append(None)
            del merge
            return None
        active = sc.getActiveSubmap()
        res, inserted = self.backend.step(active.handle, rawScanF32, odometryMotion)
        return self._after_step(k, res, inserted)

    def addRangeScan(self, rawScanF32: np.ndarray, t: int):
        """One scan of SlamWrapper's odometry and mapping workers from the raw scan and its timestamp alone (UniversalTimeScaleClock
        ticks, increasing): the backend runs the scan-to-scan odometry and the scan-to-map step with the prediction read from the
        odometry's buffer (DeviceBackend: one b2s_slam_step_host_async).  The first scan initialises both."""
        sc = self.submaps
        k = self._k
        self._k += 1
        if not sc.submaps:
            sc.createNewSubmap(self.mapToRangeSensor)
            self.backend.first_scan_with_odometry(sc.getActiveSubmap().handle, rawScanF32, t)
            sc.numScansMergedInActiveSubmap += 1
            self.poses.append(self.mapToRangeSensor.copy())
            self.results.append(None)
            return None
        res, inserted = self.backend.step_with_odometry(sc.getActiveSubmap().handle, rawScanF32, t)
        return self._after_step(k, res, inserted)

    def loopClosureUpdate(self, loopClosureCorrection: np.ndarray) -> None:
        """Mapper::loopClosureUpdate (src/Mapper.cpp:44-47): mapToRangeSensor_ = dT * mapToRangeSensor_.  The device keeps one pose
        slot per submap for both the reference's Submap::mapToRangeSensor_ (which SubmapCollection.transform right-multiplies) and
        Mapper::mapToRangeSensor_, and the next step predicts from it: after the update the active submap's slot holds dT * (the mapper
        pose before the update).  The odometry's pose buffer is left alone, as in the reference."""
        self.mapToRangeSensor = np.asarray(loopClosureCorrection, dtype=np.float64) @ self.mapToRangeSensor
        if self.submaps.submaps:
            self.backend.loop_closure_update(self.submaps.getActiveSubmap().handle, self.mapToRangeSensor)

    def _after_step(self, k: int, res, inserted: bool):
        sc = self.submaps
        self.results.append(res)
        if self.isNewInitialValueSet:   # Mapper.cpp:143-149: the result is discarded, the pose stays the initial value, nothing is inserted
            self.isNewInitialValueSet = False
        elif inserted:
            self.mapToRangeSensor = np.array(res.transformation_, dtype=np.float64)
            if not (self.isUseInitialMap and not self.isMergeScansIntoMap):   # :163-167: pure localisation never inserts
                sc.afterInsertion(k, self.backend.last_merge_cloud(), self.mapToRangeSensor)
        self.poses.append(self.mapToRangeSensor.copy())
        return res


def refineLoopClosures(backend, source_handle, target_handles, initial_guesses, mapVoxelSize: float, p: LoopClosureParameters | None = None):
    """The refinement half of PlaceRecognition::buildLoopClosureConstraints for one finished (source) submap against its
    candidate (target) submaps, src/PlaceRecognition.cpp:96-149: overlap selection with voxel = 20 x map voxel, ICP of the
    overlapping parts from the proposal, fitness gate, information matrix.  The n registrations run as one batch.
    Returns a list of dicts {overlap sizes, result, accepted, information}."""
    p = p or LoopClosureParameters()
    voxel = p.voxelExpansionFactorOverlapComputation * mapVoxelSize
    pairs = [backend.overlap(source_handle, t, T0, voxel, p.minNumPointsPerVoxel) for t, T0 in zip(target_handles, initial_guesses)]
    results = backend.register_batch([so for so, _to in pairs], [to for _so, to in pairs], initial_guesses, p.maxIcpCorrespondenceDistance, p.maxNumIter)
    out = []
    for (so, to), r in zip(pairs, results):
        acc = not (r.fitness_ < p.minRefinementFitness)
        info = backend.information_matrix(so, to, p.maxIcpCorrespondenceDistance, r.transformation_) if acc else None
        out.append({"n_source_overlap": backend.cloud_size(so), "n_target_overlap": backend.cloud_size(to), "result": r, "accepted": acc,
                    "information": info})
    return out


@dataclass
class LoopClosureConsistencyCheck:
    """PlaceRecognitionConsistencyCheckParameters (Parameters.hpp:108-115) with the Lua values (parameter_structure_definitions.lua:
    142-147): 30 deg roll / pitch / yaw, 80 / 80 / 40 m.  The C++ struct's own defaults differ (90 deg, 10 / 10 / 15 m)."""
    maxDriftRoll: float = np.deg2rad(30.0)
    maxDriftPitch: float = np.deg2rad(30.0)
    maxDriftYaw: float = np.deg2rad(30.0)
    maxDriftX: float = 80.0
    maxDriftY: float = 80.0
    maxDriftZ: float = 40.0

    def isRegistrationConsistent(self, T) -> bool:
        """PlaceRecognition::isRegistrationConsistent (src/PlaceRecognition.cpp:182-229): |roll|, |pitch|, |yaw| of toRPY and |x|, |y|,
        |z| of the translation within the limits (a NaN angle passes, as the reference's comparisons do)."""
        T = np.asarray(T, dtype=np.float64)
        r, p, y = toRPY(T[:3, :3])
        return not (abs(r) > self.maxDriftRoll or abs(p) > self.maxDriftPitch or abs(y) > self.maxDriftYaw or abs(T[0, 3]) > self.maxDriftX
                    or abs(T[1, 3]) > self.maxDriftY or abs(T[2, 3]) > self.maxDriftZ)


def toRPY(R) -> tuple[float, float, float]:
    """src/math.cpp:39-46 on Eigen::Quaterniond(R): normalise, then getRoll/Pitch/YawFromQuat (math.hpp:30-42).  The quaternion's sign
    does not matter: every term is a product of two components."""
    R = np.asarray(R, dtype=np.float64)
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    if tr > 0.0:                                     # Eigen's quaternion from a rotation matrix (the larger-diagonal branches)
        t = np.sqrt(tr + 1.0); w = 0.5 * t; t = 0.5 / t
        x, y, z = (R[2, 1] - R[1, 2]) * t, (R[0, 2] - R[2, 0]) * t, (R[1, 0] - R[0, 1]) * t
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        q = [0.0, 0.0, 0.0]
        q[i] = 0.5 * t; t = 0.5 / t
        w = (R[k, j] - R[j, k]) * t
        q[j] = (R[j, i] + R[i, j]) * t; q[k] = (R[k, i] + R[i, k]) * t
        x, y, z = q
    n = np.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    roll = np.arctan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y))
    pitch = np.arcsin(2 * (w * y - x * z)) if abs(2 * (w * y - x * z)) <= 1.0 else np.nan
    yaw = np.arctan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))
    return float(roll), float(pitch), float(yaw)


@dataclass
class Constraint:
    """include/open3d_slam/Constraint.hpp:14-20 (the timestamp stays with the caller)"""
    sourceToTarget: np.ndarray
    sourceSubmapIdx: int
    targetSubmapIdx: int
    informationMatrix: np.ndarray
    isInformationMatrixValid: bool = True
    isOdometryConstraint: bool = False


def buildLoopClosureConstraints(backend, collection: SubmapCollection, sourceIdx: int, candidateIdxs, params: E.PlaceRecognitionParameters,
                                mapVoxelSize: float, lc: LoopClosureParameters | None = None,
                                consistency: LoopClosureConsistencyCheck | None = None):
    """PlaceRecognition::buildLoopClosureConstraints (src/PlaceRecognition.cpp:50-176) for a source submap and the candidates the caller
    selected (getLoopClosureCandidatesIdxs stays with the caller).  Every candidate: RANSAC proposal (all candidates in one batched
    call, :81-84) -> correspondence-set gate (:86) -> consistency of the RANSAC T (:92) -> refineLoopClosures on the survivors (one
    batch, :96-118) -> consistency of the ICP T (:124).  The records need sparse / feature (SubmapCollection.computeFeatures).
    Returns (constraints, log): log holds one entry per candidate, (target index, decision, RANSAC inliers), decision one of
    "accepted", "rejected_correspondences", "rejected_ransac_inconsistent", "rejected_refinement_fitness", "rejected_icp_inconsistent"."""
    lc = lc or LoopClosureParameters()
    consistency = consistency or LoopClosureConsistencyCheck()
    src = collection.submaps[sourceIdx]
    cands = list(candidateIdxs)
    if not cands:
        return [], []
    if src.feature is None or any(collection.submaps[i].feature is None for i in cands):
        raise RuntimeError("Feature ptr is nullptr")   # Submap.cpp:250 assert_nonNullptr: computeFeatures has not run
    tg = [collection.submaps[i] for i in cands]
    proposals = backend.ransac(src.sparse, src.feature, [t.sparse for t in tg], [t.feature for t in tg], params)
    decision, survivors = {}, []
    for i, r in zip(cands, proposals):
        if r.n_corr < params.ransacMinCorrespondenceSetSize:
            decision[i] = "rejected_correspondences"
        elif not consistency.isRegistrationConsistent(r.transformation_):
            decision[i] = "rejected_ransac_inconsistent"
        else:
            survivors.append((i, r))
    constraints = []
    if survivors:
        sc = backend.submap_as_cloud(src.handle)
        tcs = [backend.submap_as_cloud(collection.submaps[i].handle) for i, _ in survivors]
        refined = refineLoopClosures(backend, sc, tcs, [r.transformation_ for _, r in survivors], mapVoxelSize, lc)
        for (i, _r), o in zip(survivors, refined):
            T = np.array(o["result"].transformation_, dtype=np.float64)
            if not o["accepted"]:
                decision[i] = "rejected_refinement_fitness"
            elif not consistency.isRegistrationConsistent(T):
                decision[i] = "rejected_icp_inconsistent"
            else:
                decision[i] = "accepted"
                constraints.append(Constraint(T, src.id, collection.submaps[i].id, np.array(o["information"])))
    log = [(i, decision[i], int(r.n_corr)) for i, r in zip(cands, proposals)]
    return constraints, log


def hasConstraint(sourceIdx: int, targetIdx: int, constraints) -> bool:
    """src/constraint_builders.cpp:23-30"""
    return any(c.sourceSubmapIdx == sourceIdx and c.targetSubmapIdx == targetIdx for c in constraints)


def _odometry_constraint(collection: SubmapCollection, sourceIdx: int, targetIdx: int, r) -> Constraint:
    """buildConstraint's record (src/constraint_builders.cpp:75-82) from a backend result (T, information, ...)"""
    return Constraint(np.array(r.sourceToTarget_, dtype=np.float64), collection.submaps[sourceIdx].id, collection.submaps[targetIdx].id,
                      np.array(r.informationMatrix_, dtype=np.float64), isInformationMatrixValid=True, isOdometryConstraint=True)


def buildOdometryConstraint(backend, collection: SubmapCollection, sourceIdx: int, targetIdx: int,
                            params: E.OdometryConstraintParameters | None = None) -> Constraint:
    """buildOdometryConstraint(sourceIdx = parent, targetIdx = child, submaps) (src/constraint_builders.cpp:33-41): overlap of the two
    whole maps at the identity, optional point-to-plane refinement, information matrix."""
    params = params or E.OdometryConstraintParameters()
    (r,) = backend.odometry_constraints([(collection.submaps[sourceIdx].handle, collection.submaps[targetIdx].handle)], params)
    return _odometry_constraint(collection, sourceIdx, targetIdx, r)


def computeOdometryConstraints(backend, collection: SubmapCollection, constraints: list, finishedIds=None,
                               params: E.OdometryConstraintParameters | None = None) -> list:
    """Both overloads of computeOdometryConstraints (src/constraint_builders.cpp:92-118), appending to `constraints`:
        finishedIds given (SubmapCollection::computeFeatures, :92-106): every listed submap but submap 0, from its parent;
        finishedIds None  (SlamWrapper::loopClosureWorker, :108-118): every submap 1.. from its parent, except pairs that touch the
                          active submap.
    A (parent, child) pair already in `constraints` is not rebuilt (hasConstraint).  The missing pairs go to the backend in ONE batched
    call.  Returns the constraints added, in the reference's order."""
    params = params or E.OdometryConstraintParameters()
    active = collection.activeSubmapIdx
    pairs = []
    targets = finishedIds if finishedIds is not None else range(1, len(collection.submaps))
    for t in targets:
        if t < 1:
            continue
        s = collection.submaps[t].parent
        if finishedIds is None and (s == active or t == active):
            continue
        if hasConstraint(s, t, constraints) or (s, t) in pairs:   # the pending ones count: the reference appends as it goes
            continue
        pairs.append((s, t))
    if not pairs:
        return []
    res = backend.odometry_constraints([(collection.submaps[s].handle, collection.submaps[t].handle) for s, t in pairs], params)
    added = [_odometry_constraint(collection, s, t, r) for (s, t), r in zip(pairs, res)]
    constraints.extend(added)
    return added


# ----------------------------------------------------------------------------------------------------------------------
# pose-graph optimisation and the loop-closure correction
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class GlobalOptimizationParameters:
    """Parameters.hpp:138-143 with the Lua values (parameter_structure_definitions.lua:45-50); the C++ struct's own
    maxCorrespondenceDistance default is 10"""
    edgePruneThreshold: float = 0.2
    loopClosurePreference: float = 2.0
    maxCorrespondenceDistance: float = 1000.0
    referenceNode: int = 0

    def option(self) -> E.GlobalOptimizationOption:
        return E.GlobalOptimizationOption(self.maxCorrespondenceDistance, self.edgePruneThreshold, self.loopClosurePreference, self.referenceNode)


@dataclass
class OptimizedTransform:
    """OptimizedTransform (OptimizationProblem.hpp): the increment dT_ of submap submapId_"""
    dT_: np.ndarray
    submapId_: int


class OptimizationProblem:
    """src/OptimizationProblem.cpp (without the mutexes, timers and JSON I/O).  The solve runs on the backend
    (DeviceBackend.global_optimization: one b2s_global_optimization call)."""

    def __init__(self, backend, params: GlobalOptimizationParameters | None = None):
        self.backend = backend
        self.params = params or GlobalOptimizationParameters()
        self.odometryConstraints_: list = []
        self.loopClosureConstraints_: list = []
        self.poseGraph_ = E.PoseGraph()
        self.poseGraphOptimized_ = E.PoseGraph()
        self.poseGraphNonOptimized_ = E.PoseGraph()
        self.numOdometryEdgesPrev_ = 0
        self.numLoopClosuresPrev_ = 0
        self.lastStats = None

    def clearOdometryConstraints(self):
        self.odometryConstraints_.clear()

    def clearLoopClosureConstraints(self):
        self.loopClosureConstraints_.clear()

    def insertOdometryConstraints(self, cs):
        self.odometryConstraints_.extend(cs)

    def insertLoopClosureConstraints(self, cs):   # :177-189: a (source, target) pair already held is not inserted again
        for c in cs:
            if not any(c.sourceSubmapIdx == c2.sourceSubmapIdx and c.targetSubmapIdx == c2.targetSubmapIdx for c2 in self.loopClosureConstraints_):
                self.loopClosureConstraints_.append(c)

    def getLoopClosureConstraints(self) -> list:
        return self.loopClosureConstraints_

    def updateLoopClosureConstraint(self, idx: int, c) -> None:
        self.loopClosureConstraints_[idx] = c

    def buildOptimizationProblem(self) -> None:   # :49-61
        self.poseGraph_.edges_ = []
        self.setupOdometryEdgesAndPoseGraphNodes()
        self.setupLoopClosureEdges()

    def setupOdometryEdgesAndPoseGraphNodes(self) -> None:   # :63-95
        # The reference sorts with `c1.sourceSubmapIdx_ < c2.targetSubmapIdx_`, which is not a strict weak ordering (std::sort's result
        # is then unspecified); the intent, "sources in increasing order", is a stable sort by source.
        self.odometryConstraints_.sort(key=lambda c: c.sourceSubmapIdx)
        for c in self.odometryConstraints_:
            if not c.targetSubmapIdx > c.sourceSubmapIdx:
                raise RuntimeError("id_source should always be less than id_target for the odometry constraints")
            self.poseGraph_.edges_.append(E.PoseGraphEdge(c.sourceSubmapIdx, c.targetSubmapIdx, np.array(c.sourceToTarget), np.array(c.informationMatrix), False))
        if len(self.poseGraphOptimized_.edges_) > 0:
            odometry = np.linalg.inv(self.poseGraphOptimized_.nodes_[-1].pose_)
        else:
            self.poseGraph_.nodes_.append(E.PoseGraphNode(np.eye(4)))
            odometry = np.eye(4)
        for i in range(self.numOdometryEdgesPrev_, len(self.odometryConstraints_)):
            odometry = np.asarray(self.odometryConstraints_[i].sourceToTarget) @ odometry
            self.poseGraph_.nodes_.append(E.PoseGraphNode(np.linalg.inv(odometry)))
        self.numOdometryEdgesPrev_ = len(self.odometryConstraints_)

    def setupLoopClosureEdges(self) -> None:   # :97-120
        self.numLoopClosuresPrev_ = len(self.loopClosureConstraints_)
        for c in self.loopClosureConstraints_:
            if not c.isInformationMatrixValid:
                raise RuntimeError(f"Invalid information matrix between: {c.sourceSubmapIdx} and {c.targetSubmapIdx}")
            if not c.sourceSubmapIdx > c.targetSubmapIdx:
                raise RuntimeError("Optimization problem, loop closure constraints: ")
            self.poseGraph_.edges_.append(E.PoseGraphEdge(c.sourceSubmapIdx, c.targetSubmapIdx, np.array(c.sourceToTarget), np.array(c.informationMatrix), True))

    def solve(self) -> None:   # :25-44 with [O3D]'s default criteria
        self.poseGraphNonOptimized_ = copy.deepcopy(self.poseGraph_)
        self.lastStats = self.backend.global_optimization(self.poseGraph_, E.GlobalOptimizationConvergenceCriteria(), self.params.option())
        self.poseGraphOptimized_ = copy.deepcopy(self.poseGraph_)

    def getOptimizedTransformIncrements(self) -> list:   # :191-202: the increment is the optimised node pose itself
        if len(self.poseGraphOptimized_.nodes_) != len(self.poseGraph_.nodes_):
            raise RuntimeError("Graphs are not of same size, did you run the optimization?")
        return [OptimizedTransform(np.array(n.pose_), i) for i, n in enumerate(self.poseGraphOptimized_.nodes_)]


def updateSubmapsAndTrajectory(mapper: "SegmentMapper", problem: OptimizationProblem, lastLoopClosureConstraints) -> np.ndarray:
    """SlamWrapper::updateSubmapsAndTrajectory (src/SlamWrapper.cpp:450-485).  The latest loop closure is the last one in
    lastLoopClosureConstraints (the caller appends them in time order; the timestamps stay with the caller).  Returns its dT."""
    inc = problem.getOptimizedTransformIncrements()
    mapper.submaps.transform(inc)
    latest = lastLoopClosureConstraints[-1]
    if not latest.sourceSubmapIdx > latest.targetSubmapIdx:
        raise RuntimeError("Wrapper ros, update submaps and trajectory: ")
    dT = inc[latest.sourceSubmapIdx].dT_
    mapper.loopClosureUpdate(dT)
    lcs = problem.getLoopClosureConstraints()
    for i, old in enumerate(list(lcs)):
        c = copy.copy(old)
        c.sourceToTarget = np.eye(4)
        problem.updateLoopClosureConstraint(i, c)
    mapper.submaps.updateAdjacencyMatrix(problem.getLoopClosureConstraints())
    return dT


def loopClosureCycle(backend, mapper: "SegmentMapper", problem: OptimizationProblem, loopClosureConstraints,
                     odometryParams: E.OdometryConstraintParameters | None = None) -> np.ndarray:
    """One loop closure of SlamWrapper (src/SlamWrapper.cpp:425-445, 450-485) for constraints the caller built
    (buildLoopClosureConstraints): the missing odometry constraints (one batched device call), insert, build, solve, then the
    correction of the submaps and of the mapper.  The mapper never calls this on its own.  Returns the dT applied to the mapper."""
    sc = mapper.submaps
    odometryConstraints = sc.getOdometryConstraints()
    computeOdometryConstraints(backend, sc, odometryConstraints, None, odometryParams)
    problem.clearOdometryConstraints()
    problem.insertLoopClosureConstraints(loopClosureConstraints)
    problem.insertOdometryConstraints(odometryConstraints)
    problem.buildOptimizationProblem()
    problem.solve()
    return updateSubmapsAndTrajectory(mapper, problem, list(loopClosureConstraints))


# ----------------------------------------------------------------------------------------------------------------------
# device backend
# ----------------------------------------------------------------------------------------------------------------------
class DeviceBackend:
    """All arithmetic on libb2s.so (one handle / one CUDA stream = one robot)."""

    def __init__(self, params: E.MapperParameters | None = None, device: int = 0, cuda_stream: int | None = None, submap_capacity: int = 900_000,
                 carving: bool = True, dense: bool = True, graph: bool = True, raw_capacity: int = 65536,
                 odometry: E.OdometryParameters | None = None, motionCompensation: E.ConstantVelocityMotionCompensationParameters | None = None):
        self.params = params or E.MapperParameters()
        self.odometry_params = odometry or E.OdometryParameters()   # the device odometry of SegmentMapper.addRangeScan
        self.motion_compensation = motionCompensation                # de-skew of both inputs of SegmentMapper.addRangeScan (None: off)
        self._odo = None
        self._odo_initial = None   # SlamWrapper::setInitialTransform's odometry half, applied when the odometry is created
        self.eng = E.Engine(self.params, device=device, cuda_stream=cuda_stream)
        self.mapper = E.Mapper(self.eng, 1024)     # its own first submap is a placeholder: submaps are created by new_submap()
        self.mapper.submap.free()
        self.mapper.submap = None
        self.submap_capacity = submap_capacity
        self.carving, self.dense, self.graph, self.raw_capacity = carving, dense, graph, raw_capacity
        self._voxel_maps = {}
        self._stagings = {}
        self._pin = None

    # -- submaps
    def new_submap(self):
        p = self.params
        sm = E.Submap(self.eng, self.submap_capacity)
        sm.setMapperOptions(minMovement=p.minMovementBetweenMappingSteps, carving=p.mapBuilder.carving if self.carving else None,
                            dense=self.dense, denseCarving=p.denseMapCarving if (self.dense and self.carving) else None,
                            denseCropper=p.denseMapCropper)
        if p.isUseInitialMap and not p.isMergeScansIntoMap:
            sm.setMergeScans(False)    # pure localisation: the chain neither carves nor fuses
        return sm

    # -- localisation against a prior map
    def initial_map(self, sm, xyz: np.ndarray):
        """prepareInitialMap (normals on the full map) and Submap::insertScan's initial branch (voxelized load); returns the prepared
        cloud, which SubmapCollection keeps in its overlap buffer"""
        c = self.eng.cloud(np.ascontiguousarray(xyz, dtype=np.float64))
        self.mapper.scan2MapReg_.prepareInitialMap(c)
        sm.setInitialMap(c, self.params.mapBuilder.mapVoxelSize)
        return c

    def set_initial_transform(self, sm, T):
        """Mapper::setMapToRangeSensorInitial on the submap's device pose slot, and LidarOdometry's initial transform once it exists"""
        sm.setInitialTransform(T)
        self._odo_initial = np.array(T, dtype=np.float64)
        if self._odo is not None:
            self._odo.setInitialTransform(T)

    def _activate(self, sm):
        self.mapper.submap = sm
        if self.graph:
            if id(sm) not in self._stagings:
                self._stagings[id(sm)] = self.mapper.enableGraph(self.raw_capacity)
            self.mapper._staging = self._stagings[id(sm)]

    def _pinned(self, raw: np.ndarray):
        import torch
        raw = np.ascontiguousarray(raw, dtype=np.float32)
        if self._pin is None or self._pin.shape[0] < raw.shape[0]:
            self._pin = torch.empty((max(raw.shape[0], self.raw_capacity), 3), dtype=torch.float32).pin_memory()
        self._pin[:raw.shape[0]].copy_(torch.from_numpy(raw))
        return self._pin.data_ptr(), raw.shape[0]

    def first_scan(self, sm, raw: np.ndarray):
        """Mapper.cpp:109-112: pre-process and insert at Identity (carving is a no-op on the empty map)."""
        icp = self.mapper.scan2MapReg_
        raw_c = self.eng.cloud(np.ascontiguousarray(raw, dtype=np.float32))
        ps = icp.processForScanMatchingAndMerging(raw_c)
        sm.insertScan(raw_c, ps.merge_, np.eye(4))
        sm.setPose(np.eye(4))
        raw_c.free()
        return ps.merge_

    def step(self, sm, raw: np.ndarray, odometryMotion: np.ndarray):
        self._activate(sm)
        ptr, n = self._pinned(raw)
        res = self.mapper.addRangeMeasurementHost(ptr, n, odometryMotion)
        p = self.params
        accepted = p.isIgnoreMinRefinementFitness or not (res.fitness_ < p.minRefinementFitness)
        return res, bool(accepted)     # minMovementBetweenMappingSteps = 0 in every preset: accepted scans are inserted

    # -- scan-to-scan odometry on the device, feeding the mapper step its prediction (SegmentMapper.addRangeScan)
    def odometry(self) -> E.DeviceLidarOdometry:
        if self._odo is None:
            import torch
            self._odo = E.DeviceLidarOdometry(self.eng, self.odometry_params, self.raw_capacity)
            if self.motion_compensation is not None:
                self._odo.setMotionCompensation(self.motion_compensation)
            if self._odo_initial is not None:
                self._odo.setInitialTransform(self._odo_initial)
            if self.graph:
                self._odo.enableGraph(self.raw_capacity)
            self._slam_pin = torch.empty(C.sizeof(L.SlamResult), dtype=torch.uint8).pin_memory()
            self._slam_out = L.SlamResult.from_address(self._slam_pin.data_ptr())
        return self._odo

    def first_scan_with_odometry(self, sm, raw: np.ndarray, t: int):
        """Mapper.cpp:109-112 for the map, with mapToRangeSensorBuffer_.push(t, mapToRangeSensor_ = I), and LidarOdometry::addRangeScan
        for the odometry, on the same scan and timestamp.  Both buffers are empty here, so a de-skew would leave the scan as it is."""
        merge = self.first_scan(sm, raw)
        c = self.eng.cloud(np.ascontiguousarray(raw, dtype=np.float32))
        odo = self.odometry()
        odo.addRangeScan(c, t)
        odo.pushMapToRangeSensor(t, np.eye(4))
        c.free()
        return merge

    def step_with_odometry(self, sm, raw: np.ndarray, t: int):
        odo = self.odometry()
        self.mapper.submap = sm
        ptr, n = self._pinned(raw)
        self.mapper.addRangeMeasurementWithOdometryHostAsync(odo, ptr, n, t, C.addressof(self._slam_out))
        self.eng.synchronize()
        self.last_slam_result = E._slam_res(self._slam_out)
        return self.last_slam_result.mapper, self.last_slam_result.mapperAccepted

    def last_merge_cloud(self):
        # ring of pre-allocated clouds (no cudaMalloc per scan); longer than SubmapCollection's overlap buffer, so a buffered cloud is
        # never overwritten while it can still be replayed into a new submap
        if not hasattr(self, "_merge_ring"):
            self._merge_ring = [E.Cloud(self.eng) for _ in range(16)]
            self._merge_pos = 0
        c = self._merge_ring[self._merge_pos % len(self._merge_ring)]
        self._merge_pos += 1
        return self.mapper.lastProcessedScan(merge_into=c).merge_

    def insert_scan(self, sm, cloud, T):
        sm.insertScan(None, cloud, T, isPerformCarving=False)

    def set_pose(self, sm, T):
        sm.setPose(T)

    def map_cloud(self, sm):
        return sm.getMapPointCloud()

    def map_center(self, sm) -> np.ndarray:
        xyz, _ = sm.getMapPointCloud()
        return xyz.mean(axis=0) if len(xyz) else np.zeros(3)   # [O3D] GetCenter

    def build_voxel_map(self, sm) -> None:
        v = VOXEL_EXPANSION_ADJACENCY_REVISITING * self.params.mapBuilder.mapVoxelSize
        vm = self._voxel_maps.get(id(sm))
        if vm is None:
            vm = E.VoxelMap(self.eng, v, 1 << 18)
            self._voxel_maps[id(sm)] = vm
        vm.clear()
        c = sm.toCloud()
        vm.insertCloud(VOXEL_MAP_LAYER, c)
        c.free()

    def compute_features(self, sm, params: E.PlaceRecognitionParameters):
        """Submap::computeFeatures on the device: (sparse cloud, Feature), both owned by the submap object"""
        sm.computeFeatures(params)
        return sm.getSparseMapPointCloud(), sm.getFeatures()

    def revisit_fitness(self, sm, scan, mapToRangeSensor) -> float:
        vm = self._voxel_maps[id(sm)]
        n = len(scan)
        if n == 0:
            return 0.0
        _flags, hits = vm.hasVoxelContainingPoint(scan, mapToRangeSensor)
        return hits / n

    # -- loop-closure refinement
    def submap_as_cloud(self, sm):
        return sm.toCloud()

    def overlap(self, source, target, T0, voxel, min_pts):
        return E.computeOverlappingClouds(self.eng, source, target, T0, voxel, min_pts)

    def register_batch(self, sources, targets, inits, max_corr, max_iter):
        pc = E.CloudRegistrationParameters(icp=E.IcpParameters(maxNumIter=max_iter, maxCorrespondenceDistance=max_corr, knn=self.params.icp.knn,
                                                              maxDistanceKnn=self.params.icp.maxDistanceKnn))
        reg = E.RegistrationIcpPointToPlane(self.eng, pc)
        out = reg.registerCloudsBatch(sources, targets, inits)
        self.eng.set_parameters(self.params)   # the scan-to-map chain keeps its own ICP parameters
        return out

    def information_matrix(self, source, target, max_corr, T):
        return E.getInformationMatrixFromPointClouds(self.eng, source, target, max_corr, T)

    def ransac(self, source_sparse, source_feature, target_sparses, target_features, params: E.PlaceRecognitionParameters):
        """RegistrationRANSACBasedOnFeatureMatching of the source against every candidate in one call (mutual filter on, :82)"""
        return E.registrationRANSACBasedOnFeatureMatchingBatch(self.eng, source_sparse, target_sparses, source_feature, target_features, params)

    def odometry_constraints(self, pairs, params: E.OdometryConstraintParameters):
        """buildOdometryConstraint for every (parent, child) pair of submaps in one b2s_submap_odometry_constraints call"""
        return E.buildOdometryConstraintsBatch(self.eng, [s for s, _t in pairs], [t for _s, t in pairs], params)

    def global_optimization(self, poseGraph, criteria, option):
        """[O3D] GlobalOptimization on the device (b2s_global_optimization); poseGraph is updated in place"""
        return E.globalOptimization(self.eng, poseGraph, criteria, option)

    def transform_submap(self, sm, sparse, T):
        """Submap::transform: map, dense map and pose slot (b2s_submap_transform), then the sparse feature cloud"""
        sm.transform(T)
        sm.transformSparseMapCloud(T)

    def loop_closure_update(self, sm, mapToRangeSensor):
        sm.setPose(mapToRangeSensor)

    def cloud_size(self, c) -> int:
        return len(c)

    def dense_map(self, sm):
        return sm.getDenseMap()

    def counters(self, sm) -> dict:
        return sm.mapperCounters()

    def close(self):
        for vm in self._voxel_maps.values():
            vm.free()
        self._voxel_maps.clear()
