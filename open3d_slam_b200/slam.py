"""Host control flow of the full mapper (config 5 of BASELINE.json) around the device hot path.

What stays on the host in the reference and is restated here as plain control flow (paths relative to
/root/reference/open3d_slam/open3d_slam/):
    Mapper::addRangeMeasurement                                   src/Mapper.cpp:101-181
    SubmapCollection::insertScan / updateActiveSubmap / createNewSubmap / insertBufferedScans / findClosestSubmap /
    isSwitchingSubmapsConsistant                                  src/SubmapCollection.cpp:83-131,133-158,172-207,352-364
    Submap::computeSubmapCenter / computeFeatures (voxel map part) src/Submap.cpp:228-259
    PlaceRecognition::buildLoopClosureConstraints for given candidates: RANSAC proposal -> correspondence gate -> consistency
    check -> refinement (overlap -> ICP -> information matrix, one batched device call) -> consistency check
                                                                  src/PlaceRecognition.cpp:50-229
    computeOdometryConstraints / buildOdometryConstraint: the constraints between consecutive submaps, all missing pairs in one
    batched device call                                           src/constraint_builders.cpp:23-118
    AdjacencyMatrix                                               src/AdjacencyMatrix.cpp:16-71
    PlaceRecognition::getLoopClosureCandidatesIdxs                src/PlaceRecognition.cpp:231-284
    SlamWrapper's loop-closure schedule (SegmentMapper.isAttemptLoopClosures, finishProcessing), run synchronously
                                                                  src/SlamWrapper.cpp:126-166,319-335,388-485
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
import math
import pickle
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
    """the PlaceRecognitionParameters the refinement half reads (Parameters.hpp:132-135) + magic.hpp:14, and the refinement's
    estimator.  registrationType defaults to point-to-plane; the reference refines with the scan matcher's type, which
    fromMapperParameters takes over."""
    maxIcpCorrespondenceDistance: float = 0.3
    minRefinementFitness: float = 0.7
    maxNumIter: int = 100                       # magic::icpRunUntilConvergenceNumberOfIterations
    voxelExpansionFactorOverlapComputation: float = 20.0
    minNumPointsPerVoxel: int = 1
    registrationType: str = "PointToPlaneIcp"   # CloudRegistrationType of the refinement ICP

    @classmethod
    def fromMapperParameters(cls, mapperParams: E.MapperParameters, maxIcpCorrespondenceDistance: float = 0.3,
                             minRefinementFitness: float = 0.7) -> "LoopClosureParameters":
        """PlaceRecognition::updateRegistrationAlgorithm (src/PlaceRecognition.cpp:44-48): the loop-closure ICP is the scan matcher's
        registration type with maxNumIter = magic::icpRunUntilConvergenceNumberOfIterations and maxCorrespondenceDistance =
        placeRecognition.maxIcpCorrespondenceDistance (passed here with minRefinementFitness: MapperParameters does not hold them)."""
        E.regTypeOf(mapperParams.scanToMapRegType)   # an unknown type throws, as cloudRegistrationFactory does
        return cls(maxIcpCorrespondenceDistance=maxIcpCorrespondenceDistance, minRefinementFitness=minRefinementFitness, maxNumIter=100,
                   registrationType=mapperParams.scanToMapRegType)


VOXEL_EXPANSION_ADJACENCY_REVISITING = 2.5     # magic::voxelExpansionFactorAdjacencyBasedRevisiting
VOXEL_MAP_LAYER = "map"                        # Submap::voxelMapLayer
INT_MAX = 2**31 - 1                            # std::numeric_limits<int>::max()


class AdjacencyMatrix:
    """src/AdjacencyMatrix.cpp:16-71, quirks included:
      - addEdge inserts both directions and resets the loop-closure mark of both ends, so a hand-over edge unmarks a submap an
        earlier loop closure had marked;
      - markAsLoopClosureSubmap of an id without an edge throws (std::map::at), here KeyError;
      - isAdjacent(id, id) is true;
      - getDistanceToNearestLoopClosureSubmap is INT_MAX while no edge was ever added; otherwise a BFS (neighbours in increasing
        id order, std::set) that stops at the first marked node, or, when none is reachable, at the last node it dequeued; the
        result is max(0, path length to that node - 1).  An id without an edge throws, here KeyError."""

    def __init__(self):
        self.adjacency_: dict[int, set[int]] = {}
        self.isLoopClosureSubmap_: dict[int, bool] = {}

    def addEdge(self, id1: int, id2: int) -> None:
        self.adjacency_.setdefault(id1, set()).add(id2)
        self.adjacency_.setdefault(id2, set()).add(id1)
        self.isLoopClosureSubmap_[id1] = False
        self.isLoopClosureSubmap_[id2] = False

    def getDistanceToNearestLoopClosureSubmap(self, id: int) -> int:
        if not self.isLoopClosureSubmap_:
            return INT_MAX
        toProcess = collections.deque([id])
        visited, parents = {id}, {}
        v = id
        while toProcess:
            v = toProcess.popleft()
            if self.isLoopClosureSubmap_[v]:
                break
            for adj in sorted(self.adjacency_[v]):
                if adj not in visited:
                    visited.add(adj)
                    toProcess.append(adj)
                    parents[adj] = v
        distance = 0
        while v != id:
            v = parents[v]
            distance += 1
        return max(0, distance - 1)

    def markAsLoopClosureSubmap(self, id: int) -> None:
        if id not in self.isLoopClosureSubmap_:
            raise KeyError(id)
        self.isLoopClosureSubmap_[id] = True

    def isAdjacent(self, id1: int, id2: int) -> bool:
        return id1 == id2 or id2 in self.adjacency_.get(id1, ())


@dataclass
class LoopClosureCandidateParameters:
    """The two PlaceRecognitionParameters fields candidate selection reads (Parameters.hpp:134-135, the same in the Lua defaults).
    Kept apart from engine.PlaceRecognitionParameters, which is copied field by field into the ABI's parameter struct."""
    loopClosureSearchRadius: float = 20.0
    minSubmapsBetweenLoopClosures: int = 2


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
        self.pendingFinishedSubmapIds: list[tuple[int, int]] = []   # finishedSubmapsIdxs_ of the reference: (id, timestamp), popped
        self.adjacency: set[tuple[int, int]] = set()
        self.loopClosureSubmaps: set[int] = set()   # adjacencyMatrix_.markAsLoopClosureSubmap
        self.adjacencyMatrix = AdjacencyMatrix()    # adjacencyMatrix_, what candidate selection reads
        self.odometryConstraints: list = []          # odometryConstraints_ (SubmapCollection::computeFeatures appends to it)
        self.isUseInitialMap = False                 # MapperParameters::isUseInitialMap_: localisation mode never hands over (:105-107)
        self.isForceNewSubmapCreation = False        # isForceNewSubmapCreation_ (:163-170)
        self.mapToRangeSensor_ = np.eye(4)           # the pose and timestamp of the last insertion (insertScan, :172-175)
        self.timestamp_ = 0
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
        if self.isForceNewSubmapCreation:
            self.createNewSubmap(mapToRangeSensor)
            self.isForceNewSubmapCreation = False
            return
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

    def popFinishedSubmapIds(self) -> list[tuple[int, int]]:
        """popFinishedSubmapIds: the (id, timestamp) of every submap finished since the last call, in finishing order"""
        out, self.pendingFinishedSubmapIds = self.pendingFinishedSubmapIds, []
        return out

    def computeFeaturesOf(self, finishedSubmapIds, params: E.PlaceRecognitionParameters,
                          odometryParams: E.OdometryConstraintParameters | None = None) -> None:
        """SubmapCollection::computeFeatures(finishedSubmapIds) (:219-243) as SlamWrapper::computeFeaturesIfReady calls it: the features
        of the listed submaps, then their odometry constraints into odometryConstraints (one batched backend call)."""
        ids = [i for i, _t in finishedSubmapIds]
        for idx in ids:
            rec = self.submaps[idx]
            rec.sparse, rec.feature = self.backend.compute_features(rec.handle, params)
        computeOdometryConstraints(self.backend, self, self.odometryConstraints, ids, odometryParams)

    def forceNewSubmapCreation(self, scan_index: int) -> None:
        """SubmapCollection::forceNewSubmapCreation (:163-170): insertScan of an empty scan at the last insertion's pose and time with
        isForceNewSubmapCreation_ set, so the active submap is finished and a new one created there.  The empty scan goes through the
        overlap buffer like any other (it evicts the oldest buffered scan); Submap::insertScan skips it (Submap.cpp:41-43)."""
        if not self.submaps:
            return
        self.isForceNewSubmapCreation = True
        self.afterInsertion(scan_index, None, self.mapToRangeSensor_, self.timestamp_)
        self.isForceNewSubmapCreation = False

    def getOdometryConstraints(self) -> list:
        return list(self.odometryConstraints)

    def getTotalNumPoints(self) -> int:   # :69-73
        return sum(self.backend.map_size(s.handle) for s in self.submaps)

    def updateAdjacencyMatrix(self, loopClosureConstraints) -> None:   # :75-81
        for c in loopClosureConstraints:
            self.adjacency.add((min(c.sourceSubmapIdx, c.targetSubmapIdx), max(c.sourceSubmapIdx, c.targetSubmapIdx)))
            self.loopClosureSubmaps.update((c.sourceSubmapIdx, c.targetSubmapIdx))
            self.adjacencyMatrix.addEdge(c.sourceSubmapIdx, c.targetSubmapIdx)
            self.adjacencyMatrix.markAsLoopClosureSubmap(c.sourceSubmapIdx)
            self.adjacencyMatrix.markAsLoopClosureSubmap(c.targetSubmapIdx)

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
    # A preProcessedScan of None is the empty scan of forceNewSubmapCreation.  timestamp stamps the finished submap (the scan index
    # when None).
    def afterInsertion(self, scan_index: int, preProcessedScan, mapToRangeSensor: np.ndarray, timestamp: int | None = None) -> None:
        if len(self.submaps) == 0:
            raise RuntimeError("SubmapCollection: no submap")
        self.mapToRangeSensor_ = np.array(mapToRangeSensor)
        self.timestamp_ = scan_index if timestamp is None else timestamp
        self.overlapScansBuffer.append((preProcessedScan, np.array(mapToRangeSensor)))   # addScanToBuffer :83-85
        prev = self.activeSubmapIdx
        self.updateActiveSubmap(mapToRangeSensor, preProcessedScan)
        if prev != self.activeSubmapIdx:
            self.finishSubmap(prev)
            self.finishedSubmapsIdxs.append(prev)
            self.pendingFinishedSubmapIds.append((prev, self.timestamp_))
            self.numScansMergedInActiveSubmap = 0
            a, b = self.submaps[prev].id, self.submaps[self.activeSubmapIdx].id
            self.adjacency.add((min(a, b), max(a, b)))
            self.adjacencyMatrix.addEdge(a, b)
            self.events.append(("active_submap_changed", scan_index, prev, self.activeSubmapIdx))
            while self.overlapScansBuffer:   # insertBufferedScans :87-92 (no carving)
                cloud, T = self.overlapScansBuffer.popleft()
                if cloud is not None:
                    self.backend.insert_scan(self.submaps[self.activeSubmapIdx].handle, cloud, T)
            self.backend.set_pose(self.submaps[self.activeSubmapIdx].handle, mapToRangeSensor)
        self.numScansMergedInActiveSubmap += 1


class SegmentMapper:
    """Mapper::addRangeMeasurement over a SubmapCollection, one scan per call (src/Mapper.cpp:101-181).

    With isAttemptLoopClosures (MapperParameters::isAttemptLoopClosures_, true in the reference; off here by default, so that a mapper
    built as before maps as before), every call also runs SlamWrapper's loop-closure schedule (src/SlamWrapper.cpp:319-335, 388-448,
    450-485) once the scan is mapped: the submaps finished since the last attempt get their features and odometry constraints
    (SubmapCollection::computeFeatures); each of them, in finishing order, gets its candidates (getLoopClosureCandidatesIdxs) and its
    loop-closure constraints (buildLoopClosureConstraints, stamped with the finishing scan's timestamp); if any was accepted,
    loopClosureCycle solves the pose graph and corrects the submaps and the mapper.  The reference runs these steps on worker threads,
    so when its correction lands depends on their timing; here they run synchronously before the next scan, which is the reference's
    schedule with zero worker latency.  Each step is logged in submaps.events: ("features", k, ids), ("loop_closure_candidates", k,
    source, candidates), ("loop_closure_decisions", k, source, log), ("pose_graph_solve", k, stats of both passes) and
    ("loop_closure_correction", k, source of the latest constraint, dT).  The timestamp is the scan index for addRangeMeasurement and
    t for addRangeScan."""

    def __init__(self, backend, submapParams: SubmapParameters | None = None, isAttemptLoopClosures: bool = False,
                 loopClosing: LoopClosingParameters | None = None):
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
        self.isRelocalized = False          # relocalize has re-entered the map (finishing order no longer follows submap order)
        self.isAttemptLoopClosures = isAttemptLoopClosures
        self.loopClosing = loopClosing or (LoopClosingParameters.fromMapperParameters(mp) if mp is not None else LoopClosingParameters())
        self.optimizationProblem = OptimizationProblem(backend, self.loopClosing.globalOptimization)

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

    def globalLocalization(self, rawScanF32: np.ndarray, params=None):
        """Localise the raw scan in the loaded prior map with no pose given (b2s_submap_global_localization, DESIGN.md row M3) -- what
        SlamMapInitializer's marker pose does in the reference.  When the winner passes the mapper's fitness gate, setInitialTransform(T)
        follows, so the next step keeps T (rule 3 of M2).  Logged as ("global_localization", k, found, T, fitness, runner_up) in
        submaps.events, k = the index of the next scan.  Returns the backend's GlobalLocalizationResult."""
        if not self.submaps.submaps:
            raise RuntimeError("globalLocalization: no map loaded (call setInitialMap first)")
        r = self.backend.global_localization(self.submaps.getActiveSubmap().handle, rawScanF32, params)
        self.submaps.events.append(("global_localization", self._k, r.found, r.T.copy(), r.fitness, r.runner_up_fitness))
        if r.found:
            self.setInitialTransform(r.T)
        return r

    def relocalize(self, rawScanF32: np.ndarray, t: int | None = None, params=None):
        """Find the raw scan in the union of every submap with no pose given and re-enter the mapper there (one
        b2s_submaps_global_localization call, DESIGN.md row M4): after loadSession, after losing track, or on an initial-map mapper.
        Each candidate is refined in the submap findClosestSubmap picks for it.  When the winner passes the fitness gate
        (minRefinementFitness):
          1. the active submap becomes the winner's submap when the found pose T lies within SubmapParameters.radius of its centre;
             otherwise a new submap is created at T with the winner's submap as its parent (and adjacent to it), and the scan is
             inserted into it at T as its first scan (Mapper.cpp:105-114 at T).  A submap left behind is finished as at a hand-over,
             stamped with t (the next scan index when None).  Localisation mode (isUseInitialMap) never creates or finishes submaps:
             the winner's submap becomes active wherever T lies;
          2. the overlap buffer is cleared: its scans were taken at the old pose;
          3. setInitialTransform(T) on the active submap: the next step keeps T and inserts nothing (rule 3 of M2);
          4. the odometry starts over: the next addRangeScan is its first scan, at T, with empty pose buffers;
          5. from then on a finished submap's loop-closure candidates are the older submaps only: a re-entered submap can finish
             after newer ones, and the pose graph takes loop-closure edges only from a newer submap to an older one.
        A winner that fails the gate changes nothing.  Logged as ("relocalization", k, found, T, fitness, runner_up, submap) in
        submaps.events, k = the index of the next scan.  Returns the backend's result (with winner_submap)."""
        sc = self.submaps
        if not sc.submaps:
            raise RuntimeError("relocalize: the mapper holds no submap")
        centers = np.array([s.mapToSubmapCenter() for s in sc.submaps], dtype=np.float64)
        r = self.backend.global_localization_submaps([s.handle for s in sc.submaps], centers, rawScanF32, params)
        sc.events.append(("relocalization", self._k, r.found, r.T.copy(), r.fitness, r.runner_up_fitness, r.winner_submap))
        if not r.found:
            return r
        T = np.array(r.T, dtype=np.float64)
        w, prev = r.winner_submap, sc.activeSubmapIdx
        inside = np.linalg.norm(T[:3, 3] - sc.submaps[w].mapToSubmapCenter()) < sc.params.radius
        sc.overlapScansBuffer.clear()
        sc.activeSubmapIdx = w
        sc.numScansMergedInActiveSubmap = 0
        if not inside and not self.isUseInitialMap:
            sc.createNewSubmap(T)   # parent: the winner's submap
            a, b = sc.submaps[w].id, sc.getActiveSubmap().id
            sc.adjacency.add((min(a, b), max(a, b)))
            sc.adjacencyMatrix.addEdge(a, b)
            self.backend.first_scan_at(sc.getActiveSubmap().handle, rawScanF32, T)
            sc.numScansMergedInActiveSubmap = 1
        if sc.activeSubmapIdx != prev and not self.isUseInitialMap:   # the hand-over of afterInsertion, without the buffered scans
            sc.finishSubmap(prev)
            sc.finishedSubmapsIdxs.append(prev)
            sc.pendingFinishedSubmapIds.append((prev, self._k if t is None else t))
        self.backend.restart_odometry(T)
        self.setInitialTransform(T)
        self.isRelocalized = True
        return r

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
        return self._after_step(k, res, inserted, t)

    def loopClosureUpdate(self, loopClosureCorrection: np.ndarray) -> None:
        """Mapper::loopClosureUpdate (src/Mapper.cpp:44-47): mapToRangeSensor_ = dT * mapToRangeSensor_.  The device keeps one pose
        slot per submap for both the reference's Submap::mapToRangeSensor_ (which SubmapCollection.transform right-multiplies) and
        Mapper::mapToRangeSensor_, and the next step predicts from it: after the update the active submap's slot holds dT * (the mapper
        pose before the update).  The odometry's pose buffer is left alone, as in the reference."""
        self.mapToRangeSensor = np.asarray(loopClosureCorrection, dtype=np.float64) @ self.mapToRangeSensor
        if self.submaps.submaps:
            self.backend.loop_closure_update(self.submaps.getActiveSubmap().handle, self.mapToRangeSensor)

    def getAssembledMapPointCloud(self, voxelSize: float = 0.0):
        """Mapper::getAssembledMapPointCloud (src/Mapper.cpp:183-208): the maps of every submap in submap order, with normals, then
        o3d_slam::voxelize(voxelSize) as SlamWrapperRos::publishMaps applies assembledMapVoxelSize_ (no-op for voxelSize <= 0;
        SlamWrapper::saveMap keeps the plain assembly).  The mapper never calls it on its own."""
        return self.backend.assembled_map([s.handle for s in self.submaps.submaps], voxelSize)

    def assembleColoredPointCloud(self, voxelSize: float):
        """assembleColoredPointCloud (ros/open3d_slam_ros/src/helpers_ros.cpp:51-70) + voxelize(submapVoxelSize_): (cloud, rgb)"""
        return self.backend.assembled_colored_map([s.handle for s in self.submaps.submaps], voxelSize)

    def getDenseSubmapPointClouds(self) -> list:
        """SubmapCollection::dumpToFile(dir, "denseSubmap", true) (src/SubmapCollection.cpp:269-283), which SlamWrapper::saveDenseSubmaps
        calls: getDenseMapCopy().toPointCloud() of every submap, one n x 3 array per submap in submap order (a submap without a dense
        map gives an empty one).  Writing the files stays with the caller.  The mapper never calls it on its own."""
        return self.backend.dense_map_clouds([s.handle for s in self.submaps.submaps])

    def getActiveDenseMapPointCloud(self):
        """The active submap's getDenseMapCopy().toPointCloud(), as SlamWrapperRos::publishDenseMap publishes it
        (ros/open3d_slam_ros/src/SlamWrapperRos.cpp:213-220): an n x 3 array"""
        if not self.submaps.submaps:
            return np.zeros((0, 3))
        return self.backend.dense_map_clouds([self.submaps.getActiveSubmap().handle])[0]

    def _after_step(self, k: int, res, inserted: bool, t: int | None = None):
        sc = self.submaps
        self.results.append(res)
        if self.isNewInitialValueSet:   # Mapper.cpp:143-149: the result is discarded, the pose stays the initial value, nothing is inserted
            self.isNewInitialValueSet = False
        elif inserted:
            self.mapToRangeSensor = np.array(res.transformation_, dtype=np.float64)
            if not (self.isUseInitialMap and not self.isMergeScansIntoMap):   # :163-167: pure localisation never inserts
                sc.afterInsertion(k, self.backend.last_merge_cloud(), self.mapToRangeSensor, t)
        self.poses.append(self.mapToRangeSensor.copy())
        if self.isAttemptLoopClosures:
            self.attemptLoopClosures(k)
        return res

    def attemptLoopClosures(self, k: int) -> int:
        """One pass of the schedule (the class docstring) as after scan k: computeFeaturesIfReady, attemptLoopClosuresIfReady, the
        loop-closure worker and checkIfOptimizedGraphAvailable with no latency between them.  Returns the number of loop-closure
        constraints built (numLatesLoopClosureConstraints_), or -1 when no submap was finished since the last attempt."""
        sc, lp = self.submaps, self.loopClosing
        finished = sc.popFinishedSubmapIds()
        if not finished:
            return -1
        sc.computeFeaturesOf(finished, lp.placeRecognition, lp.odometryConstraints)
        sc.events.append(("features", k, [i for i, _t in finished]))
        constraints = []
        for idx, t in finished:   # SubmapCollection::buildLoopClosureConstraints (src/SubmapCollection.cpp:253-267)
            cands = getLoopClosureCandidatesIdxs(sc, sc.adjacencyMatrix, idx, sc.activeSubmapIdx, lp.candidates)
            if self.isRelocalized:
                # an older submap re-entered by relocalize can finish after newer ones, but the pose graph takes loop-closure edges only
                # from a newer submap to an older one (setupLoopClosureEdges)
                cands = [i for i in cands if i < idx]
            sc.events.append(("loop_closure_candidates", k, idx, cands))
            cs, log = buildLoopClosureConstraints(self.backend, sc, idx, cands, lp.placeRecognition, lp.mapVoxelSize, lp.refinement,
                                                  lp.consistency, timestamp=t)
            sc.events.append(("loop_closure_decisions", k, idx, log))
            constraints.extend(cs)
        if constraints:
            dT = loopClosureCycle(self.backend, self, self.optimizationProblem, constraints, lp.odometryConstraints)
            stats = self.optimizationProblem.lastStats
            sc.events.append(("pose_graph_solve", k, [(s.valid, s.n_edges, s.lm_tries, s.accepted_steps, s.stop_reason) for s in stats]))
            latest = max(constraints, key=lambda c: c.timestamp)
            sc.events.append(("loop_closure_correction", k, latest.sourceSubmapIdx, np.array(dT)))
        return len(constraints)

    # -- session state: save a mapping session to one .npz file and continue it later, on another backend or GPU
    SESSION_VERSION = 1

    def saveSession(self, path: str) -> None:
        """Writes everything the next scan depends on to path (.npz): the backend's state blobs of every submap and of the odometry
        (DeviceBackend: the device blobs of include/b2s.h "session state"), the SubmapCollection (records, active index and merge count,
        the overlap buffer's clouds and poses, finished and pending ids, adjacency and loop-closure marks, AdjacencyMatrix, odometry
        constraints, the hand-over flag and the last insertion's pose and timestamp), the OptimizationProblem's constraints and counters,
        this mapper's pose, scan count, initial-value flag and poses, and every finished submap's feature cloud and FPFH.  results and
        events are history and are not written.  The host state is pickled: load only session files you wrote."""
        sc, be = self.submaps, self.backend
        arrays = {}

        def put(name, obj):   # a backend's state: bytes go into the file as arrays, anything else (the oracle's copies) is pickled
            if isinstance(obj, (bytes, bytearray)):
                arrays[name] = np.frombuffer(bytes(obj), dtype=np.uint8)
                return ("array", name)
            return ("object", obj)

        records = []
        for i, (r, blob) in enumerate(zip(sc.submaps, be.export_submaps([r.handle for r in sc.submaps]))):
            rec = dict(id=r.id, parent=r.parent, origin=r.origin, center=r.center, has_voxel_map=r.has_voxel_map, state=put(f"submap_{i}", blob),
                       features=r.sparse is not None)
            if r.sparse is not None:
                arrays[f"sparse_xyz_{i}"], arrays[f"sparse_nrm_{i}"], arrays[f"feature_{i}"] = be.feature_arrays(r.sparse, r.feature)
            records.append(rec)
        overlap = []
        for j, (cloud, T) in enumerate(sc.overlapScansBuffer):
            if cloud is not None:
                xyz, nrm = be.cloud_arrays(cloud)
                arrays[f"overlap_xyz_{j}"] = xyz
                if nrm is not None:
                    arrays[f"overlap_nrm_{j}"] = nrm
            overlap.append((cloud is not None, np.array(T)))
        op = self.optimizationProblem
        host = dict(
            version=self.SESSION_VERSION, submapParams=sc.params, isAttemptLoopClosures=self.isAttemptLoopClosures, loopClosing=self.loopClosing,
            records=records, odometry=put("odometry", be.export_odometry()),
            activeSubmapIdx=sc.activeSubmapIdx, numScansMergedInActiveSubmap=sc.numScansMergedInActiveSubmap, overlap=overlap,
            finishedSubmapsIdxs=list(sc.finishedSubmapsIdxs), pendingFinishedSubmapIds=list(sc.pendingFinishedSubmapIds),
            adjacency=set(sc.adjacency), loopClosureSubmaps=set(sc.loopClosureSubmaps), adjacencyMatrix=sc.adjacencyMatrix,
            collectionOdometryConstraints=list(sc.odometryConstraints), isForceNewSubmapCreation=sc.isForceNewSubmapCreation,
            collectionMapToRangeSensor=np.array(sc.mapToRangeSensor_), timestamp=sc.timestamp_,
            optimization={k: v for k, v in vars(op).items() if k not in ("backend", "lastStats")},
            mapToRangeSensor=np.array(self.mapToRangeSensor), k=self._k, isNewInitialValueSet=self.isNewInitialValueSet,
            isRelocalized=self.isRelocalized,
            poses=[np.array(T) for T in self.poses])
        arrays["host"] = np.frombuffer(pickle.dumps(host), dtype=np.uint8)
        with open(path, "wb") as f:
            np.savez(f, **arrays)

    @classmethod
    def loadSession(cls, path: str, backend) -> "SegmentMapper":
        """A SegmentMapper on backend continuing the session saveSession wrote: the next addRangeMeasurement / addRangeScan goes on
        where the saved mapper stopped.  results and events start empty; the revisit check's voxel maps are rebuilt from the restored
        maps (backend.build_voxel_map)."""
        with np.load(path, allow_pickle=False) as z:
            arrays = {k: z[k] for k in z.files}
        host = pickle.loads(arrays["host"].tobytes())
        if host["version"] != cls.SESSION_VERSION:
            raise ValueError(f"session format {host['version']}, this version reads {cls.SESSION_VERSION}")

        def get(ref):
            kind, v = ref
            return arrays[v].tobytes() if kind == "array" else v

        m = cls(backend, host["submapParams"], host["isAttemptLoopClosures"], host["loopClosing"])
        sc = m.submaps
        for i, rec in enumerate(host["records"]):
            r = SubmapRecord(backend.import_submap(get(rec["state"])), rec["id"], rec["parent"], np.array(rec["origin"]),
                             None if rec["center"] is None else np.array(rec["center"]))
            if rec["features"]:
                r.sparse, r.feature = backend.restore_features(r.handle, arrays[f"sparse_xyz_{i}"], arrays[f"sparse_nrm_{i}"], arrays[f"feature_{i}"])
            if rec["has_voxel_map"]:
                backend.build_voxel_map(r.handle)
                r.has_voxel_map = True
            sc.submaps.append(r)
        odo = get(host["odometry"])
        if odo is not None:
            backend.import_odometry(odo)
        sc.activeSubmapIdx, sc.numScansMergedInActiveSubmap = host["activeSubmapIdx"], host["numScansMergedInActiveSubmap"]
        for j, (has_cloud, T) in enumerate(host["overlap"]):
            cloud = backend.make_cloud(arrays[f"overlap_xyz_{j}"], arrays.get(f"overlap_nrm_{j}")) if has_cloud else None
            sc.overlapScansBuffer.append((cloud, T))
        sc.finishedSubmapsIdxs, sc.pendingFinishedSubmapIds = host["finishedSubmapsIdxs"], host["pendingFinishedSubmapIds"]
        sc.adjacency, sc.loopClosureSubmaps, sc.adjacencyMatrix = host["adjacency"], host["loopClosureSubmaps"], host["adjacencyMatrix"]
        sc.odometryConstraints, sc.isForceNewSubmapCreation = host["collectionOdometryConstraints"], host["isForceNewSubmapCreation"]
        sc.mapToRangeSensor_, sc.timestamp_ = host["collectionMapToRangeSensor"], host["timestamp"]
        for k, v in host["optimization"].items():
            setattr(m.optimizationProblem, k, v)
        m.mapToRangeSensor, m._k, m.isNewInitialValueSet, m.poses = host["mapToRangeSensor"], host["k"], host["isNewInitialValueSet"], host["poses"]
        m.isRelocalized = host.get("isRelocalized", False)
        return m

    def finishProcessing(self) -> None:
        """SlamWrapper::finishProcessing (src/SlamWrapper.cpp:126-166) once every scan has been mapped: forceNewSubmapCreation finishes
        the active submap, then, with isAttemptLoopClosures, attempts run until one builds no constraint or one correction has been
        applied.  With no worker latency the first attempt does one or the other, so that is one attempt."""
        self.submaps.forceNewSubmapCreation(self._k)
        if self.isAttemptLoopClosures:
            self.attemptLoopClosures(self._k)


def refineLoopClosures(backend, source_handle, target_handles, initial_guesses, mapVoxelSize: float, p: LoopClosureParameters | None = None):
    """The refinement half of PlaceRecognition::buildLoopClosureConstraints for one finished (source) submap against its
    candidate (target) submaps, src/PlaceRecognition.cpp:96-149: overlap selection with voxel = 20 x map voxel, ICP of the
    overlapping parts from the proposal with p.registrationType, fitness gate, information matrix.  The n registrations run as one
    batch.  Returns a list of dicts {overlap sizes, result, accepted, information}."""
    p = p or LoopClosureParameters()
    voxel = p.voxelExpansionFactorOverlapComputation * mapVoxelSize
    pairs = [backend.overlap(source_handle, t, T0, voxel, p.minNumPointsPerVoxel) for t, T0 in zip(target_handles, initial_guesses)]
    # point-to-plane is what register_batch does without a regType, so a backend that only registers point-to-plane needs none;
    # any other estimator is asked for by name, and a backend that cannot take it fails instead of registering point-to-plane
    kw = {} if p.registrationType == "PointToPlaneIcp" else {"regType": p.registrationType}
    results = backend.register_batch([so for so, _to in pairs], [to for _so, to in pairs], initial_guesses, p.maxIcpCorrespondenceDistance, p.maxNumIter,
                                     **kw)
    out = []
    for (so, to), r in zip(pairs, results):
        acc = not (r.fitness_ < p.minRefinementFitness)
        info = backend.information_matrix(so, to, p.maxIcpCorrespondenceDistance, r.transformation_) if acc else None
        out.append({"n_source_overlap": backend.cloud_size(so), "n_target_overlap": backend.cloud_size(to), "result": r, "accepted": acc,
                    "information": info})
    return out


def refineLoopClosuresOfSubmaps(backend, source_sm, target_sms, initial_guesses, mapVoxelSize: float, p: LoopClosureParameters | None = None):
    """refineLoopClosures on the whole maps of the source and candidate submaps (getMapPointCloudCopy, src/PlaceRecognition.cpp:64,95),
    with the map voxel through getMapVoxelSize(mapVoxelSize, 0.04) (:98).  A backend that refines submaps itself (DeviceBackend:
    one batched call on the resident maps) gets the call; a backend that only has the per-cloud operations (the oracle's) gets their
    composition.  The records are refineLoopClosures'; a backend may fill `information` for rejected pairs too."""
    batched = getattr(backend, "refine_loop_closures", None)
    if batched is not None:
        return batched(source_sm, list(target_sms), initial_guesses, mapVoxelSize, p)
    v = E.getMapVoxelSize(mapVoxelSize, E.LoopClosureRefinementParameters.voxelSizeIfMapVoxelSizeIsZero)
    return refineLoopClosures(backend, backend.submap_as_cloud(source_sm), [backend.submap_as_cloud(t) for t in target_sms], initial_guesses, v, p)


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
    """include/open3d_slam/Constraint.hpp:14-20.  timestamp_ is optional here: None on a constraint built without one, which
    updateSubmapsAndTrajectory then treats by list order."""
    sourceToTarget: np.ndarray
    sourceSubmapIdx: int
    targetSubmapIdx: int
    informationMatrix: np.ndarray
    isInformationMatrixValid: bool = True
    isOdometryConstraint: bool = False
    timestamp: int | None = None


def getLoopClosureCandidatesIdxs(collection: SubmapCollection, adjacency: AdjacencyMatrix, lastFinishedIdx: int, activeIdx: int,
                                 params: LoopClosureCandidateParameters | None = None) -> list[int]:
    """PlaceRecognition::getLoopClosureCandidatesIdxs (src/PlaceRecognition.cpp:231-284): every submap i, in order, except
      - the active submap;
      - a submap adjacent to the active one;
      - |i - last| == 1, or i adjacent to last (which excludes last itself);
      - a centre (getMapToSubmapCenter) farther than loopClosureSearchRadius from last's;
      - |i - last| <= ceil(loopClosureSearchRadius / submap radius);
      - any i while the BFS distance of last to the nearest loop-closure submap is below minSubmapsBetweenLoopClosures."""
    params = params or LoopClosureCandidateParameters()
    radius = params.loopClosureSearchRadius
    lastCenter = collection.submaps[lastFinishedIdx].mapToSubmapCenter()
    consecutiveThreshold = math.ceil(radius / collection.params.radius)
    idxs = []
    for i, rec in enumerate(collection.submaps):
        if i == activeIdx:
            continue
        if adjacency.isAdjacent(rec.id, collection.submaps[activeIdx].id):
            continue
        if abs(i - lastFinishedIdx) == 1 or adjacency.isAdjacent(i, lastFinishedIdx):
            continue
        if np.linalg.norm(lastCenter - rec.mapToSubmapCenter()) > radius:
            continue
        if abs(i - lastFinishedIdx) <= consecutiveThreshold:
            continue
        if adjacency.getDistanceToNearestLoopClosureSubmap(lastFinishedIdx) < params.minSubmapsBetweenLoopClosures:
            continue
        idxs.append(i)
    return idxs


def buildLoopClosureConstraints(backend, collection: SubmapCollection, sourceIdx: int, candidateIdxs, params: E.PlaceRecognitionParameters,
                                mapVoxelSize: float, lc: LoopClosureParameters | None = None,
                                consistency: LoopClosureConsistencyCheck | None = None, timestamp: int | None = None):
    """PlaceRecognition::buildLoopClosureConstraints (src/PlaceRecognition.cpp:50-176) for a source submap and its candidates
    (getLoopClosureCandidatesIdxs selects them in SegmentMapper's schedule).  Every candidate: RANSAC proposal (all candidates in one
    batched call, :81-84) -> correspondence-set gate (:86) -> consistency of the RANSAC T (:92) -> refineLoopClosuresOfSubmaps on the
    survivors' maps (one batch, :96-118) -> consistency of the ICP T (:124).  The records need sparse / feature
    (SubmapCollection.computeFeatures).  Every constraint carries `timestamp` (:142, the source submap's finishing scan).
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
        refined = refineLoopClosuresOfSubmaps(backend, src.handle, [collection.submaps[i].handle for i, _ in survivors],
                                              [r.transformation_ for _, r in survivors], mapVoxelSize, lc)
        for (i, _r), o in zip(survivors, refined):
            T = np.array(o["result"].transformation_, dtype=np.float64)
            if not o["accepted"]:
                decision[i] = "rejected_refinement_fitness"
            elif not consistency.isRegistrationConsistent(T):
                decision[i] = "rejected_icp_inconsistent"
            else:
                decision[i] = "accepted"
                constraints.append(Constraint(T, src.id, collection.submaps[i].id, np.array(o["information"]), timestamp=timestamp))
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
    """SlamWrapper::updateSubmapsAndTrajectory (src/SlamWrapper.cpp:450-485).  The latest loop closure is the one with the greatest
    timestamp, the first of them on a tie (std::max_element, :457-459); when a constraint has no timestamp, the last one in
    lastLoopClosureConstraints.  Returns its dT."""
    inc = problem.getOptimizedTransformIncrements()
    mapper.submaps.transform(inc)
    if all(c.timestamp is not None for c in lastLoopClosureConstraints):
        latest = max(lastLoopClosureConstraints, key=lambda c: c.timestamp)   # max keeps the first maximum
    else:
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
    correction of the submaps and of the mapper.  SegmentMapper calls it when isAttemptLoopClosures is on.  Returns the dT applied to
    the mapper."""
    sc = mapper.submaps
    odometryConstraints = sc.getOdometryConstraints()
    computeOdometryConstraints(backend, sc, odometryConstraints, None, odometryParams)
    problem.clearOdometryConstraints()
    problem.insertLoopClosureConstraints(loopClosureConstraints)
    problem.insertOdometryConstraints(odometryConstraints)
    problem.buildOptimizationProblem()
    problem.solve()
    return updateSubmapsAndTrajectory(mapper, problem, list(loopClosureConstraints))


@dataclass
class LoopClosingParameters:
    """What SegmentMapper's loop-closure schedule reads.  mapVoxelSize is the mapper's mapBuilder.mapVoxelSize (the refinement's voxel,
    src/PlaceRecognition.cpp:98); fromMapperParameters takes it and the refinement's ICP type from the backend's MapperParameters."""
    mapVoxelSize: float = 0.1
    placeRecognition: E.PlaceRecognitionParameters = field(default_factory=E.PlaceRecognitionParameters)
    candidates: LoopClosureCandidateParameters = field(default_factory=LoopClosureCandidateParameters)
    refinement: LoopClosureParameters = field(default_factory=LoopClosureParameters)
    consistency: LoopClosureConsistencyCheck = field(default_factory=LoopClosureConsistencyCheck)
    odometryConstraints: E.OdometryConstraintParameters = field(default_factory=E.OdometryConstraintParameters)
    globalOptimization: GlobalOptimizationParameters = field(default_factory=GlobalOptimizationParameters)

    @classmethod
    def fromMapperParameters(cls, mp: E.MapperParameters) -> "LoopClosingParameters":
        v = mp.mapBuilder.mapVoxelSize
        return cls(mapVoxelSize=v, refinement=LoopClosureParameters.fromMapperParameters(mp),
                   odometryConstraints=E.OdometryConstraintParameters(mapVoxelSize=v))


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

    def global_localization(self, sm, raw: np.ndarray, params: E.GlobalLocalizationParameters | None = None) -> E.GlobalLocalizationResult:
        """b2s_submap_global_localization of a raw float32 scan in the submap's map, judged by the mapper's fitness gate
        (MapperParameters::minRefinementFitness_); the submap is left as it was"""
        raw_c = self.eng.cloud(np.ascontiguousarray(raw, dtype=np.float32))
        try:
            return sm.globalLocalization(raw_c, params, self.params.minRefinementFitness)
        finally:
            raw_c.free()

    def global_localization_submaps(self, sms, centers, raw: np.ndarray,
                                    params: E.GlobalLocalizationParameters | None = None) -> E.SubmapsGlobalLocalizationResult:
        """b2s_submaps_global_localization of a raw float32 scan in the union of the submaps (centers: getMapToSubmapCenter of each),
        judged by the mapper's fitness gate; the submaps are left as they were"""
        raw_c = self.eng.cloud(np.ascontiguousarray(raw, dtype=np.float32))
        try:
            return E.globalLocalizationInSubmaps(self.eng, sms, centers, raw_c, params, self.params.minRefinementFitness)
        finally:
            raw_c.free()

    def restart_odometry(self, T) -> None:
        """LidarOdometry starts over at T: the odometry object is dropped, so the next step_with_odometry creates a new one (this
        backend's odometry and de-skew parameters, initial transform T) whose first scan is an initialisation, with no previous cloud
        and both pose buffers (odometry and map poses) empty"""
        if self._odo is not None:
            self._odo.free()
            self._odo = None
        self._odo_initial = np.array(T, dtype=np.float64)

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
        return self.first_scan_at(sm, raw, np.eye(4))

    def first_scan_at(self, sm, raw: np.ndarray, T):
        """the first scan of an empty submap, pre-processed and inserted at T, which becomes the submap's pose"""
        icp = self.mapper.scan2MapReg_
        raw_c = self.eng.cloud(np.ascontiguousarray(raw, dtype=np.float32))
        ps = icp.processForScanMatchingAndMerging(raw_c)
        sm.insertScan(raw_c, ps.merge_, T)
        sm.setPose(T)
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
            odo = E.DeviceLidarOdometry(self.eng, self.odometry_params, self.raw_capacity)
            if self.motion_compensation is not None:
                odo.setMotionCompensation(self.motion_compensation)
            if self._odo_initial is not None:
                odo.setInitialTransform(self._odo_initial)
            self._use_odometry(odo)
        return self._odo

    def _use_odometry(self, odo: E.DeviceLidarOdometry) -> None:
        import torch
        if self.graph:
            odo.enableGraph(self.raw_capacity)
        self._slam_pin = torch.empty(C.sizeof(L.SlamResult), dtype=torch.uint8).pin_memory()
        self._slam_out = L.SlamResult.from_address(self._slam_pin.data_ptr())
        self._odo = odo

    # -- session state (include/b2s.h "session state"): device blobs of the submaps and of the odometry, restored on this backend
    def export_submaps(self, sms) -> list:
        return E.exportSubmapStates(self.eng, sms)

    def import_submap(self, blob: bytes):
        return E.importSubmapState(self.eng, blob)

    def export_odometry(self) -> bytes | None:
        """None while SegmentMapper.addRangeScan has not created the odometry"""
        return None if self._odo is None else self._odo.exportState()

    def import_odometry(self, blob: bytes) -> None:
        """the odometry of the next addRangeScan steps becomes the exported one (its parameters, buffers and de-skew settings)"""
        if self._odo is not None:
            self._odo.free()
        self._use_odometry(E.DeviceLidarOdometry.importState(self.eng, blob, self.odometry_params))

    def cloud_arrays(self, c):
        """a cloud's points and normals (None without), exact fp64 copies"""
        return c.download()

    def make_cloud(self, xyz, nrm=None):
        return self.eng.cloud(xyz, nrm)

    def feature_arrays(self, sparse, feature):
        """a finished submap's feature cloud (points, normals) and FPFH rows, exact fp64 copies"""
        xyz, nrm = sparse.download()
        return xyz, nrm, feature.data_

    def restore_features(self, sm, xyz, nrm, data):
        """the feature cloud and FPFH of compute_features, uploaded into the submap that owns them"""
        sm.sparseMapCloud_ = self.eng.cloud(xyz, nrm)
        sm.feature_ = E.Feature(self.eng, data)
        return sm.getSparseMapPointCloud(), sm.getFeatures()

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

    def map_size(self, sm) -> int:
        return sm.size()

    def assembled_map(self, sms, voxelSize: float):
        """the assembled (and voxelized) map in one b2s_assemble_map call: a device Cloud"""
        return E.getAssembledMapPointCloud(self.eng, sms, voxelSize)

    def assembled_colored_map(self, sms, voxelSize: float):
        """(device Cloud, host rgb) of one b2s_assemble_colored_map call"""
        return E.assembleColoredPointCloud(self.eng, sms, voxelSize)

    def dense_map_clouds(self, sms) -> list:
        """toPointCloud of every submap's dense map: one b2s_assemble_dense_maps call and one download, split by its offsets"""
        c, offsets = E.assembleDenseMaps(self.eng, sms)
        xyz, _ = c.download()
        c.free()
        return [xyz[offsets[k]:offsets[k + 1]] for k in range(len(sms))]

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

    def register_batch(self, sources, targets, inits, max_corr, max_iter, regType: str = "PointToPlaneIcp"):
        pc = E.CloudRegistrationParameters(regType=regType, icp=E.IcpParameters(maxNumIter=max_iter, maxCorrespondenceDistance=max_corr,
                                                                               knn=self.params.icp.knn, maxDistanceKnn=self.params.icp.maxDistanceKnn))
        reg = E.cloudRegistrationFactory(self.eng, pc)
        out = reg.registerCloudsBatch(sources, targets, inits)
        self.eng.set_parameters(self.params)   # the scan-to-map chain keeps its own ICP parameters
        return out

    def information_matrix(self, source, target, max_corr, T):
        return E.getInformationMatrixFromPointClouds(self.eng, source, target, max_corr, T)

    def refine_loop_closures(self, source_sm, target_sms, inits, mapVoxelSize: float, lc: LoopClosureParameters | None = None):
        """refineLoopClosures on the resident maps of the source and candidate submaps in one b2s_submap_loop_closure_refinement call
        (getMapVoxelSize applied to mapVoxelSize, :98).  The same records as refineLoopClosures; the information matrix is there for
        every candidate."""
        lc = lc or LoopClosureParameters()
        prm = E.LoopClosureRefinementParameters(mapVoxelSize=mapVoxelSize, voxelExpansionFactorOverlapComputation=lc.voxelExpansionFactorOverlapComputation,
                                                minNumPointsPerVoxel=lc.minNumPointsPerVoxel, maxNumIter=lc.maxNumIter,
                                                maxIcpCorrespondenceDistance=lc.maxIcpCorrespondenceDistance, minRefinementFitness=lc.minRefinementFitness,
                                                regType=lc.registrationType)
        res = E.refineLoopClosuresBatch(self.eng, source_sm, list(target_sms), inits, prm)
        return [{"n_source_overlap": r.nSourceOverlap, "n_target_overlap": r.nTargetOverlap, "result": r.result, "accepted": r.accepted,
                 "information": r.information} for r in res]

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
