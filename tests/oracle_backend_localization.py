"""The oracle backend (tests/oracle_backend.py) with the reference's localisation mode restated (TEST INFRASTRUCTURE).

Paths relative to open3d_slam/open3d_slam/ (MapperParameters::isUseInitialMap_ / isMergeScansIntoMap_, Parameters.hpp:173-174):
    1. initial map      SlamWrapper::setInitialMap (src/SlamWrapper.cpp:209-220): prepareInitialMap estimates the normals on the full map;
                        addRangeMeasurement's first-scan branch (src/Mapper.cpp:105-108) hands it to SubmapCollection::insertScan, whose
                        Submap::insertScan takes the initial branch: mapCloud_ = map; voxelize(mapVoxelSize) (src/Submap.cpp:47-52)
    2. initial pose     Mapper::setMapToRangeSensorInitial (src/Mapper.cpp:87-91): pose = T, isNewInitialValueSet_
    3. next step        (src/Mapper.cpp:130-149): guess = pose, ICP result discarded, pose kept, no fitness gate, no insertion, the step
                        counts as accepted (the dense map is fed at T), and the step after it predicts without odometry too
    4. pure mode        (src/Mapper.cpp:163-167): an accepted scan updates the pose only; no carving, no insertion
    5. merge mode       merges as in mapping; SubmapCollection never hands over (src/SubmapCollection.cpp:101-107, in slam.py)
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as O
from oracle_backend import OracleBackend, OracleCloud


class OracleLocalizationBackend(OracleBackend):
    def __init__(self, params, carving=True, dense=True):
        super().__init__(params, carving=carving, dense=dense)
        self.params = params
        self.pure = params.isUseInitialMap and not params.isMergeScansIntoMap
        self.isNewInitialValueSet = False
        self.isIgnoreOdometryPrediction = False
        self.guesses: list[np.ndarray] = []   # the initial guess of every registration (pinned by the host-flow tests)

    def initial_map(self, sm, xyz):
        p = self.p
        xyz = np.ascontiguousarray(xyz, dtype=np.float64).reshape(-1, 3)
        nrm = O.estimate_normals(xyz, p.icp.knn, p.icp.maxDistanceKnn)                 # prepareInitialMap
        sm.xyz, sm.nrm = O.voxel_down_sample(xyz, p.mapBuilder.mapVoxelSize, nrm)    # Submap.cpp:47-52
        return OracleCloud(xyz, nrm)

    def set_initial_transform(self, sm, T):
        self.pose = np.array(T, dtype=np.float64)
        self.isNewInitialValueSet = True

    def step(self, sm, raw, odometryMotion):
        p = self.p
        raw64 = np.asarray(raw, dtype=np.float32).astype(np.float64)
        (mx, mn), (ax, an) = self._process(raw)
        self._merge = OracleCloud(mx, mn)
        predict = not self.isNewInitialValueSet and not self.isIgnoreOdometryPrediction
        guess = self.pose @ np.asarray(odometryMotion) if predict else self.pose.copy()
        self.isIgnoreOdometryPrediction = False
        self.guesses.append(guess)
        patch = self._cropper(p.scanProcessing.cropper, center=self.pose[:3, 3])
        px, pn = O.crop(patch, sm.xyz, sm.nrm)
        res = O.registration_icp_p2plane(ax, px, pn, p.icp.maxCorrespondenceDistance, guess, max_iter=p.icp.maxNumIter)
        res.transformation_ = res.T; res.fitness_ = res.fitness; res.inlier_rmse_ = res.inlier_rmse
        if self.isNewInitialValueSet:   # rule 3
            self.isNewInitialValueSet = False
            self.isIgnoreOdometryPrediction = True
            if self.dense:
                self._dense(sm, raw64, self.pose)
            return res, True
        accepted = p.isIgnoreMinRefinementFitness or not (res.fitness < p.minRefinementFitness)
        if accepted:
            self.pose = np.array(res.T)
            if not self.pure:           # rule 4
                if self.carving:
                    self._carve(sm, raw64, self.pose)
                self._insert(sm, mx, mn, self.pose)
            if self.dense:
                self._dense(sm, raw64, self.pose)
        return res, bool(accepted)
