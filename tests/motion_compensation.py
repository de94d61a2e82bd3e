"""numpy restatement of ConstantVelocityMotionCompensation::estimateLinearAndAngularVelocity (src/MotionCompensation.cpp:32-57) over the
numpy TransformInterpolationBuffer, and the oracle composition of SlamWrapper's two workers with both de-skews
(src/SlamWrapper.cpp:266-268,298-304): the reference the device de-skew of the combined step is checked against (TEST INFRASTRUCTURE).

The de-skewed clouds stay fp64 all the way down, as on the device: the oracle pre-processing below never rounds them to float32."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S

from odometry_buffer import TransformInterpolationBuffer
from oracle_backend import OracleBackend, OracleCloud
from test_gpu_odometry import OracleOdometry


def _fp64(raw) -> np.ndarray:
    """a float32 wire scan widened as the upload widens it; an fp64 (de-skewed) cloud as it is"""
    x = np.asarray(raw)
    return x.astype(np.float64) if x.dtype == np.float64 else np.asarray(x, dtype=np.float32).astype(np.float64)


def iso_inv(T) -> np.ndarray:
    """Eigen's inverse of an isometry: (R^T, -(R^T t))"""
    T = np.asarray(T, dtype=np.float64)
    out = np.eye(4)
    out[:3, :3] = T[:3, :3].T
    out[:3, 3] = -(T[:3, :3].T @ T[:3, 3])
    return out


def estimate_velocity(buf: TransformInterpolationBuffer, t: int, offset: int):
    """:32-57 -> (linear velocity, angular velocity rpy).  size <= offset or latest_time >= t: zeros; else dT = start^-1 * finish of
    the latest entry and the one `offset` before it, v = dT.translation / (dt + 1e-6), w = toRPY(dT.rotation) / (dt + 1e-6)"""
    e = buf.entries
    zero = (np.zeros(3), np.zeros(3))
    if len(e) <= offset or not e[-1][0] < t:
        return zero
    (ts, Ts), (tf, Tf) = e[-1 - offset], e[-1]
    dT = iso_inv(Ts) @ Tf
    den = (tf - ts) / 1e7 + 1e-6
    return dT[:3, 3] / den, np.array(S.toRPY(dT[:3, :3])) / den


def deskew(raw, buf: TransformInterpolationBuffer, t: int, mc: E.ConstantVelocityMotionCompensationParameters):
    """undistortInputPointCloud with the velocities of `buf` at t -> (fp64 cloud, v, w)"""
    v, w = estimate_velocity(buf, t, mc.numPosesVelocityEstimation)
    return O.undistort(_fp64(raw), v, w, mc.scanDuration, mc.isSpinningClockwise), v, w


class DeskewOdometry(OracleOdometry):
    """odometryWorker: the odometry composition on the scan de-skewed from its own buffer (when mc is enabled)"""

    def __init__(self, op: E.OdometryParameters, mc: E.ConstantVelocityMotionCompensationParameters):
        super().__init__(op)
        self.mc = mc
        self.velocity = (np.zeros(3), np.zeros(3))

    def preprocess(self, raw):
        sp, ic = self.op.scanProcessing, self.op.scanMatcher.icp
        cx, _ = O.crop(self.crop, _fp64(raw))
        if len(cx) == 0:
            return np.zeros((0, 3)), np.zeros((0, 3))
        vx, _ = O.voxel_down_sample(cx, sp.voxelSize)
        vn = O.estimate_normals(vx, ic.knn, ic.maxDistanceKnn)
        return O.random_down_sample(vx, sp.downSamplingRatio, self.op.seed, vn)

    def step(self, raw, t, deskewed=None):
        """deskewed: the cloud to go on with instead of this composition's own de-skew, which is kept in self.deskewed for the caller
        to compare (see DeskewBackend.step_with_odometry)"""
        if self.mc.isUndistortInputCloud:
            own, v, w = deskew(raw, self.buf, t, self.mc)
            self.velocity, self.deskewed = (v, w), own
            raw = own if deskewed is None else deskewed
        return super().step(raw, t)


class DeskewBackend(OracleBackend):
    """OracleBackend + DeskewOdometry + the mapper's mapToRangeSensorBuffer_ and its de-skew (mappingWorker): the oracle side of
    SegmentMapper.addRangeScan on a DeviceBackend with motionCompensation"""

    def __init__(self, params, op: E.OdometryParameters, mc: E.ConstantVelocityMotionCompensationParameters, **kw):
        super().__init__(params, **kw)
        self.mc = mc
        self.odo = DeskewOdometry(op, mc)
        self.map_buf = TransformInterpolationBuffer(op.bufferSize)
        self.t_last = 0
        self.velocity = (np.zeros(3), np.zeros(3))
        self.deskewed = None

    def _process(self, raw):
        p = self.p
        return O.process_scan(_fp64(raw), self.wide, self.narrow, p.scanProcessing.voxelSize, p.icp.knn, p.icp.maxDistanceKnn,
                              p.scanProcessing.downSamplingRatio, p.seed)

    def step(self, sm, raw, odometryMotion):
        """OracleBackend.step on an fp64 scan"""
        p = self.p
        raw64 = _fp64(raw)
        (mx, mn), (ax, an) = self._process(raw64)
        self._merge = OracleCloud(mx, mn)
        patch = self._cropper(p.scanProcessing.cropper, center=self.pose[:3, 3])
        px, pn = O.crop(patch, sm.xyz, sm.nrm)
        res = O.registration_icp_p2plane(ax, px, pn, p.icp.maxCorrespondenceDistance, self.pose @ np.asarray(odometryMotion), max_iter=p.icp.maxNumIter)
        res.transformation_ = res.T; res.fitness_ = res.fitness; res.inlier_rmse_ = res.inlier_rmse
        accepted = p.isIgnoreMinRefinementFitness or not (res.fitness < p.minRefinementFitness)
        if accepted:
            self.pose = np.array(res.T)
            if self.carving:
                self._carve(sm, raw64, self.pose)
            self._insert(sm, mx, mn, self.pose)
            if self.dense:
                self._dense(sm, raw64, self.pose)
        return res, bool(accepted)

    def first_scan_with_odometry(self, sm, raw, t):
        """Mapper.cpp:105-114 (the push at :112) and the odometry's first scan; both buffers are empty, so no de-skew moves a point"""
        merge = self.first_scan(sm, raw)
        self.odo.step(raw, t)
        self.map_buf.push(t, np.eye(4))
        return merge

    def step_with_odometry(self, sm, raw, t):
        """self.inject = (odometry input, mapper input): go on with these de-skewed clouds (a device step's, compared step by step)
        instead of this composition's own, which stay in self.odo.deskewed / self.deskewed.  The device's RandomDownSample selects
        points by a hash of their bits, so a de-skewed point one ulp away (libm, or poses that differ in their last bits) selects
        another subset: a comparison with the device that is to be exact downstream of the de-skew starts from the same bits."""
        inject, self.inject = getattr(self, "inject", None), None
        self.odo_result = self.odo.step(raw, t, None if inject is None else inject[0])
        b = self.odo.buf
        motion = np.linalg.inv(b.get_transform(self.t_last)) @ b.get_transform(t) if b.has(t) else np.eye(4)
        if self.mc.isUndistortInputCloud:
            own, v, w = deskew(raw, self.map_buf, t, self.mc)
            self.velocity, self.deskewed = (v, w), own
            raw = own if inject is None else inject[1]
        res, acc = self.step(sm, raw, motion)
        if acc:
            self.map_buf.push(t, res.T)    # Mapper.cpp:160, before the minimum-motion gate
            self.t_last = t
        return res, acc
