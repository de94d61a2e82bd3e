"""The synthetic workloads of BASELINE.json's configs 2-5 (SURVEY.md section 8d), shared by bench.py, tools/ and tests/ so that
every one of them measures / checks the same inputs.  numpy + the device engine only (nothing here touches the oracle).

    ClosedLoop          config 2 / 5: one exact lap of the rounded-rectangle trajectory (scan k + L is cast from the pose of scan
                        k), ray casts cached, one noise realisation per (chain, position); odometry deltas with a small error
    config3_cloud()     config 3: 2^20 returns of 21 scans in the map frame
    Config4             config 4: P scan-submap pairs over T shared 20 m-radius target submaps (pair i -> target i % T), the
                        batched loop-closure ICP of src/PlaceRecognition.cpp:45-46,111 (r = 0.3, <= 100 iterations)
"""
from __future__ import annotations

import copy

import numpy as np

from . import synth


# ----------------------------------------------------------------------------------------------------------------------
# config 2 / 5: closed lap
# ----------------------------------------------------------------------------------------------------------------------
class ClosedLoop:
    def __init__(self, step: float = 0.5, noise: float = 0.02, odom_seed: int = 12345):
        self.scene = synth.Scene()
        perimeter = synth.loop_length()
        self.L = int(round(perimeter / step))
        self.step = perimeter / self.L
        self.poses = synth.loop_trajectory(self.L, step=self.step)
        self.noise = noise
        self._casts = {}
        self._casts_moving = {}
        rng = np.random.default_rng(odom_seed)
        self._pert = [synth.se3(0.0, 0.0, rng.normal(0, 2e-3), rng.normal(0, 0.02, 3)) for _ in range(self.L)]   # stands in for the odometry error

    def pose(self, k: int) -> np.ndarray:
        return self.poses[k % self.L]

    def cast(self, k: int):
        k %= self.L
        if k not in self._casts:
            self._casts[k] = synth.lidar_cast(self.scene, self.poses[k])
        return self._casts[k]

    def scan(self, k: int, seed: int) -> np.ndarray:
        """float32 sensor-frame scan of lap position k % L with the noise realisation `seed`"""
        return synth.lidar_from_cast(self.cast(k), self.noise, seed=seed)

    def pose_between(self, k: int, phase: float) -> np.ndarray:
        """the sensor pose a fraction `phase` of the way from pose(k) to pose(k + 1): translation linear, yaw slerped (the loop is
        planar, so the slerp of two yaw rotations is the yaw rotation by the interpolated angle)"""
        A, B = self.pose(k), self.pose(k + 1)
        if phase == 0.0:
            return A.copy()
        ya, yb = np.arctan2(A[1, 0], A[0, 0]), np.arctan2(B[1, 0], B[0, 0])
        dy = (yb - ya + np.pi) % (2 * np.pi) - np.pi
        return synth.se3(0.0, 0.0, ya + phase * dy, A[:3, 3] + phase * (B[:3, 3] - A[:3, 3]))

    def cast_moving(self, k: int, clockwise: bool = True):
        """rolling-shutter cast of scan k: the sensor moves from pose(k) to pose(k + 1) during the scan (one scan period = one
        scan_duration), each azimuth column is measured at its computePhase"""
        key = (k % self.L, bool(clockwise))
        if key not in self._casts_moving:
            self._casts_moving[key] = synth.lidar_cast_moving(self.scene, lambda ph: self.pose_between(k, ph), clockwise=clockwise)
        return self._casts_moving[key]

    def scan_moving(self, k: int, seed: int, clockwise: bool = True) -> np.ndarray:
        """float32 scan of lap position k taken while moving on to k + 1 (noise realisation `seed`); its timestamp's ground truth
        stays pose(k)"""
        return synth.lidar_from_cast(self.cast_moving(k, clockwise), self.noise, seed=seed)

    def delta(self, k: int) -> np.ndarray:
        """odometry motion between scan k-1 and scan k (identity for k = 0)"""
        if k == 0:
            return np.eye(4)
        return np.linalg.inv(self.pose(k - 1)) @ self.pose(k) @ self._pert[k % self.L]

    def map_frame_pose(self, k: int) -> np.ndarray:
        """ground truth mapToRangeSensor of scan k when scan 0 defines the map frame"""
        return np.linalg.inv(self.poses[0]) @ self.pose(k)


# ----------------------------------------------------------------------------------------------------------------------
# config 3
# ----------------------------------------------------------------------------------------------------------------------
def config3_cloud(n_points: int = 1 << 20, n_scans: int = 21) -> np.ndarray:
    sc = synth.Scene(); poses = synth.loop_trajectory(600)
    parts = []
    for i in range(n_scans):
        T = poses[(i * 37) % 600]
        s = synth.lidar_scan(sc, T, seed=1000 + i).astype(np.float64)
        parts.append(s @ T[:3, :3].T + T[:3, 3])
    return np.ascontiguousarray(np.vstack(parts)[:n_points])   # scans lose their sky rays: 21 scans give > 2^20 returns


# ----------------------------------------------------------------------------------------------------------------------
# config 4
# ----------------------------------------------------------------------------------------------------------------------
class Config4:
    """P pairs, T shared targets.  Target t = the scans at lap positions c_t - 10, c_t - 6, ..., c_t + 10 (every 4th = 2 m apart,
    6 scans) fused at their true poses with the engine's own S1 (ratio 1) + F1: a 20 m-radius submap of the courtyard.  Pair i:
    target t = i % T, source = the pre-processed (match_) scan at position c_t + ((i // T) % 8 - 4) with noise seed 7000 + i,
    initial guess = its true pose displaced by a random SE(3) within (+-0.5 m, +-5 deg) (seed = pair id)."""

    R_ICP, MAX_ITER = 0.3, 100

    def __init__(self, loop: ClosedLoop, n_pairs: int = 512, n_targets: int = 64, scans_per_target: int = 6, spacing: int = 4):
        self.loop, self.P, self.T = loop, n_pairs, n_targets
        self.scans_per_target, self.spacing = scans_per_target, spacing

    def center(self, t: int) -> int:
        return int(round(t * self.loop.L / self.T))

    def target_of(self, i: int) -> int:
        return i % self.T

    def target_positions(self, t: int):
        c = self.center(t)
        half = (self.scans_per_target - 1) * self.spacing // 2
        return [c - half + j * self.spacing for j in range(self.scans_per_target)]

    def source_position(self, i: int) -> int:
        return self.center(self.target_of(i)) + ((i // self.T) % 8 - 4)

    def truth(self, i: int) -> np.ndarray:
        return self.loop.pose(self.source_position(i))

    def init(self, i: int) -> np.ndarray:
        rng = np.random.default_rng(i)
        return self.truth(i) @ synth.se3(*np.deg2rad(rng.uniform(-5, 5, 3)), rng.uniform(-0.5, 0.5, 3))

    # -- device builders (E = open3d_slam_b200.engine, passed in to keep this module importable without the library)
    def build_target(self, E, eng, icp, params, t: int, capacity: int = 700_000):
        """returns a device Cloud (xyz + normals) holding target submap t"""
        p_full = copy.deepcopy(params); p_full.scanProcessing.downSamplingRatio = 1.0   # submaps keep every voxel of the scans they fuse
        eng.set_parameters(p_full)
        sm = E.Submap(eng, capacity)
        for k in self.target_positions(t):
            raw = eng.cloud(self.loop.scan(k, seed=5000 + (k % self.loop.L)))
            ps = icp.processForScanMatchingAndMerging(raw)
            sm.insertScan(None, ps.merge_, self.loop.pose(k))
            raw.free(); ps.merge_.free(); ps.match_.free()
        xyz, nrm = sm.getMapPointCloud()
        sm.free()
        eng.set_parameters(params)
        return eng.cloud(xyz, nrm)

    def build_source(self, E, eng, icp, i: int):
        raw = eng.cloud(self.loop.scan(self.source_position(i), seed=7000 + i))
        ps = icp.processForScanMatchingAndMerging(raw)
        raw.free(); ps.merge_.free()
        return ps.match_

    def registration(self, E, eng, params):
        pc = E.CloudRegistrationParameters(icp=copy.deepcopy(params.icp))
        pc.icp.maxCorrespondenceDistance = self.R_ICP
        pc.icp.maxNumIter = self.MAX_ITER
        return E.RegistrationIcpPointToPlane(eng, pc)
