"""CPU tests of the de-skew references (-m "not gpu"): the numpy velocity estimate of tests/motion_compensation.py against independent
answers, the rolling-shutter cast of synth.lidar_cast_moving, and oracle.undistort with the true velocity on a straight segment."""
import numpy as np

from oracle import oracle as O
from open3d_slam_b200 import synth
from open3d_slam_b200 import workloads as W

from motion_compensation import estimate_velocity
from odometry_buffer import TransformInterpolationBuffer

TICK = 10_000_000


def _buffer(poses, times, limit=2000):
    b = TransformInterpolationBuffer(limit)
    for t, T in zip(times, poses):
        b.push(t, T)
    return b


def test_pure_translation_gives_displacement_over_dt():
    step = np.array([0.5, -0.1, 0.02])
    poses = [synth.se3(t=k * step) for k in range(6)]
    times = [1000 + k * TICK // 10 for k in range(6)]
    b = _buffer(poses, times)
    v, w = estimate_velocity(b, times[-1] + 1, 3)
    dp = poses[-1][:3, 3] - poses[-4][:3, 3]
    assert np.array_equal(v, dp / ((times[-1] - times[-4]) / 1e7 + 1e-6))
    assert np.array_equal(w, np.zeros(3))


def test_pure_yaw_at_constant_rate():
    rate = 0.8   # rad/s
    times = [k * TICK // 10 for k in range(5)]
    poses = [synth.se3(yaw=rate * t / 1e7) for t in times]
    v, w = estimate_velocity(_buffer(poses, times), times[-1] + 5, 2)
    dt = (times[-1] - times[-3]) / 1e7
    assert np.abs(v).max() < 1e-15
    assert abs(w[2] - rate * dt / (dt + 1e-6)) < 1e-12 and abs(w[0]) < 1e-15 and abs(w[1]) < 1e-15


def test_too_few_poses_or_a_stamp_not_before_the_latest_gives_zeros():
    poses = [synth.se3(yaw=0.1 * k, t=(k, 0.0, 0.0)) for k in range(4)]
    times = [10, 20, 30, 40]
    for offset in (3, 4, 7):                                   # size <= offset
        v, w = estimate_velocity(_buffer(poses[:offset], times[:offset]), 100, offset)
        assert not v.any() and not w.any()
    b = _buffer(poses, times)
    assert np.abs(estimate_velocity(b, 41, 3)[0]).max() > 0
    for t in (40, 39, 5):                                      # latest_time >= t: "Warning buffer has this already", zeros
        v, w = estimate_velocity(b, t, 3)
        assert not v.any() and not w.any()


def test_evicting_buffer_uses_the_entry_offset_before_the_latest():
    acc = np.array([0.0, 0.0, 0.0])
    poses, times = [], []
    for k in range(9):                                         # accelerating along x: every pair of entries gives another velocity
        acc = acc + np.array([0.1 * (k + 1), 0.0, 0.0])
        poses.append(synth.se3(t=acc.copy())); times.append(k * 1_000_000)
    b = _buffer(poses, times, limit=5)
    assert len(b.entries) == 5 and b.entries[0][0] == times[4]
    v, _ = estimate_velocity(b, times[-1] + 1, 3)
    assert np.array_equal(v, (poses[8][:3, 3] - poses[5][:3, 3]) / ((times[8] - times[5]) / 1e7 + 1e-6))
    v, w = estimate_velocity(_buffer(poses, times, limit=3), times[-1] + 1, 3)   # eviction keeps the size at the offset: zeros
    assert not v.any() and not w.any()


def test_moving_cast_without_motion_is_lidar_cast():
    sc = synth.Scene()
    pose = synth.loop_trajectory(40)[17]
    d0, r0 = synth.lidar_cast(sc, pose)
    for cw in (True, False):
        d1, r1 = synth.lidar_cast_moving(sc, lambda ph: pose, clockwise=cw)
        assert np.array_equal(d0, d1) and np.array_equal(r0, r1)


def test_phase_follows_compute_phase():
    az = np.array([0.0, np.pi / 2, np.pi, 1.5 * np.pi])
    assert np.array_equal(synth.scan_phase(az, True), [0.0, 0.75, 0.5, 0.25])
    assert np.array_equal(synth.scan_phase(az, False), [0.0, 0.25, 0.5, 0.75])


def _surface_distance(scene, w):
    cyl = np.min(np.abs(np.linalg.norm(w[:, None, :2] - scene.cylinders[None], axis=2) - scene.cyl_r), axis=1)
    return np.minimum.reduce([np.abs(w[:, 2] - scene.ground_z), np.abs(np.abs(w[:, 0]) - scene.half_x), np.abs(np.abs(w[:, 1]) - scene.half_y), cyl])


def test_undistort_with_true_velocity_puts_a_straight_moving_scan_back_on_the_surfaces():
    """on a straight segment (pure translation: constant velocity is exact) the noise-free rolling-shutter scan, de-skewed with the
    true body velocity and moved by pose(k), lies on the ground, the walls and the cylinders to 1e-9; the raw scan does not"""
    lp = W.ClosedLoop(noise=0.0)
    for k in (14, 22):
        A, B = lp.pose(k), lp.pose(k + 1)
        assert np.array_equal(A[:3, :3], B[:3, :3])              # straight: no rotation
        for cw in (True, False):
            d, r = lp.cast_moving(k, clockwise=cw)
            raw = d * r[:, None]
            v = A[:3, :3].T @ (B[:3, 3] - A[:3, 3]) / 0.1
            out = O.undistort(raw, v, np.zeros(3), 0.1, cw)
            w = out @ A[:3, :3].T + A[:3, 3]
            dist = _surface_distance(lp.scene, w)
            assert dist.max() < 1e-9, (k, cw, dist.max())
            on_ground = np.abs(w[:, 2] - lp.scene.ground_z) < 1e-9
            on_walls = (np.abs(np.abs(w[:, 0]) - lp.scene.half_x) < 1e-9) | (np.abs(np.abs(w[:, 1]) - lp.scene.half_y) < 1e-9)
            assert on_ground.sum() > 1000 and on_walls.sum() > 1000 and (~on_ground & ~on_walls).sum() > 100   # cylinders too
            raw_dist = _surface_distance(lp.scene, raw @ A[:3, :3].T + A[:3, 3])
            assert raw_dist.max() > 0.3
