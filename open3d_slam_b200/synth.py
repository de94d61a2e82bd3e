"""Synthetic inputs for the configs of BASELINE.json (SURVEY.md section 8d): the reference ships no data.

numpy only; used by tests/ and bench.py on both the CPU and the GPU box.
  - planar_cloud_config1(): 2 000-point three-plane cloud + displaced noisy copy (config 1)
  - Scene / lidar_scan():   64-beam x 1024-azimuth spinning LiDAR ray-cast against ground + courtyard walls
                            + cylinders, float32 xyz like the ROS wire format (configs 2-5)
  - loop_trajectory():      rounded-rectangle trajectory, 0.5 m per scan
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np


def rot_zyx(roll, pitch, yaw):
    ca, sa, cb, sb, cg, sg = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cg, -sg, 0], [sg, cg, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def se3(roll=0.0, pitch=0.0, yaw=0.0, t=(0.0, 0.0, 0.0)):
    T = np.eye(4)
    T[:3, :3] = rot_zyx(roll, pitch, yaw)
    T[:3, 3] = t
    return T


def planar_cloud_config1(n=2000, seed=1, noise=0.01, noise_seed=2):
    """Config 1 (SURVEY.md 8d): three mutually orthogonal 10 m planes (n/2, n/4, n/4 points) with analytic
    normals = target; source = target moved by yaw 3 deg, pitch 1 deg, t=(0.10,-0.05,0.02) + N(0, noise)."""
    rng = np.random.default_rng(seed)
    n0 = n // 2; n1 = n // 4; n2 = n - n0 - n1
    a = rng.uniform(0.0, 10.0, size=(n0, 2)); b = rng.uniform(0.0, 10.0, size=(n1, 2)); c = rng.uniform(0.0, 10.0, size=(n2, 2))
    tgt = np.vstack([np.c_[a[:, 0], a[:, 1], np.zeros(n0)],      # z = 0 plane
                     np.c_[b[:, 0], np.zeros(n1), b[:, 1]],      # y = 0 plane
                     np.c_[np.zeros(n2), c[:, 0], c[:, 1]]])     # x = 0 plane
    nrm = np.vstack([np.tile([0.0, 0.0, 1.0], (n0, 1)), np.tile([0.0, 1.0, 0.0], (n1, 1)), np.tile([1.0, 0.0, 0.0], (n2, 1))])
    T_true = se3(0.0, np.deg2rad(1.0), np.deg2rad(3.0), (0.10, -0.05, 0.02))
    src = tgt @ T_true[:3, :3].T + T_true[:3, 3]
    if noise > 0:
        src = src + np.random.default_rng(noise_seed).normal(0.0, noise, size=src.shape)
    return src, tgt, nrm, T_true


@dataclass
class Scene:
    """Ground plane z = ground_z, a rectangular courtyard of 4 walls and vertical cylinders."""
    ground_z: float = -1.8
    half_x: float = 20.0
    half_y: float = 20.0
    wall_h: float = 6.0
    cylinders: np.ndarray = field(default_factory=lambda: Scene.default_cylinders())
    cyl_r: float = 0.4

    @staticmethod
    def default_cylinders(n=12, seed=7):
        rng = np.random.default_rng(seed)
        ang = np.linspace(0, 2 * np.pi, n, endpoint=False) + rng.uniform(-0.1, 0.1, n)
        rad = rng.uniform(6.0, 15.0, n)
        return np.c_[rad * np.cos(ang), rad * np.sin(ang)]


def _ray_dirs(n_beams=64, n_az=1024, fov_deg=45.0):
    el = np.deg2rad(np.linspace(-fov_deg / 2, fov_deg / 2, n_beams))
    az = np.linspace(0.0, 2 * np.pi, n_az, endpoint=False)
    ce, se = np.cos(el)[:, None], np.sin(el)[:, None]
    d = np.stack([ce * np.cos(az)[None, :], ce * np.sin(az)[None, :], np.broadcast_to(se, (n_beams, n_az))], axis=-1)
    return d.reshape(-1, 3)


def lidar_scan(scene: Scene, pose: np.ndarray, n_beams=64, n_az=1024, max_range=60.0, noise=0.02, seed=0, dtype=np.float32):
    """Ray-cast one scan. pose = map->sensor 4x4. Returns (n_hits, 3) points in the SENSOR frame (dtype float32 like
    sensor_msgs/PointCloud2, open3d_conversions.cpp:61-67). Rays without a hit within max_range are dropped."""
    dl = _ray_dirs(n_beams, n_az)
    R = pose[:3, :3]; o = pose[:3, 3]
    d = dl @ R.T
    t_best = _hit_distances(scene, d, o)
    hit = np.isfinite(t_best) & (t_best <= max_range)
    rng = np.random.default_rng(seed)
    rr = t_best[hit] + (rng.normal(0.0, noise, size=int(hit.sum())) if noise > 0 else 0.0)
    pts = dl[hit] * rr[:, None]
    return np.ascontiguousarray(pts.astype(dtype))


def _hit_distances(scene: Scene, d: np.ndarray, o) -> np.ndarray:
    """distance along every map-frame ray direction d[i] to the first surface (inf: none); o = the rays' origin, (x, y, z) as
    scalars (one sensor pose) or as per-ray arrays (lidar_cast_moving): the arithmetic per ray is the same either way"""
    t_best = np.full(len(d), np.inf)
    # ground
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (scene.ground_z - o[2]) / d[:, 2]
    t = np.where((t > 0) & np.isfinite(t), t, np.inf)
    with np.errstate(invalid="ignore"):   # inf * 0 for rays parallel to the plane: those rows are rejected below
        hx = o[0] + t * d[:, 0]; hy = o[1] + t * d[:, 1]
    okg = (np.abs(hx) <= scene.half_x) & (np.abs(hy) <= scene.half_y)
    t_best = np.minimum(t_best, np.where(okg, t, np.inf))
    # walls
    for axis, val, other_half in ((0, scene.half_x, scene.half_y), (0, -scene.half_x, scene.half_y),
                                  (1, scene.half_y, scene.half_x), (1, -scene.half_y, scene.half_x)):
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (val - o[axis]) / d[:, axis]
        t = np.where((t > 0) & np.isfinite(t), t, np.inf)
        oth = 1 - axis
        with np.errstate(invalid="ignore"):
            ho = o[oth] + t * d[:, oth]; hz = o[2] + t * d[:, 2]
        ok = (np.abs(ho) <= other_half) & (hz >= scene.ground_z) & (hz <= scene.ground_z + scene.wall_h)
        t_best = np.minimum(t_best, np.where(ok, t, np.inf))
    # cylinders (infinite in z, clipped to wall height)
    a = d[:, 0] ** 2 + d[:, 1] ** 2
    for cx, cy in scene.cylinders:
        fx = o[0] - cx; fy = o[1] - cy
        b = 2 * (fx * d[:, 0] + fy * d[:, 1])
        c = fx * fx + fy * fy - scene.cyl_r ** 2
        disc = b * b - 4 * a * c
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (-b - np.sqrt(np.where(disc >= 0, disc, np.nan))) / (2 * a)
        hz = o[2] + t * d[:, 2]
        ok = np.isfinite(t) & (t > 0) & (hz >= scene.ground_z) & (hz <= scene.ground_z + scene.wall_h)
        t_best = np.minimum(t_best, np.where(ok, t, np.inf))
    return t_best


def _loop_path(half=8.0, corner_r=3.0):
    """closed rounded-rectangle polyline and its cumulative arc length"""
    segs = []
    s = half - corner_r
    corners = [(s, -s, -np.pi / 2), (s, s, 0.0), (-s, s, np.pi / 2), (-s, -s, np.pi)]
    for (cx, cy, a0) in corners:
        th = np.linspace(a0, a0 + np.pi / 2, 64)
        segs.append(np.c_[cx + corner_r * np.cos(th), cy + corner_r * np.sin(th)])
    path = np.vstack(segs + [segs[0][:1]])
    seglen = np.linalg.norm(np.diff(path, axis=0), axis=1)
    cum = np.r_[0.0, np.cumsum(seglen)]
    return path, seglen, cum


def loop_length(half=8.0, corner_r=3.0) -> float:
    """length of one lap of loop_trajectory()'s path"""
    return float(_loop_path(half, corner_r)[2][-1])


def loop_trajectory(n_scans=600, step=0.5, half=8.0, corner_r=3.0, z=0.0):
    """Rounded-rectangle loop (config 2): poses map->sensor, heading along the path, `step` metres per scan."""
    # the closed path is a dense polyline, resampled by arc length
    path, seglen, cum = _loop_path(half, corner_r)
    total = cum[-1]
    poses = []
    for k in range(n_scans):
        sarc = (k * step) % total
        i = np.searchsorted(cum, sarc, side="right") - 1
        i = min(i, len(seglen) - 1)
        f = (sarc - cum[i]) / seglen[i]
        p = path[i] * (1 - f) + path[i + 1] * f
        dvec = path[i + 1] - path[i]
        yaw = np.arctan2(dvec[1], dvec[0])
        poses.append(se3(0.0, 0.0, yaw, (p[0], p[1], z)))
    return poses


def lidar_cast(scene: Scene, pose: np.ndarray, n_beams=64, n_az=1024, max_range=60.0):
    """Noise-free part of lidar_scan(): returns (unit directions in the sensor frame of the rays that hit, ranges)."""
    clean = lidar_scan(scene, pose, n_beams, n_az, max_range, noise=0.0, seed=0, dtype=np.float64)
    r = np.linalg.norm(clean, axis=1)
    return clean / r[:, None], r


def scan_phase(az: np.ndarray, clockwise: bool = True) -> np.ndarray:
    """ConstantVelocityMotionCompensation::computePhase (core/src/MotionCompensation.cpp:120-139) of azimuths in [0, 2 pi): the fraction
    of the scan period after the scan's timestamp at which that azimuth is measured; 0 at az = 0"""
    az = np.asarray(az, dtype=np.float64)
    ph = 1.0 - az / (2 * np.pi) if clockwise else az / (2 * np.pi)
    return np.where(az == 0.0, 0.0, ph)


def lidar_cast_moving(scene: Scene, pose_at, n_beams=64, n_az=1024, max_range=60.0, clockwise=True):
    """Rolling-shutter lidar_cast(): azimuth column j is cast from its own pose pose_at(phase_j) (map -> sensor), phase_j =
    scan_phase(2 pi j / n_az).  Every return is expressed in the sensor frame of its own column, as a spinning sensor reports it.
    Returns (unit directions, ranges) of the rays that hit, in lidar_cast's order; lidar_from_cast adds the noise.  With a constant
    pose_at this is lidar_cast exactly."""
    dl = _ray_dirs(n_beams, n_az)
    az = np.linspace(0.0, 2 * np.pi, n_az, endpoint=False)
    phases = scan_phase(az, clockwise)
    d = np.empty_like(dl)
    o = np.empty_like(dl)
    for j, ph in enumerate(phases):          # rows of column j: beam * n_az + j
        P = np.asarray(pose_at(float(ph)), dtype=np.float64)
        d[j::n_az] = dl[j::n_az] @ P[:3, :3].T
        o[j::n_az] = P[:3, 3]
    t_best = _hit_distances(scene, d, (o[:, 0], o[:, 1], o[:, 2]))
    hit = np.isfinite(t_best) & (t_best <= max_range)
    clean = dl[hit] * (t_best[hit] + 0.0)[:, None]
    r = np.linalg.norm(clean, axis=1)
    return clean / r[:, None], r


def lidar_from_cast(cast, noise=0.02, seed=0, dtype=np.float32):
    """Apply range noise N(0, noise) (seeded) to a lidar_cast() result; identical to lidar_scan() up to rounding."""
    d, r = cast
    rr = r + (np.random.default_rng(seed).normal(0.0, noise, size=len(r)) if noise > 0 else 0.0)
    return np.ascontiguousarray((d * rr[:, None]).astype(dtype))
