"""Child process of tests/test_gpu_boundaries.py for the cases that depend on process-wide knobs.

The library reads B2S_GRID_CAP and B2S_SORT once per process, so each setting needs a process of its own.

    python tests/boundary_child.py ops OUT.npz        -- a fixed set of operations, every output written to OUT.npz

It also holds the clouds and parameters that reach every exit of the normals select kernel (imported by the tests).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import synth  # noqa: E402


def exits_scan(seed=21):
    """A LiDAR scan plus a dense 1 m blob (more candidates than the select kernel's buffer holds) and isolated points far from
    everything (fewer than k neighbours inside the radius)."""
    rng = np.random.default_rng(seed)
    raw = synth.lidar_scan(synth.Scene(), synth.loop_trajectory(4)[1], seed=seed).astype(np.float64)
    blob = np.array([4.0, 3.0, 0.5]) + rng.uniform(0.0, 1.0, (6000, 3))
    lonely = np.c_[rng.uniform(-20.0, 20.0, (40, 2)), rng.uniform(6.0, 9.0, 40)]
    return np.ascontiguousarray(np.vstack([raw, blob, lonely]))


def exits_params(knn=20):
    """Radius 4 at the 0.4 m index cell of process_scan: the whole ball does not fit the kernel's largest block, so a sparse query
    can leave the last block unresolved."""
    p = E.MapperParameters(seed=4)
    p.scanProcessing.downSamplingRatio = 1.0
    p.scanProcessing.cropper = E.ScanCroppingParameters("MinMaxRadius", 0.0, 30.0)
    p.mapBuilder.cropper = E.ScanCroppingParameters("MinMaxRadius", 0.0, 30.0)
    p.icp.knn = knn
    p.icp.maxDistanceKnn = 4.0
    return p


def two_patches(seed=5, n=3000, offset=(2500.0, 1500.0, 400.0)):
    """Two small room corners kilometres apart: the grid over both has to coarsen its cells many times."""
    rng = np.random.default_rng(seed)
    k = n // 3
    a = np.vstack([np.c_[rng.uniform(-2, 2, (n - 2 * k, 2)), 0.01 * rng.standard_normal(n - 2 * k)],
                   np.c_[rng.uniform(-2, 2, k), np.full(k, 2.0) + 0.01 * rng.standard_normal(k), rng.uniform(0, 1.5, k)],
                   np.c_[np.full(k, -2.0) + 0.01 * rng.standard_normal(k), rng.uniform(-2, 2, k), rng.uniform(0, 1.5, k)]])
    return np.ascontiguousarray(np.vstack([a, a[::-1] + np.asarray(offset)]))


def run_ops(out_path):
    """crop, voxel down-sample, normals, process_scan, registration, submap insertion with carving, three asynchronous mapper steps."""
    from open3d_slam_b200 import _lib as L
    import ctypes as C
    out = {}
    sc = synth.Scene(); poses = synth.loop_trajectory(8)
    raw = synth.lidar_scan(sc, poses[0], seed=70).astype(np.float64)
    p = E.MapperParameters(seed=9)
    p.scanProcessing.downSamplingRatio = 0.5
    eng = E.Engine(p)
    cl = eng.cloud(raw)
    cp = E.ScanCroppingParameters(cropperName="MinMaxRadius", croppingMinRadius=3.0, croppingMaxRadius=15.0)
    out["crop"] = E.crop(eng, cl, cp.to_c(center=(1.0, -2.0, 0.5))).download()[0]
    vx = E.voxelize(eng, cl, 0.1)
    out["voxel"] = vx.download()[0]
    L.check(L.lib().b2s_estimate_normals(eng._h, vx._c, 20, C.c_double(3.0)))
    out["normals_xyz"], out["normals"] = vx.download()
    s2m = E.ScanToMapIcp(eng)
    ps = s2m.processForScanMatchingAndMerging(cl)
    out["merge_xyz"], out["merge_nrm"] = ps.merge_.download()
    out["match_xyz"], out["match_nrm"] = ps.match_.download()
    sm = E.Submap(eng, 600_000)
    sm.insertScan(None, ps.merge_, np.eye(4))
    raw1 = eng.cloud(synth.lidar_scan(sc, poses[1], seed=71).astype(np.float64))
    ps1 = s2m.processForScanMatchingAndMerging(raw1)
    guess = np.linalg.inv(poses[0]) @ poses[1] @ synth.se3(0.002, -0.001, 0.01, (0.03, -0.02, 0.0))
    r = s2m.scanToMapRegistration(ps1.match_, sm, np.eye(4), guess)
    out["reg"] = np.r_[r.transformation_.ravel(), r.fitness_, r.inlier_rmse_, r.n_corr, r.iters]
    sm.insertScan(None, ps1.merge_, r.transformation_)
    out["carved"] = np.array([sm.carve(raw1, r.transformation_, E.SpaceCarvingParameters(), force=True)], dtype=np.float64)
    out["map_xyz"], out["map_nrm"] = sm.getMapPointCloud()
    mp = E.Mapper(eng, 600_000)
    mp.addRangeMeasurement(eng.cloud(synth.lidar_scan(sc, poses[0], seed=80)), None)
    for k in range(1, 4):
        mp.addRangeMeasurementAsync(eng.cloud(synth.lidar_scan(sc, poses[k], seed=80 + k)), np.linalg.inv(poses[k - 1]) @ poses[k], slot=k)
        rk = mp.fetchResult(k)
        out[f"step{k}"] = np.r_[rk.transformation_.ravel(), rk.fitness_, rk.inlier_rmse_, rk.n_corr, rk.iters]
    out["mapper_map"] = mp.submap.getMapPointCloud()[0]
    eng.close()
    np.savez(out_path, **out)


if __name__ == "__main__":
    if sys.argv[1] == "ops":
        run_ops(sys.argv[2])
    else:
        raise SystemExit(f"unknown mode {sys.argv[1]}")
