"""Child process of tests/test_gpu_renorm_worklist.py: the same mapping runs under the worklist K3 and, with B2S_RENORM_FULL=1,
under the pass over every map slot.  The library reads B2S_RENORM_FULL once per process, so each setting needs a process of its own.

    python tests/renorm_child.py OUT.npz     -- every run's per-scan results and final map, written to OUT.npz
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import synth  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402

EXTRA = 20   # scans past one lap of the closed loop: the map is re-visited and every kind of normal update happens


def mapper_run(lp, graph, out, tag):
    """The benchmark's chain (ratio 0.3) with carving every 10 insertions (each carve rehashes the map) over a lap and a bit."""
    p = E.MapperParameters(seed=3)
    p.scanProcessing.downSamplingRatio = 0.3
    eng = E.Engine(p)
    mp = E.Mapper(eng, 760_000)
    mp.submap.setMapperOptions(carving=E.SpaceCarvingParameters())
    clouds = [eng.cloud(lp.scan(k, seed=k)) for k in range(lp.L)]
    mp.addRangeMeasurement(clouds[0], None)
    mp.submap.setPose(np.eye(4))
    eng.synchronize()
    staging = mp.enableGraph(65536) if graph else None
    res = []
    for k in range(1, lp.L + EXTRA):
        if staging is not None:
            mp.stageCopy(clouds[k % lp.L])
            slot = mp.addRangeMeasurementAsync(staging, lp.delta(k))
        else:
            slot = mp.addRangeMeasurementAsync(clouds[k % lp.L], lp.delta(k), slot=k % 256)
        r = mp.fetchResult(slot)
        res.append(np.r_[r.transformation_.ravel(), r.fitness_, r.n_corr, r.iters])
    out[f"{tag}_res"] = np.array(res)
    out[f"{tag}_xyz"], out[f"{tag}_nrm"] = mp.submap.getMapPointCloud()
    out[f"{tag}_counters"] = np.array(list(mp.submap.mapperCounters().values()), dtype=np.int64)
    eng.close()


def fixed_pose_run(lp, out):
    """Scans of the closed loop (every 4th return, host-made normals that are not yet fixed points of the device's normalized())
    fused at their ground-truth poses over a lap and a bit, with a carve (a rehash of the map) every 10 insertions.  No device
    estimate enters and the cropper holds every point, so no merge depends on the order of the map's slots: the two settings
    must give the same map bit for bit."""
    p = E.MapperParameters(seed=3)
    p.mapBuilder.cropper = E.ScanCroppingParameters("MaxRadius", 0.0, 1000.0)
    eng = E.Engine(p)
    sm = E.Submap(eng, 760_000)
    rng = np.random.default_rng(11)
    for k in range(lp.L + EXTRA):
        raw = lp.scan(k, seed=k)
        xyz = np.ascontiguousarray(raw[::4].astype(np.float64))
        nrm = rng.normal(size=xyz.shape)
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        T = lp.map_frame_pose(k)
        if k % 10 == 9:
            sm.carve(eng.cloud(raw), T, E.SpaceCarvingParameters(), force=True)
        sm.insertScan(None, eng.cloud(xyz, nrm), T)
    out["fixed_xyz"], out["fixed_nrm"] = sm.getMapPointCloud()
    eng.close()


CROP_R = 6.0   # map builder cropper of cropped_run (MaxRadius)


def cropped_run(out):
    """A loaded map (one point per voxel, normals of arbitrary length, a tenth of them NaN) crossed by a sensor whose 6 m cropper
    covers a strip of it at a time: most map points start outside the cropper with a normal that is not a fixed point, and enter
    it later.  Small scans (every point well inside the cropper, host-made normals) are fused at fixed poses; no voxel ever holds
    three map points, so no merge depends on the order of the map's slots and the map is reproducible bit for bit."""
    p = E.MapperParameters(seed=3)
    p.mapBuilder.cropper = E.ScanCroppingParameters("MaxRadius", 0.0, CROP_R)
    eng = E.Engine(p)
    sm = E.Submap(eng, 200_000)
    rng = np.random.default_rng(17)
    gx, gy, gz = np.meshgrid(np.arange(-20.0, 20.0, 0.3), np.arange(-4.0, 4.0, 0.3), [0.05, 1.25], indexing="ij")
    mxyz = np.c_[gx.ravel(), gy.ravel(), gz.ravel()] + rng.uniform(-0.02, 0.02, (gx.size, 3))
    mnrm = rng.normal(size=mxyz.shape) * rng.uniform(0.5, 2.0, (len(mxyz), 1))
    mnrm[rng.random(len(mnrm)) < 0.1] = np.nan
    sm.setMapPointCloud(eng.cloud(mxyz, mnrm))
    poses, world = [], []
    for k in range(40):
        T = synth.se3(0.0, 0.0, 0.003 + 0.01 * k, (-18.0 + 0.9 * k, 0.0, 0.5))
        d = rng.normal(size=(100, 3))
        xyz = d / np.linalg.norm(d, axis=1, keepdims=True) * (3.0 * rng.random((100, 1)) ** (1 / 3))
        nrm = rng.normal(size=xyz.shape) * rng.uniform(0.5, 2.0, (len(xyz), 1))
        sm.insertScan(None, eng.cloud(xyz, nrm), T)
        poses.append(T); world.append(xyz @ T[:3, :3].T + T[:3, 3])
    out["crop_map0_xyz"], out["crop_map0_nrm"] = mxyz, mnrm
    out["crop_poses"] = np.array(poses); out["crop_r"] = np.array(CROP_R)
    out["crop_scan_world"] = np.concatenate(world)
    out["crop_xyz"], out["crop_nrm"] = sm.getMapPointCloud()
    eng.close()


def point_to_point_run(out):
    """A point-to-point submap: a map loaded without normals (NaN), scans without normals fused into it, a scan with normals of
    several lengths, a moved map (Submap::transform) and scans from a sensor that leaves part of the map outside the cropper."""
    p = E.MapperParameters(seed=5)
    p.scanToMapRegType = "PointToPointIcp"
    p.mapBuilder.cropper = E.ScanCroppingParameters("MaxRadius", 0.0, 12.0)
    eng = E.Engine(p)
    sc = synth.Scene(); poses = synth.loop_trajectory(40)
    sm = E.Submap(eng, 600_000)
    base = np.ascontiguousarray(synth.lidar_scan(sc, poses[0], seed=300).astype(np.float64)[::4])
    sm.setMapPointCloud(eng.cloud(base))
    rng = np.random.default_rng(7)
    for k in range(1, 30):
        T = np.linalg.inv(poses[0]) @ poses[k % 40]
        xyz = np.ascontiguousarray(synth.lidar_scan(sc, poses[k % 40], seed=300 + k).astype(np.float64)[::8])
        if k % 7 == 3:   # normals of random direction and length: many are not a fixed point of normalized() yet
            nrm = rng.normal(size=xyz.shape) * rng.uniform(0.1, 10.0, (len(xyz), 1))
            sm.insertScan(None, eng.cloud(xyz, nrm), T)
        else:
            sm.insertScan(None, eng.cloud(xyz), T)
        if k == 15:
            sm.transform(synth.se3(0.01, -0.02, 0.03, (0.25, -0.5, 0.125)))
    out["p2p_xyz"], out["p2p_nrm"] = sm.getMapPointCloud()
    eng.close()


def main(out_path):
    out = {}
    lp = W.ClosedLoop()
    mapper_run(lp, False, out, "eager")
    mapper_run(lp, True, out, "graph")
    fixed_pose_run(lp, out)
    cropped_run(out)
    point_to_point_run(out)
    np.savez(out_path, **out)


if __name__ == "__main__":
    main(sys.argv[1])
