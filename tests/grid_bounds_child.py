"""Child process of tests/test_gpu_grid_bounds.py: the same runs with the scan-to-map index's grid box taken from the submap's box and,
with B2S_GRID_BBOX_PASS=1, measured by a pass over the map.  The library reads the switch once per process, so each setting needs a
process of its own.

    python tests/grid_bounds_child.py OUT.npz     -- every run's results, written to OUT.npz
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from open3d_slam_b200 import _lib as L  # noqa: E402
from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402

EXTRA = 20   # scans past one lap of the closed loop: the map is re-visited


def nn_index(eng):
    """(origin + cell, dims + ncell + n), cell starts and original indices of the index the last registration built"""
    oc = (C.c_double * 4)(); dn = (C.c_int32 * 5)()
    L.check(L.lib().b2s_debug_nn_index(eng._h, oc, dn, None, C.c_size_t(0), None, C.c_size_t(0)))
    ncell, n = dn[3], dn[4]
    starts = np.zeros(ncell + 1, dtype=np.int32); orig = np.zeros(max(n, 1), dtype=np.int32)
    L.check(L.lib().b2s_debug_nn_index(eng._h, oc, dn, starts.ctypes.data_as(C.POINTER(C.c_int32)), C.c_size_t(ncell + 1),
                                       orig.ctypes.data_as(C.POINTER(C.c_int32)), C.c_size_t(len(orig))))
    return np.array(oc[:]), np.array(dn[:]), starts, orig[:n]


def mapper_run(lp, graph, out, tag):
    """The benchmark's chain (ratio 0.3) with carving every 10 insertions over a lap and a bit, eager or replayed from a graph."""
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
    oc, dn, _s, _o = nn_index(eng)
    out[f"{tag}_hdr"] = np.r_[oc, dn]   # the last scan's index: origin, cell, dims, ncell, n
    eng.close()


def lap_map(lp):
    """A map of known slot order: the first return per map voxel of the first 24 scans at their true poses, unit normals of a fixed seed"""
    pts = []
    for k in range(24):
        T = lp.map_frame_pose(k)
        s = lp.scan(k, seed=k)[::4].astype(np.float64)
        pts.append(s @ T[:3, :3].T + T[:3, 3])
    xyz = np.concatenate(pts)
    _u, first = np.unique(np.floor(xyz * 10.0).astype(np.int64), axis=0, return_index=True)   # one point per 0.1 m map voxel
    xyz = np.ascontiguousarray(xyz[np.sort(first)])
    nrm = np.random.default_rng(5).normal(size=xyz.shape)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return xyz, nrm


CROPPERS = [("MinMaxRadius", 30.0, 2.0, -50.0, 50.0), ("MaxRadius", 20.0, 0.0, -50.0, 50.0), ("Cylinder", 20.0, 0.0, -2.0, 1.0)]
# sensor offsets from the true pose: on it, inside the map, at the rim (the cropper's box cuts the map's), beyond the map
OFFSETS = [(0.0, 0.0, 0.0), (2.5, -1.5, 0.5), (0.0, 24.0, 0.0), (-31.0, 0.0, 1.0), (60.0, 0.0, 0.0)]


def patch_run(lp, out):
    """Registrations of lap scans against one loaded map, with every bounded cropper kind and sensor positions from the middle of the
    map to beyond its border: per case the index's header, cell starts and original indices, and the ICP outcome (code -1: the patch
    was empty)."""
    xyz, nrm = lap_map(lp)
    out["patch_map"] = xyz
    for ci, (kind, rmax, rmin, zmin, zmax) in enumerate(CROPPERS):
        p = E.MapperParameters(seed=3)
        c = p.scanProcessing.cropper
        c.cropperName, c.croppingMaxRadius, c.croppingMinRadius, c.croppingMinZ, c.croppingMaxZ = kind, rmax, rmin, zmin, zmax
        eng = E.Engine(p)
        reg = E.scanToMapRegistrationFactory(eng, p)
        sm = E.Submap(eng, 400_000)
        sm.setMapPointCloud(eng.cloud(xyz, nrm))
        for k in (1, 6, 11):
            scan = reg.processForScanMatchingAndMerging(eng.cloud(lp.scan(k + lp.L, seed=40 + k))).match_
            T = lp.map_frame_pose(k)
            for oi, off in enumerate(OFFSETS):
                P = T.copy(); P[:3, 3] += off
                tag = f"patch_{ci}_{k}_{oi}"
                try:
                    r = reg.scanToMapRegistration(scan, sm, P, T)
                except L.B2SError as e:
                    assert e.code == L.E_EMPTY, e
                    out[f"{tag}_res"] = np.array([-1.0])
                    continue
                out[f"{tag}_res"] = np.r_[r.transformation_.ravel(), r.fitness_, r.n_corr, r.iters]
                oc, dn, starts, orig = nn_index(eng)
                out[f"{tag}_hdr"] = np.r_[oc, dn]
                out[f"{tag}_starts"], out[f"{tag}_orig"] = starts, orig
                out[f"{tag}_pose"] = P
        eng.close()


def main(out_path):
    out = {}
    lp = W.ClosedLoop()
    mapper_run(lp, False, out, "eager")
    mapper_run(lp, True, out, "graph")
    patch_run(lp, out)
    np.savez(out_path, **out)


if __name__ == "__main__":
    main(sys.argv[1])
