"""-m gpu: the static map patch (K-patch, grid_index.cu) against the full path.  The same map sits in a submap with merge off (tile path)
and in one with merge on (full path: every map slot through the cropper inside the index build); every registration of a lap scan,
at many sensor poses and with every bounded cropper kind, must index the same points: the same grid header and, per cell, the same set
of original indices (map slots).  The ICP outcome must then be the same: iterations, correspondences and fitness equal, T within 1e-12.
After b2s_submap_set_cloud, b2s_submap_transform or merge switched on and off around an insertion, the tile path follows the new map."""
import ctypes as C

import numpy as np
import pytest

from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E

from test_localization_host import prior  # noqa: F401  (the module's fixture: closed lap, oracle-built map)

pytestmark = pytest.mark.gpu


def nn_index(eng):
    """header, {cell: sorted original indices} of the NN index the last registration built"""
    oc = (C.c_double * 4)(); dn = (C.c_int32 * 5)()
    L.check(L.lib().b2s_debug_nn_index(eng._h, oc, dn, None, C.c_size_t(0), None, C.c_size_t(0)))
    ncell, n = dn[3], dn[4]
    starts = np.zeros(ncell + 1, dtype=np.int32); orig = np.zeros(max(n, 1), dtype=np.int32)
    L.check(L.lib().b2s_debug_nn_index(eng._h, oc, dn, starts.ctypes.data_as(C.POINTER(C.c_int32)), C.c_size_t(ncell + 1),
                                       orig.ctypes.data_as(C.POINTER(C.c_int32)), C.c_size_t(len(orig))))
    cells = np.repeat(np.arange(ncell), np.diff(starts))
    o = np.lexsort((orig[:n], cells))
    return (tuple(oc), tuple(dn)), cells[o], orig[:n][o]


def params(kind, rmax=20.0, rmin=2.0, zmin=-3.0, zmax=8.0):
    p = E.MapperParameters(seed=3)
    c = p.scanProcessing.cropper
    c.cropperName, c.croppingMaxRadius, c.croppingMinRadius, c.croppingMinZ, c.croppingMaxZ = kind, rmax, rmin, zmin, zmax
    return p


class Pair:
    """one engine, the same map in a merge-off (tile) and a merge-on (full) submap"""

    def __init__(self, p, xyz, offset=np.zeros(3)):
        self.eng = E.Engine(p)
        self.reg = E.scanToMapRegistrationFactory(self.eng, p)
        self.offset = np.asarray(offset, dtype=np.float64)
        self.tile, self.full = E.Submap(self.eng, 400_000), E.Submap(self.eng, 400_000)
        self.tile.setMergeScans(False)
        self.load(xyz)

    def load(self, xyz):
        c = self.eng.cloud(np.ascontiguousarray(xyz + self.offset))
        self.reg.prepareInitialMap(c)
        for sm in (self.tile, self.full):
            sm.setMapPointCloud(c)

    def register(self, sm, scan, pose, guess):
        r = self.reg.scanToMapRegistration(scan, sm, pose, guess)
        return r, nn_index(self.eng)

    def compare(self, scan, pose, guess):
        return same(self.register(self.tile, scan, pose, guess), self.register(self.full, scan, pose, guess))


def same(a, b):
    """the same indexed points (header, per-cell original indices) and the same ICP outcome; T within 1e-12 relative to the largest
    entry (the reductions' order varies between runs: 2 ulps of a 5 km translation are 1.8e-12)"""
    (rt, (ht, ct, ot)), (rf, (hf, cf, of)) = a, b
    assert ht == hf                                                           # origin, cell, dims, ncell, n: identical
    assert np.array_equal(ct, cf) and np.array_equal(ot, of)                  # per cell, the same original indices
    assert (rt.iters, rt.n_corr, rt.fitness_) == (rf.iters, rf.n_corr, rf.fitness_)
    assert np.abs(rt.transformation_ - rf.transformation_).max() <= 1e-12 * max(1.0, np.abs(rf.transformation_).max())
    return rt, hf[1][4]


def _scans(pair, lp, ks):
    out = []
    for k in ks:
        ps = pair.reg.processForScanMatchingAndMerging(pair.eng.cloud(lp.scan(k + lp.L, seed=40 + k)))
        out.append((k, ps.match_))
    return out


@pytest.mark.parametrize("kind", ["MaxRadius", "MinMaxRadius", "Cylinder"])
@pytest.mark.parametrize("offset", [(0.0, 0.0, 0.0), (5000.0, -3000.0, 0.0)])   # the cylinder's z range is absolute
def test_tile_path_indexes_what_the_full_path_indexes(prior, kind, offset):
    lp, xyz = prior
    pair = Pair(params(kind), xyz, offset)
    rng = np.random.default_rng(7)
    sizes = []
    for k, scan in _scans(pair, lp, range(0, 10, 2)):
        T = lp.map_frame_pose(k).copy()
        T[:3, 3] += pair.offset
        # the true pose, then poses on tile faces / corners (the table's 2 m grid is anchored at the map's minimum) and far off the map
        poses = [T]
        for _ in range(3):
            P = T.copy(); P[:3, 3] += rng.uniform(-3, 3, 3); poses.append(P)
        for P in poses:
            _r, n = pair.compare(scan, P, T)
            sizes.append(n)
        Pfar = T.copy(); Pfar[:3, 3] += (60.0, 0.0, 0.0)                       # the box beyond the map border: few or no points
        try:
            pair.compare(scan, Pfar, T)
        except L.B2SError as e:                                              # both paths: "map patch size is zero"
            assert e.code == L.E_EMPTY
    assert min(sizes) > 1000


def test_tile_faces_and_corners(prior):
    """sensor positions exactly on tile faces and corners of the table (origin = the map's bbox minimum, edge 2 m)"""
    lp, xyz = prior
    pair = Pair(params("MaxRadius"), xyz)
    (k, scan), = _scans(pair, lp, [4])
    T = lp.map_frame_pose(k)
    mn = xyz.min(axis=0)
    base = mn + 2.0 * np.floor((T[:3, 3] - mn) / 2.0)
    for d in ([0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 1], [2, -1, 0]):
        P = T.copy(); P[:3, 3] = base + 2.0 * np.asarray(d, dtype=np.float64)
        pair.compare(scan, P, T)


def test_table_follows_set_cloud_transform_and_reenabled_merge(prior):
    lp, xyz = prior
    pair = Pair(params("MaxRadius"), xyz)
    (k, scan), = _scans(pair, lp, [3])
    T = lp.map_frame_pose(k)
    pair.compare(scan, T, T)                                                  # builds the table
    half = xyz[xyz[:, 0] < np.median(xyz[:, 0])]
    pair.load(half)                                                           # set_cloud: another map
    _r, n_half = pair.compare(scan, T, T)
    M = np.eye(4); M[:3, 3] = (0.3, -0.2, 0.05)
    for sm in (pair.tile, pair.full):
        sm.transform(M)                                                       # transform: the map moves
    pair.compare(scan, T, T)
    # merge on, one insertion, merge off again: the same submap through the full path (merge on) and the rebuilt table (merge off).
    # Fusion numbers the new slots in atomic order, so only the same submap has the same original indices on both paths.
    pair.tile.setMergeScans(True)
    ps = pair.reg.processForScanMatchingAndMerging(pair.eng.cloud(lp.scan(k, seed=9)))
    pair.tile.insertScan(None, ps.merge_, T)
    full = pair.register(pair.tile, scan, T, T)
    pair.tile.setMergeScans(False)
    _r, n_after = same(pair.register(pair.tile, scan, T, T), full)
    assert n_after != n_half
