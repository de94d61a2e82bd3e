"""CPU tests of the FPFH restatements (tests/oracle_features.c and its numpy twin): the two agree on random clouds and on a LiDAR
scan at the 0.5 m feature voxel (identical neighbour lists, rows within 1e-12), and the C one gives the known
answers of small constructed clouds (pair features and bins, an isolated point, coincident points, a planar patch)."""
import numpy as np
import pytest

import oracle_features as OF
from oracle import oracle as O
from open3d_slam_b200 import synth


def unit(v):
    v = np.asarray(v, dtype=np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def random_cloud(n, seed, extent=4.0):
    rng = np.random.default_rng(seed)
    return rng.uniform(-extent, extent, (n, 3)), unit(rng.normal(size=(n, 3)))


def feature_cloud(seed=0):
    """a scan of the synthetic scene, voxelised at featureVoxelSize 0.5 with normals (r 2.0, k 20): the size and density of the
    sparse cloud Submap::computeFeatures hands to FPFH"""
    pose = synth.loop_trajectory(40)[5]
    raw = synth.lidar_scan(synth.Scene(), pose, seed=seed).astype(np.float64)
    xyz, _ = O.voxel_down_sample(raw, 0.5)
    return xyz, O.estimate_normals(xyz, 20, 2.0)


def assert_same(xyz, nrm, radius, knn, max_flipped=0):
    got, det = OF.fpfh(xyz, nrm, radius, knn, details=True)
    ref, nbs = OF.np_fpfh(xyz, nrm, radius, knn)
    for i, (idx, d2) in enumerate(nbs):
        k = det["nb_cnt"][i]
        assert k == len(idx) and np.array_equal(det["nb_idx"][i, :k], idx) and np.array_equal(det["nb_d2"][i, :k], d2), i
    # every row agrees to 1e-12 (the sums are taken in another order: counts * hist_incr, numpy reductions) except where numpy's
    # arccos / arctan2, which are not glibc's, put a pair on the other side of a bin boundary or of an exact acos tie; such a
    # row must be explained by a margin below 1e-9, and only the caller's expected number of them is allowed
    diff, unexplained = OF.differing_rows(got, ref, det, tol=1e-12)
    assert len(unexplained) == 0, unexplained[:10]
    assert len(diff) <= max_flipped, len(diff)
    return got, det


@pytest.mark.parametrize("n,radius,knn,seed", [(1500, 1.0, 12, 0), (3000, 1.5, 100, 1), (800, 3.0, 128, 2)])
def test_c_and_numpy_agree_on_random_clouds(n, radius, knn, seed):
    xyz, nrm = random_cloud(n, seed)
    got, det = assert_same(xyz, nrm, radius, knn)
    assert (det["nb_cnt"] == knn).any()            # the knn cap binds somewhere ...
    assert (det["nb_cnt"] < knn).any()             # ... and the radius elsewhere
    has = det["nb_cnt"] > 1
    assert np.abs(got[has].reshape(-1, 3, 11).sum(axis=2) - 200.0).max() < 1e-9
    assert np.all(got[~has] == 0.0)


def test_c_and_numpy_agree_on_a_feature_cloud():
    xyz, nrm = feature_cloud()
    assert len(xyz) > 1000
    # the scan's flat surfaces give pairs with a zero margin (an exact acos tie or a feature on a boundary): 17 of 6 976 rows flip
    got, det = assert_same(xyz, nrm, 2.5, 100, max_flipped=len(xyz) // 200)
    has = det["nb_cnt"] > 1
    # every 11-bin block of a point with a neighbour at d2 > 0 sums to 100 (normalised neighbour sum) + 100 (own SPFH)
    blocks = got[has].reshape(-1, 3, 11).sum(axis=2)
    assert np.abs(blocks - 200.0).max() < 1e-9


def test_two_points_pair_features_and_bins():
    s = 1 / np.sqrt(2.0)
    xyz = np.array([[0.0, 0, 0], [1.0, 0, 0]])
    # no swap: f = (atan2(0, 0) = 0, v.n2 = -1, angle1 = 0) -> bins 5, 11 + 0, 22 + 5
    _, det = OF.fpfh(xyz, np.array([[0.0, 0, 1], [0.0, 1, 0]]), 2.0, 10, details=True)
    assert np.flatnonzero(det["spfh"][0]).tolist() == [5, 11, 27] and np.all(det["spfh"][0][[5, 11, 27]] == 100.0)
    # swap (acos|angle1| = pi/2 > acos|angle2| = pi/4): f = (pi/4, 0, -1/sqrt2) -> bins 6 (6.875), 16 (5.5), 22 + 1 (1.61)
    _, det = OF.fpfh(xyz, np.array([[0.0, 0, 1], [s, 0, s]]), 2.0, 10, details=True)
    assert np.flatnonzero(det["spfh"][0]).tolist() == [6, 16, 23]
    # zero cross product (n1 along dp): all three features 0 -> bins 5, 16, 27
    _, det = OF.fpfh(xyz, np.array([[1.0, 0, 0], [0.0, 0, 1]]), 2.0, 10, details=True)
    assert np.flatnonzero(det["spfh"][0]).tolist() == [5, 16, 27]
    # FPFH of a pair: the other point's SPFH (d2 = 1, block sums 100 -> scale 1) plus its own
    feat = OF.fpfh(xyz, np.array([[0.0, 0, 1], [0.0, 1, 0]]), 2.0, 10)
    assert np.flatnonzero(feat[0]).tolist() == [5, 11, 27] and np.all(feat[0][[5, 11, 27]] == 200.0)
    ref, _ = OF.np_fpfh(xyz, np.array([[0.0, 0, 1], [s, 0, s]]), 2.0, 10)
    assert np.abs(ref - OF.fpfh(xyz, np.array([[0.0, 0, 1], [s, 0, s]]), 2.0, 10)).max() < 1e-12


def test_isolated_point_gets_a_zero_row():
    xyz = np.array([[0.0, 0, 0], [0.3, 0, 0], [0.0, 0.3, 0], [50.0, 0, 0]])
    nrm = unit([[0, 0, 1], [0, 0.1, 1], [0.1, 0, 1], [0, 0, 1]])
    feat, det = OF.fpfh(xyz, nrm, 1.0, 10, details=True)
    assert det["nb_cnt"][3] == 1 and np.all(feat[3] == 0.0)
    assert np.all(feat[:3].sum(axis=1) > 0)


def test_coincident_points_skip_zero_distances():
    # points 0 and 1 coincide: the list of 1 is [0 (d2 0), 1 (d2 0), 2]; SPFH skips entry 0 (the quirk: here not the point itself)
    # and pairs 1 with itself (zero features -> bins 5, 16, 27); FPFH skips both d2 == 0 entries and stays finite
    xyz = np.array([[0.0, 0, 0], [0.0, 0, 0], [0.5, 0, 0]])
    nrm = np.array([[0.0, 0, 1], [0.0, 0, 1], [0.0, 1, 0]])
    feat, det = OF.fpfh(xyz, nrm, 1.0, 10, details=True)
    assert det["nb_idx"][1, :3].tolist() == [0, 1, 2] and det["nb_d2"][1, 0] == 0.0
    assert np.all(det["spfh"][1][[5, 16, 27]] >= 50.0)
    assert np.isfinite(feat).all()
    assert np.abs(feat[:2].reshape(2, 3, 11).sum(axis=2) - 200.0).max() < 1e-12
    ref, _ = OF.np_fpfh(xyz, nrm, 1.0, 10)
    assert np.abs(ref - feat).max() < 1e-12


def test_planar_patch_puts_the_mass_in_the_flat_bins():
    g = np.arange(-5, 6) * 0.2
    X, Y = np.meshgrid(g, g)
    xyz = np.c_[X.ravel(), Y.ravel(), np.zeros(X.size)]
    nrm = np.tile([0.0, 0.0, 1.0], (len(xyz), 1))
    feat = OF.fpfh(xyz, nrm, 0.5, 30)
    # coplanar pairs with parallel normals: f = (0, 0, 0) -> every SPFH and FPFH row is 100 / 200 in bins 5, 16, 27
    assert np.all(feat[:, [5, 16, 27]] == pytest.approx(200.0, abs=1e-12))
    assert np.all(np.delete(feat, [5, 16, 27], axis=1) == 0.0)


def test_empty_cloud():
    assert OF.fpfh(np.zeros((0, 3)), np.zeros((0, 3)), 1.0, 10).shape == (0, 33)
