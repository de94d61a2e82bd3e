"""-m gpu: b2s_compute_fpfh (row K-fpfh) against the C restatement tests/oracle_features.c.  Rows must be BIT-IDENTICAL; a row may
differ only where the device's atan2 / acos and the host libm can disagree -- the row's point or a neighbour has an SPFH pair within
1e-9 of a bin boundary or of the acos swap decision -- and every such row is reported.  Covered: random clouds up to knn 128, a
LiDAR scan at the 0.5 m feature voxel, a dense cloud with far more than 128 candidates in the radius, lattice clouds full of exact
distance ties, coincident points, empty and single-point clouds, the error codes, a feature passed with another handle and the
feature upload / download round trip."""
import ctypes as C

import numpy as np
import pytest

import oracle_features as OF
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from test_fpfh_oracle import feature_cloud, random_cloud, unit

pytestmark = pytest.mark.gpu


def check(eng, xyz, nrm, radius, knn):
    f = E.computeFPFHFeature(eng, eng.cloud(xyz, nrm), radius, knn)
    assert f.Num() == len(xyz) and f.Dimension() == 33
    got = f.data_.T
    ref, det = OF.fpfh(xyz, nrm, radius, knn, details=True)
    diff, unexplained = OF.differing_rows(got, ref, det)
    if len(diff):
        print(f"K-fpfh: {len(diff)} of {len(xyz)} rows differ, all next to a bin boundary / acos tie "
              f"(smallest margin {det['margin'].min():.3g})")
    assert len(unexplained) == 0, (unexplained[:10], np.abs(got - ref).max())
    assert len(diff) <= max(1, len(xyz) // 100)
    return got, det


@pytest.mark.parametrize("n,radius,knn,seed", [(1500, 1.0, 12, 0), (3000, 1.5, 100, 1), (800, 3.0, 128, 2), (2000, 1.2, 33, 3)])
def test_random_clouds(engine_factory, n, radius, knn, seed):
    eng = engine_factory()
    xyz, nrm = random_cloud(n, seed)
    _, det = check(eng, xyz, nrm, radius, knn)
    assert (det["nb_cnt"] == knn).any() and (det["nb_cnt"] < knn).any()


def test_feature_cloud_lua_parameters(engine_factory):
    eng = engine_factory()
    xyz, nrm = feature_cloud()
    check(eng, xyz, nrm, 2.5, 100)   # featureRadius 2.5, featureKnn 100 (parameter_structure_definitions.lua)


def test_dense_cloud_far_more_candidates_than_knn(engine_factory):
    eng = engine_factory()
    xyz, nrm = random_cloud(20000, 4, extent=1.0)
    _, det = check(eng, xyz, nrm, 0.5, 128)
    assert (det["nb_cnt"] == 128).mean() > 0.9    # ~1300 points inside the radius of most queries: the search must select


def test_lattice_distance_ties(engine_factory):
    eng = engine_factory()
    g = np.arange(8) * 0.25
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    xyz = np.c_[X.ravel(), Y.ravel(), Z.ravel()]
    rng = np.random.default_rng(5)
    xyz = xyz[rng.permutation(len(xyz))]            # tie order is by index, not by position
    nrm = unit(rng.normal(size=xyz.shape))
    for radius, knn in ((0.6, 20), (0.26, 5), (0.55, 128)):   # the k-th neighbour sits inside a shell of equal distances
        check(eng, xyz, nrm, radius, knn)


def test_coincident_points(engine_factory):
    eng = engine_factory()
    xyz, nrm = random_cloud(400, 6, extent=1.0)
    xyz = np.vstack([xyz, xyz[:50], xyz[10:20]])    # duplicates with higher indices, some three-fold
    nrm = np.vstack([nrm, unit(nrm[:50] + 0.3), nrm[10:20]])
    got, _ = check(eng, xyz, nrm, 0.5, 30)
    assert np.isfinite(got).all()


def test_empty_and_single_point(engine_factory):
    eng = engine_factory()
    f = E.computeFPFHFeature(eng, eng.cloud(np.zeros((0, 3)), np.zeros((0, 3))), 2.5, 100)
    assert f.Num() == 0 and f.data_.shape == (33, 0)
    f = E.computeFPFHFeature(eng, eng.cloud(np.zeros((0, 3))), 2.5, 100)   # empty without normals: zero features, no error
    assert f.Num() == 0
    f = E.computeFPFHFeature(eng, eng.cloud(np.array([[1.0, 2.0, 3.0]]), np.array([[0.0, 0.0, 1.0]])), 2.5, 100)
    assert f.Num() == 1 and np.all(f.data_ == 0.0)


def test_errors(engine_factory):
    eng = engine_factory()
    xyz, nrm = random_cloud(100, 7)
    c = eng.cloud(xyz, nrm)
    for radius, knn, code in ((2.5, 0, L.E_INVALID), (0.0, 10, L.E_INVALID), (-1.0, 10, L.E_INVALID), (2.5, 129, L.E_UNSUPPORTED)):
        with pytest.raises(L.B2SError) as e:
            E.computeFPFHFeature(eng, c, radius, knn)
        assert e.value.code == code
    with pytest.raises(L.B2SError) as e:
        E.computeFPFHFeature(eng, eng.cloud(xyz), 2.5, 10)
    assert e.value.code == L.E_NO_NORMALS


def test_feature_of_another_handle_is_rejected(engine_factory):
    a, b = engine_factory(), engine_factory()
    xyz, nrm = random_cloud(100, 9)
    f = E.Feature(a, np.zeros((33, 4)))
    cb = b.cloud(xyz, nrm)
    for call in (lambda: L.lib().b2s_compute_fpfh(b._h, cb._c, C.c_double(2.5), C.c_int32(10), f._f),
                 lambda: L.lib().b2s_feature_size(b._h, f._f, C.byref(C.c_size_t()))):
        assert call() == L.E_INVALID
    assert f.Num() == 4


def test_feature_upload_download_round_trip(engine_factory):
    eng = engine_factory()
    data = np.random.default_rng(8).uniform(0, 200, (33, 257))
    f = E.Feature(eng, data)
    assert f.Num() == 257 and np.array_equal(f.data_, data)
    f.upload(data[:, :3])
    assert f.Num() == 3 and np.array_equal(f.data_, data[:, :3])
