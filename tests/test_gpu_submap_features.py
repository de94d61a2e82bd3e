"""-m gpu: b2s_submap_compute_features (row K-features), the feature-cloud front end of Submap::computeFeatures on the device,
against the C restatement in tests/oracle_submap_features.c.  Real submaps built by the device mapper on the closed lap: sparse cloud
bit-identical to the oracle's voxel down-sample (keyed), normals within 1e-9 (widened by the conditioning of the eigenproblem
at the few ill-conditioned points: the covariance is summed in another order), FPFH
rows bit-identical to the restatement on the device's own sparse cloud under the margin rule of the K-fpfh tests.  Constructed
maps on exact ties of the camera orientation (a plane through the origin, isolated points at z = 0) with priors of both signs:
normals bit-identical.  Edge cases: empty submap, a point-to-point map without normals, error codes, outputs of another handle,
repeated calls on the same outputs."""
import copy
import ctypes as C

import numpy as np
import pytest

import oracle_features as OF
import oracle_submap_features as OSF
from oracle import oracle as O
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W
from test_features_front_end import isolated_points, lidar_map, signed_priors, tie_plane

pytestmark = pytest.mark.gpu

P = E.PlaceRecognitionParameters()


def lex(x):
    return np.lexsort((x[:, 2], x[:, 1], x[:, 0]))


def check_fpfh(xyz, nrm, got):
    ref, det = OF.fpfh(xyz, nrm, P.featureRadius, P.featureKnn, details=True)
    diff, unexplained = OF.differing_rows(got, ref, det)
    if len(diff):
        print(f"K-features: {len(diff)} of {len(xyz)} FPFH rows differ, all next to a bin boundary / acos tie")
    assert len(unexplained) == 0, (unexplained[:10], np.abs(got - ref).max())
    # the 0.5 m cloud of a map is full of flat surfaces whose pairs sit exactly on a bin boundary: 1-3 % of the rows flip there
    assert len(diff) <= max(1, len(xyz) // 20)


def check_normals(xyz, got, ref):
    """device normals against the restatement's, both in the order of xyz: 1e-9, widened only where the eigenproblem is
    ill-conditioned -- the covariance is summed in another order (warp butterfly), and a small gap between the two smallest
    eigenvalues amplifies that last-bit difference by max eigenvalue / gap.  Reordering the cumulant sums of these 0.5 m clouds on
    the CPU moves a normal by at most 1.7e-12 / gap (up to 5e-8 in absolute terms); the bar is 1e-11 / gap.  The sign must agree
    everywhere."""
    _, cov = O.estimate_normals(xyz, P.normalKnn, P.normalEstimationRadius, return_cov=True)
    w = np.linalg.eigvalsh(cov)
    gap = (w[:, 1] - w[:, 0]) / np.maximum(np.abs(w[:, 2]), 1e-300)
    tol = np.maximum(1e-9, 1e-11 / np.maximum(gap, 1e-300))
    err = np.abs(got - ref).max(axis=1)
    assert (err <= tol).all(), (err.max(), tol[np.argmax(err - tol)])
    assert (err > 1e-9).mean() < 1e-3 and ((got * ref).sum(axis=1) > 0.5).all()


def check_submap(eng, sm, map_xyz, map_nrm, exact_normals):
    """sm.computeFeatures has run; map_xyz / map_nrm: the map as the restatement sees it (map_nrm None: no normals)"""
    ref = OSF.submap_features(map_xyz, map_nrm, P)
    dx, dn = sm.getSparseMapPointCloud().download()
    got = sm.getFeatures().data_.T
    assert len(dx) == len(ref["xyz"]) == len(got)
    a, b = lex(dx), lex(ref["xyz"])
    assert np.array_equal(dx[a], ref["xyz"][b])                      # same voxels, bit-identical means
    if exact_normals:
        assert np.array_equal(dn[a], ref["nrm"][b])
    else:
        check_normals(ref["xyz"][b], dn[a], ref["nrm"][b])
    check_fpfh(dx, dn, got)
    return ref


def test_real_submaps_through_the_collection(engine_factory):
    """120 scans of the closed lap through the device mapper with 5 m submaps: several finished submaps, then
    SubmapCollection.computeFeatures and every finished submap against the restatement run on its downloaded map"""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=False, graph=True)
    m = S.SegmentMapper(dev, S.SubmapParameters(radius=5.0))
    for k in range(120):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    sc = m.submaps
    assert len(sc.finishedSubmapsIdxs) >= 3 and all(r.feature is None for r in sc.submaps)   # the mapper never computes them
    done = sc.computeFeatures(P)
    assert done == sc.finishedSubmapsIdxs
    for idx in set(done):
        rec = sc.submaps[idx]
        sm = rec.handle
        assert rec.sparse is sm.getSparseMapPointCloud() and rec.feature is sm.getFeatures()
        x, n = dev.map_cloud(sm)
        ref = check_submap(dev.eng, sm, x, n, exact_normals=False)
        assert len(ref["xyz"]) > 500
        # the voxel-mean normals (the priors, overwritten by the estimate on the device) through the plain down-sample
        v = E.voxelize(dev.eng, sm.toCloud(), P.featureVoxelSize)
        vx, vn = v.download()
        a, b = lex(vx), lex(ref["xyz"])
        assert np.array_equal(vx[a], ref["xyz"][b]) and np.array_equal(vn[a], ref["prior"][b])
    dev.close()


@pytest.mark.parametrize("cloud", ["plane", "isolated", "both"])
def test_constructed_ties_keep_the_prior_sign(engine_factory, cloud):
    eng = engine_factory()
    xyz = {"plane": tie_plane, "isolated": isolated_points}[cloud]() if cloud != "both" else np.vstack([tie_plane(), isolated_points() + [40.0, 0, 0]])
    prior, s = signed_priors(len(xyz), 7)
    sm = E.Submap(eng, 4096)
    sm.setMapPointCloud(eng.cloud(xyz, prior))
    sm.computeFeatures(P)
    ref = check_submap(eng, sm, xyz, prior, exact_normals=True)
    assert ref["tie"].sum() > 0 and ref["tie"].all()
    dx, dn = sm.getSparseMapPointCloud().download()
    a, q = lex(dx), lex(xyz)
    assert np.array_equal(dn[a][:, 2], s[q])                          # the prior's sign, exactly +-z
    plain = O.estimate_normals(dx, P.normalKnn, P.normalEstimationRadius)
    assert (dn[:, 2] != plain[:, 2]).any()                            # the no-prior answer differs


def test_empty_submap(engine_factory):
    eng = engine_factory()
    sm = E.Submap(eng, 1024)
    sm.computeFeatures(P)
    assert len(sm.getSparseMapPointCloud()) == 0 and sm.getFeatures().Num() == 0
    sm.setMapPointCloud(eng.cloud(np.zeros((0, 3)), np.zeros((0, 3))))
    sm.computeFeatures(P)
    assert len(sm.getSparseMapPointCloud()) == 0 and sm.getFeatures().Num() == 0


def test_point_to_point_map_without_normals(engine_factory):
    """set_cloud stores missing normals as NaN; the down-sample skips them, the zero priors change nothing: the result is the
    restatement run without priors"""
    eng = engine_factory(E.MapperParameters(scanToMapRegType="PointToPointIcp"))
    xyz, _ = lidar_map(1)
    sm = E.Submap(eng, 100_000)
    sm.setMapPointCloud(eng.cloud(xyz))
    sm.computeFeatures(P)
    check_submap(eng, sm, xyz, None, exact_normals=False)


def test_errors(engine_factory):
    eng = engine_factory()
    xyz, nrm = lidar_map(2)
    sm = E.Submap(eng, 100_000)
    sm.setMapPointCloud(eng.cloud(xyz, nrm))
    bad = [(dict(featureVoxelSize=0.0), L.E_INVALID), (dict(featureVoxelSize=-0.5), L.E_INVALID), (dict(normalEstimationRadius=0.0), L.E_INVALID),
           (dict(featureRadius=-1.0), L.E_INVALID), (dict(normalKnn=0), L.E_INVALID), (dict(featureKnn=0), L.E_INVALID),
           (dict(normalKnn=33), L.E_UNSUPPORTED), (dict(featureKnn=129), L.E_UNSUPPORTED)]
    for kw, code in bad:
        with pytest.raises(L.B2SError) as e:
            sm.computeFeatures(E.PlaceRecognitionParameters(**kw))
        assert e.value.code == code, kw
    sm.computeFeatures(E.PlaceRecognitionParameters(normalKnn=32, featureKnn=128))   # the limits themselves are fine
    assert sm.getFeatures().Num() == len(sm.getSparseMapPointCloud()) > 0


def test_outputs_of_another_handle(engine_factory):
    a, b = engine_factory(), engine_factory()
    xyz, nrm = lidar_map(3)
    sm = E.Submap(a, 100_000)
    sm.setMapPointCloud(a.cloud(xyz, nrm))
    ca, fa, cb, fb = E.Cloud(a), E.Feature(a), E.Cloud(b), E.Feature(b)
    prm = P.to_c()
    call = lambda h, c, f: L.lib().b2s_submap_compute_features(h._h, sm._s, C.byref(prm), c._c, f._f)
    assert call(a, cb, fa) == L.E_INVALID and call(a, ca, fb) == L.E_INVALID and call(b, cb, fb) == L.E_INVALID
    assert call(a, ca, fa) == L.OK and fa.Num() == len(ca) > 0


def test_repeated_calls_reuse_the_outputs(engine_factory):
    eng = engine_factory()
    x1, n1 = lidar_map(4)
    sm = E.Submap(eng, 200_000)
    sm.setMapPointCloud(eng.cloud(x1, n1))
    sm.computeFeatures(P)
    c, f = sm.getSparseMapPointCloud(), sm.getFeatures()
    first = c.download()
    sm.computeFeatures(P)
    assert sm.getSparseMapPointCloud() is c and sm.getFeatures() is f
    # the same cloud again (the normals only up to the summation order, which the grid's atomic cell fill leaves open)
    again = c.download()
    assert np.array_equal(first[0], again[0]) and np.abs(first[1] - again[1]).max() < 1e-6
    check_submap(eng, sm, x1, n1, exact_normals=False)
    # a smaller map into the same outputs, then a coarser voxel
    x2, n2 = x1[: len(x1) // 3], n1[: len(x1) // 3]
    sm.setMapPointCloud(eng.cloud(x2, n2))
    sm.computeFeatures(P)
    check_submap(eng, sm, x2, n2, exact_normals=False)
    sm.setMapPointCloud(eng.cloud(x1, n1))
    sm.computeFeatures(P)
    check_submap(eng, sm, x1, n1, exact_normals=False)
