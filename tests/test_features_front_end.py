"""CPU tests of the feature-cloud front end of Submap::computeFeatures (tests/oracle_submap_features.c and its numpy twin): voxel
down-sample of the map with its normals, normals estimated on a cloud that already has normals (the voxel means are the priors),
FPFH.  The C restatement and the twin agree on a LiDAR map; constructed clouds show the prior branch of [O3D] EstimateNormals is
taken (exact ties of the camera orientation keep the prior's sign, where the no-prior restatement gives +z); the control flow
SubmapCollection.computeFeatures runs over the oracle backend."""
import copy

import numpy as np
import pytest

import oracle_features as OF
import oracle_submap_features as OSF
from oracle import oracle as O
from oracle_backend_features import FeatureOracleBackend
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import synth
from open3d_slam_b200 import workloads as W

P = E.PlaceRecognitionParameters()


def lidar_map(seed=0):
    """two scans of the synthetic scene at the map voxel (0.1 m) with their scan normals (k 20, r 3.0): a small submap map"""
    poses = synth.loop_trajectory(40)
    xs, ns = [], []
    for k in (5, 6):
        raw = synth.lidar_scan(synth.Scene(), poses[k], seed=seed + k).astype(np.float64)
        x, _ = O.voxel_down_sample(raw, 0.1)
        xs.append(x); ns.append(O.estimate_normals(x, 20, 3.0))
    return np.vstack(xs), np.vstack(ns)


def by_key(keys):
    return np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))


def test_c_and_numpy_agree_on_the_front_end():
    xyz, nrm = lidar_map()
    c = OSF.submap_features(xyz, nrm, P)
    t = OSF.np_submap_features(xyz, nrm, P)
    assert len(c["xyz"]) > 1000
    # identical sparse cloud, keyed: same voxels, bit-identical means of the points and of the normals
    oc, ot = by_key(c["keys"]), by_key(t["keys"])
    assert np.array_equal(c["keys"][oc], t["keys"][ot])
    assert np.array_equal(c["xyz"][oc], t["xyz"][ot]) and np.array_equal(c["prior"][oc], t["prior"][ot])
    assert np.abs(c["nrm"][oc] - t["nrm"][ot]).max() < 1e-12
    # FPFH of the C cloud (C order) with the twin's normals, under the margin rule of the FPFH tests
    nrm_t = np.empty_like(c["nrm"]); nrm_t[oc] = t["nrm"][ot]
    ref, _ = OF.np_fpfh(c["xyz"], nrm_t, P.featureRadius, P.featureKnn)
    diff, unexplained = OF.differing_rows(c["feature"], ref, c, tol=1e-12)
    assert len(unexplained) == 0, unexplained[:10]
    assert len(diff) <= len(ref) // 200
    # the priors matter here only at ties: away from them the result equals the no-prior restatement's
    plain = O.estimate_normals(c["xyz"], P.normalKnn, P.normalEstimationRadius)
    assert np.array_equal(c["nrm"][~c["tie"]], plain[~c["tie"]])


def tie_plane(spacing=0.5, half=6):
    """grid on z = 0 through the camera (the map-frame origin): every normal is exactly +-z and n . (-p) == 0 everywhere"""
    g = np.arange(-half, half + 1) * spacing
    X, Y = np.meshgrid(g, g)
    return np.c_[X.ravel(), Y.ravel(), np.zeros(X.size)]


def isolated_points():
    """points at z = 0 further apart than the normal radius: identity covariance -> (0,0,1), a tie with any camera direction"""
    return np.array([[5.0 * i, 3.0 - 7.0 * (i % 2), 0.0] for i in range(8)])


def signed_priors(n, seed):
    rng = np.random.default_rng(seed)
    s = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    s[0], s[1] = 1.0, -1.0                                          # both signs, whatever the draw
    tilt = rng.uniform(-0.3, 0.3, (n, 2))
    return np.c_[tilt, s] / np.linalg.norm(np.c_[tilt, s], axis=1, keepdims=True), s


@pytest.mark.parametrize("cloud", ["plane", "isolated"])
def test_prior_sign_survives_exact_ties(cloud):
    xyz = tie_plane() if cloud == "plane" else isolated_points()
    prior, s = signed_priors(len(xyz), 3)
    got, tie = OSF.estimate_normals(xyz, P.normalKnn, P.normalEstimationRadius, prior)
    assert tie.all()
    assert np.array_equal(got, np.c_[np.zeros((len(xyz), 2)), s])    # exactly +-z, the prior's sign
    # without priors the tie leaves the solver's sign (isolated points: +z from the identity covariance)
    plain = O.estimate_normals(xyz, P.normalKnn, P.normalEstimationRadius)
    assert np.array_equal(np.abs(plain), np.tile([0.0, 0.0, 1.0], (len(xyz), 1)))
    changed = got[:, 2] != plain[:, 2]
    assert changed.sum() > 0 and np.array_equal(changed, s != plain[:, 2])   # the prior branch decided every sign
    twin, ttie = OSF.np_estimate_normals(xyz, P.normalKnn, P.normalEstimationRadius, prior)
    assert np.array_equal(twin, got) and np.array_equal(ttie, tie)
    # without priors the restatement is orc_estimate_normals
    none, _ = OSF.estimate_normals(xyz, P.normalKnn, P.normalEstimationRadius)
    assert np.array_equal(none, plain)


def test_front_end_keeps_prior_signs_of_a_map_on_the_tie_plane():
    """one map point per feature voxel: the sparse cloud is the map, the priors are the map's normals"""
    xyz = tie_plane()
    prior, s = signed_priors(len(xyz), 4)
    r = OSF.submap_features(xyz, prior, P)
    o = by_key(r["keys"])
    assert len(r["xyz"]) == len(xyz) and r["tie"].all()
    m = np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0])); q = np.lexsort((r["xyz"][:, 2], r["xyz"][:, 1], r["xyz"][:, 0]))
    assert np.array_equal(r["xyz"][q], xyz[m]) and np.array_equal(r["prior"][q], prior[m])
    assert np.array_equal(r["nrm"][q][:, 2], s[m]) and o.size == len(xyz)
    assert (r["nrm"][q][:, 2] != O.estimate_normals(r["xyz"], P.normalKnn, P.normalEstimationRadius)[q][:, 2]).any()
    # without normals (a point-to-point map): the no-prior branch, orc_estimate_normals
    r0 = OSF.submap_features(xyz, None, P)
    assert r0["prior"] is None and np.array_equal(r0["nrm"], O.estimate_normals(r0["xyz"], P.normalKnn, P.normalEstimationRadius))


def test_empty_map():
    r = OSF.submap_features(np.zeros((0, 3)), np.zeros((0, 3)), P)
    assert len(r["xyz"]) == 0 and r["feature"].shape == (0, 33)


def test_submap_collection_compute_features_on_the_oracle_backend():
    """12 scans with a 2 m submap radius (hand-overs), then SubmapCollection.computeFeatures: every finished submap gets its
    sparse cloud and features, equal to the restatement run on its map; the mapper itself never computed them."""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    ora = FeatureOracleBackend(copy.deepcopy(p), carving=True, dense=False)
    m = S.SegmentMapper(ora, S.SubmapParameters(radius=2.0))
    for k in range(12):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    sc = m.submaps
    assert len(sc.finishedSubmapsIdxs) >= 1 and all(r.feature is None for r in sc.submaps)
    done = sc.computeFeatures(P)
    assert done == sc.finishedSubmapsIdxs
    for i, rec in enumerate(sc.submaps):
        if i not in done:
            assert rec.feature is None and rec.sparse is None
            continue
        x, n = ora.map_cloud(rec.handle)
        ref = OSF.submap_features(x, n, P)
        assert np.array_equal(rec.sparse.xyz, ref["xyz"]) and np.array_equal(rec.sparse.nrm, ref["nrm"])
        assert np.array_equal(rec.feature, ref["feature"]) and len(rec.feature) > 100
        has = ref["nb_cnt"] > 1
        assert np.abs(rec.feature[has].reshape(-1, 3, 11).sum(axis=2) - 200.0).max() < 1e-9
