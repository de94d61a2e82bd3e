"""-m gpu parity tests: the CUDA path (through the C ABI) against the CPU oracle on identical seeded inputs.

Tolerances: the north star asks for 1e-4 relative on the converged SE(3); because the device path is fp64 and
reproduces the oracle's neighbour decisions bit-for-bit, the tests hold it to 1e-9 (transform) / 1e-12 (voxel means).

The inputs here are typical ones.  The size switches of the kernels (ICP cluster size, 64-point tiles, shared or global memory,
batch cluster shrink, certificates; normals knn, select exits, coarsened grid; voxel key width, one-cluster or multi-kernel sort,
wide grid, grid-size independence) are crossed from both sides in test_gpu_boundaries.py.
"""
import ctypes as C

import numpy as np
import pytest

import normals_checks as NC
from oracle import oracle as O
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import synth
from open3d_slam_b200 import _lib as L

pytestmark = pytest.mark.gpu


def rel_rot(Ta, Tb):
    return np.linalg.norm(Ta[:3, :3] - Tb[:3, :3]) / np.linalg.norm(Tb[:3, :3])


def rel_trans(Ta, Tb):
    return np.linalg.norm(Ta[:3, 3] - Tb[:3, 3]) / max(np.linalg.norm(Tb[:3, 3]), 1.0)


def sort_by_key(xyz, voxel, origin=None):
    """Sort points of a voxelised cloud canonically (by their quantised coordinates) to compare as sets."""
    q = np.floor(xyz / (voxel * 0.5)).astype(np.int64) if origin is None else np.floor((xyz - origin) / voxel).astype(np.int64)
    order = np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0], q[:, 2], q[:, 1], q[:, 0]))
    return order


def lua_params(**kw):
    p = E.MapperParameters()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def test_icp_sixteen_sm_clusters_give_the_same_registration(engine_factory):
    """b2s_config.icp_cluster_ctas = 16 (latency mode: one registration over 16 SMs, non-portable cluster size) must change nothing but
    the summation order: same iterations / correspondences, T to 1e-10 of the default 8-SM clusters, on a scan-sized source."""
    sc = synth.Scene(); poses = synth.loop_trajectory(8)
    results = []
    for ctas in (0, 16, 4):
        p = lua_params()
        p.icpClusterCtas = ctas
        eng = engine_factory(p)
        icp = E.ScanToMapIcp(eng)
        sm = E.Submap(eng, 400_000)
        for k in range(3):
            ps = icp.processForScanMatchingAndMerging(eng.cloud(synth.lidar_scan(sc, poses[k], seed=k)))
            sm.insertScan(None, ps.merge_, np.linalg.inv(poses[0]) @ poses[k])
        ps = icp.processForScanMatchingAndMerging(eng.cloud(synth.lidar_scan(sc, poses[3], seed=3)))
        assert len(ps.match_) > 8 * 768                      # enough points for the launch to pick the largest cluster allowed
        guess = np.linalg.inv(poses[0]) @ poses[3] @ synth.se3(0.004, -0.003, 0.01, (0.03, -0.02, 0.01))
        results.append(icp.scanToMapRegistration(ps.match_, sm, np.linalg.inv(poses[0]) @ poses[2], guess))
    a = results[0]
    for b in results[1:]:
        assert a.iters == b.iters and a.n_corr == b.n_corr and abs(a.fitness_ - b.fitness_) < 1e-14
        assert np.abs(a.transformation_ - b.transformation_).max() < 1e-10
    assert a.fitness_ > 0.9


def test_icp_source_larger_than_shared_memory(engine_factory):
    """A source cloud too large for the cluster's shared memory (8 CTAs x ~4.9 k points) takes the kernel's other path: working copy
    and per-point state in global memory, no phase-2 queue, no certificates.  Same answers as the oracle."""
    rng = np.random.default_rng(11)
    n_t, n_s = 30_000, 60_000
    tgt = np.c_[rng.uniform(-8, 8, (n_t, 2)), 0.05 * rng.standard_normal(n_t)]
    tgt[: n_t // 3] = np.c_[rng.uniform(-8, 8, n_t // 3), np.full(n_t // 3, 8.0) + 0.05 * rng.standard_normal(n_t // 3), rng.uniform(0, 4, n_t // 3)]
    tgt[n_t // 3: 2 * n_t // 3, 0] = -8.0 + 0.05 * rng.standard_normal(2 * n_t // 3 - n_t // 3)
    tgt[n_t // 3: 2 * n_t // 3, 2] = rng.uniform(0, 4, 2 * n_t // 3 - n_t // 3)
    nrm = O.estimate_normals(tgt, 10, 1.0)
    T_true = synth.se3(0.01, -0.015, 0.02, (0.06, -0.04, 0.03))
    pick = rng.integers(0, n_t, n_s)
    src = (tgt[pick] + 0.01 * rng.standard_normal((n_s, 3)) - T_true[:3, 3]) @ T_true[:3, :3]      # inverse motion of noisy target samples
    p = lua_params()
    p.icp.maxCorrespondenceDistance = 0.5
    p.icp.maxNumIter = 4
    eng = engine_factory(p)
    reg = E.cloudRegistrationFactory(eng, E.CloudRegistrationParameters(icp=p.icp))
    res = reg.registerClouds(eng.cloud(src), eng.cloud(tgt, nrm), np.eye(4))
    ref = O.registration_icp_p2plane(src, tgt, nrm, 0.5, np.eye(4), max_iter=4)
    assert res.iters == ref.iters and res.n_corr == ref.n_corr
    assert abs(res.fitness_ - ref.fitness) < 1e-12
    assert rel_rot(res.transformation_, ref.T) < 1e-9 and rel_trans(res.transformation_, ref.T) < 1e-9


# ----------------------------------------------------------------------------------------------------------------------
# R1-R5: config 1 -- scan-to-scan point-to-plane ICP on the 2k-pt three-plane cloud
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("noise", [0.0, 0.01])
def test_icp_config1(engine_factory, noise):
    src, tgt, nrm, T_true = synth.planar_cloud_config1(noise=noise)
    p = lua_params()
    p.icp.maxCorrespondenceDistance = 1.0
    p.icp.maxNumIter = 50
    eng = engine_factory(p)
    reg = E.cloudRegistrationFactory(eng, E.CloudRegistrationParameters(icp=p.icp))
    res = reg.registerClouds(eng.cloud(src), eng.cloud(tgt, nrm), np.eye(4))
    ref = O.registration_icp_p2plane(src, tgt, nrm, 1.0, np.eye(4), max_iter=50)
    assert res.iters == ref.iters
    assert res.n_corr == ref.n_corr
    assert abs(res.fitness_ - ref.fitness) < 1e-12
    assert abs(res.inlier_rmse_ - ref.inlier_rmse) < 1e-10
    assert rel_rot(res.transformation_, ref.T) < 1e-9
    assert rel_trans(res.transformation_, ref.T) < 1e-9
    # and the registration actually recovers the displacement (source = T_true * target)
    assert rel_trans(res.transformation_, np.linalg.inv(T_true)) < (1e-6 if noise == 0 else 5e-3)


def test_icp_init_and_iteration_cap(engine_factory):
    src, tgt, nrm, T_true = synth.planar_cloud_config1(noise=0.01)
    init = synth.se3(0.01, -0.02, 0.03, (0.05, 0.02, -0.01))
    for max_iter in (0, 1, 2, 30):
        p = lua_params()
        p.icp.maxCorrespondenceDistance = 0.5
        p.icp.maxNumIter = max_iter
        eng = engine_factory(p)
        reg = E.RegistrationIcpPointToPlane(eng)
        res = reg.registerClouds(eng.cloud(src), eng.cloud(tgt, nrm), init)
        ref = O.registration_icp_p2plane(src, tgt, nrm, 0.5, init, max_iter=max_iter)
        assert res.iters == ref.iters and res.n_corr == ref.n_corr
        assert np.abs(res.transformation_ - ref.T).max() < 1e-9
        assert abs(res.inlier_rmse_ - ref.inlier_rmse) < 1e-10


def test_icp_no_overlap_and_missing_normals(engine_factory):
    src, tgt, nrm, _ = synth.planar_cloud_config1()
    eng = engine_factory(lua_params())
    reg = E.RegistrationIcpPointToPlane(eng)
    far = src + np.array([500.0, 0.0, 0.0])
    res = reg.registerClouds(eng.cloud(far), eng.cloud(tgt, nrm), np.eye(4))
    ref = O.registration_icp_p2plane(far, tgt, nrm, 1.0, np.eye(4), max_iter=50)
    assert res.n_corr == 0 and res.fitness_ == 0.0 and res.inlier_rmse_ == 0.0 and res.iters == ref.iters
    assert np.array_equal(res.transformation_, np.eye(4))
    with pytest.raises(L.B2SError) as ei:
        reg.registerClouds(eng.cloud(src), eng.cloud(tgt), np.eye(4))
    assert ei.value.code == L.E_NO_NORMALS


def test_icp_batch_matches_single(engine_factory):
    rng = np.random.default_rng(5)
    src, tgt, nrm, _ = synth.planar_cloud_config1(noise=0.01)
    p = lua_params()
    p.icp.maxCorrespondenceDistance = 0.6
    eng = engine_factory(p)
    reg = E.RegistrationIcpPointToPlane(eng)
    tcloud = eng.cloud(tgt, nrm)
    sources, inits = [], []
    for k in range(6):
        d = synth.se3(*rng.uniform(-0.02, 0.02, 3), rng.uniform(-0.05, 0.05, 3))
        s = src @ d[:3, :3].T + d[:3, 3]
        sources.append(s)
        inits.append(np.eye(4))
    clouds = [eng.cloud(s) for s in sources]
    batch = reg.registerCloudsBatch(clouds, [tcloud] * len(clouds), inits)
    for s, b in zip(sources, batch):
        ref = O.registration_icp_p2plane(s, tgt, nrm, 0.6, np.eye(4), max_iter=50)
        assert b.iters == ref.iters and b.n_corr == ref.n_corr
        assert np.abs(b.transformation_ - ref.T).max() < 1e-9


# ----------------------------------------------------------------------------------------------------------------------
# P1 / P2 / P4 / F0
# ----------------------------------------------------------------------------------------------------------------------
def _scan(k=0, seed=0):
    sc = synth.Scene()
    poses = synth.loop_trajectory(8)
    return synth.lidar_scan(sc, poses[k], seed=seed).astype(np.float64), poses[k]


def test_crop_all_kinds(engine_factory):
    raw, _ = _scan()
    eng = engine_factory(lua_params())
    cl = eng.cloud(raw)
    for kind, kw in (("MaxRadius", {}), ("MinRadius", {}), ("MinMaxRadius", {}), ("Cylinder", {})):
        for invert in (False, True):
            cp = E.ScanCroppingParameters(cropperName=kind, croppingMinRadius=3.0, croppingMaxRadius=15.0, croppingMinZ=-1.0, croppingMaxZ=2.0)
            c = cp.to_c(center=(1.0, -2.0, 0.5), invert=invert)
            out, _n = E.crop(eng, cl, c).download()
            oc = O.cropper(kind, 3.0, 15.0, -1.0, 2.0, (1.0, -2.0, 0.5), invert)
            ref, _ = O.crop(oc, raw)
            assert out.shape == ref.shape and np.array_equal(out, ref)   # same points, same order, bit-exact


@pytest.mark.parametrize("voxel", [0.1, 0.3])
def test_voxel_down_sample_bit_exact(engine_factory, voxel):
    raw, _ = _scan()
    eng = engine_factory(lua_params())
    out, _n = E.voxelize(eng, eng.cloud(raw), voxel).download()
    ref, _, keys = O.voxel_down_sample(raw, voxel, return_keys=True)
    assert len(out) == len(ref)
    vmin = raw.min(axis=0) - 0.5 * voxel
    ko = np.floor((out - vmin) / voxel).astype(np.int64)
    # every output point lies in a distinct reference voxel; compare as keyed sets
    o1 = np.lexsort((ko[:, 2], ko[:, 1], ko[:, 0])); o2 = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    # a mean can fall on a voxel face, so match by nearest reference mean instead of by key when keys disagree
    a, b = out[o1], ref[o2]
    if not np.array_equal(a, b):
        from scipy.spatial import cKDTree
        d, j = cKDTree(ref).query(out)
        assert d.max() == 0.0 and len(np.unique(j)) == len(ref)
    else:
        assert np.array_equal(a, b)


def test_voxel_negative_coordinates_and_faces(engine_factory):
    # points exactly on voxel faces, negative coordinates, duplicates
    g = np.arange(-5, 6) * 0.25
    pts = np.array([[x, y, z] for x in g for y in g[:5] for z in (-0.5, 0.0, 0.25)], dtype=np.float64)
    pts = np.vstack([pts, pts[:50], pts[:7] + 1e-12])
    eng = engine_factory(lua_params())
    out, _n = E.voxelize(eng, eng.cloud(pts), 0.25).download()
    ref, _ = O.voxel_down_sample(pts, 0.25)
    assert len(out) == len(ref)
    from scipy.spatial import cKDTree
    d, j = cKDTree(ref).query(out)
    assert d.max() == 0.0 and len(np.unique(j)) == len(ref)


def test_random_down_sample(engine_factory):
    raw, _ = _scan()
    eng = engine_factory(lua_params())
    vx = E.voxelize(eng, eng.cloud(raw), 0.2)
    xyz, _n = vx.download()
    for ratio, seed in ((0.3, 0), (0.25, 7), (1.0, 3), (0.0, 1)):
        out, _ = E.random_down_sample(eng, vx, ratio, seed).download()
        ref, _ = O.random_down_sample(xyz, ratio, seed)
        assert out.shape == ref.shape and np.array_equal(out, ref)


def test_transform_with_identity_quirk(engine_factory):
    raw, _ = _scan()
    raw = raw[:5000]
    nrm = np.random.default_rng(0).normal(size=raw.shape)
    eng = engine_factory(lua_params())
    cl = eng.cloud(raw, nrm)
    for T in (synth.se3(0.1, -0.2, 0.7, (3.0, -1.0, 0.2)), np.eye(4), synth.se3(0, 0, 5e-5, (2e-5, 0, 0))):
        ox, on = E.transform(eng, T, cl).download()
        rx, rn = O.transform(T, raw, nrm)
        assert ox.shape == rx.shape
        assert np.array_equal(ox, rx) and np.array_equal(on, rn)


# ----------------------------------------------------------------------------------------------------------------------
# P3: normals
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knn,radius", [(20, 3.0), (5, 10.0), (10, 0.35)])
def test_estimate_normals(engine_factory, knn, radius):
    raw, _ = _scan()
    eng = engine_factory(lua_params())
    vx = E.voxelize(eng, eng.cloud(raw), 0.1)
    xyz, _n = vx.download()
    reg = E.RegistrationIcpPointToPlane(eng)
    reg.knnNormalEstimation_ = knn; reg.maxRadiusNormalEstimation_ = radius
    reg.estimateNormalsOrCovariancesIfNeeded(vx)
    _x, got = vx.download()
    ref = O.estimate_normals(xyz, knn, radius)
    # same neighbour sets, same covariance arithmetic, the cumulants summed in another order: per point within the gap-aware bound
    # of tests/normals_checks.py (far below the 1e-6 rad of SURVEY 8c test 4 wherever the eigenproblem is well conditioned)
    worst = NC.assert_normals_close(got, ref, xyz, knn, radius)
    print(f"normals knn {knn} r {radius}: worst {worst:.3g} of the gap-aware bound")


def test_normals_degenerate_few_neighbours(engine_factory):
    pts = np.array([[1.0, 0, 0], [1.05, 0, 0], [50.0, 3, 1], [-20, 4, 2.0], [1.0, 0.05, 0.0]])
    eng = engine_factory(lua_params())
    cl = eng.cloud(pts)
    reg = E.RegistrationIcpPointToPlane(eng)
    reg.knnNormalEstimation_ = 5; reg.maxRadiusNormalEstimation_ = 0.5
    reg.estimateNormalsOrCovariancesIfNeeded(cl)
    _x, got = cl.download()
    ref = O.estimate_normals(pts, 5, 0.5)
    assert np.allclose(got, ref, atol=1e-12)
    with pytest.raises(L.B2SError):
        reg.maxRadiusNormalEstimation_ = 0.0
        reg.estimateNormalsOrCovariancesIfNeeded(cl)


# ----------------------------------------------------------------------------------------------------------------------
# S1: processForScanMatchingAndMerging
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ratio", [1.0, 0.3])
def test_process_scan(engine_factory, ratio):
    raw32 = synth.lidar_scan(synth.Scene(), synth.loop_trajectory(4)[1], seed=11)
    raw = raw32.astype(np.float64)
    p = lua_params(seed=5)
    p.scanProcessing.downSamplingRatio = ratio
    p.scanProcessing.cropper = E.ScanCroppingParameters("MinMaxRadius", 2.0, 25.0)
    eng = engine_factory(p)
    s2m = E.scanToMapRegistrationFactory(eng, p)
    ps = s2m.processForScanMatchingAndMerging(eng.cloud(raw32))
    (mx, mn), (ax, an) = O.process_scan(raw, O.cropper("MinMaxRadius", 2.0, 30.0), O.cropper("MinMaxRadius", 2.0, 25.0), 0.1, 20, 3.0, ratio, 5)
    gx, gn = ps.merge_.download()
    hx, hn = ps.match_.download()
    assert len(gx) == len(mx) and len(hx) == len(ax)
    from scipy.spatial import cKDTree
    d, j = cKDTree(mx).query(gx)
    assert d.max() == 0.0 and len(np.unique(j)) == len(mx)      # identical point sets (bit-exact voxel means)
    assert ((gn * mn[j]).sum(axis=1)).min() > 1 - 1e-6
    d, j = cKDTree(ax).query(hx)
    assert d.max() == 0.0 and len(np.unique(j)) == len(ax)


# ----------------------------------------------------------------------------------------------------------------------
# F1 / S2 / M1: map fusion, scan-to-map registration, odometry loop
# ----------------------------------------------------------------------------------------------------------------------
def _keyed(xyz, nrm, voxel):
    k = np.floor(xyz * (1.0 / voxel)).astype(np.int64)
    order = np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0], k[:, 2], k[:, 1], k[:, 0]))
    return xyz[order], nrm[order]


def test_submap_insert_matches_reference_fusion(engine_factory):
    p = lua_params(seed=1)
    p.scanProcessing.downSamplingRatio = 1.0
    eng = engine_factory(p)
    sc = synth.Scene(); poses = synth.loop_trajectory(6)
    s2m = E.ScanToMapIcp(eng)
    sm = E.Submap(eng, 600_000)
    map_x = np.zeros((0, 3)); map_n = np.zeros((0, 3))
    crop = O.cropper("MinMaxRadius", 2.0, 30.0)
    for k in range(4):
        raw = synth.lidar_scan(sc, poses[k], seed=k)
        ps = s2m.processForScanMatchingAndMerging(eng.cloud(raw))
        mx, mn = ps.merge_.download()
        T = np.eye(4) if k == 0 else poses[k]     # first insertion with identity exercises the duplication quirk
        sm.insertScan(None, ps.merge_, T)
        map_x, map_n = O.submap_insert_scan(map_x, map_n, mx, mn, T, 0.1, crop)
        gx, gn = sm.getMapPointCloud()
        assert len(gx) == len(map_x)
        a, an = _keyed(gx, gn, 0.1); b, bn = _keyed(map_x, map_n, 0.1)
        assert np.array_equal(a, b)
        assert np.abs(an - bn).max() < 1e-12


def test_scan_to_map_registration_and_mapper_loop(engine_factory):
    """Config-2 style loop, 8 scans: device Mapper vs an oracle-only restatement of the same control flow."""
    p = lua_params(seed=3)
    p.scanProcessing.downSamplingRatio = 1.0
    eng = engine_factory(p)
    sc = synth.Scene(); poses = synth.loop_trajectory(10)
    mapper = E.Mapper(eng, 800_000)
    wide = O.cropper("MinMaxRadius", 2.0, 30.0); narrow = O.cropper("MinMaxRadius", 2.0, 30.0)
    map_x = np.zeros((0, 3)); map_n = np.zeros((0, 3)); pose = np.eye(4)
    rng = np.random.default_rng(0)
    for k in range(8):
        raw = synth.lidar_scan(sc, poses[k], seed=100 + k)
        delta = np.eye(4) if k == 0 else np.linalg.inv(poses[k - 1]) @ poses[k] @ synth.se3(0, 0, rng.normal(0, 2e-3), rng.normal(0, 0.02, 3))
        ok = mapper.addRangeMeasurement(eng.cloud(raw), delta)
        (mx, mn), (ax, an) = O.process_scan(raw.astype(np.float64), wide, narrow, 0.1, 20, 3.0, 1.0, 3)
        if k == 0:
            map_x, map_n = O.submap_insert_scan(map_x, map_n, mx, mn, np.eye(4), 0.1, wide)
            continue
        assert ok
        guess = pose @ delta
        c = O.cropper("MinMaxRadius", 2.0, 30.0, center=pose[:3, 3])
        px, pn = O.crop(c, map_x, map_n)
        ref = O.registration_icp_p2plane(ax, px, pn, 1.0, guess, max_iter=50)
        got = mapper.lastResult
        assert got.iters == ref.iters and got.n_corr == ref.n_corr
        assert rel_rot(got.transformation_, ref.T) < 1e-9 and rel_trans(got.transformation_, ref.T) < 1e-9
        assert ref.fitness > 0.7
        pose = ref.T
        map_x, map_n = O.submap_insert_scan(map_x, map_n, mx, mn, pose, 0.1, wide)
    # trajectory is sane w.r.t. ground truth expressed in the first sensor frame
    gt = np.linalg.inv(poses[0]) @ poses[7]
    assert np.linalg.norm(pose[:3, 3] - gt[:3, 3]) < 0.15


@pytest.mark.parametrize("reg_type", ["GeneralizedIcp", "PointToPointIcp"])
def test_scan_to_map_loop_with_the_other_estimators(engine_factory, reg_type):
    """ScanToMapIcp serves all three registration types (src/ScanToMapRegistration.cpp:91-129): the device Mapper against the
    oracle-only restatement of the loop with the matching oracle estimator."""
    p = lua_params(seed=3)
    p.scanToMapRegType = reg_type
    p.scanProcessing.downSamplingRatio = 0.5
    eng = engine_factory(p)
    assert isinstance(E.scanToMapRegistrationFactory(eng, p), E.ScanToMapIcp)
    sc = synth.Scene(); poses = synth.loop_trajectory(8)
    mapper = E.Mapper(eng, 600_000)
    wide = O.cropper("MinMaxRadius", 2.0, 30.0)
    map_x = np.zeros((0, 3)); map_n = np.zeros((0, 3)); pose = np.eye(4)
    for k in range(4):
        raw = synth.lidar_scan(sc, poses[k], seed=300 + k)
        delta = np.eye(4) if k == 0 else np.linalg.inv(poses[k - 1]) @ poses[k] @ synth.se3(0, 0, 1e-3, (0.02, -0.01, 0.005))
        ok = mapper.addRangeMeasurement(eng.cloud(raw), delta)
        (mx, mn), (ax, an) = O.process_scan(raw.astype(np.float64), wide, wide, 0.1, 20, 3.0, 0.5, 3)
        if k == 0:
            map_x, map_n = O.submap_insert_scan(map_x, map_n, mx, mn, np.eye(4), 0.1, wide)
            continue
        assert ok
        guess = pose @ delta
        px, pn = O.crop(O.cropper("MinMaxRadius", 2.0, 30.0, center=pose[:3, 3]), map_x, map_n)
        if reg_type == "GeneralizedIcp":
            ref = O.registration_gicp(ax, an, px, pn, 1.0, guess, max_iter=50)
        else:
            ref = O.registration_icp_p2point(ax, px, 1.0, guess, max_iter=50)
        got = mapper.lastResult
        assert got.iters == ref.iters and got.n_corr == ref.n_corr
        assert rel_rot(got.transformation_, ref.T) < 1e-7 and rel_trans(got.transformation_, ref.T) < 1e-7
        assert ref.fitness > 0.7
        pose = ref.T
        map_x, map_n = O.submap_insert_scan(map_x, map_n, mx, mn, pose, 0.1, O.cropper("MinMaxRadius", 2.0, 30.0, center=pose[:3, 3]))
    gt = np.linalg.inv(poses[0]) @ poses[3]
    assert np.linalg.norm(pose[:3, 3] - gt[:3, 3]) < 0.15


def test_mapper_async_chain_matches_sync(engine_factory):
    p = lua_params(seed=3)
    p.scanProcessing.downSamplingRatio = 0.5
    sc = synth.Scene(); poses = synth.loop_trajectory(8)
    e1, e2 = engine_factory(p), engine_factory(p)
    m1, m2 = E.Mapper(e1, 800_000), E.Mapper(e2, 800_000)
    for k in range(6):
        raw = synth.lidar_scan(sc, poses[k], seed=7 + k)
        delta = np.eye(4) if k == 0 else np.linalg.inv(poses[k - 1]) @ poses[k]
        m1.addRangeMeasurement(e1.cloud(raw), delta)
        if k == 0:
            m2.addRangeMeasurement(e2.cloud(raw), delta)
            continue
        m2.addRangeMeasurementAsync(e2.cloud(raw), delta, slot=k)
        r2 = m2.fetchResult(k)
        # the initial guess is composed on the host (numpy) in one path and on the device in the other: last-bit
        # differences in the guess are allowed, the converged results must agree far below the 1e-4 target
        assert np.abs(r2.transformation_ - m1.lastResult.transformation_).max() < 1e-10
        assert r2.n_corr == m1.lastResult.n_corr and r2.iters == m1.lastResult.iters
    assert np.abs(m2.submap.getPose() - m1.mapToRangeSensor_).max() < 1e-10
    a = m1.submap.getMapPointCloud()[0]; b = m2.submap.getMapPointCloud()[0]
    assert a.shape == b.shape
    ka, kb = _keyed(a, a, 0.1)[0], _keyed(b, b, 0.1)[0]
    assert np.abs(ka - kb).max() < 1e-9


def test_mapper_graph_replay_matches_eager(engine_factory):
    """b2s_mapper_graph_enable: the captured-and-replayed chain gives bit-identical results to eager launches."""
    p = lua_params(seed=3)
    sc = synth.Scene(); poses = synth.loop_trajectory(12)
    e1, e2 = engine_factory(p), engine_factory(p)
    m1, m2 = E.Mapper(e1, 600_000), E.Mapper(e2, 600_000)
    raw0 = synth.lidar_scan(sc, poses[0], seed=50)
    for m, e in ((m1, e1), (m2, e2)):
        m.addRangeMeasurement(e.cloud(raw0), None)
        m.submap.setPose(np.eye(4))
    st = m2.enableGraph(65536)
    for k in range(1, 10):      # steps 1-2 run eagerly (warm-up), step 3 captures, the rest replay
        raw = synth.lidar_scan(sc, poses[k], seed=50 + k)
        delta = np.linalg.inv(poses[k - 1]) @ poses[k]
        m1.addRangeMeasurementAsync(e1.cloud(raw), delta, slot=k)
        st.upload(raw)
        sl = m2.addRangeMeasurementAsync(st, delta)
        r1, r2 = m1.fetchResult(k), m2.fetchResult(sl)
        assert r1.iters == r2.iters and r1.n_corr == r2.n_corr
        # the order in which the ICP kernel's phase-2 queue is drained (atomics) differs from run to run, so the fp64 sums
        # agree to the last few bits only
        assert np.abs(r1.transformation_ - r2.transformation_).max() < 1e-12
        assert r1.fitness_ > 0.9
    assert np.abs(m1.submap.getPose() - m2.submap.getPose()).max() < 1e-12
    a = m1.submap.getMapPointCloud()[0]; b = m2.submap.getMapPointCloud()[0]
    assert a.shape == b.shape and np.abs(_keyed(a, a, 0.1)[0] - _keyed(b, b, 0.1)[0]).max() < 1e-11


@pytest.mark.parametrize("graph", [False, True])
def test_mapper_step_host_matches_device_chain(engine_factory, graph):
    """b2s_mapper_step_host (float32 host scan in, result out, one call) == upload + b2s_mapper_step_async + fetch."""
    p = lua_params(seed=5)
    sc = synth.Scene(); poses = synth.loop_trajectory(10)
    e1, e2 = engine_factory(p), engine_factory(p)
    m1, m2 = E.Mapper(e1, 600_000), E.Mapper(e2, 600_000)
    raw0 = synth.lidar_scan(sc, poses[0], seed=80).astype(np.float32)
    for m, e in ((m1, e1), (m2, e2)):
        m.addRangeMeasurement(e.cloud(raw0.astype(np.float64)), None)
        m.submap.setPose(np.eye(4))
    if graph:
        m2.enableGraph(65536)
    for k in range(1, 8):
        raw = np.ascontiguousarray(synth.lidar_scan(sc, poses[k], seed=80 + k).astype(np.float32))
        delta = np.linalg.inv(poses[k - 1]) @ poses[k]
        m1.addRangeMeasurementAsync(e1.cloud(raw.astype(np.float64)), delta, slot=k)
        r1 = m1.fetchResult(k)
        r2 = m2.addRangeMeasurementHost(raw.ctypes.data, raw.shape[0], delta)
        assert r1.iters == r2.iters and r1.n_corr == r2.n_corr
        assert np.abs(r1.transformation_ - r2.transformation_).max() < 1e-12
    assert np.abs(m1.submap.getPose() - m2.submap.getPose()).max() < 1e-12
    assert m1.submap.size() == m2.submap.size()
    with pytest.raises(L.B2SError):   # a scan larger than the staging capacity is refused, not truncated
        if not graph:
            raise L.B2SError(L.E_CAPACITY, "eager mode grows the staging cloud")
        big = np.zeros((65537, 3), np.float32)
        m2.addRangeMeasurementHost(big.ctypes.data, big.shape[0], np.eye(4))


def test_mapper_step_host_async_results_land_in_pinned_memory(engine_factory):
    import torch
    p = lua_params(seed=5)
    sc = synth.Scene(); poses = synth.loop_trajectory(10)
    e1, e2 = engine_factory(p), engine_factory(p)
    m1, m2 = E.Mapper(e1, 600_000), E.Mapper(e2, 600_000)
    raw0 = synth.lidar_scan(sc, poses[0], seed=80).astype(np.float32)
    for m, e in ((m1, e1), (m2, e2)):
        m.addRangeMeasurement(e.cloud(raw0.astype(np.float64)), None)
        m.submap.setPose(np.eye(4))
    m2.enableGraph(65536)
    n = 6
    scans = [torch.from_numpy(np.ascontiguousarray(synth.lidar_scan(sc, poses[k], seed=80 + k).astype(np.float32))).pin_memory() for k in range(1, n)]
    out = torch.zeros((n, C.sizeof(L.Result)), dtype=torch.uint8).pin_memory()
    for k in range(1, n):      # enqueue everything, synchronise once
        m2.addRangeMeasurementHostAsync(scans[k - 1].data_ptr(), scans[k - 1].shape[0], np.linalg.inv(poses[k - 1]) @ poses[k], out[k].data_ptr())
    e2.synchronize()
    for k in range(1, n):
        r1 = m1.addRangeMeasurementHost(scans[k - 1].data_ptr(), scans[k - 1].shape[0], np.linalg.inv(poses[k - 1]) @ poses[k])
        r2 = L.Result.from_buffer_copy(out[k].numpy().tobytes())
        assert r1.iters == r2.iters and r1.n_corr == r2.n_corr
        assert np.abs(r1.transformation_ - np.array(r2.T).reshape(4, 4)).max() < 1e-12


def test_config3_voxel_normals_1m(engine_factory):
    """BASELINE config 3 at full size: 21 scans in the map frame cut to 1 048 576 points, voxel 0.1, knn 20, radius 3.0."""
    sc = synth.Scene(); poses = synth.loop_trajectory(600)
    parts = []
    for i in range(21):
        T = poses[(i * 37) % 600]
        s = synth.lidar_scan(sc, T, seed=1000 + i).astype(np.float64)
        parts.append(s @ T[:3, :3].T + T[:3, 3])
    xyz = np.ascontiguousarray(np.vstack(parts)[:1 << 20])   # scans lose their sky rays: 21 scans give > 2^20 returns
    assert xyz.shape[0] == 1 << 20
    eng = engine_factory(lua_params())
    vox = E.voxelize(eng, eng.cloud(xyz), 0.1)
    gx, _ = vox.download()
    ox, _ = O.voxel_down_sample(xyz, 0.1)
    assert gx.shape == ox.shape
    og, gg = np.lexsort(ox.T[::-1]), np.lexsort(gx.T[::-1])
    assert np.array_equal(ox[og], gx[gg])          # same voxels, same members summed in the same order: bit-identical means
    L.check(L.lib().b2s_estimate_normals(eng._h, vox._c, 20, C.c_double(3.0)))
    gx2, gn = vox.download()
    assert np.array_equal(gx2, gx)
    on = O.estimate_normals(gx, 20, 3.0)
    assert np.abs(on - gn).max() < 1e-9
    assert np.abs(np.linalg.norm(gn, axis=1) - 1.0).max() < 1e-12
    assert np.all(np.sum(gn * gx, axis=1) <= 0.0)   # oriented towards the origin (OrientNormalsTowardsCameraLocation)


def test_config4_scan_submap_pairs_batch(engine_factory):
    """BASELINE config 4 (a handful of its 512 pairs): oracle-built 20 m submaps, sources displaced by a random SE(3)
    within (+-0.5 m, +-5 deg), r = 0.3, max_iter = 100 (core/src/PlaceRecognition.cpp:45-46,111), one batched launch."""
    p = lua_params()
    p.icp.maxCorrespondenceDistance = 0.3
    p.icp.maxNumIter = 100
    eng = engine_factory(p)
    reg = E.RegistrationIcpPointToPlane(eng)
    sc = synth.Scene(); poses = synth.loop_trajectory(600)
    wide = O.cropper("MinMaxRadius", 2.0, 30.0); mapc = O.cropper("MaxRadius", 0.0, 20.0)
    rng = np.random.default_rng(44)
    srcs, tgts, inits, refs = [], [], [], []
    for pair in range(5):
        k0 = 97 * pair
        mx = np.zeros((0, 3)); mn = np.zeros((0, 3))
        for k in range(k0, k0 + 3):       # submap from three consecutive scans at their true poses
            (ax, an), _ = O.process_scan(synth.lidar_scan(sc, poses[k], seed=k), wide, wide, 0.1, 20, 3.0, 1.0, 0)
            c = O.cropper("MaxRadius", 0.0, 20.0, center=tuple(poses[k][:3, 3]))
            mx, mn = O.submap_insert_scan(mx, mn, ax, an, poses[k], 0.1, c)
        _, (sx, sn) = O.process_scan(synth.lidar_scan(sc, poses[k0 + 3], seed=k0 + 3), wide, wide, 0.1, 20, 3.0, 0.3, 7)
        d = synth.se3(*np.deg2rad(rng.uniform(-5, 5, 3)), rng.uniform(-0.5, 0.5, 3) * (0.2 if pair < 3 else 1.0))
        init = poses[k0 + 3] @ d
        srcs.append(sx); tgts.append((mx, mn)); inits.append(init)
        refs.append(O.registration_icp_p2plane(sx, mx, mn, 0.3, init, max_iter=100))
    res = reg.registerCloudsBatch([eng.cloud(s) for s in srcs], [eng.cloud(x, n) for x, n in tgts], inits)
    for r, ref in zip(res, refs):
        assert r.iters == ref.iters and r.n_corr == ref.n_corr
        assert abs(r.fitness_ - ref.fitness) < 1e-12 and abs(r.inlier_rmse_ - ref.inlier_rmse) < 1e-9
        assert rel_rot(r.transformation_, ref.T) < 1e-8 and rel_trans(r.transformation_, ref.T) < 1e-8


def test_point_to_point_icp_matches_oracle(engine_factory):
    """R1' (SURVEY 8f rank 3): RegistrationIcpPointToPoint -- [O3D] RegistrationICP with Eigen::umeyama updates."""
    src, tgt, nrm, T_true = synth.planar_cloud_config1(noise=0.01)
    p = lua_params()
    p.icp.maxCorrespondenceDistance = 1.0
    p.icp.maxNumIter = 50
    eng = engine_factory(p)
    reg = E.cloudRegistrationFactory(eng, E.CloudRegistrationParameters(regType="PointToPointIcp", icp=p.icp))
    assert isinstance(reg, E.RegistrationIcpPointToPoint)
    tcloud = eng.cloud(tgt)                                   # no normals: point-to-point does not need them
    for init in (np.eye(4), synth.se3(0.01, -0.02, 0.03, (0.05, 0.02, -0.01))):
        res = reg.registerClouds(eng.cloud(src), tcloud, init)
        ref = O.registration_icp_p2point(src, tgt, 1.0, init, max_iter=50)
        assert res.iters == ref.iters and res.n_corr == ref.n_corr
        assert abs(res.fitness_ - ref.fitness) < 1e-12 and abs(res.inlier_rmse_ - ref.inlier_rmse) < 1e-9
        assert rel_rot(res.transformation_, ref.T) < 1e-8 and rel_trans(res.transformation_, ref.T) < 1e-8
    # iteration cap and the batched launch (one scan-submap-sized pair among them)
    sc = synth.Scene(); poses = synth.loop_trajectory(600)
    wide = O.cropper("MinMaxRadius", 2.0, 30.0)
    (mx, mn), _ = O.process_scan(synth.lidar_scan(sc, poses[0], seed=0), wide, wide, 0.1, 20, 3.0, 1.0, 0)
    _, (sx, sn) = O.process_scan(synth.lidar_scan(sc, poses[1], seed=1), wide, wide, 0.1, 20, 3.0, 0.3, 7)
    init1 = np.linalg.inv(poses[0]) @ poses[1] @ synth.se3(0.0, 0.0, np.deg2rad(1.0), (0.1, -0.05, 0.0))
    reg.max_iteration_ = 7
    batch = reg.registerCloudsBatch([eng.cloud(src), eng.cloud(sx)], [tcloud, eng.cloud(mx, mn)], [np.eye(4), init1])
    refs = [O.registration_icp_p2point(src, tgt, 1.0, np.eye(4), max_iter=7), O.registration_icp_p2point(sx, mx, 1.0, init1, max_iter=7)]
    for b, ref in zip(batch, refs):
        assert b.iters == ref.iters and b.n_corr == ref.n_corr
        assert rel_rot(b.transformation_, ref.T) < 1e-8 and rel_trans(b.transformation_, ref.T) < 1e-8
    # the plane estimator still refuses a target without normals on the same engine
    with pytest.raises(L.B2SError) as ei:
        E.RegistrationIcpPointToPlane(eng).registerClouds(eng.cloud(src), tcloud, np.eye(4))
    assert ei.value.code == L.E_NO_NORMALS


def test_icp_properties_permutation_and_rigid_invariance(engine_factory):
    """SURVEY 8c test 7 on the device: the result does not depend on the order of the points (the grid index re-orders the
    target, the cluster splits the source) and is covariant under a common rigid motion of source, target and guess."""
    rng = np.random.default_rng(31)
    src, tgt, nrm, _ = synth.planar_cloud_config1(noise=0.01)
    p = lua_params()
    p.icp.maxCorrespondenceDistance = 0.8
    eng = engine_factory(p)
    reg = E.RegistrationIcpPointToPlane(eng)
    init = synth.se3(0.005, -0.01, 0.01, (0.02, 0.01, -0.01))
    base = reg.registerClouds(eng.cloud(src), eng.cloud(tgt, nrm), init)
    assert 0.0 <= base.fitness_ <= 1.0 and base.inlier_rmse_ <= 0.8
    ps, pt = rng.permutation(len(src)), rng.permutation(len(tgt))
    perm = reg.registerClouds(eng.cloud(src[ps]), eng.cloud(tgt[pt], nrm[pt]), init)
    assert perm.iters == base.iters and perm.n_corr == base.n_corr
    assert np.abs(perm.transformation_ - base.transformation_).max() < 1e-9
    G = synth.se3(0.3, -0.2, 1.1, (4.0, -7.0, 2.5))                    # common rigid motion
    R = G[:3, :3]
    moved = reg.registerClouds(eng.cloud(src @ R.T + G[:3, 3]), eng.cloud(tgt @ R.T + G[:3, 3], nrm @ R.T), G @ init @ np.linalg.inv(G))
    assert moved.n_corr == base.n_corr and abs(moved.inlier_rmse_ - base.inlier_rmse_) < 1e-9
    assert np.abs(moved.transformation_ - G @ base.transformation_ @ np.linalg.inv(G)).max() < 1e-7


def test_generalized_icp_matches_oracle(engine_factory):
    """R1'' (SURVEY 8f rank 3, second half): RegistrationIcpGeneralized -- [O3D] RegistrationGeneralizedICP with the
    covariances derived from the normals (what the reference's estimateNormalsOrCovariancesIfNeeded leaves on the clouds)."""
    src, tgt, nrm, T_true = synth.planar_cloud_config1(noise=0.01)
    snrm = O.estimate_normals(src, 10, 2.0)
    p = lua_params()
    p.icp.maxCorrespondenceDistance = 1.0
    p.icp.maxNumIter = 30
    eng = engine_factory(p)
    reg = E.cloudRegistrationFactory(eng, E.CloudRegistrationParameters(regType="GeneralizedIcp", icp=p.icp))
    assert isinstance(reg, E.RegistrationIcpGeneralized)
    tcloud = eng.cloud(tgt, nrm)
    for init in (np.eye(4), synth.se3(0.01, -0.02, 0.03, (0.05, 0.02, -0.01))):
        res = reg.registerClouds(eng.cloud(src, snrm), tcloud, init)
        ref = O.registration_gicp(src, snrm, tgt, nrm, 1.0, init, max_iter=30)
        assert res.iters == ref.iters and res.n_corr == ref.n_corr
        assert abs(res.fitness_ - ref.fitness) < 1e-12 and abs(res.inlier_rmse_ - ref.inlier_rmse) < 1e-9
        assert rel_rot(res.transformation_, ref.T) < 1e-8 and rel_trans(res.transformation_, ref.T) < 1e-8
    # a scan against a submap-sized target, batched with the small pair, iteration cap 6
    sc = synth.Scene(); poses = synth.loop_trajectory(600)
    wide = O.cropper("MinMaxRadius", 2.0, 30.0)
    (mx, mn), _ = O.process_scan(synth.lidar_scan(sc, poses[0], seed=0), wide, wide, 0.1, 20, 3.0, 1.0, 0)
    _, (sx, sn) = O.process_scan(synth.lidar_scan(sc, poses[1], seed=1), wide, wide, 0.1, 20, 3.0, 0.3, 7)
    init1 = np.linalg.inv(poses[0]) @ poses[1] @ synth.se3(0.0, 0.0, np.deg2rad(1.0), (0.1, -0.05, 0.0))
    reg.max_iteration_ = 6
    batch = reg.registerCloudsBatch([eng.cloud(src, snrm), eng.cloud(sx, sn)], [tcloud, eng.cloud(mx, mn)], [np.eye(4), init1])
    refs = [O.registration_gicp(src, snrm, tgt, nrm, 1.0, np.eye(4), max_iter=6), O.registration_gicp(sx, sn, mx, mn, 1.0, init1, max_iter=6)]
    for b, ref in zip(batch, refs):
        assert b.iters == ref.iters and b.n_corr == ref.n_corr
        assert rel_rot(b.transformation_, ref.T) < 1e-8 and rel_trans(b.transformation_, ref.T) < 1e-8
    with pytest.raises(L.B2SError) as ei:                       # covariances come from normals: both clouds need them
        reg.registerClouds(eng.cloud(src), tcloud, np.eye(4))
    assert ei.value.code == L.E_NO_NORMALS


def test_edge_cases_empty_inputs_and_capacity(engine_factory):
    """Empty and overflowing inputs: the reference's asserts become error codes, everything else degrades like [O3D]."""
    src, tgt, nrm, _ = synth.planar_cloud_config1()
    p = lua_params()
    eng = engine_factory(p)
    empty = eng.cloud(np.zeros((0, 3)))
    assert len(E.voxelize(eng, empty, 0.1)) == 0
    assert len(E.random_down_sample(eng, empty, 0.5, 1)) == 0
    assert len(E.transform(eng, synth.se3(0.1, 0, 0, (1, 2, 3)), empty)) == 0
    assert len(E.crop(eng, empty, E.ScanCroppingParameters().to_c())) == 0
    L.check(L.lib().b2s_estimate_normals(eng._h, empty._c, 20, C.c_double(3.0)))       # no points: nothing to do, no error
    reg = E.RegistrationIcpPointToPlane(eng)
    # empty source: no correspondences -> identity updates, fitness 0, one iteration until the criteria see 0 == 0
    r = reg.registerClouds(empty, eng.cloud(tgt, nrm), np.eye(4))
    ref = O.registration_icp_p2plane(np.zeros((0, 3)), tgt, nrm, 1.0, np.eye(4), max_iter=50)
    assert (r.iters, r.n_corr, r.fitness_, r.inlier_rmse_) == (ref.iters, 0, 0.0, 0.0) and np.array_equal(r.transformation_, np.eye(4))
    # empty target (with a normals array of length 0): same outcome, the initial guess comes back untouched
    init = synth.se3(0.0, 0.0, 0.1, (1.0, 0.0, 0.0))
    r = reg.registerClouds(eng.cloud(src), eng.cloud(np.zeros((0, 3)), np.zeros((0, 3))), init)
    assert r.n_corr == 0 and r.fitness_ == 0.0 and np.array_equal(r.transformation_, init)
    # everything cropped away: ScanToMapIcp's assert_gt(cropped size, 0)  (ScanToMapRegistration.cpp:51-52)
    far = eng.cloud(np.array([[100.0, 0, 0], [0, 120.0, 1.0], [90.0, 90.0, 0.0]]))
    with pytest.raises(L.B2SError) as ei:
        E.ScanToMapIcp(eng).processForScanMatchingAndMerging(far)
    assert ei.value.code == L.E_EMPTY
    # a submap that cannot hold the scan answers B2S_E_CAPACITY instead of writing out of bounds
    sc = synth.Scene(); poses = synth.loop_trajectory(4)
    ps = E.ScanToMapIcp(eng).processForScanMatchingAndMerging(eng.cloud(synth.lidar_scan(sc, poses[0], seed=0).astype(np.float64)))
    small = E.Submap(eng, 2000)
    with pytest.raises(L.B2SError) as ei:
        small.insertScan(None, ps.merge_, np.eye(4))
        small.size()      # only NEW voxels take slots, so the overflow is detected on the device and raised at the next synchronising call
    assert ei.value.code == L.E_CAPACITY
    # invalid parameters are refused like the reference's asserts (CloudRegistration.cpp:50-51, [O3D] r <= 0)
    with pytest.raises(L.B2SError):
        L.check(L.lib().b2s_estimate_normals(eng._h, eng.cloud(src)._c, 0, C.c_double(3.0)))
    bad = lua_params(); bad.icp.maxCorrespondenceDistance = 0.0
    with pytest.raises(L.B2SError) as ei:
        E.RegistrationIcpPointToPlane(engine_factory(bad)).registerClouds(eng.cloud(src), eng.cloud(tgt, nrm), np.eye(4))
    assert ei.value.code == L.E_INVALID


def test_loop_closure_overlap_and_information_matrix(engine_factory):
    """L1 (SURVEY 8f rank 2): overlap selection -> ICP on the overlap -> information matrix, the sequence of
    PlaceRecognition::buildLoopClosureConstraints (src/PlaceRecognition.cpp:103-148) on two oracle-built submaps."""
    sc = synth.Scene(); poses = synth.loop_trajectory(600)
    wide = O.cropper("MinMaxRadius", 2.0, 30.0)
    subs = []
    for k0 in (0, 8):                       # two submaps 4 m apart
        mx = np.zeros((0, 3)); mn = np.zeros((0, 3))
        for k in range(k0, k0 + 3):
            (ax, an), _ = O.process_scan(synth.lidar_scan(sc, poses[k], seed=k), wide, wide, 0.1, 20, 3.0, 1.0, 0)
            mx, mn = O.submap_insert_scan(mx, mn, ax, an, poses[k], 0.1, O.cropper("MaxRadius", 0.0, 20.0, center=tuple(poses[k][:3, 3])))
        subs.append((mx, mn))
    (sx, sn), (tx, tn) = subs
    guess = synth.se3(0.0, 0.0, np.deg2rad(0.8), (0.08, -0.05, 0.02))          # stands in for the RANSAC result
    p = lua_params()
    p.icp.maxCorrespondenceDistance = 0.3
    p.icp.maxNumIter = 100
    eng = engine_factory(p)
    src, tgt = eng.cloud(sx, sn), eng.cloud(tx, tn)
    for voxel, m in ((0.3, 1), (0.5, 4)):                                        # 3 x map voxel, minNumPointsPerVoxel = 1 is the reference's call
        so, to = E.computeOverlappingClouds(eng, src, tgt, guess, voxel, m)
        fs, ft = O.overlap_flags(sx, tx, guess, voxel, m)
        gsx, gsn = so.download(); gtx, gtn = to.download()
        assert 0 < fs.sum() < len(sx) and 0 < ft.sum() < len(tx)
        assert np.array_equal(gsx, sx[fs]) and np.array_equal(gsn, sn[fs]) and np.array_equal(gtx, tx[ft]) and np.array_equal(gtn, tn[ft])
    so, to = E.computeOverlappingClouds(eng, src, tgt, guess, 0.3, 1)
    fs, ft = O.overlap_flags(sx, tx, guess, 0.3, 1)
    res = E.RegistrationIcpPointToPlane(eng).registerClouds(so, to, guess)
    ref = O.registration_icp_p2plane(sx[fs], tx[ft], tn[ft], 0.3, guess, max_iter=100)
    assert res.iters == ref.iters and res.n_corr == ref.n_corr and np.abs(res.transformation_ - ref.T).max() < 1e-8
    G = E.getInformationMatrixFromPointClouds(eng, so, to, 0.3, ref.T)      # the same transformation on both sides
    Gref = O.information_matrix(sx[fs], tx[ft], 0.3, ref.T)
    assert G[3, 3] == Gref[3, 3] > 1000 and np.abs(G - Gref).max() < 1e-9 * np.abs(Gref).max()
    assert np.array_equal(G, G.T)
    # identity transformation: [O3D] skips the Transform (isIdentity) -- same matrix as with an explicit identity
    G0 = E.getInformationMatrixFromPointClouds(eng, so, to, 0.3, np.eye(4))
    assert np.abs(G0 - O.information_matrix(sx[fs], tx[ft], 0.3, np.eye(4))).max() < 1e-9 * np.abs(Gref).max()
    with pytest.raises(L.B2SError):
        E.computeOverlappingClouds(eng, src, tgt, guess, 0.3, 0)


def test_dense_map_carving_matches_oracle(engine_factory):
    """C2: Submap::carve on the dense map -- first-point-per-voxel ray set, neighbourhood enumeration with the reference's
    floating loops, removal of every nominated voxel that exists.  Same surviving voxel set and sums as the oracle."""
    p = lua_params()
    eng = engine_factory(p)
    sc = synth.Scene(); poses = synth.loop_trajectory(8)
    sm = E.Submap(eng, 10_000)
    dm = O.DenseMap(0.05, 1 << 21)
    cp = E.ScanCroppingParameters("MaxRadius", 0.0, 15.0)
    for k in range(2):
        raw = synth.lidar_scan(sc, poses[k], seed=k).astype(np.float64)
        sm.insertScanDenseMap(eng.cloud(raw), poses[k], cp.to_c())
        kept, _ = O.crop(O.cropper("MaxRadius", 0.0, 15.0), raw)
        dm.insert(O.transform(poses[k], kept)[0])
    clutter = np.random.default_rng(1).uniform([-4, -4, -1], [4, 4, 1], (3000, 3))
    Tc = synth.se3(0.0, 0.0, 0.2, (0.5, -0.3, 0.1))                  # floating clutter in free space, to be carved
    sm.insertScanDenseMap(eng.cloud(clutter), Tc, None)
    dm.insert(O.transform(Tc, clutter)[0])
    n0 = sm.denseSize()
    raw = synth.lidar_scan(sc, poses[2], seed=2).astype(np.float64)[::4]
    scan = raw @ poses[2][:3, :3].T + poses[2][:3, 3]
    prm = E.SpaceCarvingParameters(maxRaytracingLength=20.0, truncationDistance=0.3, neighborhoodRadiusDenseMap=0.1)
    removed = sm.carveDenseMap(eng.cloud(scan), poses[2][:3, 3], prm)
    ref_removed = dm.carve(scan, poses[2][:3, 3], 0.05, 0.1, 0.3, 20.0)
    assert removed == ref_removed and 0 < removed < n0
    gx, gk = sm.getDenseMap(); rx, _rn, rk = dm.to_cloud()
    o1 = np.lexsort((gk[:, 2], gk[:, 1], gk[:, 0])); o2 = np.lexsort((rk[:, 2], rk[:, 1], rk[:, 0]))
    assert np.array_equal(gk[o1], rk[o2]) and np.abs(gx[o1] - rx[o2]).max() < 1e-12
    assert sm.denseSize() == n0 - removed


def test_constant_velocity_deskew_matches_oracle(engine_factory):
    """D1 (SURVEY 8f rank 4): undistortInputPointCloud on a full 64x1024 scan, float32 wire input, both spin directions."""
    sc = synth.Scene(); poses = synth.loop_trajectory(8)
    raw32 = np.ascontiguousarray(synth.lidar_scan(sc, poses[2], seed=2))
    raw = raw32.astype(np.float64)
    raw[0] = [3.0, 0.0, 1.0]                                   # azimuth exactly 0 -> phase 0 -> untouched
    eng = engine_factory(lua_params())
    lv, av = E.ConstantVelocityMotionCompensation.estimateLinearAndAngularVelocity(poses[0], poses[2], 0.2)
    assert abs(np.linalg.norm(lv) - 5.0) < 0.1                 # the synthetic trajectory moves 0.5 m per 0.1 s scan
    av = av + np.array([0.03, -0.02, 0.4])                     # some rotation too
    for cw in (True, False):
        mc = E.ConstantVelocityMotionCompensation(eng, isSpinningClockwise=cw, scanDuration=0.1)
        out, _ = mc.undistortInputPointCloud(eng.cloud(raw), lv, av).download()
        ref = O.undistort(raw, lv, av, 0.1, cw)
        assert out.shape == ref.shape and np.abs(out - ref).max() < 1e-12     # libm (atan2, sincos) is the only difference
        assert np.array_equal(out[0], raw[0])
        assert 0.05 < np.abs(out - raw).max() < 10.0           # it actually moved points (translation + lever arm of the rotation)
    zero = E.ConstantVelocityMotionCompensation(eng).undistortInputPointCloud(eng.cloud(raw), np.zeros(3), np.zeros(3)).download()[0]
    assert np.array_equal(zero, raw)
    with pytest.raises(RuntimeError):
        E.ConstantVelocityMotionCompensation(eng, scanDuration=0.0)


def _carving_case():
    """A three-scan oracle submap plus floating clutter in free space, and the next raw scan with its pose."""
    sc = synth.Scene(); poses = synth.loop_trajectory(600)
    wide = O.cropper("MinMaxRadius", 2.0, 30.0)
    mx = np.zeros((0, 3)); mn = np.zeros((0, 3))
    for k in range(3):
        (ax, an), _ = O.process_scan(synth.lidar_scan(sc, poses[k], seed=k), wide, wide, 0.1, 20, 3.0, 1.0, 0)
        mx, mn = O.submap_insert_scan(mx, mn, ax, an, poses[k], 0.1, O.cropper("MaxRadius", 0.0, 20.0, center=tuple(poses[k][:3, 3])))
    rng = np.random.default_rng(0)
    clutter = rng.uniform([-6, -6, -1.5], [6, 6, 1.5], (800, 3)); cn = rng.normal(size=(800, 3))
    cn[:50] = 0.0                                    # zero normals: normalized() leaves them, |dir . 0| = 0 never exceeds the threshold
    return np.vstack([mx, clutter]), np.vstack([mn, cn]), synth.lidar_scan(sc, poses[3], seed=3).astype(np.float64), poses[3], poses[2]


@pytest.mark.parametrize("voxel,min_dot,trunc", [(0.1, 0.5, 0.1), (0.25, 0.2, 0.5)])
def test_space_carving_matches_oracle(engine_factory, voxel, min_dot, trunc):
    """C1 (SURVEY 8f rank 1): Submap::carve -> getIdxsOfCarvedPoints; the surviving map must be the oracle's, in order, bit-exact."""
    mx, mn, raw, T, Tprev = _carving_case()
    p = lua_params()
    p.mapBuilder.cropper = E.ScanCroppingParameters(cropperName="MaxRadius", croppingMaxRadius=20.0)
    p.mapBuilder.carving = E.SpaceCarvingParameters(voxelSize=voxel, maxRaytracingLength=20.0, truncationDistance=trunc, minDotProductWithNormal=min_dot)
    eng = engine_factory(p)
    sm = E.Submap(eng, 400_000)
    sm.setMapPointCloud(eng.cloud(mx, mn))
    sm._cropperPose = Tprev                       # mapBuilderCropper_ still sits at the previous insertion (Submap.cpp:59 vs :71)
    n_removed = sm.carve(eng.cloud(raw), T, p.mapBuilder.carving, force=True)
    scan_map, _ = O.transform(T, raw)
    rem = O.carve(mx, mn, scan_map, T[:3, 3], O.cropper("MaxRadius", 0.0, 20.0, center=tuple(Tprev[:3, 3])), voxel, 20.0, trunc, min_dot)
    assert 0 < rem.sum() < len(mx) and rem[len(mx) - 800:].sum() > 0
    assert n_removed == int(rem.sum())
    gx, gn = sm.getMapPointCloud()
    assert np.array_equal(gx, mx[~rem]) and np.array_equal(gn, mn[~rem])


def test_insert_scan_with_carving_schedule(engine_factory):
    """Submap.insertScan(isPerformCarving=True) carves only when nScansInsertedMap_ % carveSpaceEveryNscans_ == 1."""
    p = lua_params()
    p.mapBuilder.carving.carveSpaceEveryNscans = 2
    eng = engine_factory(p)
    icp = E.ScanToMapIcp(eng)
    sc = synth.Scene(); poses = synth.loop_trajectory(8)
    sm = E.Submap(eng, 400_000)
    carved = []
    for k in range(4):
        raw = eng.cloud(synth.lidar_scan(sc, poses[k], seed=k).astype(np.float64))
        ps = icp.processForScanMatchingAndMerging(raw)
        sm.lastCarvedCount = -1
        sm.insertScan(raw, ps.merge_, poses[k], isPerformCarving=True)
        carved.append(sm.lastCarvedCount)
    assert carved[0] == -1 and carved[2] == -1          # 0 % 2, 2 % 2 != 1: skipped
    assert carved[1] >= 0 and carved[3] >= 0            # 1 % 2 == 1, 3 % 2 == 1: carved
    assert sm.size() > 0


def test_dense_map_running_sums(engine_factory):
    p = lua_params()
    eng = engine_factory(p)
    sc = synth.Scene(); poses = synth.loop_trajectory(4)
    sm = E.Submap(eng, 10_000)
    dm = O.DenseMap(0.05, 1 << 20)
    cp = E.ScanCroppingParameters("MaxRadius", 0.0, 15.0)
    for k in range(3):
        raw = synth.lidar_scan(sc, poses[k], seed=k).astype(np.float64)
        sm.insertScanDenseMap(eng.cloud(raw), poses[k], cp.to_c())
        kept, _ = O.crop(O.cropper("MaxRadius", 0.0, 15.0), raw)
        tx, _ = O.transform(poses[k], kept)
        dm.insert(tx)
    gx, gk = sm.getDenseMap()
    rx, _rn, rk = dm.to_cloud()
    assert len(gx) == len(rx)
    o1 = np.lexsort((gk[:, 2], gk[:, 1], gk[:, 0])); o2 = np.lexsort((rk[:, 2], rk[:, 1], rk[:, 0]))
    assert np.array_equal(gk[o1], rk[o2])
    assert np.abs(gx[o1] - rx[o2]).max() < 1e-12      # atomics change the summation order, not the members
    # F2: the VoxelHashMap query interface, batched -- has / content / remove / size / clear against the oracle's voxel set
    assert sm.denseSize() == len(rx)
    table = {tuple(k): x for k, x in zip(rk, rx)}
    rng = np.random.default_rng(9)
    q = np.vstack([rx[::7] + rng.uniform(-0.02, 0.02, (len(rx[::7]), 3)), rng.uniform(-30, 30, (2000, 3))])
    counts, means = sm.denseQuery(eng.cloud(q))
    keys = np.floor(q * (1.0 / 0.05)).astype(np.int64)
    has = np.array([tuple(k) in table for k in keys])
    assert np.array_equal(counts > 0, has) and has.sum() > 1000 and (~has).sum() > 1000
    exp = np.array([table[tuple(k)] if h else np.zeros(3) for k, h in zip(keys, has)])
    assert np.abs(means - exp).max() < 1e-12
    victims = q[has][::3]
    sm.denseRemove(eng.cloud(victims))
    gone = {tuple(k) for k in np.floor(victims * (1.0 / 0.05)).astype(np.int64)}
    assert sm.denseSize() == len(rx) - len(gone)
    counts2, _ = sm.denseQuery(eng.cloud(q), with_means=False)
    assert np.array_equal(counts2 > 0, np.array([h and tuple(k) not in gone for k, h in zip(keys, has)]))
    gx2, gk2 = sm.getDenseMap()
    assert {tuple(k) for k in gk2} == set(table) - gone
    sm.insertScanDenseMap(eng.cloud(raw), poses[2], cp.to_c())          # removed voxels can be populated again
    assert sm.denseSize() > len(rx) - len(gone)
    sm.denseClear()
    assert sm.denseSize() == 0 and len(sm.getDenseMap()[0]) == 0


def test_device_against_committed_golden_fixtures(engine_factory):
    """The CUDA path against tests/golden/*.npz directly (no oracle call): config-1 ICP, scan pre-processing, two-scan fusion
    and the "next" rows.  The fixtures are written by tests/golden/make_golden.py."""
    import os
    from scipy.spatial import cKDTree
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    # config 1
    g = np.load(os.path.join(gold, "config1_icp.npz"))
    p = lua_params(); p.icp.maxCorrespondenceDistance = 1.0; p.icp.maxNumIter = 50
    eng = engine_factory(p)
    for tag, noise in (("clean", 0.0), ("noisy", 0.01)):
        src, tgt, nrm, _ = synth.planar_cloud_config1(noise=noise)
        r = E.RegistrationIcpPointToPlane(eng).registerClouds(eng.cloud(src), eng.cloud(tgt, nrm), np.eye(4))
        assert r.iters == int(g[f"{tag}_iters"]) and r.n_corr == int(g[f"{tag}_ncorr"])
        assert np.abs(r.transformation_ - g[f"{tag}_T"]).max() < 1e-9 and abs(r.inlier_rmse_ - float(g[f"{tag}_rmse"])) < 1e-10
    # scan pre-processing (16 x 512 scan stored in the fixture)
    g = np.load(os.path.join(gold, "scan_preprocess.npz"))
    p2 = lua_params(seed=5); p2.scanProcessing.downSamplingRatio = 0.3
    p2.scanProcessing.cropper = E.ScanCroppingParameters("MinMaxRadius", 2.0, 25.0)
    e2 = engine_factory(p2)
    raw = g["raw"].astype(np.float64)
    vx, _ = E.voxelize(e2, e2.cloud(raw), 0.1).download()
    o = np.lexsort(vx.T[::-1]); og = np.lexsort(g["voxel_means"].T[::-1])
    assert np.array_equal(vx[o], g["voxel_means"][og])
    ps = E.ScanToMapIcp(e2).processForScanMatchingAndMerging(e2.cloud(raw))
    for got, (rx, rn) in ((ps.merge_, (g["merge_xyz"], g["merge_nrm"])), (ps.match_, (g["match_xyz"], g["match_nrm"]))):
        gx, gn = got.download()
        d, j = cKDTree(rx).query(gx)
        assert len(gx) == len(rx) and d.max() == 0.0 and len(np.unique(j)) == len(rx) and np.abs(gn - rn[j]).max() < 1e-8
    # fusion of two scans (first insertion with the identity: duplication quirk)
    g = np.load(os.path.join(gold, "fusion_two_scans.npz"))
    p3 = lua_params(); p3.scanProcessing.downSamplingRatio = 1.0
    e3 = engine_factory(p3)
    scene = synth.Scene(); poses = synth.loop_trajectory(4)
    sm = E.Submap(e3, 200_000); s2m = E.ScanToMapIcp(e3)
    for k in range(2):
        raw = synth.lidar_scan(scene, poses[k], n_beams=16, n_az=512, seed=20 + k).astype(np.float64)
        sm.insertScan(None, s2m.processForScanMatchingAndMerging(e3.cloud(raw)).merge_, np.eye(4) if k == 0 else np.linalg.inv(poses[0]) @ poses[1])
    mx, mn = sm.getMapPointCloud()
    d, j = cKDTree(g["map_xyz"]).query(mx)
    # the identity insertion doubles every point (quirk): the voxel sums run over the same members in a different order -> last bit
    assert len(mx) == len(g["map_xyz"]) and d.max() < 1e-12 and len(np.unique(j)) == len(mx) and np.abs(mn - g["map_nrm"][j]).max() < 1e-8
    # "next" rows
    g = np.load(os.path.join(gold, "next_rows.npz"))
    src, tgt, nrm, _ = synth.planar_cloud_config1(n=800, noise=0.01)
    init = synth.se3(0.01, -0.02, 0.03, (0.05, 0.02, -0.01))
    p4 = lua_params(); p4.icp.maxCorrespondenceDistance = 1.0; p4.icp.maxNumIter = 50; p4.icp.knn = 10; p4.icp.maxDistanceKnn = 2.0
    e4 = engine_factory(p4)
    r = E.RegistrationIcpPointToPoint(e4).registerClouds(e4.cloud(src), e4.cloud(tgt), init)
    assert r.iters == int(g["p2p_iters"]) and r.n_corr == int(g["p2p_ncorr"]) and np.abs(r.transformation_ - g["p2p_T"]).max() < 1e-8
    gicp = E.RegistrationIcpGeneralized(e4); gicp.max_iteration_ = 30
    sc = e4.cloud(src); gicp.estimateNormalsOrCovariancesIfNeeded(sc)          # knn 10, radius 2.0 like the fixture's source normals
    r = gicp.registerClouds(sc, e4.cloud(tgt, nrm), init)
    assert r.iters == int(g["gicp_iters"]) and r.n_corr == int(g["gicp_ncorr"]) and np.abs(r.transformation_ - g["gicp_T"]).max() < 1e-7
    so, to = E.computeOverlappingClouds(e4, e4.cloud(src), e4.cloud(tgt), init, 0.5, 2)
    fs = np.unpackbits(g["overlap_src"])[:len(src)].astype(bool); ft = np.unpackbits(g["overlap_tgt"])[:len(tgt)].astype(bool)
    assert np.array_equal(so.download()[0], src[fs]) and np.array_equal(to.download()[0], tgt[ft])
    G = E.getInformationMatrixFromPointClouds(e4, e4.cloud(src), e4.cloud(tgt), 0.3, init)
    assert np.abs(G - g["info"]).max() < 1e-9 * np.abs(g["info"]).max()
    rng = np.random.default_rng(77)
    raw = rng.normal(size=(300, 3)); raw = raw / np.linalg.norm(raw, axis=1)[:, None] * rng.uniform(3, 9, (300, 1))   # sensor frame
    p5 = lua_params(); p5.mapBuilder.cropper = E.ScanCroppingParameters(cropperName="MaxRadius", croppingMaxRadius=8.0)
    e5 = engine_factory(p5)
    smc = E.Submap(e5, 10_000); smc.setMapPointCloud(e5.cloud(tgt, nrm))
    smc._cropperPose = synth.se3(t=(5.0, 5.0, 0.0))
    Ts = synth.se3(t=(5.0, 5.0, 1.0))                                            # sensor at (5, 5, 1)
    smc.carve(e5.cloud(raw), Ts, E.SpaceCarvingParameters(voxelSize=0.25, truncationDistance=0.1, minDotProductWithNormal=0.3), force=True)
    rem = np.unpackbits(g["carved"])[:len(tgt)].astype(bool)
    assert np.array_equal(smc.getMapPointCloud()[0], tgt[~rem])
    out = E.ConstantVelocityMotionCompensation(e5).undistortInputPointCloud(e5.cloud(src[:50]), [5.0, -0.4, 0.1], [0.02, -0.05, 0.8]).download()[0]
    assert np.abs(out - g["deskew"]).max() < 1e-12


def test_submap_transform_matches_oracle(engine_factory):
    """Submap::transform (src/Submap.cpp:94-107): [O3D] PointCloud::Transform of the map in place (no duplication quirk),
    VoxelizedPointCloud::transform of the dense map (sums moved, keys kept) and mapToRangeSensor_ * T."""
    eng = engine_factory(lua_params())
    sc = synth.Scene(); poses = synth.loop_trajectory(4)
    wide = O.cropper("MinMaxRadius", 2.0, 30.0)
    (mx, mn), _ = O.process_scan(synth.lidar_scan(sc, poses[0], seed=0), wide, wide, 0.1, 20, 3.0, 0.5, 1)
    sm = E.Submap(eng, 100_000)
    sm.setMapPointCloud(eng.cloud(mx, mn))
    sm.setPose(poses[1])
    raw = synth.lidar_scan(sc, poses[1], seed=1).astype(np.float64)[::8]
    sm.insertScanDenseMap(eng.cloud(raw), poses[1], None)
    dm = O.DenseMap(0.05, 1 << 18); dm.insert(O.transform(poses[1], raw)[0])
    for T in (synth.se3(0.01, -0.02, 0.3, (0.5, -0.25, 0.1)), np.eye(4) + 0.0):   # the identity must NOT duplicate anything here
        sm.transform(T)
        mx, mn = O.pointcloud_transform(T, mx, mn)
        dm.transform(T)
    gx, gn = sm.getMapPointCloud()
    assert np.array_equal(gx, mx) and np.array_equal(gn, mn)                      # same expressions, same order: bit-identical
    assert np.abs(sm.getPose() - poses[1] @ synth.se3(0.01, -0.02, 0.3, (0.5, -0.25, 0.1))).max() < 1e-12
    dx, dk = sm.getDenseMap(); rx, _rn, rk = dm.to_cloud()
    o1 = np.lexsort((dk[:, 2], dk[:, 1], dk[:, 0])); o2 = np.lexsort((rk[:, 2], rk[:, 1], rk[:, 0]))
    assert np.array_equal(dk[o1], rk[o2]) and np.abs(dx[o1] - rx[o2]).max() < 1e-9
