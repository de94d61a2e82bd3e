"""GPU: b2s_submap_loop_closure_refinement with the estimator the caller chooses (reg_type), as PlaceRecognition::
updateRegistrationAlgorithm (src/PlaceRecognition.cpp:44-48) takes the scan matcher's.  Generalized and point-to-point ICP against the
device composition (b2s_submap_to_cloud x 2 + b2s_overlap(T0) + b2s_register_batch of that type + b2s_information_matrix) and the
oracle, from the identity, a translation and a 30 deg yaw (the source covariances rotated by T0), K = 1 / 4 / 16 / 17 against single
calls; the normals rules, an unknown type, the default against an explicit point-to-plane, the odometry constraints after a
generalized refinement on the same handle, and slam.buildLoopClosureConstraints over the device and the oracle backends."""
import copy
import ctypes as C
import os

import numpy as np
import pytest

from oracle import oracle as O
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from test_gpu_loop_closure_refinement import GUESS, HERE, TRUTH, fields, odometry_records, refine, rel, source, submap, target
from test_loop_closure_host import P, collection, room
from test_ransac_oracle import rigid

pytestmark = pytest.mark.gpu

REGS = ["GeneralizedIcp", "PointToPointIcp"]


def prm(reg, **kw):
    return E.LoopClosureRefinementParameters(regType=reg, **kw)


def composed(eng, src, tgt, T0, p):
    """the device composition with the estimator of p: two map copies, b2s_overlap at T0, b2s_register_batch, b2s_information_matrix"""
    v = E.getMapVoxelSize(p.mapVoxelSize, p.voxelSizeIfMapVoxelSizeIsZero)
    params = eng.params
    sc, tc = src.toCloud(), tgt.toCloud()
    so, to = E.computeOverlappingClouds(eng, sc, tc, T0, p.voxelExpansionFactorOverlapComputation * v, p.minNumPointsPerVoxel)
    reg = E.cloudRegistrationFactory(eng, E.CloudRegistrationParameters(regType=p.regType, icp=E.IcpParameters(
        maxNumIter=p.maxNumIter, maxCorrespondenceDistance=p.maxIcpCorrespondenceDistance)))
    (r,) = reg.registerCloudsBatch([so], [to], [T0])
    eng.set_parameters(params)
    info = E.getInformationMatrixFromPointClouds(eng, so, to, p.maxIcpCorrespondenceDistance, r.transformation_)
    return so, to, r, info, not (r.fitness_ < p.minRefinementFitness)


def check_against_composition(eng, src, tgt, T0, g, so, to, p):
    """the bar of the point-to-plane tests: the same overlap sets, T / fitness / rmse within 1e-12, n_corr / iters equal, information"""
    cso, cto, r, info, acc = composed(eng, src, tgt, T0, p)
    for x, y in ((so, cso), (to, cto)):
        (xx, xn), (yx, yn) = x.download(), y.download()
        assert np.array_equal(xx, yx) and np.array_equal(xn, yn, equal_nan=True)
    assert (g.nSourceOverlap, g.nTargetOverlap) == (len(cso), len(cto))
    assert np.abs(g.result.transformation_ - r.transformation_).max() <= 1e-12
    assert abs(g.result.fitness_ - r.fitness_) <= 1e-12 and abs(g.result.inlier_rmse_ - r.inlier_rmse_) <= 1e-12
    assert (g.result.n_corr, g.result.iters, g.accepted) == (r.n_corr, r.iters, acc)
    assert rel(g.information, info) <= 1e-12


def oracle_icp(reg, sx, sn, tx, tn, T0, p):
    if reg == "GeneralizedIcp":
        return O.registration_gicp(sx, sn, tx, tn, p.maxIcpCorrespondenceDistance, T0, max_iter=p.maxNumIter)
    return O.registration_icp_p2point(sx, tx, p.maxIcpCorrespondenceDistance, T0, max_iter=p.maxNumIter)


@pytest.mark.parametrize("reg", REGS)
@pytest.mark.parametrize("kind", ["identity", "translation", "yaw30"])
def test_against_device_composition_and_oracle(engine_factory, reg, kind):
    eng = engine_factory()
    p = prm(reg)
    src, tgt = source(eng), target(eng, kind)
    T0 = GUESS[kind]
    (g,), (so,), (to,) = refine(eng, src, [tgt], [T0], p, overlaps=True)
    assert g.accepted and g.nSourceOverlap > 3000
    check_against_composition(eng, src, tgt, T0, g, so, to, p)
    # the oracle on the device's maps: the overlap sets in order, the registration of that type from T0 (the generalized one rotates
    # the source covariances by T0 first), the information matrix at the device's T
    (sx, sn), (tx, tn) = src.getMapPointCloud(), tgt.getMapPointCloud()
    fs, ft = O.overlap_flags(sx, tx, T0, p.voxelExpansionFactorOverlapComputation * p.mapVoxelSize, p.minNumPointsPerVoxel)
    assert np.array_equal(so.download()[0], sx[fs]) and np.array_equal(to.download()[0], tx[ft])
    ref = oracle_icp(reg, sx[fs], sn[fs], tx[ft], tn[ft], T0, p)
    assert np.abs(g.result.transformation_ - ref.T).max() < 1e-8 and g.result.n_corr == ref.n_corr
    assert rel(g.information, O.information_matrix(sx[fs], tx[ft], p.maxIcpCorrespondenceDistance, g.result.transformation_)) < 1e-9
    assert np.abs(g.result.transformation_ - TRUTH[kind]).max() < 0.02
    # another estimator, another refinement
    (d,) = refine(eng, src, [tgt], [T0])
    assert not np.array_equal(d.result.transformation_, g.result.transformation_)


@pytest.mark.parametrize("reg", REGS)
@pytest.mark.parametrize("K", [1, 4, 16, 17])
def test_k_targets_equal_single_calls(engine_factory, reg, K):
    eng = engine_factory()
    p = prm(reg)
    src = source(eng)
    kinds = list(TRUTH)
    tgts = [target(eng, kinds[k % 3], seed=1 + k, parts=3 if k % 5 == 4 else 5) for k in range(K)]
    inits = [GUESS[kinds[k % 3]] for k in range(K)]
    res, so, to = refine(eng, src, tgts, inits, p, overlaps=True)
    again = refine(eng, src, tgts, inits, p)
    singles = [refine(eng, src, [t], [T0], p)[0] for t, T0 in zip(tgts, inits)]
    assert [fields(r) for r in res] == [fields(r) for r in again] == [fields(r) for r in singles]
    for k in (0, K // 2, K - 1):
        check_against_composition(eng, src, tgts[k], inits[k], res[k], so[k], to[k], p)


@pytest.mark.parametrize("reg", REGS)
def test_same_target_twice_and_empty_overlap(engine_factory, reg):
    eng = engine_factory()
    p = prm(reg)
    src, a = source(eng), target(eng, "yaw30")
    far = submap(eng, *(lambda x, n: (x + [0.0, 0.0, 100.0], n))(*room(3)))
    res = refine(eng, src, [a, far, a], [GUESS["yaw30"], GUESS["translation"], GUESS["yaw30"]], p)
    assert fields(res[0]) == fields(res[2]) and res[0].accepted
    assert (res[1].nSourceOverlap, res[1].nTargetOverlap, res[1].result.fitness_, res[1].accepted) == (0, 0, 0.0, False)
    assert not res[1].information.any()


def code(fn):
    with pytest.raises(L.B2SError) as e:
        fn()
    return e.value.code


def test_point_to_point_needs_no_normals(engine_factory):
    """a point-to-point mapper's maps carry no normals (stored as NaN): PointToPointIcp refines them, as source and as target, and
    equals the composition and the oracle"""
    eng = engine_factory(E.MapperParameters(scanToMapRegType="PointToPointIcp"))
    p = prm("PointToPointIcp")
    T0 = GUESS["yaw30"]
    x, _ = room(1)
    tx = x @ TRUTH["yaw30"][:3, :3].T + TRUTH["yaw30"][:3, 3]
    bare_src, bare_tgt = E.Submap(eng, 16384), E.Submap(eng, 16384)
    bare_src.setMapPointCloud(eng.cloud(room(0)[0]))
    bare_tgt.setMapPointCloud(eng.cloud(tx))
    assert code(lambda: refine(eng, source(eng), [bare_tgt], [T0])) == L.E_NO_NORMALS   # point-to-plane still needs them
    for src, tgt in ((source(eng), bare_tgt), (bare_src, bare_tgt), (bare_src, target(eng, "yaw30"))):
        (g,), (so,), (to,) = refine(eng, src, [tgt], [T0], p, overlaps=True)
        assert g.accepted
        check_against_composition(eng, src, tgt, T0, g, so, to, p)
        (sx, _), (tgx, _) = src.getMapPointCloud(), tgt.getMapPointCloud()
        fs, ft = O.overlap_flags(sx, tgx, T0, p.voxelExpansionFactorOverlapComputation * p.mapVoxelSize, p.minNumPointsPerVoxel)
        ref = O.registration_icp_p2point(sx[fs], tgx[ft], p.maxIcpCorrespondenceDistance, T0, max_iter=p.maxNumIter)
        assert np.abs(g.result.transformation_ - ref.T).max() < 1e-8 and g.result.n_corr == ref.n_corr


def test_generalized_needs_normals_on_both_sides(engine_factory):
    eng = engine_factory(E.MapperParameters(scanToMapRegType="PointToPointIcp"))
    p = prm("GeneralizedIcp")
    bare = E.Submap(eng, 16384)
    bare.setMapPointCloud(eng.cloud(room(1)[0]))
    I = [np.eye(4)]
    assert code(lambda: refine(eng, bare, [source(eng)], I, p)) == L.E_NO_NORMALS   # the source
    assert code(lambda: refine(eng, source(eng), [bare], I, p)) == L.E_NO_NORMALS   # a target
    assert code(lambda: refine(eng, source(eng), [target(eng, "identity"), bare], I * 2, p)) == L.E_NO_NORMALS
    refine(eng, bare, [source(eng)], I)   # point-to-plane: a source without normals is fine


def raw_call(eng, src, tgt, T0, c_params):
    out = (L.LoopClosureRefinement * 1)()
    T = np.ascontiguousarray(np.asarray(T0, dtype=np.float64).reshape(16))
    rc = L.lib().b2s_submap_loop_closure_refinement(eng._h, src._s, C.c_int32(1), (C.c_void_p * 1)(tgt._s), E._pd(T), C.byref(c_params),
                                                    None, None, out)
    return rc, bytes(out)


def test_unknown_type_and_explicit_point_to_plane(engine_factory):
    eng = engine_factory()
    src, tgt = source(eng), target(eng, "yaw30")
    T0 = GUESS["yaw30"]
    d = L.LoopClosureRefinementParams()
    L.lib().b2s_default_loop_closure_refinement_params(C.byref(d))
    assert d.reg_type == L.REG_POINT_TO_PLANE
    rc_d, out_d = raw_call(eng, src, tgt, T0, d)
    e = E.LoopClosureRefinementParameters(regType="PointToPlaneIcp").to_c()
    rc_e, out_e = raw_call(eng, src, tgt, T0, e)
    assert rc_d == rc_e == L.OK and out_d == out_e   # bit for bit
    bad = L.LoopClosureRefinementParams()
    L.lib().b2s_default_loop_closure_refinement_params(C.byref(bad))
    bad.reg_type = 99
    assert raw_call(eng, src, tgt, T0, bad)[0] == L.E_UNSUPPORTED
    assert b"registration type" in L.lib().b2s_last_error()
    assert code(lambda: refine(eng, src, [tgt], [T0], prm("Ndt"))) == L.E_UNSUPPORTED


def test_odometry_constraints_unchanged_after_a_generalized_refinement(engine_factory):
    """b2s_submap_odometry_constraints on the handle that just refined with GeneralizedIcp: every record bit for bit as before it, and
    as the library recorded them before the driver was shared"""
    eng = engine_factory()
    before = odometry_records(eng)
    src, tgt = source(eng), target(eng, "yaw30")
    (g,) = refine(eng, src, [tgt], [GUESS["yaw30"]], prm("GeneralizedIcp"))
    assert g.accepted
    after = odometry_records(eng)
    ref = np.load(os.path.join(HERE, "golden", "odometry_constraints_records.npz"))
    assert sorted(before) == sorted(after) == sorted(ref.files)
    for k in ref.files:
        assert np.array_equal(before[k], after[k]) and np.array_equal(after[k], ref[k]), k


@pytest.mark.parametrize("reg", REGS)
def test_build_loop_closure_constraints_device_and_oracle_backends(reg):
    """slam.buildLoopClosureConstraints with LoopClosureParameters.fromMapperParameters on the room scene (the target map another
    sample of the room, so the estimators differ): the device backend (one batched call) and the oracle backend (its composition)
    give the same decisions and constraints; the device's per-cloud composition of refineLoopClosures gives the same records"""
    from oracle_backend import OracleSubmap
    from oracle_backend_estimators import EstimatorOracleBackend
    mp = E.MapperParameters(scanToMapRegType=reg)
    lc = S.LoopClosureParameters.fromMapperParameters(mp)
    T = rigid(0.4, [3.0, -1.5, 0.2], 0.02, -0.01)
    ora, co = collection(T)
    ora.__class__ = EstimatorOracleBackend
    x, n = room(1)
    co.submaps[1].handle.xyz, co.submaps[1].handle.nrm = x @ T[:3, :3].T + T[:3, 3], n @ T[:3, :3].T
    dev = S.DeviceBackend(copy.deepcopy(mp), carving=False, dense=False, graph=False)
    eng = dev.eng
    cd = S.SubmapCollection(dev, S.SubmapParameters())
    for k, q in enumerate(co.submaps):
        sm = submap(eng, q.handle.xyz, q.handle.nrm)
        r = S.SubmapRecord(sm, k, 0, np.zeros(3))
        r.sparse, r.feature = eng.cloud(q.sparse.xyz), E.Feature(eng, np.asarray(q.feature, dtype=np.float64).reshape(-1, 33).T)
        cd.submaps.append(r)
        om = OracleSubmap(None)
        om.xyz, om.nrm = dev.map_cloud(sm)   # the oracle reads the device's maps
        q.handle = om
    gd, ld = S.buildLoopClosureConstraints(dev, cd, 0, [1], P, mp.mapBuilder.mapVoxelSize, lc)
    go, lo = S.buildLoopClosureConstraints(ora, co, 0, [1], P, mp.mapBuilder.mapVoxelSize, lc)
    assert ld == lo and ld[0][1] == "accepted" and len(gd) == len(go) == 1
    for a, b in zip(gd, go):
        assert np.abs(a.sourceToTarget - b.sourceToTarget).max() < 1e-8
        assert rel(a.informationMatrix, b.informationMatrix) < 1e-9
        assert np.abs(a.sourceToTarget - T).max() < 0.02
    # DeviceBackend.register_batch with the same estimator: refineLoopClosures on the two map copies
    src, tgt = cd.submaps[0].handle, cd.submaps[1].handle
    T0 = [dev.ransac(cd.submaps[0].sparse, cd.submaps[0].feature, [cd.submaps[1].sparse], [cd.submaps[1].feature], P)[0].transformation_]
    one = S.refineLoopClosuresOfSubmaps(dev, src, [tgt], T0, mp.mapBuilder.mapVoxelSize, lc)[0]
    per = S.refineLoopClosures(dev, dev.submap_as_cloud(src), [dev.submap_as_cloud(tgt)], T0, mp.mapBuilder.mapVoxelSize, lc)[0]
    assert (one["n_source_overlap"], one["n_target_overlap"], one["accepted"]) == (per["n_source_overlap"], per["n_target_overlap"], per["accepted"])
    assert np.abs(one["result"].transformation_ - per["result"].transformation_).max() <= 1e-12
    assert (one["result"].n_corr, one["result"].iters) == (per["result"].n_corr, per["result"].iters)
    assert rel(one["information"], per["information"]) <= 1e-12
    assert np.array_equal(one["result"].transformation_, gd[0].sourceToTarget)
    dev.close()
