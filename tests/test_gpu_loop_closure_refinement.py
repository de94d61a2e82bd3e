"""GPU: b2s_submap_loop_closure_refinement (the refinement half of PlaceRecognition::buildLoopClosureConstraints, src/PlaceRecognition.cpp:
96-149), one source submap against K candidates in one call on the resident maps -- against the device composition it replaces
(b2s_submap_to_cloud x 2 + b2s_overlap(T0) + b2s_register_batch + b2s_information_matrix), against the oracle, at its boundaries (the
kind of guess, K = 1 / 4 / 16 / 17, a target listed twice, an empty overlap, the fitness gate, getMapVoxelSize, errors), K pairs in one
call against K single calls, and b2s_submap_odometry_constraints against the records of the library before the two were merged."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import oracle as O
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from test_loop_closure_host import room
from test_ransac_oracle import rigid

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
PRM = E.LoopClosureRefinementParameters()


def rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    s = np.abs(b).max()
    return np.abs(a - b).max() / (s if s > 0 else 1.0)


def submap(eng, xyz, nrm=None, cap=None):
    sm = E.Submap(eng, cap or max(2 * len(xyz), 1024))
    sm.setMapPointCloud(eng.cloud(np.asarray(xyz, dtype=np.float64).reshape(-1, 3), nrm))
    return sm


def moved(T, xyz, nrm):
    return xyz @ T[:3, :3].T + T[:3, 3], nrm @ T[:3, :3].T


# the place seen twice: a room of planes (floor, two walls, a box) and another sample of it moved by the true sourceToTarget
TRUTH = {"identity": np.eye(4), "translation": rigid(0.0, [3.0, -1.5, 0.2]), "yaw30": rigid(np.deg2rad(30.0), [4.0, -3.0, 0.3])}
GUESS = {"identity": np.eye(4),                                                           # exactly the identity
         "translation": TRUTH["translation"] @ rigid(0.0, [0.06, -0.04, 0.02]),           # pure translation, off by a few cm
         "yaw30": TRUTH["yaw30"] @ rigid(np.deg2rad(1.0), [0.05, -0.04, 0.02], np.deg2rad(0.5), np.deg2rad(-0.5))}


def target(eng, kind, seed=1, parts=5):
    """another sample of the room moved by TRUTH[kind]; parts = 3 keeps the floor and the two walls (no box)"""
    x, n = room(seed)
    k = len(x) // 5
    return submap(eng, *moved(TRUTH[kind], x[:parts * k], n[:parts * k]))


def source(eng, seed=0):
    return submap(eng, *room(seed))


def composed(eng, src, tgt, T0, prm=PRM):
    """the composition the call replaces: two map copies, b2s_overlap at T0, b2s_register_batch (point-to-plane), b2s_information_matrix"""
    v = E.getMapVoxelSize(prm.mapVoxelSize, prm.voxelSizeIfMapVoxelSizeIsZero)
    params = eng.params
    sc, tc = src.toCloud(), tgt.toCloud()
    so, to = E.computeOverlappingClouds(eng, sc, tc, T0, prm.voxelExpansionFactorOverlapComputation * v, prm.minNumPointsPerVoxel)
    reg = E.RegistrationIcpPointToPlane(eng, E.CloudRegistrationParameters(icp=E.IcpParameters(maxNumIter=prm.maxNumIter,
                                                                                               maxCorrespondenceDistance=prm.maxIcpCorrespondenceDistance)))
    (r,) = reg.registerCloudsBatch([so], [to], [T0])
    eng.set_parameters(params)
    info = E.getInformationMatrixFromPointClouds(eng, so, to, prm.maxIcpCorrespondenceDistance, r.transformation_)
    return so, to, r, info, not (r.fitness_ < prm.minRefinementFitness)


def refine(eng, src, tgts, inits, prm=PRM, overlaps=False):
    if not overlaps:
        return E.refineLoopClosuresBatch(eng, src, tgts, inits, prm)
    so, to = [E.Cloud(eng) for _ in tgts], [E.Cloud(eng) for _ in tgts]
    return E.refineLoopClosuresBatch(eng, src, tgts, inits, prm, so, to), so, to


def fields(r):
    return (r.result.transformation_.tobytes(), r.result.fitness_, r.result.inlier_rmse_, r.result.n_corr, r.result.iters, r.information.tobytes(),
            r.accepted, r.nSourceOverlap, r.nTargetOverlap)


def check_against_composition(eng, src, tgt, T0, g, so, to, prm=PRM):
    cso, cto, r, info, acc = composed(eng, src, tgt, T0, prm)
    for x, y in ((so, cso), (to, cto)):
        (xx, xn), (yx, yn) = x.download(), y.download()
        assert np.array_equal(xx, yx) and np.array_equal(xn, yn, equal_nan=True)   # bit-identical, in order
    assert (g.nSourceOverlap, g.nTargetOverlap) == (len(cso), len(cto))
    assert np.abs(g.result.transformation_ - r.transformation_).max() <= 1e-12
    assert abs(g.result.fitness_ - r.fitness_) <= 1e-12 and abs(g.result.inlier_rmse_ - r.inlier_rmse_) <= 1e-12
    assert g.accepted == acc
    assert rel(g.information, info) <= 1e-12   # K-info-wide and K-icp-iter sum in different orders


@pytest.mark.parametrize("kind", ["identity", "translation", "yaw30"])
def test_against_device_composition_and_oracle(engine_factory, kind):
    eng = engine_factory()
    src, tgt = source(eng), target(eng, kind)
    T0 = GUESS[kind]
    (g,), (so,), (to,) = refine(eng, src, [tgt], [T0], overlaps=True)
    assert g.accepted and g.nSourceOverlap > 3000 and g.result.iters >= (0 if kind == "identity" else 1)
    check_against_composition(eng, src, tgt, T0, g, so, to)
    # the oracle on the device's own maps: the overlap sets, the ICP from T0, the information matrix at the device's T
    (sx, sn), (tx, tn) = src.getMapPointCloud(), tgt.getMapPointCloud()
    fs, ft = O.overlap_flags(sx, tx, T0, PRM.voxelExpansionFactorOverlapComputation * PRM.mapVoxelSize, PRM.minNumPointsPerVoxel)
    assert np.array_equal(so.download()[0], sx[fs]) and np.array_equal(to.download()[0], tx[ft])
    ref = O.registration_icp_p2plane(sx[fs], tx[ft], tn[ft], PRM.maxIcpCorrespondenceDistance, T0, max_iter=PRM.maxNumIter)
    assert np.abs(g.result.transformation_ - ref.T).max() < 1e-8 and g.result.n_corr == ref.n_corr
    assert rel(g.information, O.information_matrix(sx[fs], tx[ft], PRM.maxIcpCorrespondenceDistance, g.result.transformation_)) < 1e-9
    assert np.abs(g.result.transformation_ - TRUTH[kind]).max() < 0.02


def test_resident_map_with_tombstones(engine_factory):
    """fusion into the target leaves tombstones in its map slots: the call skips them like b2s_submap_to_cloud does"""
    eng = engine_factory()
    src, tgt = source(eng), target(eng, "yaw30")
    x, n = room(7, 3000)
    scan = eng.cloud(*moved(TRUTH["yaw30"], x, n))
    tgt.insertScan(None, scan, np.eye(4))
    tgt.insertScan(None, scan, rigid(0.0, [0.01, 0.0, 0.0]))
    (g,), (so,), (to,) = refine(eng, src, [tgt], [GUESS["yaw30"]], overlaps=True)
    check_against_composition(eng, src, tgt, GUESS["yaw30"], g, so, to)


def test_mixed_batch_fitness_gate_and_empty_overlap(engine_factory):
    """one call: accepted; rejected by the fitness gate (the target lacks the box); an empty overlap (the target 100 m away) -- each the
    composition's record; and the batch equals one call per pair"""
    eng = engine_factory()
    src = source(eng)
    good, nobox = target(eng, "translation"), target(eng, "translation", parts=3)
    far = submap(eng, *moved(rigid(0.0, [0.0, 0.0, 100.0]), *room(3)))
    tgts, inits = [good, nobox, far], [GUESS["translation"]] * 3
    res, so, to = refine(eng, src, tgts, inits, overlaps=True)
    assert [r.accepted for r in res] == [True, False, False]
    assert 0.0 < res[1].result.fitness_ < PRM.minRefinementFitness
    assert (res[2].nSourceOverlap, res[2].nTargetOverlap, res[2].result.fitness_) == (0, 0, 0.0) and not res[2].information.any()
    for t, T0, g, a, b in zip(tgts, inits, res, so, to):
        check_against_composition(eng, src, t, T0, g, a, b)
    assert [fields(r) for r in res] == [fields(refine(eng, src, [t], [T0])[0]) for t, T0 in zip(tgts, inits)]


@pytest.mark.parametrize("K", [1, 4, 16, 17])
def test_k_targets_equal_single_calls(engine_factory, K):
    eng = engine_factory()
    src = source(eng)
    kinds = list(TRUTH)
    tgts = [target(eng, kinds[k % 3], seed=1 + k, parts=3 if k % 5 == 4 else 5) for k in range(K)]
    inits = [GUESS[kinds[k % 3]] for k in range(K)]
    res, so, to = refine(eng, src, tgts, inits, overlaps=True)
    again = refine(eng, src, tgts, inits)
    singles = [refine(eng, src, [t], [T0])[0] for t, T0 in zip(tgts, inits)]
    assert [fields(r) for r in res] == [fields(r) for r in again] == [fields(r) for r in singles]
    for k in (0, K // 2, K - 1):
        check_against_composition(eng, src, tgts[k], inits[k], res[k], so[k], to[k])


def test_same_target_twice(engine_factory):
    eng = engine_factory()
    src, a, b = source(eng), target(eng, "yaw30"), target(eng, "translation")
    res = refine(eng, src, [a, b, a], [GUESS["yaw30"], GUESS["translation"], GUESS["yaw30"]])
    assert fields(res[0]) == fields(res[2]) and res[0].accepted and res[1].accepted


@pytest.mark.parametrize("v", [0.0, 1e-3, -1e-3])
def test_map_voxel_size_rule(engine_factory, v):
    """getMapVoxelSize(mapBuilder_, 0.04), PlaceRecognition.cpp:98: |v| <= 1e-3 gives the records of an explicit 0.04"""
    eng = engine_factory()
    src, tgt = source(eng), target(eng, "translation")
    z = refine(eng, src, [tgt], [GUESS["translation"]], E.LoopClosureRefinementParameters(mapVoxelSize=v))
    e = refine(eng, src, [tgt], [GUESS["translation"]], E.LoopClosureRefinementParameters(mapVoxelSize=0.04))
    assert [fields(r) for r in z] == [fields(r) for r in e]


def test_errors(engine_factory):
    e1, e2 = engine_factory(), engine_factory()
    a, b, other = source(e1), target(e1, "identity"), source(e2)
    I = [np.eye(4)]
    assert E.refineLoopClosuresBatch(e1, a, [], []) == []

    def code(fn):
        with pytest.raises(L.B2SError) as e:
            fn()
        return e.value.code

    assert code(lambda: refine(e1, other, [b], I)) == L.E_INVALID
    assert code(lambda: refine(e1, a, [other], I)) == L.E_INVALID
    for prm in (E.LoopClosureRefinementParameters(mapVoxelSize=-0.2), E.LoopClosureRefinementParameters(mapVoxelSize=0.0, voxelSizeIfMapVoxelSizeIsZero=0.0),
                E.LoopClosureRefinementParameters(voxelExpansionFactorOverlapComputation=0.0),
                E.LoopClosureRefinementParameters(maxIcpCorrespondenceDistance=0.0), E.LoopClosureRefinementParameters(minNumPointsPerVoxel=0),
                E.LoopClosureRefinementParameters(maxNumIter=-1)):
        assert code(lambda: refine(e1, a, [b], I, prm)) == L.E_INVALID
    assert code(lambda: E.refineLoopClosuresBatch(e1, a, [b], I, None, [E.Cloud(e2)], [E.Cloud(e1)])) == L.E_INVALID
    c = E.Cloud(e1)
    assert code(lambda: E.refineLoopClosuresBatch(e1, a, [b], I, None, [c], [c])) == L.E_INVALID
    p = PRM.to_c()
    lib = L.lib()
    tg = (C.c_void_p * 1)(b._s)
    out = (L.LoopClosureRefinement * 1)()
    assert lib.b2s_submap_loop_closure_refinement(e1._h, a._s, C.c_int32(-1), tg, None, C.byref(p), None, None, out) == L.E_INVALID
    assert lib.b2s_submap_loop_closure_refinement(e1._h, a._s, C.c_int32(1), tg, None, C.byref(p), None, None, out) == L.E_INVALID   # no inits
    assert lib.b2s_submap_loop_closure_refinement(e1._h, a._s, C.c_int32(0), None, None, C.byref(p), None, None, None) == L.OK
    # a point-to-point map (normals stored as NaN) cannot be a point-to-plane target; as the source it is fine
    p2p = engine_factory(E.MapperParameters(scanToMapRegType="PointToPointIcp"))
    x, n = room(0)
    pa, ch = submap(p2p, x, n), E.Submap(p2p, 16384)
    ch.setMapPointCloud(p2p.cloud(room(1)[0]))
    assert code(lambda: refine(p2p, pa, [ch], I)) == L.E_NO_NORMALS
    refine(p2p, ch, [pa], I)


# ---- b2s_submap_odometry_constraints through the shared driver: the records of the library before it was shared --------------------
def odometry_inputs():
    """parent / child maps of three constructed pairs (uploaded, so the maps do not depend on fusion's atomics)"""
    out = []
    for k, kind in enumerate(("identity", "translation", "identity")):
        x, n = room(10 + k)
        y, m = room(20 + k)
        if kind == "translation":
            y, m = moved(rigid(0.0, [0.05, -0.03, 0.01]), y, m)
        if k == 2:   # a pair whose overlap is partial: the child shifted by 9 m
            y, m = moved(rigid(0.0, [9.0, 0.0, 0.0]), y, m)
        out.append((x, n, y, m))
    return out


def odometry_records(eng):
    pairs = [(submap(eng, x, n), submap(eng, y, m)) for x, n, y, m in odometry_inputs()]
    rec = {}
    for refine_ in (False, True):
        prm = E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=refine_)
        res = E.buildOdometryConstraintsBatch(eng, [p for p, _ in pairs], [c for _, c in pairs], prm)
        for k, r in enumerate(res):
            rec[f"T_{int(refine_)}_{k}"] = r.sourceToTarget_
            rec[f"info_{int(refine_)}_{k}"] = r.informationMatrix_
            rec[f"n_{int(refine_)}_{k}"] = np.array([r.nSourceOverlap, r.nTargetOverlap] + ([r.icp.n_corr, r.icp.iters] if r.icp else [0, 0]))
            if r.icp:
                rec[f"fit_{int(refine_)}_{k}"] = np.array([r.icp.fitness_, r.icp.inlier_rmse_])
    return rec


def test_odometry_constraints_match_the_records_before_the_shared_driver(engine_factory):
    """tests/golden/odometry_constraints_records.npz: odometry_records() by the library before the odometry constraints and the
    loop-closure refinement shared one driver, on an H100; every record bit for bit"""
    ref = np.load(os.path.join(HERE, "golden", "odometry_constraints_records.npz"))
    got = odometry_records(engine_factory())
    assert sorted(got) == sorted(ref.files)
    for k in ref.files:
        assert np.array_equal(got[k], ref[k]), k
