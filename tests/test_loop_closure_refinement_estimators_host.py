"""CPU: the estimator of the loop-closure refinement.  LoopClosureParameters.fromMapperParameters restates
PlaceRecognition::updateRegistrationAlgorithm (src/PlaceRecognition.cpp:44-48): the scan matcher's registration type, 100 iterations,
placeRecognition.maxIcpCorrespondenceDistance.  The oracle backend's register_batch dispatches on the estimator like
cloudRegistrationFactory (src/CloudRegistration.cpp:85-100), and slam.buildLoopClosureConstraints refines with it on both of
refineLoopClosuresOfSubmaps' routes; point-to-point refines maps without normals.  A backend whose register_batch takes no estimator
still refines point-to-plane, and fails when asked for another type."""
import numpy as np
import pytest

from oracle import oracle as O
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from test_loop_closure_host import P, collection, room
from test_loop_closure_refinement_host import BatchedBackend, same_constraints
from test_ransac_oracle import rigid
from oracle_backend import OracleCloud
from oracle_backend_estimators import EstimatorOracleBackend
from oracle_backend_ransac import RansacOracleBackend

TYPES = ["PointToPlaneIcp", "PointToPointIcp", "GeneralizedIcp"]
T_TRUE = rigid(0.4, [3.0, -1.5, 0.2], 0.02, -0.01)


@pytest.mark.parametrize("reg", TYPES)
def test_from_mapper_parameters_restates_update_registration_algorithm(reg):
    mp = E.MapperParameters(scanToMapRegType=reg)
    mp.icp.maxNumIter, mp.icp.maxCorrespondenceDistance = 7, 2.5   # the scan matcher's own values do not reach the refinement
    lc = S.LoopClosureParameters.fromMapperParameters(mp)
    assert (lc.registrationType, lc.maxNumIter, lc.maxIcpCorrespondenceDistance, lc.minRefinementFitness) == (reg, 100, 0.3, 0.7)
    lc = S.LoopClosureParameters.fromMapperParameters(mp, maxIcpCorrespondenceDistance=0.45, minRefinementFitness=0.6)
    assert (lc.maxIcpCorrespondenceDistance, lc.minRefinementFitness) == (0.45, 0.6)
    d = S.LoopClosureParameters()
    assert (lc.voxelExpansionFactorOverlapComputation, lc.minNumPointsPerVoxel) == (d.voxelExpansionFactorOverlapComputation, d.minNumPointsPerVoxel)


def test_defaults_are_point_to_plane_and_unknown_types_fail():
    assert S.LoopClosureParameters().registrationType == "PointToPlaneIcp"
    assert E.LoopClosureRefinementParameters().regType == "PointToPlaneIcp"
    codes = {"PointToPlaneIcp": L.REG_POINT_TO_PLANE, "PointToPointIcp": L.REG_POINT_TO_POINT, "GeneralizedIcp": L.REG_GENERALIZED}
    for name, code in codes.items():
        assert E.LoopClosureRefinementParameters(regType=name).to_c().reg_type == code
    assert E.LoopClosureRefinementParameters().to_c().reg_type == L.REG_POINT_TO_PLANE
    for fn in (lambda: E.LoopClosureRefinementParameters(regType="Ndt").to_c(),
               lambda: S.LoopClosureParameters.fromMapperParameters(E.MapperParameters(scanToMapRegType="Ndt"))):
        with pytest.raises(L.B2SError) as e:
            fn()
        assert e.value.code == L.E_UNSUPPORTED
    with pytest.raises(RuntimeError):
        EstimatorOracleBackend(E.MapperParameters()).register_batch([], [], [], 0.3, 100, "Ndt")


def pair_clouds(T0):
    """the overlap of the room and another sample of it moved by T_TRUE, at the guess T0"""
    sx, sn = room(0)
    x, n = room(1)
    tx, tn = x @ T_TRUE[:3, :3].T + T_TRUE[:3, 3], n @ T_TRUE[:3, :3].T
    fs, ft = O.overlap_flags(sx, tx, T0, 2.0, 1)
    return OracleCloud(sx[fs], sn[fs]), OracleCloud(tx[ft], tn[ft])


@pytest.mark.parametrize("reg", TYPES)
def test_oracle_backend_dispatches_on_the_estimator(reg):
    """register_batch(regType) is the oracle's registration of that type, pair by pair, with the source's normals for GeneralizedIcp"""
    T0 = T_TRUE @ rigid(np.deg2rad(1.0), [0.05, -0.04, 0.02], np.deg2rad(0.5), np.deg2rad(-0.5))
    so, to = pair_clouds(T0)
    be = EstimatorOracleBackend(E.MapperParameters())
    (r,) = be.register_batch([so], [to], [T0], 0.3, 100, reg)
    ref = {"PointToPlaneIcp": lambda: O.registration_icp_p2plane(so.xyz, to.xyz, to.nrm, 0.3, T0, max_iter=100),
           "PointToPointIcp": lambda: O.registration_icp_p2point(so.xyz, to.xyz, 0.3, T0, max_iter=100),
           "GeneralizedIcp": lambda: O.registration_gicp(so.xyz, so.nrm, to.xyz, to.nrm, 0.3, T0, max_iter=100)}[reg]()
    assert np.array_equal(r.transformation_, ref.T) and (r.fitness_, r.inlier_rmse_, r.n_corr, r.iters) == \
        (ref.fitness, ref.inlier_rmse, ref.n_corr, ref.iters)
    assert np.abs(r.transformation_ - T_TRUE).max() < 0.02 and r.fitness_ > 0.9
    if reg == "PointToPlaneIcp":   # the default of the old signature
        (d,) = be.register_batch([so], [to], [T0], 0.3, 100)
        assert np.array_equal(d.transformation_, r.transformation_)
    others = [x for x in TYPES if x != reg]
    assert all(not np.array_equal(be.register_batch([so], [to], [T0], 0.3, 100, o)[0].transformation_, r.transformation_) for o in others)


class SpyBackend(EstimatorOracleBackend):
    """the oracle backend, recording the estimator every register_batch call gets"""

    def register_batch(self, sources, targets, inits, max_corr, max_iter, regType="PointToPlaneIcp"):
        self.calls.append(regType)
        return super().register_batch(sources, targets, inits, max_corr, max_iter, regType)


def resampled(T):
    """collection(T) with the target's map replaced by another sample of the room moved by T (the sparse clouds and features stay,
    so the RANSAC proposal stays): the estimators no longer agree to the last bit"""
    be, sc = collection(T)
    be.__class__ = SpyBackend
    be.calls = []
    x, n = room(1)
    sc.submaps[1].handle.xyz, sc.submaps[1].handle.nrm = x @ T[:3, :3].T + T[:3, 3], n @ T[:3, :3].T
    return be, sc


@pytest.mark.parametrize("reg", TYPES)
def test_build_loop_closure_constraints_with_the_mapper_estimator(reg):
    """the composed route of refineLoopClosuresOfSubmaps registers with the estimator fromMapperParameters takes from the scan matcher:
    the constraint is the oracle registration of that type from the RANSAC proposal, and differs from the other types'"""
    lc = S.LoopClosureParameters.fromMapperParameters(E.MapperParameters(scanToMapRegType=reg))
    be, sc = resampled(T_TRUE)
    cons, log = S.buildLoopClosureConstraints(be, sc, 0, [1], P, 0.1, lc)
    assert be.calls == [reg] and log[0][1] == "accepted" and len(cons) == 1
    src, tgt = sc.submaps[0], sc.submaps[1]
    (prop,) = be.ransac(src.sparse, src.feature, [tgt.sparse], [tgt.feature], P)
    so, to = be.overlap(OracleCloud(src.handle.xyz, src.handle.nrm), OracleCloud(tgt.handle.xyz, tgt.handle.nrm), prop.transformation_,
                        lc.voxelExpansionFactorOverlapComputation * 0.1, 1)
    (r,) = EstimatorOracleBackend(E.MapperParameters()).register_batch([so], [to], [prop.transformation_], 0.3, 100, reg)
    assert np.array_equal(cons[0].sourceToTarget, r.transformation_)
    assert np.array_equal(cons[0].informationMatrix, O.information_matrix(so.xyz, to.xyz, 0.3, r.transformation_))
    assert np.abs(cons[0].sourceToTarget - T_TRUE).max() < 0.02
    for other in TYPES:
        if other != reg:
            be2, sc2 = resampled(T_TRUE)
            c2, _ = S.buildLoopClosureConstraints(be2, sc2, 0, [1], P, 0.1, S.LoopClosureParameters(registrationType=other))
            assert not np.array_equal(c2[0].sourceToTarget, cons[0].sourceToTarget)


def test_batched_route_gets_the_estimator():
    """a backend with its own refine_loop_closures (DeviceBackend's route) receives the parameters, estimator included"""
    lc = S.LoopClosureParameters.fromMapperParameters(E.MapperParameters(scanToMapRegType="GeneralizedIcp"))
    seen = []

    class Batched(BatchedBackend):
        def refine_loop_closures(self, source_sm, target_sms, inits, mapVoxelSize, lc=None):
            seen.append(lc.registrationType)
            return super().refine_loop_closures(source_sm, target_sms, inits, mapVoxelSize, lc)

    be, sc = collection(T_TRUE)
    be.__class__ = Batched
    be.calls = []
    S.buildLoopClosureConstraints(be, sc, 0, [1], P, 0.1, lc)
    assert seen == ["GeneralizedIcp"]


def test_point_to_point_refines_maps_without_normals():
    """a point-to-point mapper's maps carry no normals: the refinement of PointToPointIcp needs none"""
    lc = S.LoopClosureParameters.fromMapperParameters(E.MapperParameters(scanToMapRegType="PointToPointIcp"))
    be, sc = collection(T_TRUE)
    be.__class__ = EstimatorOracleBackend
    ref_c, ref_log = S.buildLoopClosureConstraints(be, sc, 0, [1], P, 0.1, lc)
    for rec in sc.submaps:
        rec.handle.nrm = None
    c, log = S.buildLoopClosureConstraints(be, sc, 0, [1], P, 0.1, lc)
    assert log == ref_log and log[0][1] == "accepted"
    same_constraints(c, ref_c)


def test_backend_without_estimator_argument():
    """the oracle backend's register_batch has no regType: point-to-plane refines through it as before, another type is refused
    instead of being registered as point-to-plane"""
    be, sc = collection(T_TRUE)
    assert type(be) is RansacOracleBackend
    cons, log = S.buildLoopClosureConstraints(be, sc, 0, [1], P, 0.1, S.LoopClosureParameters())
    be2, sc2 = collection(T_TRUE)
    be2.__class__ = EstimatorOracleBackend
    cons2, log2 = S.buildLoopClosureConstraints(be2, sc2, 0, [1], P, 0.1, S.LoopClosureParameters())
    assert log == log2 and log[0][1] == "accepted"
    same_constraints(cons, cons2)
    with pytest.raises(TypeError):
        S.buildLoopClosureConstraints(be, sc, 0, [1], P, 0.1, S.LoopClosureParameters(registrationType="GeneralizedIcp"))
