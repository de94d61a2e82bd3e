"""CPU self-test of tests/normals_checks.py: the checks accept the fp64 restatement of the normal estimation (reference neighbour sets,
list-order cumulants, the oracle's FastEigen3x3, finish_normal's prior / normalise / orient) on every family, measure the direction
constant K that the GPU tests use, and reject each one-detail mutant of the operation with a printed margin."""
import mpmath
import numpy as np
import pytest

import normals_checks as NC
from oracle import oracle as O
from open3d_slam_b200 import synth

mpmath.mp.dps = 40


def _voxel_scan(n_max=4000):
    raw = synth.lidar_scan(synth.Scene(), synth.loop_trajectory(8)[0], seed=0).astype(np.float64)
    vx, _ = O.voxel_down_sample(raw, 0.1)
    return vx[np.random.default_rng(0).permutation(len(vx))[:n_max]]


def _priors(xyz, seed=1):
    p = np.random.default_rng(seed).normal(size=xyz.shape)
    p[:, 2] = np.abs(p[:, 2]) + 0.5
    return p


# name -> (cloud, knn, radius, priors)
def families():
    pl = NC.plane_through_origin()
    lone = np.array([[5.0, 5.0, 0.0], [-5.0, 6.0, 0.0], [7.0, -7.0, 0.0]])   # isolated points at z = 0: identity covariance, n . p == 0
    plo = np.vstack([pl, lone])
    pri = np.tile([0.0, 0.0, -1.0], (len(plo), 1))
    return {
        "lattice": (NC.lattice(7, 0.25), 20, 0.6, None),
        "lattice_1e3": (NC.lattice(6, 0.25, (1000.0, -1000.0, 500.0)), 20, 0.6, None),
        "radius_edge": (NC.radius_edge(), 20, 0.5, None),
        "cluster": (NC.cluster_at_distance(), 20, 2.0, None),
        "coincident": (NC.coincident(), 5, 0.3, None),
        "coincident_prior": (NC.coincident(), 5, 0.3, _priors(NC.coincident())),
        "plane_origin_prior": (plo, 10, 0.5, pri),
        "plane_prior_only": (pl, 10, 0.5, pri[:len(pl)]),
        "knn2": (NC.lattice(5, 0.25), 2, 0.6, None),
        "scan": (_voxel_scan(), 20, 3.0, None),
        "scan_1e4": (_voxel_scan(2000) + [1e4, -1e4, 1e2], 20, 3.0, None),
        "config1": (synth.planar_cloud_config1(noise=0.01)[1][:1500].astype(np.float64), 10, 1.0, None),
    }


def restatement(xyz, knn, radius, priors, sets_kw=None, swap_xy_xz=False, orient_sign=1.0, prior_flip=1.0, diag_tie="strict"):
    """what a correct device (or a one-detail mutant) would record and return for every point"""
    _, sets = NC.neighbour_sets(xyz, knn, radius, **(sets_kw or {}))
    rec = NC.restated_cumulants(xyz, sets)
    if swap_xy_xz:
        rec[:, [4, 5]] = rec[:, [5, 4]]
    cov = NC.covariance(rec)
    kind, vec = NC.solver_branch(cov, diag_tie)
    nrm = np.empty((len(xyz), 3))
    for i in range(len(xyz)):
        v = vec[i] if kind[i] == 2 else O.fast_eigen3x3(cov[i])
        nrm[i] = NC.finish_exact(v, xyz[i], None if priors is None else priors[i], orient_sign, prior_flip)
    return rec, nrm


@pytest.fixture(scope="module")
def fams():
    return {k: v + restatement(*v) for k, v in families().items()}


def test_checks_accept_the_restatement_and_measure_k(fams):
    worst = 0.0
    for name, (xyz, knn, radius, pri, rec, nrm) in fams.items():
        path = np.ones(len(xyz), dtype=np.int32)
        s = NC.check_all(xyz, knn, radius, rec, path, nrm, pri)
        cov = NC.covariance(rec)
        kind, _ = NC.solver_branch(cov)
        ev = np.nonzero(kind == 0)[0]
        k = 0.0
        if len(ev):
            v, gap, norm = NC.smallest_eigvec(cov[ev])
            met, _ = NC.direction_metric(nrm[ev], v, gap, norm, cov[ev])
            k = float(np.nanmax(met))
        worst = max(worst, k)
        print(f"{name:20s} n {len(xyz):5d} knn {knn:2d}: cumulants {s['cum']:.3g} of bound, K {k:.3g}, exact branches {s['exact']}, "
              f"signs checked {s['signs']} (+{s['prior_signs']} by the prior)")
    print(f"measured K = {worst:.3g} (K_MEASURED {NC.K_MEASURED}, K_DIR {NC.K_DIR})")
    assert worst <= NC.K_MEASURED


def test_reference_eigenvector_against_mpmath(fams):
    """the long-double Rayleigh refinement is the eigenvector of the exact fp64 covariance to far below the direction bound"""
    rng = np.random.default_rng(0)
    covs = []
    for name in ("scan", "scan_1e4", "config1", "lattice"):
        rec = fams[name][4]
        cov = NC.covariance(rec)
        kind, _ = NC.solver_branch(cov)
        ev = np.nonzero(kind == 0)[0]
        _, gap, norm = NC.smallest_eigvec(cov[ev])
        rel = gap / norm
        ev, rel = ev[rel > 1e-6], rel[rel > 1e-6]   # a (numerically) repeated smallest eigenvalue has no single eigenvector
        pick = np.r_[ev[np.argsort(rel)[:8]], rng.choice(ev, 8, replace=False)]   # the smallest gaps and a random sample
        covs += [cov[i] for i in pick]
    covs = np.array(covs)
    v, gap, norm = NC.smallest_eigvec(covs)
    worst = 0.0
    for i, c in enumerate(covs):
        E, Q = mpmath.eigsy(mpmath.matrix(c.reshape(3, 3).tolist()))
        j = min(range(3), key=lambda t: E[t])
        ref = np.array([float(Q[t, j]) for t in range(3)])
        s = np.linalg.norm(np.cross(v[i], ref / np.linalg.norm(ref)))
        worst = max(worst, s / (NC.U * norm[i] / gap[i]))
    print(f"reference eigenvector vs mpmath: worst {worst:.3g} u||C||/gap over {len(covs)} covariances")
    assert worst < 0.25   # under 5 % of the K_DIR bound


# mutant -> (family, restatement change, the stage of check_all that must reject it)
MUTANTS = {
    "tie_to_higher_index": ("lattice", dict(sets_kw=dict(tie="higher")), "cumulant"),
    "radius_le": ("radius_edge", dict(sets_kw=dict(cut="le")), "count"),
    "k_minus_1_members": ("scan", dict(sets_kw=dict(count_delta=-1)), "count"),
    "k_plus_1th_for_kth": ("scan", dict(sets_kw=dict(replace_kth=True)), "cumulant"),
    "xy_xz_swapped": ("scan", dict(swap_xy_xz=True), "cumulant"),
    "orient_towards_p": ("cluster", dict(orient_sign=-1.0), "sign"),
    "prior_flip_inverted": ("plane_prior_only", dict(prior_flip=-1.0), "sign"),
    "prior_flip_inverted_isolated": ("plane_origin_prior", dict(prior_flip=-1.0), "exact"),
    "diagonal_tie_rule": ("knn2", dict(diag_tie="le"), "exact"),
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_checks_reject_mutant(fams, mutant):
    fam, kw, stage = MUTANTS[mutant]
    xyz, knn, radius, pri = fams[fam][:4]
    rec, nrm = restatement(xyz, knn, radius, pri, **kw)
    path = np.ones(len(xyz), dtype=np.int32)
    _, sets = NC.neighbour_sets(xyz, knn, radius)
    S, A, cnt = NC.cumulant_reference(xyz, sets)
    cw, _, badc = NC.check_cumulants(rec, S, A, cnt)
    f = NC.check_finish(rec, nrm, xyz, pri)
    margin = (f"count mismatches {len(badc)}, worst cumulant {cw:.3g} x bound, exact-branch mismatches {len(f['exact_bad'])}, "
              f"direction {f['dir_worst'] / NC.K_DIR:.3g} x bound, wrong signs {len(f['sign_bad'])}")
    print(f"{mutant}: {margin}")
    with pytest.raises(AssertionError, match=rf"^\[{stage}\]"):
        NC.check_all(xyz, knn, radius, rec, path, nrm, pri)
