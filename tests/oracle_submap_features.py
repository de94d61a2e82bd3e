"""CPU restatements of the feature-cloud front end of Submap::computeFeatures for the tests (test infrastructure, never imported by
the package): VoxelDownSample of the map with its normals averaged -> EstimateNormals with the voxel-mean normals as priors ->
NormalizeNormals -> OrientNormalsTowardsCameraLocation(0) -> ComputeFPFHFeature.

- estimate_normals(), submap_features(): the C restatement in tests/oracle_submap_features.c, linked with the FPFH restatement of
  tests/oracle_features.c and the oracle (KD-tree, voxel down-sample, eigen-solver).  It is the ground truth of the device path.
- np_estimate_normals(), np_submap_features(): a numpy + scipy cKDTree twin (own voxel grouping, neighbours, cumulants, prior and
  orientation rules, the FPFH twin of oracle_features.py) that validates the C one.  Only the 3x3 eigen-solver is the oracle's:
  LAPACK's eigh and FastEigen3x3 differ by up to ~1e-9 on ill-conditioned neighbourhoods.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O
from oracle_features import _p, np_fpfh, np_hybrid_neighbors

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "oracle_submap_features.c"), os.path.join(_HERE, "oracle_features.c")]
_lib = None


def lib():
    """Compiles oracle_submap_features.c together with oracle_features.c against libo3d_oracle.so in a temporary directory, loads it
    and removes the directory again (the loaded library stays mapped), so the tree stays untouched and nothing is left behind."""
    global _lib
    if _lib is None:
        oracle_so = O.build()
        with tempfile.TemporaryDirectory(prefix="b2s_oracle_submap_features_") as tmp:
            out = os.path.join(tmp, "liboracle_submap_features.so")
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", *_SRCS, "-o", out, oracle_so,
                                   "-Wl,-rpath," + os.path.dirname(oracle_so), "-lm"])
            C.CDLL(oracle_so, mode=C.RTLD_GLOBAL)
            _lib = C.CDLL(out)
    return _lib


def estimate_normals(xyz, knn, radius, prior=None):
    """C restatement: (normals, tie flags).  prior None = a cloud without normals (what orc_estimate_normals restates)."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float64).reshape(-1, 3)
    prior = None if prior is None else np.ascontiguousarray(prior, dtype=np.float64).reshape(-1, 3)
    n = len(xyz)
    out = np.zeros((n, 3)); tie = np.zeros(n, dtype=np.int32)
    lib().fo_estimate_normals(_p(xyz), C.c_int(n), C.c_int(knn), C.c_double(radius), _p(prior), _p(out), _p(tie))
    return out, tie.astype(bool)


def submap_features(xyz, nrm, p):
    """C restatement of the whole front end for a map cloud (nrm None: a map without normals, estimated without priors).
    p: open3d_slam_b200.engine.PlaceRecognitionParameters.  Returns a dict: xyz, prior, nrm, keys, tie, feature and the fo_fpfh
    details (spfh, margin, nb_idx, nb_d2, nb_cnt) of the sparse cloud, in the oracle's voxel order."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float64).reshape(-1, 3)
    nrm = None if nrm is None else np.ascontiguousarray(nrm, dtype=np.float64).reshape(-1, 3)
    n, k = len(xyz), int(p.featureKnn)
    m1 = max(n, 1)
    sx, sp, sn = np.zeros((m1, 3)), np.zeros((m1, 3)), np.zeros((m1, 3))
    keys, tie = np.zeros((m1, 3), dtype=np.int32), np.zeros(m1, dtype=np.int32)
    feat, spfh, margin = np.zeros((m1, 33)), np.zeros((m1, 33)), np.zeros(m1)
    nb_idx, nb_d2, nb_cnt = np.zeros((m1, k), dtype=np.int32), np.zeros((m1, k)), np.zeros(m1, dtype=np.int32)
    m = lib().fo_submap_features(_p(xyz), _p(nrm), C.c_int(n), C.c_double(p.featureVoxelSize), C.c_double(p.normalEstimationRadius),
                                 C.c_int(p.normalKnn), C.c_double(p.featureRadius), C.c_int(k), _p(sx), _p(sp), _p(sn), _p(keys), _p(tie),
                                 _p(feat), _p(spfh), _p(margin), _p(nb_idx), _p(nb_d2), _p(nb_cnt))
    if m < 0:
        raise ValueError("fo_submap_features: radius and knn must be > 0")
    return dict(xyz=sx[:m], prior=sp[:m] if nrm is not None else None, nrm=sn[:m], keys=keys[:m], tie=tie[:m].astype(bool),
                feature=feat[:m], spfh=spfh[:m], margin=margin[:m], nb_idx=nb_idx[:m], nb_d2=nb_d2[:m], nb_cnt=nb_cnt[:m])


def np_voxel_down_sample(xyz, nrm, voxel):
    """[O3D] VoxelDownSample: key floor((p - (min - v/2)) / v), per-voxel means accumulated in input order (NaN normals skipped).
    Returns (xyz, normals or None, keys), voxels in ascending key order."""
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    vmin = xyz.min(axis=0) - voxel * 0.5
    keys = np.floor((xyz - vmin) / voxel).astype(np.int64)
    uk, inv = np.unique(keys, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    cnt = np.bincount(inv, minlength=len(uk)).astype(np.float64)
    sx = np.zeros((len(uk), 3))
    np.add.at(sx, inv, xyz)                        # unbuffered, in index order: the running sum of AccumulatedPoint
    sn = None
    if nrm is not None:
        nrm = np.asarray(nrm, dtype=np.float64).reshape(-1, 3)
        ok = ~np.isnan(nrm).any(axis=1)
        sn = np.zeros((len(uk), 3))
        np.add.at(sn, inv[ok], nrm[ok])
        sn = sn / cnt[:, None]
    return sx / cnt[:, None], sn, uk


def np_estimate_normals(xyz, knn, radius, prior=None):
    """twin of estimate_normals: cKDTree neighbours, numpy covariance, the oracle's FastEigen3x3, then the prior / normalise / orient
    rules restated in numpy.  Returns (normals, tie flags)."""
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    out = np.zeros_like(xyz); tie = np.zeros(len(xyz), dtype=bool)
    for i, (idx, _d2) in enumerate(np_hybrid_neighbors(xyz, radius, knn) if len(xyz) else []):
        nr = np.array([0.0, 0.0, 1.0])            # fewer than 3 neighbours: identity covariance, FastEigen3x3 picks z
        cov = np.eye(3)
        if len(idx) >= 3:
            # ComputeCovariance's single-pass cumulants, summed in the search order (cumsum is sequential)
            p = xyz[idx]
            c = np.cumsum(np.c_[p, p[:, [0]] * p, p[:, [1]] * p[:, 1:], p[:, 2] * p[:, 2]], axis=0)[-1] / len(idx)
            mu, s = c[:3], c[3:]
            cov = np.array([[s[0] - mu[0] * mu[0], s[1] - mu[0] * mu[1], s[2] - mu[0] * mu[2]],
                            [s[1] - mu[0] * mu[1], s[3] - mu[1] * mu[1], s[4] - mu[1] * mu[2]],
                            [s[2] - mu[0] * mu[2], s[4] - mu[1] * mu[2], s[5] - mu[2] * mu[2]]])
            # the analytic solver of the oracle: eigh agrees only to ~1e-9 on ill-conditioned neighbourhoods
            nr = O.fast_eigen3x3(cov)
        if not nr.any():                           # FastEigen3x3 returned a zero vector (zero covariance)
            nr = prior[i].copy() if prior is not None else np.array([0.0, 0.0, 1.0])
        elif prior is not None and nr @ prior[i] < 0.0:
            nr = -nr
        z = nr @ nr
        if z > 0:
            nr = nr / np.sqrt(z)
        if np.isnan(nr[0]):
            nr = np.array([0.0, 0.0, 1.0])
        ref = -xyz[i]
        if not nr.any():
            rn = np.linalg.norm(ref)
            nr = ref / rn if rn > 0 else np.array([0.0, 0.0, 1.0])
        else:
            d = nr @ ref
            if d < 0.0:
                nr = -nr
            tie[i] = d == 0.0
        out[i] = nr
    return out, tie


def np_submap_features(xyz, nrm, p):
    """independent twin of submap_features: (xyz, prior, normals, keys, ties, feature, neighbour lists of the FPFH)"""
    sx, sp, keys = np_voxel_down_sample(xyz, nrm, p.featureVoxelSize)
    sn, tie = np_estimate_normals(sx, p.normalKnn, p.normalEstimationRadius, sp)
    feat, nbs = np_fpfh(sx, sn, p.featureRadius, p.featureKnn)
    return dict(xyz=sx, prior=sp, nrm=sn, keys=keys, tie=tie, feature=feat, nbs=nbs)
