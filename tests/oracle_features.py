"""Two CPU restatements of [O3D] ComputeFPFHFeature for the tests (test infrastructure, never imported by the package):

- fpfh():    the C restatement in tests/oracle_features.c, neighbour lists from the KD-tree of oracle/o3d_oracle.c.  It is the
             ground truth of the device kernels (same expressions, same summation order).
- np_fpfh(): an independent numpy + scipy cKDTree restatement (ball query + lexsort, vectorised pair features, histogram by
             counts) that validates the C one.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
from scipy.spatial import cKDTree

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oracle_features.c")
_lib = None


def lib():
    """Compiles oracle_features.c against libo3d_oracle.so in a temporary directory, loads it and removes the directory again
    (the loaded library stays mapped), so the tree stays untouched and nothing is left behind."""
    global _lib
    if _lib is None:
        oracle_so = O.build()
        with tempfile.TemporaryDirectory(prefix="b2s_oracle_features_") as tmp:
            out = os.path.join(tmp, "liboracle_features.so")
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", _SRC, "-o", out, oracle_so,
                                   "-Wl,-rpath," + os.path.dirname(oracle_so), "-lm"])
            C.CDLL(oracle_so, mode=C.RTLD_GLOBAL)
            _lib = C.CDLL(out)
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def fpfh(xyz, nrm, radius, knn, details=False):
    """(n, 33) FPFH rows.  details=True also returns a dict with spfh (n, 33), margin (n: smallest bin-boundary / swap margin of the
    point's SPFH pairs) and the neighbour lists nb_idx / nb_d2 (n, knn) with counts nb_cnt (n)."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float64).reshape(-1, 3)
    nrm = np.ascontiguousarray(nrm, dtype=np.float64).reshape(-1, 3)
    n = len(xyz)
    feat = np.zeros((n, 33)); spfh = np.zeros((n, 33)); margin = np.zeros(n)
    nb_idx = np.zeros((n, knn), dtype=np.int32); nb_d2 = np.zeros((n, knn)); nb_cnt = np.zeros(n, dtype=np.int32)
    rc = lib().fo_fpfh(_p(xyz), _p(nrm), C.c_int(n), C.c_double(radius), C.c_int(knn), _p(feat), _p(spfh), _p(margin), _p(nb_idx), _p(nb_d2),
                       _p(nb_cnt))
    if rc != 0:
        raise ValueError("fo_fpfh: radius and knn must be > 0")
    if not details:
        return feat
    return feat, dict(spfh=spfh, margin=margin, nb_idx=nb_idx, nb_d2=nb_d2, nb_cnt=nb_cnt)


def differing_rows(a, b, det, tol=0.0, margin=1e-9):
    """Rows of two FPFH results that differ by more than tol, split into those a libm difference explains -- the row's point or one of
    its neighbours has an SPFH pair within `margin` of a bin boundary or of the acos swap decision, where one ulp of atan2 / acos
    moves the pair to another bin -- and the unexplained rest.  Returns (differing, unexplained) index arrays."""
    diff = np.flatnonzero(np.abs(np.asarray(a) - np.asarray(b)).max(axis=1, initial=0.0) > tol)
    m = det["margin"]
    unexplained = [i for i in diff if min(m[i], m[det["nb_idx"][i, :det["nb_cnt"][i]]].min(initial=np.inf)) >= margin]
    return diff, np.array(unexplained, dtype=np.int64)


# ---------------------------------------------------------------------------------------------------------------------
# independent numpy restatement
# ---------------------------------------------------------------------------------------------------------------------
def np_hybrid_neighbors(xyz, radius, knn):
    """[O3D] KDTreeFlann::SearchHybrid for every point: the knn nearest with d2 < radius^2, ascending (d2, index)."""
    tree = cKDTree(xyz)
    r2 = radius * radius
    out = []
    for i, cand in enumerate(tree.query_ball_point(xyz, radius * (1 + 1e-9))):   # superset; the exact fp64 cut follows
        cand = np.asarray(cand, dtype=np.int64)
        d = xyz[i] - xyz[cand]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        keep = d2 < r2
        cand, d2 = cand[keep], d2[keep]
        o = np.lexsort((cand, d2))[:knn]
        out.append((cand[o], d2[o]))
    return out


def np_pair_features(p1, n1, p2, n2):
    """ComputePairFeatures, vectorised over rows: (m, 3) f0, f1, f2."""
    dp = p2 - p1
    ln = np.sqrt((dp[:, 0] * dp[:, 0] + dp[:, 1] * dp[:, 1]) + dp[:, 2] * dp[:, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        a1 = (n1 * dp).sum(axis=1) / ln
        a2 = (n2 * dp).sum(axis=1) / ln
        swap = np.arccos(np.abs(a1)) > np.arccos(np.abs(a2))
        a = np.where(swap[:, None], n2, n1); b = np.where(swap[:, None], n1, n2); dp = np.where(swap[:, None], -dp, dp)
        f2 = np.where(swap, -a2, a1)
        v = np.cross(dp, a)
        vn = np.linalg.norm(v, axis=1)
        v = v / vn[:, None]
        w = np.cross(a, v)
        f = np.stack([np.arctan2((w * b).sum(axis=1), (a * b).sum(axis=1)), (v * b).sum(axis=1), f2], axis=1)
    f[(ln == 0.0) | (vn == 0.0)] = 0.0
    return f


def np_bins(f):
    h0 = np.floor(11 * (f[:, 0] + np.pi) / (2.0 * np.pi))
    h1 = np.floor(11 * (f[:, 1] + 1.0) * 0.5)
    h2 = np.floor(11 * (f[:, 2] + 1.0) * 0.5)
    return np.clip(np.stack([h0, h1, h2], axis=1), 0, 10).astype(np.int64) + np.array([0, 11, 22])


def np_fpfh(xyz, nrm, radius, knn):
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3); nrm = np.asarray(nrm, dtype=np.float64).reshape(-1, 3)
    n = len(xyz)
    nbs = np_hybrid_neighbors(xyz, radius, knn) if n else []
    spfh = np.zeros((n, 33))
    for i, (idx, _d2) in enumerate(nbs):
        if len(idx) <= 1:
            continue
        j = idx[1:]
        f = np_pair_features(np.broadcast_to(xyz[i], (len(j), 3)), np.broadcast_to(nrm[i], (len(j), 3)), xyz[j], nrm[j])
        counts = np.bincount(np_bins(f).reshape(-1), minlength=33)
        spfh[i] = counts * (100.0 / (len(idx) - 1))
    feat = np.zeros((n, 33))
    for i, (idx, d2) in enumerate(nbs):
        if len(idx) <= 1:
            continue
        j, d = idx[1:], d2[1:]
        keep = d != 0.0
        acc = (spfh[j[keep]] / d[keep][:, None]).sum(axis=0)
        s = acc.reshape(3, 11).sum(axis=1)
        fac = np.where(s != 0.0, 100.0 / np.where(s != 0.0, s, 1.0), 0.0)
        feat[i] = acc * np.repeat(fac, 11) + spfh[i]
    return feat, nbs
