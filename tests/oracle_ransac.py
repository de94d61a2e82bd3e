"""CPU restatements of RegistrationRANSACBasedOnFeatureMatching (DESIGN.md row K-ransac) for the tests (test infrastructure, never
imported by the package):

- feature_corr(), ransac(): the C restatement in tests/oracle_ransac.c (KD-tree 1-NN and orc_svd3 of the oracle), one hypothesis
  after the other.  It is the ground truth of the device path.
- np_feature_corr(), np_ransac(): an independent numpy twin (brute-force argmins, brute-force validation) that validates the C one.
  Only the 3x3 SVD is the oracle's, so that T can be compared bit for bit.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import tempfile
from dataclasses import dataclass

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oracle_ransac.c")
_lib = None
GOLDEN = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1


def lib():
    """Compiles oracle_ransac.c against libo3d_oracle.so in a temporary directory and loads it (the tree stays untouched)."""
    global _lib
    if _lib is None:
        oracle_so = O.build()
        with tempfile.TemporaryDirectory(prefix="b2s_oracle_ransac_") as tmp:
            out = os.path.join(tmp, "liboracle_ransac.so")
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-Wall", _SRC, "-o", out, oracle_so,
                                   "-Wl,-rpath," + os.path.dirname(oracle_so), "-lm"])
            C.CDLL(oracle_so, mode=C.RTLD_GLOBAL)
            _lib = C.CDLL(out)
            _lib.or_stream.restype = C.c_uint64
            _lib.or_stream.argtypes = [C.c_uint64, C.c_int64, C.c_int, C.c_int, C.c_uint64]
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@dataclass
class Params:
    """the RANSAC fields of PlaceRecognitionParameters, Lua defaults"""
    mutual_filter: bool = True
    ransac_n: int = 3
    max_corr: float = 0.75
    checker_distance: float = 0.8
    checker_edge: float = 0.6
    max_iteration: int = 10_000_000
    confidence: float = 0.999
    seed: int = 1

    @classmethod
    def of(cls, p, mutual_filter=True):   # from engine.PlaceRecognitionParameters
        return cls(mutual_filter, p.ransacModelSize, p.ransacMaxCorrespondenceDistance, p.correspondenceCheckerDistance,
                   p.correspondenceCheckerEdgeLength, p.ransacNumIter, p.ransacProbability, p.ransacSeed)


@dataclass
class Result:
    T: np.ndarray
    fitness: float
    rmse: float
    inliers: int
    hypotheses: int
    validations: int
    n_feature_corr: int
    used_mutual: bool
    best_h: int
    sum_d2: float
    k_d: float          # k_d of the last update of best (0 when none)


def feature_corr(fs, ft):
    fs = np.ascontiguousarray(fs, dtype=np.float64).reshape(-1, 33); ft = np.ascontiguousarray(ft, dtype=np.float64).reshape(-1, 33)
    s2t = np.full(max(len(fs), 1), -1, dtype=np.int32); t2s = np.full(max(len(ft), 1), -1, dtype=np.int32)
    lib().or_feature_corr(_p(fs), C.c_int(len(fs)), _p(ft), C.c_int(len(ft)), _p(s2t), _p(t2s))
    return s2t[:len(fs)], t2s[:len(ft)]


def stream(seed, h, n, j, size):
    return int(lib().or_stream(seed, h, n, j, size))


def ransac(sx, sf, tx, tf, p: Params) -> Result:
    sx = np.ascontiguousarray(sx, dtype=np.float64).reshape(-1, 3); tx = np.ascontiguousarray(tx, dtype=np.float64).reshape(-1, 3)
    sf = np.ascontiguousarray(sf, dtype=np.float64).reshape(-1, 33); tf = np.ascontiguousarray(tf, dtype=np.float64).reshape(-1, 33)
    T = np.empty(16); st = np.zeros(6, dtype=np.int64); sums = np.zeros(4)
    lib().or_ransac(_p(sx), _p(sf), C.c_int(len(sx)), _p(tx), _p(tf), C.c_int(len(tx)), C.c_int(int(p.mutual_filter)), C.c_int(p.ransac_n),
                    C.c_double(p.max_corr), C.c_double(p.checker_distance), C.c_double(p.checker_edge), C.c_int64(p.max_iteration),
                    C.c_double(p.confidence), C.c_uint64(p.seed), _p(T), _p(st), _p(sums))
    return Result(T.reshape(4, 4), sums[1], sums[2], int(st[5]), int(st[0]), int(st[1]), int(st[2]), bool(st[3]), int(st[4]), sums[0], sums[3])


# ---- numpy twin ----------------------------------------------------------------------------------------------------------
def np_stream(seed, h, n, j, size):
    z = (seed + ((h * n + j + 1) * GOLDEN)) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    z ^= z >> 31
    return (z * size) >> 64


def np_feature_corr(fs, ft):
    fs = np.asarray(fs, dtype=np.float64).reshape(-1, 33); ft = np.asarray(ft, dtype=np.float64).reshape(-1, 33)
    if len(fs) == 0 or len(ft) == 0:
        return np.full(len(fs), -1, dtype=np.int32), np.full(len(ft), -1, dtype=np.int32)
    d = np.zeros((len(fs), len(ft)))
    for k in range(33):                    # ascending k
        e = fs[:, None, k] - ft[None, :, k]
        d = d + e * e
    return d.argmin(axis=1).astype(np.int32), d.argmin(axis=0).astype(np.int32)   # argmin: the first minimum


def _xf(T, p):
    p = np.atleast_2d(p)
    return np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)], axis=1)


def _norm(v):
    return np.sqrt((v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2])


def _umeyama(S, Q):
    n = len(S)
    one_over_n = 1.0 / n
    ms, mt = np.zeros(3), np.zeros(3)
    for j in range(n):
        ms = ms + S[j]; mt = mt + Q[j]
    ms, mt = ms * one_over_n, mt * one_over_n
    sigma = np.zeros((3, 3))
    for j in range(n):
        sigma = sigma + np.outer(Q[j] - mt, S[j] - ms)
    sigma = sigma * one_over_n
    U, _s, V = O.svd3(sigma)
    sgn = -1.0 if np.linalg.det(U) * np.linalg.det(V) < 0 else 1.0
    R = np.array([[U[a, 0] * V[b, 0] + U[a, 1] * V[b, 1] + sgn * U[a, 2] * V[b, 2] for b in range(3)] for a in range(3)])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = mt - np.array([(R[a, 0] * ms[0] + R[a, 1] * ms[1]) + R[a, 2] * ms[2] for a in range(3)])
    return T


def np_ransac(sx, sf, tx, tf, p: Params) -> Result:
    sx = np.asarray(sx, dtype=np.float64).reshape(-1, 3); tx = np.asarray(tx, dtype=np.float64).reshape(-1, 3)
    ns, nt, n = len(sx), len(tx), p.ransac_n
    empty = Result(np.eye(4), 0.0, 0.0, 0, 0, 0, 0, False, -1, 0.0, 0.0)
    if n < 3 or not p.max_corr > 0 or ns < n or nt == 0:
        return empty
    s2t, t2s = np_feature_corr(sf, tf)
    mutual = np.nonzero(t2s[s2t] == np.arange(ns))[0] if p.mutual_filter else np.zeros(0, dtype=np.int64)
    used_mutual = bool(p.mutual_filter and len(mutual) >= 3 * n)
    cs = mutual if used_mutual else np.arange(ns)
    ct = s2t[cs]
    m = len(cs)
    r2 = p.max_corr * p.max_corr
    est_k, h, validations = p.max_iteration, 0, 0
    best = (0, 0.0, np.eye(4), -1, 0.0)
    while h < est_k:
        ks = [np_stream(p.seed, h, n, j, m) for j in range(n)]
        S, Q = sx[cs[ks]], tx[ct[ks]]
        ok = True
        for i in range(n):
            for j in range(i + 1, n):
                ds, dt = _norm(S[i] - S[j]), _norm(Q[i] - Q[j])
                if ds < dt * p.checker_edge or dt < ds * p.checker_edge:
                    ok = False
        if ok:
            T = _umeyama(S, Q)
            ok = bool((_norm(Q - _xf(T, S)) <= p.checker_distance).all())
        if ok:
            validations += 1
            q = _xf(T, sx)
            d = ((q[:, None, 0] - tx[None, :, 0]) ** 2 + (q[:, None, 1] - tx[None, :, 1]) ** 2) + (q[:, None, 2] - tx[None, :, 2]) ** 2
            dmin = d.min(axis=1)
            hit = dmin < r2
            inl = int(hit.sum())
            s = 0.0
            for v in dmin[hit]:                 # sequential, in point order
                s += float(v)
            if inl > 0 and (inl > best[0] or (inl == best[0] and s < best[1])):
                fitness = inl / ns
                with np.errstate(divide="ignore"):      # fitness 1: log(0) = -inf, k_d = -0 (as in C)
                    k_d = float(np.log(1.0 - p.confidence) / np.log(np.float64(1.0 - fitness ** n)))
                best = (inl, s, T, h, k_d)
                if k_d < est_k:
                    est_k = int(math.ceil(k_d))
        h += 1
    inl, s, T, bh, kd = best
    return Result(T, inl / ns if inl else 0.0, math.sqrt(s / inl) if inl else 0.0, inl, h, validations, m, used_mutual, bh, s, kd)
