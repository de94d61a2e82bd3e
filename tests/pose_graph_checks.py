"""Accuracy checks of the pose-graph optimiser's linear algebra (posegraph.cu, DESIGN.md row G1), evaluated in np.longdouble and held to
the rounding bounds of the operations themselves, so that a failure names the tile or the component where a kernel went wrong:

- factor:  |A - L D L'| <= (M + 1) u (|L| |D| |L'|) entrywise over the lower triangle, exactly 0 where the right side is 0; reported
           per 64 x 64 tile (every tile up to M = 1536; above that the diagonal tiles, the first tile column, the last tile row and 32
           random tiles)
- solve:   |b - A delta| <= 2 (M + 1) u (|L| |D| |L'|) |delta| per component (components with a zeroed pivot are reported apart: their
           delta must be exactly 0)
- forward: |delta - x| / |x| <= 2 g M u kappa_inf(A) against an independent solution x (mpmath at 40 digits for 6N <= 66, LAPACK
           LU plus three steps of long-double iterative refinement above), g = ||(|L| |D| |L'|)||_inf / ||A||_inf the growth
- assembly: H, b and the confidences against a long-double evaluation of the restatement's linear_system, bounded by 64 u times
           the running magnitudes of the same sums (conf |J|' |Info| |J| and conf (|Info| |zeta|)' |J|, |J| and |zeta| carried
           through the products with absolute values)

u = 2^-53, M the padded size (a multiple of 64).  Each check returns the worst ratio to its bound (<= 1 passes) and where it is.
The matrix families the tests run (dense SPD at a given condition number, pose-graph H + lambda I, quasi-definite, decoupled rows
at the zero-pivot threshold) are built here too."""
from __future__ import annotations

import math
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import scipy.linalg as sla

import oracle_pose_graph as PG

U = 2.0 ** -53
LD = np.longdouble
NB = PG.NB
TINY = PG.TINY
NEXT_TINY = float(np.nextafter(TINY, 1.0))
FULL_TILE_CHECK_MAX = 1536
_POOL = ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1))   # long-double matmuls release the GIL


def padded(n6: int) -> int:
    return NB * ((n6 + NB - 1) // NB)


def sym_from_lower(A):
    """the symmetric matrix the device factors: its lower triangle, mirrored"""
    Lw = np.tril(A)
    return Lw + np.tril(A, -1).T


# ---- factor -----------------------------------------------------------------------------------------------------------------
def factor_tiles(n6: int, rng=None):
    nt = (n6 + NB - 1) // NB
    if padded(n6) <= FULL_TILE_CHECK_MAX:
        return [(i, j) for i in range(nt) for j in range(i + 1)]
    rng = rng or np.random.default_rng(0)
    sel = {(i, i) for i in range(nt)} | {(i, 0) for i in range(nt)} | {(nt - 1, j) for j in range(nt)}
    while len(sel) < nt + 2 * nt - 2 + 32:
        i = int(rng.integers(0, nt)); sel.add((i, int(rng.integers(0, i + 1))))
    return sorted(sel)


def _tile_ratio(A, L, d, I, J, M):
    n6 = A.shape[0]
    r0, r1, c0, c1 = NB * I, min(NB * I + NB, n6), NB * J, min(NB * J + NB, n6)
    Lr, Lc, dd = L[r0:r1, :c1].astype(LD), L[c0:c1, :c1].astype(LD), d[:c1].astype(LD)
    P = (Lr * dd) @ Lc.T
    Pa = (np.abs(Lr) * np.abs(dd)) @ np.abs(Lc).T
    R = np.abs(A[r0:r1, c0:c1].astype(LD) - P)
    if I == J:
        keep = np.tril(np.ones(R.shape, dtype=bool))
        R, Pa = np.where(keep, R, 0), np.where(keep, Pa, 0)
    bound = (M + 1) * LD(U) * Pa
    if np.any((bound == 0) & (R != 0)):
        return math.inf
    with np.errstate(invalid="ignore", divide="ignore"):
        q = np.where(bound > 0, R / np.where(bound > 0, bound, 1), 0)
    return float(q.max()) if q.size else 0.0


def factor_check(A, L, d, tiles=None):
    """worst |A - L D L'| / ((M + 1) u |L||D||L'|) over the lower triangle of the chosen tiles, and that tile (I, J)"""
    n6 = A.shape[0]
    M = padded(n6)
    tiles = tiles if tiles is not None else factor_tiles(n6)
    ratios = list(_POOL.map(lambda t: _tile_ratio(A, L, d, t[0], t[1], M), tiles))
    k = int(np.argmax(ratios))
    return ratios[k], tiles[k]


# ---- solve ------------------------------------------------------------------------------------------------------------------
def _ld_matvec(A, x, rows=512):
    xl = np.asarray(x).astype(LD)
    parts = _POOL.map(lambda r: A[r:r + rows].astype(LD) @ xl, range(0, A.shape[0], rows))
    return np.concatenate(list(parts))


def zeroed_pivots(d):
    return np.abs(d) <= TINY


def solve_check(A, L, d, b, delta):
    """worst |b - A delta| / (2 (M + 1) u (|L||D||L'|)|delta|) over the components whose pivot is not zeroed, that component, and
    the largest |delta| over the zeroed ones (must be 0)"""
    n6 = A.shape[0]
    M = padded(n6)
    r = np.abs(b.astype(LD) - _ld_matvec(A, delta))
    aL = np.abs(L)
    bound = 2 * (M + 1) * U * (aL @ (np.abs(d) * (aL.T @ np.abs(delta))))
    z = zeroed_pivots(d)
    bad = (bound == 0) & (r != 0) & ~z
    with np.errstate(invalid="ignore", divide="ignore"):
        q = np.where(bound > 0, r / np.where(bound > 0, bound, 1).astype(LD), 0).astype(np.float64)
    q[z] = 0.0
    q[bad] = math.inf
    k = int(np.argmax(q))
    return float(q[k]), k, float(np.max(np.abs(delta[z]))) if z.any() else 0.0


# ---- forward error ----------------------------------------------------------------------------------------------------------
MPMATH_MAX = 66


def reference_solution(A, b):
    """(x, kappa_inf(A)): mpmath at 40 digits up to 6N = 66, else LAPACK LU and three long-double refinement steps"""
    n = A.shape[0]
    if n <= MPMATH_MAX:
        import mpmath
        with mpmath.workdps(40):
            Am = mpmath.matrix(A.tolist())
            x = mpmath.lu_solve(Am, mpmath.matrix(b.tolist()))
            Ai = mpmath.inverse(Am)
            kappa = float(mpmath.mnorm(Am, "inf") * mpmath.mnorm(Ai, "inf"))
        return np.array([float(v) for v in x]), kappa
    lu = sla.lu_factor(A, check_finite=False)
    x = sla.lu_solve(lu, b).astype(LD)
    bl = b.astype(LD)
    for _ in range(3):
        res = bl - _ld_matvec(A, x)
        x = x + sla.lu_solve(lu, res.astype(np.float64)).astype(LD)
    anorm = float(np.abs(A).sum(axis=1).max())
    if n <= FULL_TILE_CHECK_MAX:
        kappa = anorm * float(np.abs(sla.lu_solve(lu, np.eye(n))).sum(axis=1).max())
    else:   # LAPACK's estimate of the 1-norm condition number of A' (A is symmetric: the same as kappa_inf(A))
        rc, _info = sla.lapack.dgecon(lu[0], anorm, norm="I")
        kappa = 1.0 / rc
    return x.astype(np.float64), kappa


def forward_check(A, L, d, delta, x, kappa, idx=None):
    """|delta - x|_inf / |x|_inf over idx, in units of 2 g M u kappa"""
    idx = np.arange(A.shape[0]) if idx is None else idx
    M = padded(A.shape[0])
    g = _growth(A, L, d)
    err = float(np.max(np.abs(delta[idx] - x[idx]))) / max(float(np.max(np.abs(x[idx]))), 1e-300)
    return err / (2.0 * g * M * U * kappa)


def _growth(A, L, d):
    aL = np.abs(L)
    s = aL @ (np.abs(d) * (aL.T @ np.ones(A.shape[0])))
    return max(1.0, float(s.max()) / float(np.abs(A).sum(axis=1).max()))


def check_solution(family, L, d, delta, A, b):
    """the factor, solve and forward checks plus the decoupled rows' exact rules; returns the metrics"""
    fr, tile = factor_check(A, L, d)
    sr, comp, zmax = solve_check(A, L, d, b, delta)
    n6 = A.shape[0]
    keep = np.ones(n6, dtype=bool)
    exact_ok = True
    if family in ("zero-pivot", "next-pivot"):
        rows = decoupled_rows(n6)
        keep[rows] = False
        for r in rows:
            if family == "zero-pivot":
                exact_ok &= delta[r] == 0.0 and not np.any(L[r + 1:, r])
            else:
                exact_ok &= delta[r] == b[r] / A[r, r]
    idx = np.flatnonzero(keep)
    fw = 0.0
    if idx.size:
        As = A[np.ix_(idx, idx)]
        x, kappa = reference_solution(As, b[idx])
        fw = forward_check(As, L[np.ix_(idx, idx)], d[idx], delta[idx], x, kappa)
    return dict(factor=fr, tile=tile, solve=sr, comp=comp, zero_delta=zmax, exact=bool(exact_ok), forward=fw)


def passes(m):
    return m["factor"] <= 1 and m["solve"] <= 1 and m["forward"] <= 1 and m["zero_delta"] == 0 and m["exact"]


# ---- matrix families --------------------------------------------------------------------------------------------------------
def _reflect(A, v):
    """(I - 2 v v') A (I - 2 v v'), |v| = 1"""
    w = A @ v
    s = float(v @ w)
    return A - 2.0 * np.outer(v, w) - 2.0 * np.outer(w, v) + 4.0 * s * np.outer(v, v)


def dense_spd(n, kappa, seed, reflectors=3):
    """Q diag(ev) Q' with ev geometric from 1 to 1/kappa (shuffled) and Q a product of random Householder reflectors: dense, every
    entry nonzero, eigenvalues known"""
    rng = np.random.default_rng(seed)
    ev = np.geomspace(1.0, 1.0 / kappa, n) if n > 1 else np.array([1.0])
    A = np.diag(rng.permutation(ev))
    for _ in range(reflectors if n > 1 else 0):
        v = rng.normal(size=n)
        A = _reflect(A, v / np.linalg.norm(v))
    return (A + A.T) / 2.0


def quasi_definite(n, p, seed):
    """[[A, B], [B', -C]] with A (p x p) and C SPD at condition 1e2 and B dense: unpivoted LDL' exists and is stable, the pivots
    change sign at row p"""
    rng = np.random.default_rng(seed)
    K = np.zeros((n, n))
    K[:p, :p] = dense_spd(p, 1e2, seed + 1)
    K[p:, p:] = -dense_spd(n - p, 1e2, seed + 2)
    B = rng.normal(size=(p, n - p)) * (0.5 / math.sqrt(max(n, 1)))
    K[:p, p:] = B
    K[p:, :p] = B.T
    return K


def decoupled_rows(n6):
    return sorted({r for r in (0, 63, 64, 127, n6 - 1) if r < n6})


def decoupled(n, pivot, seed):
    """dense SPD (condition 1e2) with rows / columns 0, 63, 64, 127 and n - 1 replaced by `pivot` on the diagonal and 0 elsewhere"""
    A = dense_spd(n, 1e2, seed)
    for r in decoupled_rows(n):
        A[r, :] = 0.0
        A[:, r] = 0.0
        A[r, r] = pivot
    return A


def graph_system(N, seed):
    """(H, b, lambda0) of PG.random_graph at its initial poses (confidences 1), lambda0 = 1e-5 max diag H where LM starts"""
    _t, init, edges = PG.random_graph(N, seed, loop_every=8 if N > 8 else max(N - 1, 1), odo_noise=0.01, loop_noise=0.002)
    if N == 1:
        edges = [PG.Edge(0, 0, PG.rigid([0.01, 0, 0], [0.1, 0, 0]), PG.information(np.random.default_rng(seed), 100.0), uncertain=True)]
        init = [PG.rigid([0.02, -0.01, 0.03], [0.4, 0.1, -0.2])]
    H, b = PG.linear_system(edges, [PG.zeta_of(e, init) for e in edges], init)
    if N == 1:   # a self-loop's four blocks cancel: H is rounding noise, and lambda = 1 makes the system the identity
        return H, b, 1.0
    return H, b, 1e-5 * float(np.max(np.diag(H)))


FAMILIES = ("spd-1e2", "spd-1e8", "graph", "qd-edge", "qd-inside", "zero-pivot", "next-pivot")


def family_system(family, N, seed=0):
    """(A, b, lambda): the device factors lower(A) + lambda I"""
    n6 = 6 * N
    rng = np.random.default_rng(1000 * N + seed)
    if family == "graph":
        return graph_system(N, seed + N)
    if family.startswith("spd"):
        A = dense_spd(n6, float(family[4:]), seed + N)
    elif family.startswith("qd"):
        if family == "qd-edge":
            p = NB * max(1, (n6 // 2) // NB) if n6 > NB else n6 // 2
        else:
            p = min(n6 - 1, NB * ((n6 // 2) // NB) + 37) if n6 > NB else max(1, n6 // 2 + 1)
        A = quasi_definite(n6, max(1, min(p, n6 - 1)) if n6 > 1 else 1, seed + N)
    else:
        A = decoupled(n6, TINY if family == "zero-pivot" else NEXT_TINY, seed + N)
    b = rng.normal(size=n6)
    if family in ("zero-pivot", "next-pivot"):
        b[decoupled_rows(n6)] = 1e-300 * (1.0 + rng.random(len(decoupled_rows(n6))))   # b / d stays finite for the next pivot
    return A, b, 0.0


# ---- graphs for the assembly checks -----------------------------------------------------------------------------------------
def odd_graph(seed=3, N=12):
    """parallel edges in both orientations, self-loops on interior nodes, a loop closure source > target, uncertain edges with
    zeta = 0 and with a huge zeta, nodes 5 km from the origin"""
    rng = np.random.default_rng(seed)
    truth, init, edges = PG.random_graph(N, seed, loop_every=5, odo_noise=0.01)
    off = PG.rigid([0, 0, 0], [3000.0, -4000.0, 0.0])
    init = [off @ T for T in init]
    truth = [off @ T for T in truth]
    info = lambda: PG.information(rng, 500.0)
    edges += [PG.Edge(3, 7, PG.measurement(truth[3], truth[7]) @ PG.rigid([0.01, 0, 0], [0.02, 0, 0]), info()),
              PG.Edge(7, 3, PG.measurement(truth[7], truth[3]), info()),
              PG.Edge(3, 7, PG.measurement(truth[3], truth[7]), info(), uncertain=True),
              PG.Edge(5, 5, PG.rigid([0.02, 0.01, 0], [0.1, 0, 0.05]), info()),
              PG.Edge(8, 8, PG.rigid([0, 0.01, 0], [0, 0.2, 0]), info(), uncertain=True),
              PG.Edge(9, 2, PG.measurement(init[9], init[2]), info(), uncertain=True),            # zeta = 0 at the initial poses
              PG.Edge(10, 1, PG.rigid([1.0, -2.0, 0.5], [5e3, 2e3, -1e3]), info(), uncertain=True)]   # huge zeta
    return init, edges


# ---- assembly -----------------------------------------------------------------------------------------------------------------
def _inv_rigid_ld(T):
    R = T[:3, :3].T
    out = np.zeros((4, 4), dtype=T.dtype)
    out[:3, :3] = R
    out[:3, 3] = -(R @ T[:3, 3])
    out[3, 3] = 1
    return out


def _inv_rigid_abs(T):
    R = np.abs(T[:3, :3].T)
    out = np.zeros((4, 4))
    out[:3, :3] = R
    out[:3, 3] = R @ np.abs(T[:3, 3])
    out[3, 3] = 1
    return out


def _lin_abs(M):
    return np.array([(M[2, 1] + M[1, 2]) / 2.0, (M[0, 2] + M[2, 0]) / 2.0, (M[1, 0] + M[0, 1]) / 2.0, M[0, 3], M[1, 3], M[2, 3]])


def m2v_ld(T):
    sy = np.sqrt(T[0, 0] * T[0, 0] + T[1, 0] * T[1, 0])
    if not (sy < 1e-6):
        a = (np.arctan2(T[2, 1], T[2, 2]), np.arctan2(-T[2, 0], sy), np.arctan2(T[1, 0], T[0, 0]))
    else:
        a = (np.arctan2(-T[1, 2], T[1, 1]), np.arctan2(-T[2, 0], sy), LD(0))
    return np.array([a[0], a[1], a[2], T[0, 3], T[1, 3], T[2, 3]], dtype=LD)


def linearize_reference(poses, edges, lpw, conf_in):
    """The restatement's residual, UpdateConfidence and linear_system in long double, with the running magnitudes of every sum.
    Returns dict(res, res_abs, conf, conf_abs, H, H_abs, b, b_abs, xx)."""
    N = len(poses)
    n6 = 6 * N
    P = [np.asarray(T, dtype=LD) for T in poses]
    Pa = [np.abs(np.asarray(T, dtype=np.float64)) for T in poses]
    G = [g.astype(LD) for g in PG.G]
    H = np.zeros((n6, n6), dtype=LD); Ha = np.zeros((n6, n6))
    b = np.zeros(n6, dtype=LD); ba = np.zeros(n6)
    conf = np.array(conf_in, dtype=np.float64).copy(); conf_a = np.zeros(len(edges))
    res = LD(0); res_a = 0.0
    lpw_l = LD(lpw)
    for k, e in enumerate(edges):
        Info = np.asarray(e.information, dtype=LD); Ia = np.abs(np.asarray(e.information, dtype=np.float64))
        Q = _inv_rigid_ld(np.asarray(e.T, dtype=LD)) @ _inv_rigid_ld(P[e.target])
        Qa = _inv_rigid_abs(np.asarray(e.T)) @ _inv_rigid_abs(np.asarray(poses[e.target]))
        Ts, Tsa = P[e.source], Pa[e.source]
        z = PG.lin(Q @ Ts).astype(LD)
        za = _lin_abs(Qa @ Tsa)
        q = z @ Info @ z
        qa = 2.0 * float(za @ Ia @ za)
        c_in = LD(conf_in[k])
        res += c_in * q + lpw_l * (np.sqrt(c_in) - 1) ** 2
        res_a += float(c_in) * qa + lpw * (math.sqrt(conf_in[k]) + 1.0) ** 2
        c, rel = c_in, 0.0
        if e.uncertain:
            c = (lpw_l / (lpw_l + q)) ** 2
            rel = 2.0 * qa / (lpw + float(q)) if lpw + float(q) > 0 else 0.0
        conf[k] = float(c)
        conf_a[k] = float(c) * (1.0 + rel)
        Js = np.stack([PG.lin(Q @ (G[i] @ Ts)) for i in range(6)], axis=1).astype(LD)
        Jsa = np.stack([_lin_abs(Qa @ (np.abs(PG.G[i]) @ Tsa)) for i in range(6)], axis=1)
        Hss = c * (Js.T @ Info @ Js)
        Hsa = conf_a[k] * (Jsa.T @ Ia @ Jsa)
        g = c * (z @ Info @ Js)
        gav = conf_a[k] * ((Ia @ za) @ Jsa)
        i, j = 6 * e.source, 6 * e.target
        for (r, s, sign) in ((i, i, 1), (i, j, -1), (j, i, -1), (j, j, 1)):
            H[r:r + 6, s:s + 6] += sign * Hss
            Ha[r:r + 6, s:s + 6] += Hsa
        b[i:i + 6] -= g
        b[j:j + 6] += g
        ba[i:i + 6] += gav
        ba[j:j + 6] += gav
    xx = sum(float(np.sum(m2v_ld(T) ** 2)) for T in P)
    return dict(res=float(res), res_abs=res_a, conf=conf, conf_abs=conf_a, H=H, H_abs=Ha, b=b, b_abs=ba, xx=xx)


def assembly_check(ref, conf, H, b, rec=None):
    """worst ratio to 64 u times the running magnitude, over the confidences, lower(H), b and (optionally) the record
    (residual at conf_in, signed max b, max diag H, |x|^2).  Returns dict name -> ratio (<= 1 passes)."""
    tol = 64.0 * U

    def ratio(got, want, mag):
        d = np.abs(np.asarray(got, dtype=LD) - np.asarray(want, dtype=LD)).astype(np.float64)
        bound = tol * np.asarray(mag, dtype=np.float64)
        if np.any((bound == 0) & (d != 0)):
            return math.inf
        return float(np.max(np.where(bound > 0, d / np.where(bound > 0, bound, 1.0), 0.0), initial=0.0))

    low = np.tril(np.ones(H.shape, dtype=bool))
    out = {"conf": ratio(conf, ref["conf"], ref["conf_abs"]),
           "H": ratio(np.where(low, H, 0), np.where(low, ref["H"], 0), np.where(low, ref["H_abs"], 0)),
           "b": ratio(b, ref["b"], ref["b_abs"])}
    if rec is not None:
        n6 = H.shape[0]
        out["res"] = ratio(rec[0], ref["res"], ref["res_abs"])
        out["maxb"] = ratio(rec[1], np.max(ref["b"]), np.max(ref["b_abs"]))
        out["maxdiag"] = ratio(rec[2], np.max(np.diag(ref["H"])), np.max(np.diag(ref["H_abs"])[:n6]))
        out["xx"] = ratio(rec[3], ref["xx"], 4.0 * ref["xx"] + 1e-300)
    return out
