"""CPU self-test of tests/pose_graph_checks.py: the restatement's blocked LDL' (ldl_blocked / ldl_solve, and the device's tiled
substitution order) and its linear_system pass every check on every matrix and graph family the GPU tests use, and numpy mutants
of them -- one kernel detail each, as a kernel could get it wrong -- are rejected.  Each rejection prints its margin."""
import math

import numpy as np
import pytest
import scipy.linalg as sla

import oracle_pose_graph as PG
import pose_graph_checks as PC

NB = PG.NB
SIZES = [1, 10, 11, 21, 22, 32, 33, 64]


# ---- the restatement with one detail changed (mutant=None: the restatement itself) ---------------------------------------------
def ldl_blocked(A, mutant=None):
    tiny_ok = (lambda d: np.abs(d) >= PG.TINY) if mutant == "zero-pivot-ge" else (lambda d: np.abs(d) > PG.TINY)
    A = np.tril(np.array(A, dtype=np.float64))
    n = A.shape[0]
    L, d = np.eye(n), np.zeros(n)
    for k0 in range(0, n, NB):
        k1 = min(k0 + NB, n)
        T = A[k0:k1, k0:k1].copy()
        Lk = np.eye(k1 - k0)
        for j in range(k1 - k0):
            d[k0 + j] = T[j, j]
            col = T[j + 1:, j].copy()
            l = col / T[j, j] if tiny_ok(T[j, j]) else np.zeros_like(col)
            Lk[j + 1:, j] = l
            T[j + 1:, j + 1:] -= np.outer(l, col)
        L[k0:k1, k0:k1] = Lk
        if k1 == n:
            break
        dk = d[k0:k1]
        W = sla.solve_triangular(Lk, A[k1:, k0:k1].T, lower=True, unit_diagonal=True).T
        ok = tiny_ok(dk)
        piv = np.roll(dk, 1) if mutant == "panel-wrong-pivot" else dk
        Lp = np.where(ok[None, :], W / np.where(ok, piv, 1.0)[None, :], 0.0)
        L[k1:, k0:k1] = Lp
        if mutant in ("skip-trailing-tile", "wj-li"):   # tile by tile; (2, 1) of the first trailing matrix is the odd one
            m = (n - k1 + NB - 1) // NB
            for I in range(m):
                for J in range(I + 1):
                    r, c = slice(k1 + NB * I, k1 + NB * I + NB), slice(k1 + NB * J, k1 + NB * J + NB)
                    wr, lc = slice(NB * I, NB * I + NB), slice(NB * J, NB * J + NB)
                    odd = k0 == 0 and (I, J) == (2, 1)
                    if odd and mutant == "skip-trailing-tile":
                        continue
                    if odd and mutant == "wj-li":
                        A[r, c] -= W[lc] @ Lp[wr].T
                    else:
                        A[r, c] -= W[wr] @ Lp[lc].T
            A = np.tril(A)
        else:
            A[k1:, k1:] -= W @ Lp.T
    return L, d


def ldl_solve_tiled(L, d, b, mutant=None):
    """K-pg-fwd / K-pg-bwd's order: per tile, the diagonal solve, then the update of the other tiles' right-hand sides"""
    tiny_ok = (lambda v: np.abs(v) >= PG.TINY) if mutant == "zero-pivot-ge" else (lambda v: np.abs(v) > PG.TINY)
    n = len(b)
    y = np.array(b, dtype=np.float64)
    for k0 in range(0, n, NB):
        k1 = min(k0 + NB, n)
        yk = sla.solve_triangular(L[k0:k1, k0:k1], y[k0:k1], lower=True, unit_diagonal=True)
        y[k1:] -= L[k1:, k0:k1] @ (y[k0:k1] if mutant == "fwd-rhs" else yk)
        y[k0:k1] = yk
    ok = tiny_ok(d)
    x = np.where(ok, y / np.where(ok, d, 1.0), 0.0)
    for k0 in reversed(range(0, n, NB)):
        k1 = min(k0 + NB, n)
        xk = sla.solve_triangular(L[k0:k1, k0:k1].T, x[k0:k1], lower=False, unit_diagonal=True)
        x[k0:k1] = xk
        for j0 in range(0, k0, NB):
            blk = L[k0:k1, j0:j0 + NB]
            x[j0:j0 + NB] -= (blk @ xk) if mutant == "bwd-untransposed" else (blk.T @ xk)
    return x


def linear_system(edges, zetas, poses, mutant=None):
    n6 = 6 * len(poses)
    H, b = np.zeros((n6, n6)), np.zeros(n6)
    seen = set()
    for e, z in zip(edges, zetas):
        Js, Jt = PG.jacobians(e, poses)
        c = e.confidence
        i, j = 6 * e.source, 6 * e.target
        JsI, JtI, eI = Js.T @ e.information, Jt.T @ e.information, z @ e.information
        cross = 1.0
        if mutant == "cross-sign" and e.source > e.target:
            cross = -1.0
        pair = (min(e.source, e.target), max(e.source, e.target))
        first = pair not in seen
        seen.add(pair)
        H[i:i + 6, i:i + 6] += c * (JsI @ Js)
        if mutant == "parallel-first-only" and not first and e.source != e.target:
            pass
        elif mutant == "self-loop-once" and e.source == e.target:
            H[i:i + 6, j:j + 6] += cross * c * (JsI @ Jt)
        else:
            H[i:i + 6, j:j + 6] += cross * c * (JsI @ Jt)
            H[j:j + 6, i:i + 6] += cross * c * (JtI @ Js)
        H[j:j + 6, j:j + 6] += c * (JtI @ Jt)
        b[i:i + 6] -= c * (eI @ Js)
        b[j:j + 6] -= c * (eI @ Jt)
    return H, b


# ---- assembly helpers ---------------------------------------------------------------------------------------------------------
def lpw_of(edges, p=PG.Params(max_correspondence_distance=0.1)):
    return PG.line_process_weight(edges, p)


def restatement_linearize(poses, edges, lpw, mutant=None):
    es = [PG.Edge(e.source, e.target, e.T, e.information, e.uncertain, 1.0) for e in edges]
    zetas = [PG.zeta_of(e, poses) for e in es]
    PG.update_confidence(es, zetas, lpw)
    H, b = linear_system(es, zetas, poses, mutant)
    return np.array([e.confidence for e in es]), H, b


# ---- tests ----------------------------------------------------------------------------------------------------------------------
def test_mutant_free_copies_are_the_restatement():
    A, b, lam = PC.family_system("spd-1e2", 22)
    L0, d0 = PG.ldl_blocked(A)
    L1, d1 = ldl_blocked(A)
    assert np.array_equal(L0, L1) and np.array_equal(d0, d1)
    init, edges = PC.odd_graph()
    lpw = lpw_of(edges)
    c0, H0, b0 = restatement_linearize(init, edges, lpw)
    es = [PG.Edge(e.source, e.target, e.T, e.information, e.uncertain, 1.0) for e in edges]
    zetas = [PG.zeta_of(e, init) for e in es]
    PG.update_confidence(es, zetas, lpw)
    H1, b1 = PG.linear_system(es, zetas, init)
    assert np.array_equal(H0, H1) and np.array_equal(b0, b1)


@pytest.mark.parametrize("family", PC.FAMILIES)
def test_restatement_passes_every_check(family):
    worst = {"factor": 0.0, "solve": 0.0, "forward": 0.0}
    for N in SIZES:
        A, b, lam = PC.family_system(family, N)
        A = PC.sym_from_lower(A) + lam * np.eye(A.shape[0])
        L, d = PG.ldl_blocked(A)
        for delta in (PG.ldl_solve(L, d, b), ldl_solve_tiled(L, d, b)):
            m = PC.check_solution(family, L, d, delta, A, b)
            assert PC.passes(m), (family, N, m)
            for k in worst:
                worst[k] = max(worst[k], m[k])
    print(f"{family}: worst factor {worst['factor']:.3g}, solve {worst['solve']:.3g}, forward {worst['forward']:.3g} (units of the bound)")


@pytest.mark.parametrize("mutant,family,N", [
    ("skip-trailing-tile", "spd-1e2", 64), ("wj-li", "spd-1e2", 64), ("panel-wrong-pivot", "graph", 22),
    ("zero-pivot-ge", "zero-pivot", 32), ("fwd-rhs", "spd-1e2", 32), ("bwd-untransposed", "spd-1e2", 32)])
def test_checks_reject_factor_and_solve_mutants(mutant, family, N):
    A, b, lam = PC.family_system(family, N)
    A = PC.sym_from_lower(A) + lam * np.eye(A.shape[0])
    L, d = ldl_blocked(A, mutant if mutant in ("skip-trailing-tile", "wj-li", "panel-wrong-pivot", "zero-pivot-ge") else None)
    delta = ldl_solve_tiled(L, d, b, mutant if mutant in ("fwd-rhs", "bwd-untransposed", "zero-pivot-ge") else None)
    m = PC.check_solution(family, L, d, delta, A, b)
    assert not PC.passes(m), m
    print(f"{mutant}: factor {m['factor']:.3g} at tile {m['tile']}, solve {m['solve']:.3g} at {m['comp']}, forward {m['forward']:.3g}, "
          f"zeroed-pivot |delta| {m['zero_delta']:.3g}, exact rules {'hold' if m['exact'] else 'broken'}")


def test_restatement_assembly_passes():
    init, edges = PC.odd_graph()
    lpw = lpw_of(edges)
    conf, H, b = restatement_linearize(init, edges, lpw)
    ref = PC.linearize_reference(init, edges, lpw, [1.0] * len(edges))
    r = PC.assembly_check(ref, conf, H, b)
    print("restatement assembly (units of the bound):", {k: f"{v:.3g}" for k, v in r.items()})
    assert max(r.values()) <= 1, r
    assert any(e.source > e.target for e in edges) and any(e.source == e.target for e in edges)


@pytest.mark.parametrize("mutant", ["cross-sign", "parallel-first-only", "self-loop-once"])
def test_checks_reject_assembly_mutants(mutant):
    init, edges = PC.odd_graph()
    lpw = lpw_of(edges)
    conf, H, b = restatement_linearize(init, edges, lpw, mutant)
    ref = PC.linearize_reference(init, edges, lpw, [1.0] * len(edges))
    r = PC.assembly_check(ref, conf, H, b)
    print(f"{mutant}: worst H {r['H']:.3g}, b {r['b']:.3g} (units of the bound)")
    assert r["H"] > 1 and math.isfinite(r["b"])
