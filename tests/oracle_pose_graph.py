"""CPU restatement of the submap pose-graph optimisation: [O3D] GlobalOptimization with GlobalOptimizationLevenbergMarquardt, as
OptimizationProblem::solve (core/src/OptimizationProblem.cpp:25-44) calls it.  The [O3D] source is not at hand; this file and
open3d_slam_b200/csrc/posegraph.cu hold the same list of rules (DESIGN.md row G1):

1. validation: edge ids in [0, N) (the C entry point returns B2S_E_INVALID); connected from node 0 over all edges and over the certain
   edges alone (BFS), else the poses stay and valid = False
2. lpw = preference_loop_closure * max_correspondence_distance^2 * mean_e information_e[5, 5], 0 without edges
3. zeta_e = lin(X^-1 Tt^-1 Ts), Js[:, i] = lin(X^-1 Tt^-1 G_i Ts), Jt = -Js; inverses are rigid ones
4. uncertain edges: conf = (lpw / (lpw + zeta' Info zeta))^2, certain ones keep theirs; residual = sum conf q + lpw (sqrt(conf) - 1)^2
5. the LM loop (below, literal)
6. two passes, pruning, reference-node compensation
7. delta by an unpivoted LDL' (|d| <= 1/DBL_MAX zeroes the component), blocked in 64-wide tiles like the device; no square root
"""
from __future__ import annotations

import sys
from dataclasses import dataclass, field

import numpy as np
import scipy.linalg as sla

TINY = 1.0 / sys.float_info.max
NB = 64
STOP_REASONS = ["none", "right_term", "relative_increment", "relative_residual_increment", "max_iteration_lm", "residual", "max_iteration"]

G = [np.array(m, dtype=np.float64).reshape(4, 4) for m in (
    [0, 0, 0, 0, 0, 0, -1, 0, 0, 1, 0, 0, 0, 0, 0, 0], [0, 0, 1, 0, 0, 0, 0, 0, -1, 0, 0, 0, 0, 0, 0, 0],
    [0, -1, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0], [0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0],
    [0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0], [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0])]


@dataclass
class Edge:
    source: int
    target: int
    T: np.ndarray
    information: np.ndarray
    uncertain: bool = False
    confidence: float = 1.0


@dataclass
class Params:
    max_correspondence_distance: float = 1000.0
    edge_prune_threshold: float = 0.2
    preference_loop_closure: float = 2.0
    reference_node: int = 0
    max_iteration: int = 100
    min_relative_increment: float = 1e-6
    min_relative_residual_increment: float = 1e-6
    min_right_term: float = 1e-6
    min_residual: float = 1e-6
    max_iteration_lm: int = 20
    upper_scale_factor: float = 2.0 / 3.0
    lower_scale_factor: float = 1.0 / 3.0


@dataclass
class PassStats:
    valid: bool = False
    n_edges: int = 0
    outer_iterations: int = 0
    lm_tries: int = 0
    accepted_steps: int = 0
    stop_reason: str = "none"
    initial_residual: float = 0.0
    final_residual: float = 0.0
    final_lambda: float = 0.0
    tries: list = field(default_factory=list)   # per try: (accepted, rho, margins of the decisions it took)


def inv_rigid(T):
    R = T[:3, :3].T
    out = np.eye(4)
    out[:3, :3] = R
    out[:3, 3] = -(R @ T[:3, 3])
    return out


def lin(M):
    return np.array([(M[2, 1] - M[1, 2]) / 2.0, (M[0, 2] - M[2, 0]) / 2.0, (M[1, 0] - M[0, 1]) / 2.0, M[0, 3], M[1, 3], M[2, 3]])


def v2m(x):
    """TransformVector6dToMatrix4d: Rz(x2) Ry(x1) Rx(x0), t = x[3:]"""
    sa, ca, sb, cb, sg, cg = np.sin(x[0]), np.cos(x[0]), np.sin(x[1]), np.cos(x[1]), np.sin(x[2]), np.cos(x[2])
    return np.array([[cg * cb, cg * sb * sa - sg * ca, cg * sb * ca + sg * sa, x[3]], [sg * cb, sg * sb * sa + cg * ca, sg * sb * ca - cg * sa, x[4]],
                     [-sb, cb * sa, cb * ca, x[5]], [0.0, 0.0, 0.0, 1.0]])


def m2v(T):
    """TransformMatrix4dToVector6d"""
    sy = np.sqrt(T[0, 0] * T[0, 0] + T[1, 0] * T[1, 0])
    if not (sy < 1e-6):
        a = (np.arctan2(T[2, 1], T[2, 2]), np.arctan2(-T[2, 0], sy), np.arctan2(T[1, 0], T[0, 0]))
    else:
        a = (np.arctan2(-T[1, 2], T[1, 1]), np.arctan2(-T[2, 0], sy), 0.0)
    return np.array([a[0], a[1], a[2], T[0, 3], T[1, 3], T[2, 3]])


def zeta_of(e: Edge, poses):
    return lin(inv_rigid(e.T) @ inv_rigid(poses[e.target]) @ poses[e.source])


def jacobians(e: Edge, poses):
    Q = inv_rigid(e.T) @ inv_rigid(poses[e.target])
    Ts = poses[e.source]
    Js = np.stack([lin(Q @ (G[i] @ Ts)) for i in range(6)], axis=1)
    Jt = np.stack([lin(Q @ (-G[i] @ Ts)) for i in range(6)], axis=1)
    return Js, Jt


def line_process_weight(edges, p: Params) -> float:
    if not edges:
        return 0.0
    return p.preference_loop_closure * p.max_correspondence_distance ** 2 * float(np.mean([e.information[5, 5] for e in edges]))


def residual(edges, zetas, lpw) -> float:
    terms = [e.confidence * float(z @ e.information @ z) + lpw * (np.sqrt(e.confidence) - 1.0) ** 2 for e, z in zip(edges, zetas)]
    return float(np.sum(terms)) if terms else 0.0


def update_confidence(edges, zetas, lpw):
    for e, z in zip(edges, zetas):
        if e.uncertain:
            e.confidence = (lpw / (lpw + float(z @ e.information @ z))) ** 2


def linear_system(edges, zetas, poses):
    n6 = 6 * len(poses)
    H = np.zeros((n6, n6))
    b = np.zeros(n6)
    for e, z in zip(edges, zetas):
        Js, Jt = jacobians(e, poses)
        c = e.confidence
        i, j = 6 * e.source, 6 * e.target
        JsI, JtI, eI = Js.T @ e.information, Jt.T @ e.information, z @ e.information
        H[i:i + 6, i:i + 6] += c * (JsI @ Js)
        H[i:i + 6, j:j + 6] += c * (JsI @ Jt)
        H[j:j + 6, i:i + 6] += c * (JtI @ Js)
        H[j:j + 6, j:j + 6] += c * (JtI @ Jt)
        b[i:i + 6] -= c * (eI @ Js)
        b[j:j + 6] -= c * (eI @ Jt)
    return H, b


# ---- item 7: the unpivoted LDL' --------------------------------------------------------------------------------------------
def ldl_unblocked(A):
    """Right-looking LDL' of the lower triangle of A (A_ik -= l_i col_k); a pivot with |d| <= 1/DBL_MAX gets l = 0.
    Returns (L unit lower, d)."""
    A = np.array(A, dtype=np.float64)
    n = A.shape[0]
    L = np.eye(n)
    d = np.zeros(n)
    for j in range(n):
        d[j] = A[j, j]
        col = A[j + 1:, j].copy()
        l = col / d[j] if abs(d[j]) > TINY else np.zeros_like(col)
        L[j + 1:, j] = l
        A[j + 1:, j + 1:] -= np.outer(l, col)
    return L, d


def ldl_blocked(A, nb: int = NB):
    """The device's blocked order: per 64-wide tile column, the diagonal tile (unblocked), the panel W = A L_KK^-T, L = W D^-1,
    the trailing update A -= W L'.  Returns (L, d)."""
    A = np.tril(np.array(A, dtype=np.float64))
    n = A.shape[0]
    L = np.eye(n)
    d = np.zeros(n)
    for k0 in range(0, n, nb):
        k1 = min(k0 + nb, n)
        Lk, dk = ldl_unblocked(A[k0:k1, k0:k1])
        L[k0:k1, k0:k1] = Lk
        d[k0:k1] = dk
        if k1 == n:
            break
        W = sla.solve_triangular(Lk, A[k1:, k0:k1].T, lower=True, unit_diagonal=True).T
        ok = np.abs(dk) > TINY
        Lp = np.where(ok[None, :], W / np.where(ok, dk, 1.0)[None, :], 0.0)
        L[k1:, k0:k1] = Lp
        A[k1:, k1:] -= W @ Lp.T
    return L, d


def ldl_solve(L, d, b):
    y = sla.solve_triangular(L, b, lower=True, unit_diagonal=True)
    ok = np.abs(d) > TINY
    z = np.where(ok, y / np.where(ok, d, 1.0), 0.0)
    return sla.solve_triangular(L.T, z, lower=False, unit_diagonal=True)


def solve_lm(H, b, lam, use_cholesky=False):
    A = H + lam * np.eye(H.shape[0])
    if use_cholesky:   # LAPACK on a well-conditioned system (large graphs, far from the tiny-pivot regime)
        return sla.cho_solve(sla.cho_factor(A, lower=True), b)
    L, d = ldl_blocked(A)
    return ldl_solve(L, d, b)


# ---- items 5 and 6 -----------------------------------------------------------------------------------------------------------
def connected(n, edges, certain_only):
    adj = [[] for _ in range(n)]
    for e in edges:
        if certain_only and e.uncertain:
            continue
        adj[e.source].append(e.target)
        adj[e.target].append(e.source)
    seen = {0}
    q = [0]
    while q:
        u = q.pop()
        for v in adj[u]:
            if v not in seen:
                seen.add(v)
                q.append(v)
    return len(seen) == n


def optimize_pass(poses, edges, p: Params, use_cholesky=False) -> PassStats:
    """GlobalOptimizationLevenbergMarquardt::OptimizePoseGraph; poses (list of 4x4) and the edges' confidences change in place"""
    st = PassStats(valid=True, n_edges=len(edges))
    lpw = line_process_weight(edges, p)
    zetas = [zeta_of(e, poses) for e in edges]
    cur = residual(edges, zetas, lpw)
    new = cur
    update_confidence(edges, zetas, lpw)
    H, b = linear_system(edges, zetas, poses)
    x = np.concatenate([m2v(T) for T in poses])
    lam = 1e-5 * float(np.max(np.diag(H)))
    nu, rho = 2.0, 0.0
    st.initial_residual = cur
    stop, reason = False, "none"

    def stop_on(cond, why):
        nonlocal stop, reason
        if not stop and cond:
            stop, reason = True, why

    stop_on(float(np.max(b)) < p.min_right_term, "right_term")
    it = 0
    while not stop and it < p.max_iteration:
        it += 1
        st.outer_iterations += 1
        lm = 0
        while True:
            delta = solve_lm(H, b, lam, use_cholesky)
            st.lm_tries += 1
            dn, thr = float(np.linalg.norm(delta)), p.min_relative_increment * (float(np.linalg.norm(x)) + p.min_relative_increment)
            stop_on(dn < thr, "relative_increment")
            rec = {"accepted": False, "rel_inc_margin": abs(dn - thr) / max(thr, 1e-300)}
            if not stop:
                trial = [v2m(delta[6 * i:6 * i + 6]) @ T for i, T in enumerate(poses)]
                zn = [zeta_of(e, trial) for e in edges]
                new = residual(edges, zn, lpw)
                den = float(delta @ (lam * delta + b)) + 1e-3
                rho = (cur - new) / den
                rec.update(rho=rho, rho_margin=abs(cur - new) / max(abs(cur), abs(new), 1e-300))
                if rho > 0:
                    rec["accepted"] = True
                    stop_on(cur - new < p.min_relative_residual_increment * cur, "relative_residual_increment")
                    rec["rel_res_margin"] = abs((cur - new) - p.min_relative_residual_increment * cur) / max(abs(cur), 1e-300)
                    alpha = min(1.0 - (2.0 * rho - 1.0) ** 3, p.upper_scale_factor)
                    lam *= max(p.lower_scale_factor, alpha)
                    nu = 2.0
                    cur = new
                    st.accepted_steps += 1
                    poses[:] = trial
                    zetas = zn
                    update_confidence(edges, zetas, lpw)
                    x = np.concatenate([m2v(T) for T in poses])
                    H, b = linear_system(edges, zetas, poses)
                    stop_on(float(np.max(b)) < p.min_right_term, "right_term")
                    st.tries.append(rec)
                    if stop:
                        break
                    lm += 1
                    stop_on(lm >= p.max_iteration_lm, "max_iteration_lm")
                    break
                else:
                    lam *= nu
                    nu *= 2.0
            st.tries.append(rec)
            lm += 1
            stop_on(lm >= p.max_iteration_lm, "max_iteration_lm")
            if rho > 0 or stop:
                break
        stop_on(new < p.min_residual, "residual")
    if not stop:
        reason = "max_iteration"
    st.stop_reason, st.final_residual, st.final_lambda = reason, cur, lam
    return st


def global_optimization(poses, edges, p: Params | None = None, use_cholesky=False):
    """GlobalOptimization.  poses: list/array of 4x4, edges: list of Edge (confidence 1 on entry).  Returns (new poses, kept flags,
    final confidences, [pass 1 stats, pass 2 stats]); a graph that fails validation returns the poses unchanged."""
    p = p or Params()
    n = len(poses)
    for e in edges:
        if not (0 <= e.source < n and 0 <= e.target < n):
            raise ValueError("edge id out of range")
    orig = [np.array(T, dtype=np.float64) for T in poses]
    edges = [Edge(e.source, e.target, np.asarray(e.T, dtype=np.float64), np.asarray(e.information, dtype=np.float64), bool(e.uncertain), 1.0)
             for e in edges]
    stats = [PassStats(), PassStats()]
    if not connected(n, edges, False) or not connected(n, edges, True):
        return orig, [True] * len(edges), [1.0] * len(edges), stats
    if not edges:
        stats[0].valid = stats[1].valid = True
        return orig, [], [], stats
    cur = [T.copy() for T in orig]
    stats[0] = optimize_pass(cur, edges, p, use_cholesky)
    kept = [(not e.uncertain) or e.confidence > p.edge_prune_threshold for e in edges]
    stats[1] = optimize_pass(cur, [e for e, k in zip(edges, kept) if k], p, use_cholesky)
    if 0 <= p.reference_node < n:
        C = orig[p.reference_node] @ inv_rigid(cur[p.reference_node])
        cur = [C @ T for T in cur]
    return cur, kept, [e.confidence for e in edges], stats


# ---- synthetic graphs with known truth (shared by the CPU and GPU tests and tools/pose_graph_bench.py) ----------------------
def rot(axis_angle):
    v = np.asarray(axis_angle, dtype=np.float64)
    t = float(np.linalg.norm(v))
    if t == 0.0:
        return np.eye(3)
    k = v / t
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * (K @ K)


def rigid(axis_angle, t):
    T = np.eye(4)
    T[:3, :3] = rot(axis_angle)
    T[:3, 3] = t
    return T


def information(rng, n_corr):
    """an SPD 6x6 with information[5, 5] close to n_corr, like GetInformationMatrixFromPointClouds's scale"""
    A = rng.normal(size=(6, 6)) * 0.3
    return n_corr * (np.eye(6) + A @ A.T / 6.0)


def measurement(Ts, Tt):
    """the exact source-to-target measurement X of an edge: zeta = lin(X^-1 Tt^-1 Ts) = 0"""
    return inv_rigid(Tt) @ Ts


def random_graph(n, seed, loop_every=8, n_outliers=0, odo_noise=0.01, loop_noise=0.0, n_corr=1000.0):
    """A random-walk trajectory (truth), odometry edges i -> i+1 with noise odo_noise (certain), a true loop closure every
    loop_every nodes back to a random earlier node (uncertain, noise loop_noise) and n_outliers uncertain edges with a wrong
    measurement.  The initial poses chain the noisy odometry from the true node 0.  Returns (truth, initial, edges)."""
    rng = np.random.default_rng(seed)
    truth = [np.eye(4)]
    for _ in range(1, n):
        truth.append(truth[-1] @ rigid(rng.normal(size=3) * 0.1, rng.normal(size=3) * 2.0))
    edges = []
    for i in range(n - 1):
        X = measurement(truth[i], truth[i + 1]) @ rigid(rng.normal(size=3) * odo_noise, rng.normal(size=3) * odo_noise)
        edges.append(Edge(i, i + 1, X, information(rng, n_corr)))
    initial = [truth[0].copy()]
    for i in range(n - 1):
        initial.append(initial[-1] @ inv_rigid(edges[i].T))
    for s in range(loop_every, n, loop_every):
        t = int(rng.integers(0, s - 1)) if s > 1 else 0
        X = measurement(truth[s], truth[t]) @ rigid(rng.normal(size=3) * loop_noise, rng.normal(size=3) * loop_noise)
        edges.append(Edge(s, t, X, information(rng, n_corr), uncertain=True))
    for _ in range(n_outliers):
        s, t = (int(v) for v in rng.choice(n, size=2, replace=False)) if n > 1 else (0, 0)
        edges.append(Edge(s, t, rigid(rng.normal(size=3) * 0.5, rng.normal(size=3) * 5.0), information(rng, n_corr), uncertain=True))
    return truth, initial, edges
