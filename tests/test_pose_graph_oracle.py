"""CPU tests of the pose-graph restatement (tests/oracle_pose_graph.py) against independent answers: high-precision Jacobians,
LAPACK, graphs with known solutions and hand-built cases for validation, pruning, the reference node and the signed right-term check."""
import numpy as np
import pytest
import scipy.linalg as sla

import oracle_pose_graph as PG


def _mp_v2m(x):
    sa, ca, sb, cb, sg, cg = mp.sin(x[0]), mp.cos(x[0]), mp.sin(x[1]), mp.cos(x[1]), mp.sin(x[2]), mp.cos(x[2])
    return mp.matrix([[cg * cb, cg * sb * sa - sg * ca, cg * sb * ca + sg * sa, x[3]], [sg * cb, sg * sb * sa + cg * ca, sg * sb * ca - cg * sa, x[4]],
                      [-sb, cb * sa, cb * ca, x[5]], [0, 0, 0, 1]])


def _mp_lin(M):
    return [(M[2, 1] - M[1, 2]) / 2, (M[0, 2] - M[2, 0]) / 2, (M[1, 0] - M[0, 1]) / 2, M[0, 3], M[1, 3], M[2, 3]]


def test_jacobians_match_central_differences_at_50_digits():
    """Js[:, i] and Jt[:, i] are the derivatives of lin(X^-1 (V2M(d_t) Tt)^-1 V2M(d_s) Ts) in d_s[i] and d_t[i] at 0: the sign and
    ordering conventions of the generators and of the left-multiplied update"""
    global mp
    mp = pytest.importorskip("mpmath")
    rng = np.random.default_rng(3)
    Ts, Tt = PG.rigid(rng.normal(size=3), rng.normal(size=3) * 3), PG.rigid(rng.normal(size=3), rng.normal(size=3) * 3)
    X = PG.rigid(rng.normal(size=3) * 0.2, rng.normal(size=3))
    e = PG.Edge(0, 1, X, np.eye(6))
    Js, Jt = PG.jacobians(e, [Ts, Tt])
    mp.mp.dps = 50
    Xi, Tsm, Ttm = mp.matrix(PG.inv_rigid(X).tolist()), mp.matrix(Ts.tolist()), mp.matrix(Tt.tolist())
    h = mp.mpf("1e-20")

    def f(ds, dt):
        return _mp_lin(Xi * mp.inverse(_mp_v2m(dt) * Ttm) * _mp_v2m(ds) * Tsm)

    z6 = [mp.mpf(0)] * 6
    for i in range(6):
        u = list(z6); u[i] = h
        w = list(z6); w[i] = -h
        ns = [(a - b) / (2 * h) for a, b in zip(f(u, z6), f(w, z6))]
        nt = [(a - b) / (2 * h) for a, b in zip(f(z6, u), f(z6, w))]
        assert np.allclose(Js[:, i], [float(v) for v in ns], rtol=0, atol=1e-12), i
        assert np.allclose(Jt[:, i], [float(v) for v in nt], rtol=0, atol=1e-12), i
    assert np.array_equal(Jt, -Js)


@pytest.mark.parametrize("n", [6, 60, 64, 66, 130, 200])
def test_ldl_matches_lapack_on_well_conditioned_systems(n):
    rng = np.random.default_rng(n)
    A = rng.normal(size=(n, n))
    H = A @ A.T
    lam = 1e-2 * np.max(np.diag(H))
    b = rng.normal(size=n)
    ref = sla.solve(H + lam * np.eye(n), b, assume_a="pos")
    for L, d in (PG.ldl_unblocked(H + lam * np.eye(n)), PG.ldl_blocked(H + lam * np.eye(n))):
        x = PG.ldl_solve(L, d, b)
        assert np.linalg.norm(x - ref) <= 1e-10 * np.linalg.norm(ref)


def test_ldl_zero_pivot_zeroes_the_component_and_stays_finite():
    H = np.zeros((6, 6)); H[:3, :3] = np.eye(3) * 2.0
    L, d = PG.ldl_unblocked(H)
    assert np.all(d[3:] == 0.0)
    x = PG.ldl_solve(L, d, np.ones(6))
    assert np.all(np.isfinite(x)) and np.all(x[3:] == 0.0) and np.allclose(x[:3], 0.5)


def test_exact_constraints_converge_to_the_true_poses():
    """every edge exact, node 0 at its true pose and the others perturbed: the optimum is the truth (the reference node pins the
    gauge).  Tight tolerances, so that the loop runs to the bottom instead of stopping at the default 1e-6 residual"""
    truth, _, edges = PG.random_graph(12, seed=5, loop_every=4, odo_noise=0.0)
    rng = np.random.default_rng(1)
    init = [truth[0]] + [T @ PG.rigid(rng.normal(size=3) * 0.02, rng.normal(size=3) * 0.05) for T in truth[1:]]
    p = PG.Params(min_residual=1e-30, min_right_term=1e-30, min_relative_increment=1e-15, min_relative_residual_increment=1e-15)
    out, kept, _conf, st = PG.global_optimization(init, edges, p)
    assert all(kept) and st[0].valid and st[1].valid
    for T, R in zip(out, truth):
        assert np.abs(T - R).max() < 1e-9


def test_odometry_chain_returns_unchanged_through_the_right_term_check():
    truth, _, edges = PG.random_graph(10, seed=2, loop_every=100, odo_noise=0.0)
    out, kept, _conf, st = PG.global_optimization(truth, edges)
    assert st[0].stop_reason == "right_term" and st[0].outer_iterations == 0 and st[0].lm_tries == 0
    assert st[1].stop_reason == "right_term" and all(kept)
    for T, R in zip(out, truth):
        assert np.abs(T - R).max() < 1e-12


def test_outlier_loop_closure_is_pruned_and_a_true_one_survives():
    """with the Lua max_correspondence_distance (1000) lpw dwarfs every residual and nothing is ever pruned; at 0.1 (the scale of a
    point-to-plane correspondence distance) the line process separates the two"""
    truth, init, edges = PG.random_graph(24, seed=7, loop_every=8, n_outliers=0, odo_noise=0.005)
    edges.append(PG.Edge(20, 3, PG.rigid([0.3, -0.2, 0.5], [4.0, -3.0, 1.0]), PG.information(np.random.default_rng(0), 1000.0), uncertain=True))
    p = PG.Params(max_correspondence_distance=0.1)
    out, kept, conf, st = PG.global_optimization(init, edges, p)
    assert not kept[-1] and conf[-1] <= p.edge_prune_threshold
    true_loops = [k for k, e in enumerate(edges[:-1]) if e.uncertain]
    assert true_loops and all(kept[k] for k in true_loops)
    assert st[1].n_edges == len(edges) - 1
    err = max(np.linalg.norm(T[:3, 3] - R[:3, 3]) for T, R in zip(out, truth))
    err0 = max(np.linalg.norm(T[:3, 3] - R[:3, 3]) for T, R in zip(init, truth))
    assert err < err0
    out_all, kept_all, _c, _s = PG.global_optimization(init, edges)   # the Lua value: the outlier stays
    assert all(kept_all)


def test_reference_node_keeps_its_input_pose():
    truth, init, edges = PG.random_graph(16, seed=11, loop_every=5, odo_noise=0.02)
    for ref in (0, 7, 15):
        out, _k, _c, _s = PG.global_optimization(init, edges, PG.Params(reference_node=ref))
        assert np.abs(out[ref] - init[ref]).max() < 1e-12
    out, _k, _c, _s = PG.global_optimization(init, edges, PG.Params(reference_node=-1))   # out of range: no compensation
    assert np.abs(out[0] - init[0]).max() > 1e-9


def test_disconnected_graph_is_invalid_and_unchanged():
    truth, init, edges = PG.random_graph(6, seed=1, loop_every=100)
    cut = [e for e in edges if not (e.source == 2 and e.target == 3)]
    out, kept, conf, st = PG.global_optimization(init, cut)
    assert not st[0].valid and not st[1].valid and all(np.array_equal(a, b) for a, b in zip(out, init))
    # connected only through an uncertain edge: the certain-edge BFS fails
    bridged = cut + [PG.Edge(2, 3, PG.measurement(truth[2], truth[3]), np.eye(6), uncertain=True)]
    _o, _k, _c, st = PG.global_optimization(init, bridged)
    assert not st[0].valid


def test_id_out_of_range_is_an_error():
    with pytest.raises(ValueError):
        PG.global_optimization([np.eye(4)], [PG.Edge(0, 1, np.eye(4), np.eye(6))])


def star_graph(dx):
    """node 0 linked to m leaves by edges that all disagree in x by the same amount: b of node 0 is -+m g in that component, every
    leaf +-g, so with the right sign of dx the signed maximum of b is g while max |b| is m g"""
    m = 12
    poses = [np.eye(4) for _ in range(m + 1)]
    edges = [PG.Edge(0, i, PG.rigid([0, 0, 0], [dx, 0, 0]), np.eye(6) * 10.0) for i in range(1, m + 1)]
    return poses, edges


def test_right_term_uses_the_signed_maximum():
    poses, edges = star_graph(-1e-4)   # the sign that leaves the large entry of b negative, at the hub
    H, b = PG.linear_system(edges, [PG.zeta_of(e, poses) for e in edges], poses)
    thr = 3.0 * float(np.max(b))
    assert float(np.max(b)) < thr < float(np.max(np.abs(b)))
    _o, _k, _c, st = PG.global_optimization(poses, edges, PG.Params(min_right_term=thr))
    assert st[0].stop_reason == "right_term" and st[0].lm_tries == 0
    _o, _k, _c, st = PG.global_optimization(poses, edges, PG.Params(min_right_term=float(np.max(b)) / 2))
    assert st[0].lm_tries > 0
