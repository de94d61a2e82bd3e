"""GPU tests of the pose-graph optimiser's kernels one by one (posegraph.cu, DESIGN.md row G1) through b2s_debug_pose_graph_solve and
b2s_debug_pose_graph_linearize, which run the production launches on given inputs:

- the blocked LDL' (K-pg-form, K-pg-diag, K-pg-panel, K-pg-trailing) and the substitutions (K-pg-fwd, K-pg-bwd) against the rounding
  bounds of tests/pose_graph_checks.py at N = 1 ... 1000 (1 to 94 tiles, 0 to 62 padding rows) on dense SPD, pose-graph, quasi-definite
  and zero-pivot matrices; the worst factor / solve / forward metric is printed per family and size
- K-pg-edge, K-pg-assemble and K-pg-reduce-lin against a long-double restatement at the edge-count, layout and pose edges
- the hooks against b2s_global_optimization itself, and bit-identical repeats"""
import ctypes as C

import numpy as np
import pytest

import oracle_pose_graph as PG
import pose_graph_checks as PC
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E

pytestmark = pytest.mark.gpu

SIZES = [1, 10, 11, 21, 22, 32, 33, 64, 75, 128, 171, 256, 500, 1000]


@pytest.fixture(scope="module")
def eng(engine_factory):
    return engine_factory()


def _pd(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def dev_solve(eng, A, b, lam, factors=True):
    """delta, D and L of lower(A) + lam I from the device"""
    n6 = A.shape[0]
    A = np.ascontiguousarray(A, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    delta, d = np.zeros(n6), np.zeros(n6)
    Lf = np.zeros((n6, n6)) if factors else None
    L.check(L.lib().b2s_debug_pose_graph_solve(eng._h, C.c_int32(n6 // 6), _pd(A), _pd(b), C.c_double(lam), _pd(delta),
                                               _pd(d) if factors else None, _pd(Lf) if factors else None))
    return delta, d, Lf


def edge_array(edges):
    arr = (L.PoseGraphEdge * max(len(edges), 1))()
    for k, e in enumerate(edges):
        arr[k].source, arr[k].target, arr[k].uncertain = int(e.source), int(e.target), int(bool(e.uncertain))
        arr[k].T[:] = np.asarray(e.T, dtype=np.float64).ravel().tolist()
        arr[k].information[:] = np.asarray(e.information, dtype=np.float64).ravel().tolist()
    return arr


def go_params(p: PG.Params):
    q = L.GlobalOptimizationParams()
    L.lib().b2s_default_global_optimization_params(C.byref(q))
    q.max_correspondence_distance, q.edge_prune_threshold = p.max_correspondence_distance, p.edge_prune_threshold
    q.preference_loop_closure, q.reference_node = p.preference_loop_closure, p.reference_node
    return q


def dev_linearize(eng, poses, edges, p: PG.Params, conf_in):
    N, ne = len(poses), len(edges)
    P = np.ascontiguousarray(np.stack([np.asarray(T, dtype=np.float64) for T in poses]))
    cin = np.ascontiguousarray(np.asarray(conf_in, dtype=np.float64).reshape(-1) if ne else np.zeros(1))
    cout = np.zeros(max(ne, 1))
    H, b, rec = np.zeros((6 * N, 6 * N)), np.zeros(6 * N), np.zeros(4)
    q = go_params(p)
    L.check(L.lib().b2s_debug_pose_graph_linearize(eng._h, C.c_int32(N), _pd(P), C.c_int32(ne), edge_array(edges), C.byref(q), _pd(cin),
                                                   _pd(cout), _pd(H), _pd(b), _pd(rec)))
    return cout[:ne], H, b, rec


# ---- factorisation and substitution --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", PC.FAMILIES)
def test_factor_and_solve_within_rounding_bounds(eng, family):
    worst = {"factor": 0.0, "solve": 0.0, "forward": 0.0}
    for N in SIZES:
        A, b, lam = PC.family_system(family, N)
        delta, d, Lf = dev_solve(eng, A, b, lam)
        As = PC.sym_from_lower(A) + lam * np.eye(A.shape[0])
        m = PC.check_solution(family, Lf, d, delta, As, b)
        print(f"{family} N={N} M={PC.padded(6 * N)}: factor {m['factor']:.3g} (tile {m['tile']}), solve {m['solve']:.3g} "
              f"(component {m['comp']}), forward {m['forward']:.3g}, negative pivots {int(np.sum(d < 0))}")
        assert np.all(np.isfinite(delta)) and PC.passes(m), (family, N, m)
        for k in worst:
            worst[k] = max(worst[k], m[k])
    print(f"{family}: worst factor {worst['factor']:.3g}, solve {worst['solve']:.3g}, forward {worst['forward']:.3g} (units of the bound)")


def test_decoupled_pivots_match_the_restatement_bit_for_bit(eng):
    """a pivot of exactly 1/DBL_MAX zeroes its component and its column of L; the next double above it divides"""
    for N in (11, 22, 33):
        for family in ("zero-pivot", "next-pivot"):
            A, b, _lam = PC.family_system(family, N)
            delta, d, Lf = dev_solve(eng, A, b, 0.0)
            Lr, dr = PG.ldl_blocked(A)
            xr = PG.ldl_solve(Lr, dr, b)
            for r in PC.decoupled_rows(6 * N):
                assert d[r] == dr[r] == A[r, r] and delta[r] == xr[r], (family, N, r, d[r], delta[r], xr[r])
                assert np.array_equal(Lf[:, r], Lr[:, r])


# ---- linearisation ---------------------------------------------------------------------------------------------------------------
def chain_with_extra_edges(ne, N=40, seed=0):
    truth, init, edges = PG.random_graph(N, seed, loop_every=1000, odo_noise=0.01)
    rng = np.random.default_rng(seed + 1)
    while len(edges) < ne:
        s, t = (int(v) for v in rng.integers(0, N, size=2))
        edges.append(PG.Edge(s, t, PG.measurement(truth[s], truth[t]) @ PG.rigid(rng.normal(size=3) * 0.01, rng.normal(size=3) * 0.02),
                             PG.information(rng, 300.0), uncertain=bool(rng.integers(0, 2))))
    return init, edges[:ne]


def hub_graph(N=60, hub=7, n_hub=300, seed=4):
    truth, init, edges = PG.random_graph(N, seed, loop_every=1000, odo_noise=0.01)
    rng = np.random.default_rng(seed)
    for k in range(n_hub):
        t = int(rng.integers(0, N))
        s, t = (hub, t) if k % 2 == 0 else (t, hub)
        edges.append(PG.Edge(s, t, PG.measurement(truth[s], truth[t]), PG.information(rng, 200.0), uncertain=bool(k % 3 == 0)))
    return init, edges


def gimbal_graph(seed=6):
    """poses at pitch +-pi/2 and at sy = 1e-6 (1 -+ 1e-3), both branches of TransformMatrix4dToVector6d"""
    rng = np.random.default_rng(seed)
    betas = [np.pi / 2, -np.pi / 2, np.arccos(1e-6 * (1 - 1e-3)), np.arccos(1e-6 * (1 + 1e-3)), -np.arccos(1e-6 * (1 - 1e-3)),
             -np.arccos(1e-6 * (1 + 1e-3)), 0.3, -0.2]
    poses = [PG.v2m(np.array([0.3 * k - 1.0, be, 0.5 - 0.2 * k, *rng.normal(size=3) * 3.0])) for k, be in enumerate(betas)]
    edges = [PG.Edge(k, k + 1, PG.measurement(poses[k], poses[k + 1]) @ PG.rigid(rng.normal(size=3) * 0.01, rng.normal(size=3) * 0.01),
                     PG.information(rng, 100.0)) for k in range(len(poses) - 1)]
    edges.append(PG.Edge(6, 1, PG.measurement(poses[6], poses[1]), PG.information(rng, 100.0), uncertain=True))
    return poses, edges


def far_graph(seed=8):
    _t, init, edges = PG.random_graph(20, seed, loop_every=5, odo_noise=0.01)
    off = PG.rigid([0.1, -0.2, 0.3], [4000.0, -3000.0, 0.0])   # 5 km from the origin
    return [off @ T for T in init], edges


LIN_CASES = {f"edges-{n}": (lambda n=n: chain_with_extra_edges(n)) for n in (63, 64, 65, 128, 129, 255, 256, 257)}
LIN_CASES.update({"parallel-self-loops-zeta": PC.odd_graph, "hub-300": hub_graph, "gimbal": gimbal_graph, "far-5km": far_graph})


@pytest.mark.parametrize("case", list(LIN_CASES))
def test_linearize_matches_long_double_restatement(eng, case):
    poses, edges = LIN_CASES[case]()
    p = PG.Params(max_correspondence_distance=0.1)
    lpw = PG.line_process_weight(edges, p)
    rng = np.random.default_rng(len(edges))
    for conf_in in (np.ones(len(edges)), 0.2 + 0.8 * rng.random(len(edges))):
        conf, H, b, rec = dev_linearize(eng, poses, edges, p, conf_in)
        ref = PC.linearize_reference(poses, edges, lpw, conf_in)
        r = PC.assembly_check(ref, conf, H, b, rec)
        print(f"{case}: N={len(poses)} edges={len(edges)} (units of the bound)", {k: f"{v:.3g}" for k, v in r.items()})
        assert max(r.values()) <= 1, (case, r)
        assert not np.any(np.triu(H, 1))


# ---- the hooks are the production launches --------------------------------------------------------------------------------------
def test_hooks_rebuild_the_two_accepted_steps_of_global_optimization(eng):
    """one outer iteration and one try per pass, all edges certain, no reference compensation: the call's poses are
    V2M(delta_2) V2M(delta_1) T with each delta from the hooks at lambda0 = 1e-5 max diag H"""
    _t, init, edges = PG.random_graph(12, 21, loop_every=4, odo_noise=0.005)
    edges = [PG.Edge(e.source, e.target, e.T, e.information, False) for e in edges]
    p = PG.Params(max_iteration=1, max_iteration_lm=1, reference_node=-1)
    g = E.PoseGraph([E.PoseGraphNode(np.array(T)) for T in init],
                    [E.PoseGraphEdge(e.source, e.target, np.array(e.T), np.array(e.information), False) for e in edges])
    crit = E.GlobalOptimizationConvergenceCriteria(p.max_iteration, p.min_relative_increment, p.min_relative_residual_increment, p.min_right_term,
                                                   p.min_residual, p.max_iteration_lm, p.upper_scale_factor, p.lower_scale_factor)
    opt = E.GlobalOptimizationOption(p.max_correspondence_distance, p.edge_prune_threshold, p.preference_loop_closure, p.reference_node)
    st = E.globalOptimization(eng, g, crit, opt)
    assert [(s.lm_tries, s.accepted_steps) for s in st] == [(1, 1), (1, 1)], st
    poses = [np.array(T) for T in init]
    for _pass in range(2):
        _c, H, b, rec = dev_linearize(eng, poses, edges, p, np.ones(len(edges)))
        delta, _d, _L = dev_solve(eng, H, b, 1e-5 * rec[2], factors=False)
        poses = [PG.v2m(delta[6 * i:6 * i + 6]) @ T for i, T in enumerate(poses)]
    err = max(float(np.abs(nd.pose_ - T).max()) for nd, T in zip(g.nodes_, poses))
    print(f"hooks vs b2s_global_optimization: max pose difference {err:.3g}")
    assert err < 1e-12


def test_repeated_solves_are_bit_identical_across_regrown_buffers(eng):
    A, b, lam = PC.family_system("graph", 22)
    first = dev_solve(eng, A, b, lam)
    big, bb, blam = PC.family_system("spd-1e8", 256)   # grows the factor and panel buffers
    dev_solve(eng, big, bb, blam, factors=False)
    again = dev_solve(eng, A, b, lam)
    assert all(np.array_equal(x, y) for x, y in zip(first, again))
    # the captured try: a larger call re-sizes the scratch and recaptures, the smaller one after it captures again
    runs = []
    for N in (64, 171, 64):
        _t, init, edges = PG.random_graph(N, 30 + N, loop_every=8, odo_noise=0.01)
        g = E.PoseGraph([E.PoseGraphNode(np.array(T)) for T in init],
                        [E.PoseGraphEdge(e.source, e.target, np.array(e.T), np.array(e.information), bool(e.uncertain)) for e in edges])
        st = E.globalOptimization(eng, g)
        runs.append(([nd.pose_ for nd in g.nodes_], [s.final_lambda for s in st]))
    assert all(np.array_equal(x, y) for x, y in zip(runs[0][0], runs[2][0])) and runs[0][1] == runs[2][1]
