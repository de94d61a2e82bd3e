"""High-precision references for the registration's pose solves, and checks of the references themselves (CPU).

The device's single-thread fp64 solves -- Umeyama / Kabsch from the point-to-point moments, the 6x6 LDL^T solve of point-to-plane --
are compared in test_gpu_pose_solvers.py with answers computed here at a precision that does not share their rounding:
  * kabsch_mp: Umeyama without scaling (means, demeaned cross-covariance, SVD, det sign rule) in mpmath at 50 digits;
  * solve_exact: a 6x6 linear system in exact rational arithmetic (fractions.Fraction), unobservable components set to zero the
    way the pseudo-inverse of D does for exactly zero rows and columns.
The tests below hold the references to answers known in closed form, and show on CPU emulations of the candidate fp64 formulas
why the cross-covariance must not be formed from raw moments far from the origin.
"""
from fractions import Fraction

import mpmath
import numpy as np
import pytest

DPS = 50
SKEW = np.array([1.0, 0.7, -0.4]) / np.linalg.norm([1.0, 0.7, -0.4])   # direction along which the clouds are moved off the origin


def rotation(axis, angle) -> np.ndarray:
    """Rodrigues' rotation in fp64"""
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1.0 - np.cos(angle)) * (K @ K)


def _mpmat(a):
    a = np.asarray(a, dtype=np.float64)
    return mpmath.matrix([[mpmath.mpf(float(v)) for v in row] for row in a])


def kabsch_mp(src, tgt):
    """Eigen::umeyama(src^T, tgt^T, false) in mpmath: the rotation R and translation t minimising sum |R s + t - t'|^2 over exact
    correspondences src[i] -> tgt[i].  The inputs are taken as the exact binary values they hold.  Returns (R, t) as mpmath
    matrices and the signs (det U * det V) the rule saw."""
    with mpmath.workdps(DPS):
        S, Tt = _mpmat(src), _mpmat(tgt)
        n = S.rows
        ms = [mpmath.fsum(S[i, a] for i in range(n)) / n for a in range(3)]
        mt = [mpmath.fsum(Tt[i, a] for i in range(n)) / n for a in range(3)]
        sigma = mpmath.matrix(3, 3)
        for a in range(3):
            for b in range(3):
                sigma[a, b] = mpmath.fsum((Tt[i, a] - mt[a]) * (S[i, b] - ms[b]) for i in range(n)) / n
        U, sv, V = mpmath.svd_r(sigma)                     # sigma = U diag(sv) V  (V holds the right singular vectors as rows)
        sgn = mpmath.det(U) * mpmath.det(V)
        D = mpmath.eye(3)
        if sgn < 0:
            D[int(np.argmin([float(s) for s in sv])), int(np.argmin([float(s) for s in sv]))] = -1
        R = U * D * V
        t = mpmath.matrix([mt[a] - sum(R[a, b] * ms[b] for b in range(3)) for a in range(3)])
        return R, t, float(sgn)


def mp_to_np(M) -> np.ndarray:
    return np.array([[float(M[i, j]) for j in range(M.cols)] for i in range(M.rows)])


def kabsch_pose_mp(src, tgt, G=None) -> np.ndarray:
    """The 4x4 pose [R t] of kabsch_mp composed with G on the right (what the device's T = update * init holds), rounded once"""
    R, t, _ = kabsch_mp(src, tgt)
    with mpmath.workdps(DPS):
        U = mpmath.eye(4)
        for a in range(3):
            for b in range(3):
                U[a, b] = R[a, b]
            U[a, 3] = t[a]
        if G is not None:
            U = U * _mpmat(G)
        return mp_to_np(U)


def solve_exact(A, b):
    """x with A x = b in exact rational arithmetic.  A is symmetric PSD with entries that are exact binary fractions.  Rows and columns
    that are exactly zero (with b exactly zero there) are unobservable: x is zero in them, as D^+ of an LDL^T gives.  The rest must
    be nonsingular."""
    A = [[Fraction(float(v)) for v in row] for row in np.asarray(A)]
    b = [Fraction(float(v)) for v in np.asarray(b)]
    keep = [i for i in range(len(b)) if any(A[i][j] != 0 for j in range(len(b)))]
    for i in range(len(b)):
        if i not in keep:
            assert b[i] == 0, "an exactly zero row of A with a nonzero right-hand side has no solution"
    M = [[A[i][j] for j in keep] + [b[i]] for i in keep]
    m = len(keep)
    for k in range(m):                                     # Gauss-Jordan with exact pivots (any nonzero pivot is exact)
        p = next(i for i in range(k, m) if M[i][k] != 0)
        M[k], M[p] = M[p], M[k]
        for i in range(m):
            if i != k and M[i][k] != 0:
                f = M[i][k] / M[k][k]
                M[i] = [x - f * y for x, y in zip(M[i], M[k])]
    x = [Fraction(0)] * len(b)
    for r, i in enumerate(keep):
        x[i] = M[r][m] / M[r][r]
    return x


def interpolate_mp(Ta, ta: int, Tb, tb: int, t: int) -> np.ndarray:
    """The pose Transform.cpp's interpolate aims at, in mpmath: the rotation on the SO(3) geodesic from Ra to Rb,
    Ra exp(f theta [k]x) with theta k the axis-angle of Ra^T Rb (what quaternion slerp along the shortest path traces), the
    translation on the straight line, with the reference's factor f = toSeconds(t - ta) / (toSeconds(tb - ta) + 1e-6) from the exact
    tick counts.  The relative rotation must stay clear of pi (where the geodesic stops being unique)."""
    with mpmath.workdps(DPS):
        Ra, Rb = _mpmat(np.asarray(Ta)[:3, :3]), _mpmat(np.asarray(Tb)[:3, :3])
        f = (mpmath.mpf(t - ta) / 10 ** 7) / (mpmath.mpf(tb - ta) / 10 ** 7 + mpmath.mpf(1e-6))
        rel = Ra.T * Rb
        v = [(rel[2, 1] - rel[1, 2]) / 2, (rel[0, 2] - rel[2, 0]) / 2, (rel[1, 0] - rel[0, 1]) / 2]   # sin(theta) k
        sn = mpmath.sqrt(sum(x * x for x in v))
        ang = mpmath.atan2(sn, (rel[0, 0] + rel[1, 1] + rel[2, 2] - 1) / 2)
        assert ang < 3.1, "the relative rotation must stay clear of pi"
        R = Ra
        if sn > 0:
            k = [x / sn for x in v]
            K = mpmath.matrix([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
            R = Ra * (mpmath.eye(3) + mpmath.sin(f * ang) * K + (1 - mpmath.cos(f * ang)) * K * K)
        out = mpmath.eye(4)
        for a in range(3):
            for b in range(3):
                out[a, b] = R[a, b]
            out[a, 3] = mpmath.mpf(float(Ta[a, 3])) + (mpmath.mpf(float(Tb[a, 3])) - mpmath.mpf(float(Ta[a, 3]))) * f
        return mp_to_np(out)


STAMP0 = 18_000_000_000_000_000          # 1.8e16 ticks: Unix time in 100 ns


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3] = R; T[:3, 3] = t
    return T


def buffer_pushes():
    """(stamp, T) pushes in time order for the interpolation buffer: full 3-D rotations; exactly pi about x, y, z and about the xy
    diagonal (trace -1; about z and about the diagonal R(1,1) == R(0,0), the tie of Eigen's quaternion conversion) and pi about a
    skew axis; a pair whose quaternions have a negative dot product (170 and -170 degrees about z); identical rotations; rotations
    1e-9 rad apart (slerp's linear-weight branch); an equal stamp; irregular spacing.  No two neighbours are pi apart."""
    g = [rotation([0.3, -0.5, 0.8], 0.7), rotation([1.0, 2.0, -1.0], 1.1), rotation([-0.2, 0.9, 0.4], 2.2)]
    rz170, rzm170 = rotation([0, 0, 1], np.deg2rad(170.0)), rotation([0, 0, 1], np.deg2rad(-170.0))
    rots = [g[0], np.diag([1.0, -1.0, -1.0]), g[1], np.diag([-1.0, -1.0, 1.0]), g[2],
            np.array([[0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, -1.0]]), g[0], rz170, rzm170, rzm170,
            rzm170 @ rotation([0.6, -0.64, 0.48], 1e-9), rotation([0.48, 0.6, -0.64], np.pi), g[1], np.diag([-1.0, 1.0, -1.0]),
            np.diag([-1.0, 1.0, -1.0]) @ rotation([0, 0, 1], 0.3), g[2]]
    dts = [0, 1_000_000, 1_000_000, 999_999, 1_000_001, 3, 1_000_000, 1_000_000, 1_000_000, 1_000_000, 1_000_000, 500_000,
           1_000_000, 1_000_000, 0, 1_000_000]
    rng = np.random.default_rng(17)
    out, t = [], STAMP0
    for R, dt in zip(rots, dts):
        t += dt
        out.append((t, _pose(R, rng.uniform(-20, 20, 3))))
    return out


def buffer_queries(pushes):
    ts = [t for t, _ in pushes]
    q = set(ts) | {ts[0] - 1, ts[0] - 10 ** 7, ts[-1] + 1, ts[-1] + 10 ** 7}
    for a, b in zip(ts[:-1], ts[1:]):
        if b > a:
            q |= {a + 1, b - 1, a + (b - a) // 4, a + (b - a) // 2, a + 3 * (b - a) // 4}
    return sorted(q)


def lookup_mp(entries, t: int) -> np.ndarray:
    """getTransform(t, buffer) with interpolate_mp between the bracketing entries: clamped to the ends, an exact hit returns the first
    entry with that stamp (std::find_if)"""
    t = min(max(t, entries[0][0]), entries[-1][0])
    i = next(k for k, (ti, _) in enumerate(entries) if t <= ti)
    if entries[i][0] == t:
        return entries[i][1].copy()
    (ta, Ta), (tb, Tb) = entries[i - 1], entries[i]
    return interpolate_mp(Ta, ta, Tb, tb, t)


def vec6_to_mat4(x) -> np.ndarray:
    """[O3D] TransformVector6dToMatrix4d: R = Rz(x2) Ry(x1) Rx(x0), t = x[3..5]"""
    x = [float(v) for v in x]
    sa, ca, sb, cb, sg, cg = np.sin(x[0]), np.cos(x[0]), np.sin(x[1]), np.cos(x[1]), np.sin(x[2]), np.cos(x[2])
    return np.array([[cg * cb, cg * sb * sa - sg * ca, cg * sb * ca + sg * sa, x[3]],
                     [sg * cb, sg * sb * sa + cg * ca, sg * sb * ca - cg * sa, x[4]],
                     [-sb, cb * sa, cb * ca, x[5]],
                     [0.0, 0.0, 0.0, 1.0]])


def lattice_pairs(offset, spread, angle, seed, n_side=5):
    """Point-to-point correspondences that a nearest-neighbour search recovers exactly: a jittered n_side^3 lattice of targets with
    the given spread, the source = targets rotated by `angle` about a skew axis through their centre plus noise, both moved
    `offset` metres along SKEW.  Every source point lies within 0.25 spacing of its own target and beyond 0.6 spacing of every
    other; max_corr = 0.3 spacing."""
    rng = np.random.default_rng(seed)
    spacing = spread / (n_side - 1)
    g = (np.arange(n_side) - 0.5 * (n_side - 1)) * spacing
    tgt0 = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + rng.uniform(-0.05, 0.05, (n_side ** 3, 3)) * spacing
    src0 = tgt0 @ rotation([0.3, -0.5, 0.8], angle).T + np.clip(rng.standard_normal(tgt0.shape), -3, 3) * 0.02 * spacing
    base = offset * SKEW
    return src0 + base, tgt0 + base, 0.3 * spacing


def nearest_pairs_are_exact(src, tgt, max_corr) -> bool:
    d = np.linalg.norm(src[:, None, :] - tgt[None, :, :], axis=2)
    own = np.diagonal(d).copy()
    np.fill_diagonal(d, np.inf)
    return bool(np.all(own < 0.85 * max_corr) and np.all(d.min(axis=1) > 2.0 * max_corr))


# ---- fp64 emulations of the candidate update formulas (what a single device thread computes) ----------------------------
def _rot_from_sigma(sigma):
    U, _, Vt = np.linalg.svd(sigma)
    D = np.diag([1.0, 1.0, -1.0 if np.linalg.det(U) * np.linalg.det(Vt) < 0 else 1.0])
    return U @ D @ Vt


def umeyama_two_pass(src, tgt):
    ms, mt = src.mean(0), tgt.mean(0)
    R = _rot_from_sigma((tgt - mt).T @ (src - ms) / len(src))
    return R, mt - R @ ms


def umeyama_raw_moments(src, tgt, c=np.zeros(3)):
    """One pass over the moments about the point c: sigma = E[(t - c)(s - c)^T] - (mt - c)(ms - c)^T.  c = 0 is the raw form."""
    s, t = src - c, tgt - c
    n = len(src)
    dms, dmt = s.sum(0) / n, t.sum(0) / n
    R = _rot_from_sigma(t.T @ s / n - np.outer(dmt, dms))
    ms, mt = dms + c, dmt + c
    return R, mt - R @ ms


# ---- the references against closed-form answers ---------------------------------------------------------------------------
EXACT_ROTATIONS = {
    "cyclic_120deg": np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]),
    "pi_about_x": np.diag([1.0, -1.0, -1.0]),
    "pi_about_xy_diagonal": np.array([[0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, -1.0]]),
}


@pytest.mark.parametrize("offset", [0.0, 1e3, 1e5])
@pytest.mark.parametrize("name", sorted(EXACT_ROTATIONS))
def test_kabsch_mp_recovers_an_exact_motion(offset, name):
    """Rotations with entries 0 and +-1 (120 degrees, and exactly pi about an axis and about a diagonal) and a dyadic translation
    map the source to targets that fp64 holds exactly: the reference returns that motion to its own precision."""
    rng = np.random.default_rng(1)
    src = np.round(rng.uniform(-5, 5, (40, 3)) * 64) / 64 + np.round(offset * SKEW)
    R0 = EXACT_ROTATIONS[name]
    t0 = np.array([0.5, -1.25, 3.0])
    tgt = src @ R0.T + t0
    R, t, sgn = kabsch_mp(src, tgt)
    assert sgn > 0
    assert np.abs(mp_to_np(R) - R0).max() < 1e-40
    assert np.abs(mp_to_np(t)[:, 0] - t0).max() < 1e-40 * max(1.0, offset)


def test_kabsch_mp_reflection_rule():
    """A source mirrored through the targets' thin mid-plane: the best orthogonal map is the reflection, det U * det V < 0, and the
    rule flips the smallest singular direction: the rotation is the identity."""
    g = np.arange(-2.0, 2.5, 0.5)
    xy = np.stack(np.meshgrid(g, 2.0 * g, indexing="ij"), -1).reshape(-1, 2)
    tgt = np.r_[np.c_[xy, np.full(len(xy), 0.0625)], np.c_[xy, np.full(len(xy), -0.0625)]]
    src = tgt * np.array([1.0, 1.0, -1.0])
    R, t, sgn = kabsch_mp(src, tgt)
    assert sgn < 0
    assert np.abs(mp_to_np(R) - np.eye(3)).max() < 1e-40
    assert np.abs(mp_to_np(t)).max() < 1e-17


def test_solve_exact_on_a_dyadic_system():
    rng = np.random.default_rng(3)
    J = rng.integers(-8, 9, (20, 6)) / 4.0
    A = J.T @ J
    b = J.T @ (rng.integers(-8, 9, 20) / 8.0)
    x = solve_exact(A, b)
    Af = [[Fraction(float(v)) for v in row] for row in A]
    assert all(sum(Af[i][j] * x[j] for j in range(6)) == Fraction(float(b[i])) for i in range(6))
    assert np.allclose([float(v) for v in x], np.linalg.solve(A, b), rtol=1e-9, atol=1e-12)


def test_solve_exact_leaves_unobservable_components_at_zero():
    A = np.diag([2.0, 0.0, 3.0, 0.0, 0.0, 1.0]); A[0, 2] = A[2, 0] = 1.0
    b = np.array([1.0, 0.0, 2.0, 0.0, 0.0, -0.5])
    x = solve_exact(A, b)
    assert x[1] == x[3] == x[4] == 0
    assert x[5] == Fraction(-1, 2) and 2 * x[0] + x[2] == 1 and x[0] + 3 * x[2] == 2


def test_vec6_to_mat4_is_a_rotation_with_the_zyx_angles():
    x = [0.3, -0.2, 1.1, 1.0, 2.0, 3.0]
    T = vec6_to_mat4(x)
    Rz = rotation([0, 0, 1], x[2]); Ry = rotation([0, 1, 0], x[1]); Rx = rotation([1, 0, 0], x[0])
    assert np.abs(T[:3, :3] - Rz @ Ry @ Rx).max() < 1e-15
    assert np.all(T[:3, 3] == [1.0, 2.0, 3.0])


# ---- why the point-to-point cross-covariance is accumulated about a point near the clouds --------------------------------
def _bound_ok(R, t, Rr, tr, offset):
    return np.abs(R - Rr).max() <= 1e-13 and np.abs(t - tr).max() <= 1e-14 * max(1.0, offset)


@pytest.mark.parametrize("offset", [0.0, 1e2, 1e3, 1e4, 1e5])
@pytest.mark.parametrize("spread", [0.5, 5.0, 30.0])
def test_fp64_umeyama_about_a_nearby_point_meets_the_bound(offset, spread):
    """The fp64 forms that stay within |dR| <= 1e-13, |dt| <= 1e-14 max(1, |offset|) of the 50-digit answer at any offset: two passes
    (the oracle, RANSAC), and one pass over moments about a point inside the targets' box (the device: the grid's box centre)."""
    src, tgt, mc = lattice_pairs(offset, spread, 0.04, seed=int(offset) % 97 + int(spread * 10))
    assert nearest_pairs_are_exact(src, tgt, mc)
    R, t, _ = kabsch_mp(src, tgt)
    Rr, tr = mp_to_np(R), mp_to_np(t)[:, 0]
    assert _bound_ok(*umeyama_two_pass(src, tgt), Rr, tr, offset)
    c = 0.5 * (tgt.min(0) + tgt.max(0)) + np.array([0.1, -0.2, 0.3]) * spread   # any point near the box will do
    assert _bound_ok(*umeyama_raw_moments(src, tgt, c), Rr, tr, offset)


def test_fp64_umeyama_from_raw_moments_fails_the_bound_far_from_the_origin():
    """The raw-moment form sigma = E[t s^T] - mt ms^T loses the covariance to cancellation: at 1e4 m with a 5 m spread it is far
    outside the bound the tests hold the device to (so those tests can tell the two forms apart)."""
    src, tgt, _ = lattice_pairs(1e4, 5.0, 0.04, seed=5)
    R, t, _ = kabsch_mp(src, tgt)
    Rb, tb = umeyama_raw_moments(src, tgt)
    assert np.abs(Rb - mp_to_np(R)).max() > 1e-11


# ---- the 3x3 SVD of the oracle (the same algorithm as the device's svd3_dev) ---------------------------------------------------
SVD_CASES = {
    "zero_row": np.array([[0.7, -0.2, 0.1], [0.3, 1.1, -0.4], [0.0, 0.0, 0.0]]),
    "zero_row_rank_one": np.array([[0.0, 0.0, 0.0], [0.6, -0.3, 0.2], [1.2, -0.6, 0.4]]),
    "repeated_rows": np.array([[0.5, -1.0, 0.25], [0.5, -1.0, 0.25], [0.1, 0.3, -0.7]]),
    "planar_cross_covariance": np.array([[0.31, 0.02, 1e-17], [-0.01, 0.27, 0.0], [0.0, 0.0, 0.0]]),
    "general": np.array([[0.9, 0.1, -0.3], [0.2, -0.7, 0.5], [0.4, 0.6, 0.8]]),
}


@pytest.mark.parametrize("name", sorted(SVD_CASES))
def test_oracle_svd3_is_orthonormal_on_rank_deficient_inputs(name):
    """orc_svd3 at inputs whose exactly zero or repeated rows keep one-sided Jacobi's columns in a plane: U and V orthonormal to
    1e-15, U diag(S) V^T = A, and the singular values those of the 50-digit SVD"""
    from oracle import oracle as O
    A = SVD_CASES[name]
    U, S, V = O.svd3(A)
    assert np.abs(U.T @ U - np.eye(3)).max() < 1e-15 and np.abs(V.T @ V - np.eye(3)).max() < 1e-15
    assert abs(abs(np.linalg.det(U)) - 1.0) < 1e-15
    assert np.abs(U @ np.diag(S) @ V.T - A).max() < 1e-15
    with mpmath.workdps(DPS):
        sv = sorted((float(s) for s in mpmath.svd_r(_mpmat(A), compute_uv=False)), reverse=True)
    assert np.abs(S - sv).max() < 1e-15


# ---- interpolation of poses ---------------------------------------------------------------------------------------------------
def test_interpolate_mp_on_a_closed_form_geodesic():
    Ta, Tb = _pose(rotation([0, 0, 1], 0.2), [1.0, 2.0, 3.0]), _pose(rotation([0, 0, 1], 1.0), [3.0, 2.0, -1.0])
    ta, tb, t = STAMP0, STAMP0 + 10 ** 7, STAMP0 + 2_500_000
    f = 0.25 / (1.0 + 1e-6)
    T = interpolate_mp(Ta, ta, Tb, tb, t)
    assert np.abs(T[:3, :3] - rotation([0, 0, 1], 0.2 + 0.8 * f)).max() < 1e-15
    assert np.abs(T[:3, 3] - (np.array([1.0, 2.0, 3.0]) + f * np.array([2.0, 0.0, -4.0]))).max() < 1e-15


def test_buffer_pushes_cover_the_quaternion_branches():
    """the pushes reach every branch of Eigen's conversion and slerp that the buffer tests mean to cover"""
    from odometry_buffer import EPS, quat_from_rot
    pushes = buffer_pushes()
    Rs = [T[:3, :3] for _, T in pushes]
    traces = [np.trace(R) for R in Rs]
    assert sum(abs(tr + 1.0) < 1e-15 for tr in traces) >= 5
    assert any(R[1, 1] == R[0, 0] and np.trace(R) <= 0 for R in Rs)
    dots = [float(np.dot(quat_from_rot(a), quat_from_rot(b))) for a, b in zip(Rs[:-1], Rs[1:])]
    assert any(d < 0 for d in dots)
    assert any(abs(d) >= 1.0 - EPS for d in dots)
    ts = [t for t, _ in pushes]
    assert any(a == b for a, b in zip(ts[:-1], ts[1:]))


@pytest.mark.parametrize("size", [2000, 5, 1])
def test_numpy_buffer_follows_the_geodesic(size):
    """tests/odometry_buffer.py (Eigen's quaternion conversion and slerp) against the 50-digit geodesic at 1e-12 on every query: exact
    hits, clamping at both ends, interpolation across pi-rotated poses, a negative quaternion dot product, identical rotations,
    rotations 1e-9 rad apart and an equal stamp.  size < the number of pushes evicts (size 1: every query is the latest pose)."""
    from odometry_buffer import TransformInterpolationBuffer
    pushes = buffer_pushes()
    buf = TransformInterpolationBuffer(size)
    for t, T in pushes:
        buf.push(t, T)
    kept = pushes[-size:]
    for q in buffer_queries(pushes):
        got = buf.get_transform(q)
        ref = lookup_mp(kept, q)
        assert np.abs(got - ref).max() < 1e-12, q
        if size == 1:
            assert np.array_equal(got, pushes[-1][1])
