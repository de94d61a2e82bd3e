"""Accuracy checks of the normal estimation (normals.cu, DESIGN.md K-normals) one stage at a time, against references of the operation
itself, held to the rounding bounds of the arithmetic, so that a failure names the stage and the point where a kernel went wrong:

- neighbour set: the candidates within the radius, at most k of them, in (d2, original index) order.  d2 is fp64 with dist2_exact's
  association (dx^2 + dy^2) + dz^2 and the cut is strict, d2 < r^2: the reference's KD-tree compares the same rounded values, so this
  rounded d2 is the definition.  Candidates come from cKDTree with a slightly enlarged radius and are filtered exactly.
- cumulants: the nine sums x, y, z, xx, xy, xz, yy, yz, zz of that set in long double next to the running magnitudes sum |term|.  The
  device's count must be exact and each cumulant within the (k + 1)-term fp64 summation bound (k + 1) u sum |term| (plus the long double
  reference's own error).  A wrong member moves a coordinate sum by a coordinate difference, orders of magnitude above that bound.
- finish: the covariance is formed from the device's own cumulants with finish_normal's rounding (bit-exact here: every step is one
  correctly rounded fp64 operation, and the library is built with -fmad=false).  Then
    * the solver's exact branches -- fewer than 3 neighbours (identity covariance), max coefficient 0 (zero solver result: the prior,
      or (0,0,1)), a diagonal covariance (the axis of the strict minimum, ties -> z), NaN -- are restated and must match bit for bit,
      normalisation and orientation included;
    * otherwise the direction must lie within K u ||C|| (1 + 1 / sqrt(1 - h^2)) / (lambda_1 - lambda_0) of the eigenvector of the
      smallest eigenvalue of that covariance (h: the solver's clamped det / 2 p^3, whose acos turns rounding into eigenvalue error
      when two eigenvalues are close -- a planar patch) (two Rayleigh-quotient steps in long double from LAPACK's vector; tests/test_normals_checks.py holds it to mpmath);
    * the sign follows the orientation rule n . p < 0 wherever |n_ref . p| / |p| is above the direction bound, and the prior rule
      n . prior > 0 where the orientation is an exact tie (n . p == 0, a plane through the origin) and |n_ref . prior| is above it.

u = 2^-53.  K was measured with the fp64 restatement of the solver (oracle orc_fast_eigen3x3) on the families below
(tests/test_normals_checks.py prints it); K_DIR is that measurement times a safety factor for the device's acos / cos, which are
not the host's.  Each check returns the worst ratio to its bound (<= 1 passes) and where it is.

The clouds the tests run are built here too: lattices (ties at every shell), a dense cluster at a distance (more than 32 members in the
k-th key's histogram bin), the scan families of tests/boundary_child.py, coincident points, offsets far from the origin."""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

U = 2.0 ** -53
LD = np.longdouble
ULD = float(np.finfo(np.longdouble).eps) / 2
K_MEASURED = 2.0   # max over the CPU families of the direction metric of orc_fast_eigen3x3 (measured 1.77), rounded up
K_DIR = 4.0 * K_MEASURED
# cumulant order: x, y, z, xx, xy, xz, yy, yz, zz (finish_normal's c[0..8])
PAIRS = [(0, None), (1, None), (2, None), (0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]


# ---- neighbour sets -----------------------------------------------------------------------------------------------------------
def dist2(q, P):
    """dist2_exact: fp64, (dx^2 + dy^2) + dz^2"""
    d = q[None, :] - P
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def neighbour_sets(xyz, knn, radius, queries=None, tie="lower", cut="strict", count_delta=0, replace_kth=False):
    """Reference neighbour set of every query (original indices, ascending (d2, index)).  The keyword arguments are the one-detail
    mutants the self-test feeds to the checks: tie="higher" (equal d2 -> higher index first), cut="le" (d2 <= r2), count_delta=-1
    (k - 1 members), replace_kth (the (k + 1)-th key in place of the k-th)."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float64)
    n = len(xyz)
    queries = np.arange(n) if queries is None else np.asarray(queries)
    tree = cKDTree(xyz)
    r2 = radius * radius
    want = knn + 1 if replace_kth else knn
    kq = min(want, n)
    dk, _ = tree.query(xyz[queries], k=kq, distance_upper_bound=radius * (1 + 1e-9))
    dk = dk.reshape(len(queries), -1)[:, -1]
    reach = np.where(np.isfinite(dk), np.minimum(dk, radius), radius) * (1 + 1e-7) + 1e-300
    cands = tree.query_ball_point(xyz[queries], reach)
    out = []
    for qn, q in enumerate(queries):
        c = np.asarray(cands[qn], dtype=np.int64)
        d2 = dist2(xyz[q], xyz[c])
        keep = d2 < r2 if cut == "strict" else d2 <= r2
        c, d2 = c[keep], d2[keep]
        o = np.lexsort((c if tie == "lower" else -c, d2))
        sel = c[o[:want]]
        if replace_kth and len(sel) == knn + 1:
            sel = np.r_[sel[:knn - 1], sel[knn]]
        else:
            sel = sel[:knn]
        if count_delta and len(sel) > 0:
            sel = sel[:len(sel) + count_delta]
        out.append(sel)
    return queries, out


def cumulant_reference(xyz, sets):
    """(exact-ish sums in long double, running magnitudes sum |term|, counts) of the nine cumulants of each set"""
    m = len(sets)
    kmax = max((len(s) for s in sets), default=0)
    P = np.zeros((m, max(kmax, 1), 3), dtype=LD)
    cnt = np.array([len(s) for s in sets], dtype=np.int64)
    for i, s in enumerate(sets):
        P[i, :len(s)] = xyz[s]
    S = np.zeros((m, 9), dtype=LD)
    A = np.zeros((m, 9), dtype=LD)
    for t, (a, b) in enumerate(PAIRS):
        term = P[:, :, a] if b is None else P[:, :, a] * P[:, :, b]
        S[:, t] = term.sum(axis=1)
        A[:, t] = np.abs(term).sum(axis=1)
    return S, A, cnt


def restated_cumulants(xyz, sets):
    """the sums in fp64, in list order: what the phase-2 kernel and the reference's ComputeCovariance compute"""
    m = len(sets)
    cnt = np.array([len(s) for s in sets], dtype=np.int64)
    kmax = int(cnt.max(initial=0))
    idx = np.zeros((m, max(kmax, 1)), dtype=np.int64)
    for i, s in enumerate(sets):
        idx[i, :len(s)] = s
    rec = np.zeros((m, 10))
    for j in range(kmax):   # column j = the j-th neighbour of every set: left-to-right fp64 sums, vectorised over the sets
        live = cnt > j
        P = xyz[idx[live, j]]
        for t, (a, b) in enumerate(PAIRS):
            rec[live, t] += P[:, a] if b is None else P[:, a] * P[:, b]
    rec[:, 9] = cnt
    return rec


def check_cumulants(rec, S, A, cnt):
    """rec: device records (m x 10) of the queries.  Returns (worst ratio to the bound, row of it, count mismatches)."""
    bad_count = np.nonzero(rec[:, 9] != cnt)[0]
    k = cnt.astype(np.float64)[:, None]
    bound = ((k + 1) * U / (1 - (k + 1) * U)) * A.astype(np.float64) + (k + 2) * ULD * A.astype(np.float64)
    err = np.abs(rec[:, :9].astype(LD) - S).astype(np.float64)
    ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    ratio[~np.isfinite(rec[:, :9])] = np.inf
    worst = ratio.max(axis=1) if len(ratio) else np.zeros(0)
    j = int(np.argmax(worst)) if len(worst) else -1
    return (float(worst[j]) if j >= 0 else 0.0), j, bad_count


# ---- finish ---------------------------------------------------------------------------------------------------------------------
def covariance(rec):
    """finish_normal's covariance from the recorded cumulants and count, bit-exact (identity below 3 neighbours)"""
    m = len(rec)
    kk = rec[:, 9]
    cov = np.tile(np.eye(3).ravel(), (m, 1))
    big = kk >= 3
    with np.errstate(all="ignore"):
        c = rec[big, :9] / kk[big, None]
        cv = np.empty((int(big.sum()), 9))
        cv[:, 0] = c[:, 3] - c[:, 0] * c[:, 0]
        cv[:, 4] = c[:, 6] - c[:, 1] * c[:, 1]
        cv[:, 8] = c[:, 8] - c[:, 2] * c[:, 2]
        cv[:, 1] = cv[:, 3] = c[:, 4] - c[:, 0] * c[:, 1]
        cv[:, 2] = cv[:, 6] = c[:, 5] - c[:, 0] * c[:, 2]
        cv[:, 5] = cv[:, 7] = c[:, 7] - c[:, 1] * c[:, 2]
    cov[big] = cv
    return cov


def solver_branch(cov, diag_tie="strict"):
    """FastEigen3x3's exact branches: (kind, vector) per row, kind 0 = eigen path (vector unused), 1 = zero result (max coefficient 0),
    2 = diagonal (the axis).  diag_tie="le" is the self-test's mutant of the tie rule."""
    m = len(cov)
    mc = cov[:, 0].copy()
    for i in range(1, 9):
        gt = cov[:, i] > mc
        mc[gt] = cov[gt, i]
    kind = np.zeros(m, dtype=np.int64)
    vec = np.zeros((m, 3))
    with np.errstate(all="ignore"):
        A = cov / mc[:, None]
        norm = (A[:, 1] * A[:, 1] + A[:, 2] * A[:, 2]) + A[:, 5] * A[:, 5]
        a0, a1, a2 = A[:, 0] * mc, A[:, 4] * mc, A[:, 8] * mc
    zero = mc == 0
    diag = ~zero & ~(norm > 0)
    kind[zero] = 1
    kind[diag] = 2
    if diag_tie == "strict":
        x = (a0 < a1) & (a0 < a2)
        y = ~x & (a1 < a0) & (a1 < a2)
    else:
        x = (a0 <= a1) & (a0 <= a2)
        y = ~x & (a1 <= a0) & (a1 <= a2)
    vec[diag] = np.where(x[diag, None], [1.0, 0, 0], np.where(y[diag, None], [0, 1.0, 0], [0, 0, 1.0]))
    return kind, vec


def finish_exact(v, q, prior=None, orient_sign=1.0, prior_flip=1.0):
    """finish_normal after the solver for a solver result v (fp64, bit-exact): prior rule, NormalizeNormals, orientation towards the
    origin.  orient_sign / prior_flip = -1 are the self-test's mutants (towards +p; the prior flip inverted)."""
    nr = np.array(v, dtype=np.float64)
    dot = lambda a, b: (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]
    with np.errstate(all="ignore"):
        if prior is not None:
            if np.sqrt(dot(nr, nr)) == 0.0:
                nr = np.array(prior, dtype=np.float64)
            elif prior_flip * dot(nr, prior) < 0.0:
                nr = -nr
        elif np.sqrt(dot(nr, nr)) == 0.0:
            nr = np.array([0.0, 0.0, 1.0])
        zz = dot(nr, nr)
        if zz > 0:
            nr = nr / np.sqrt(zz)
        if nr[0] != nr[0]:
            nr = np.array([0.0, 0.0, 1.0])
        ref = -orient_sign * np.asarray(q, dtype=np.float64)
        if np.sqrt(dot(nr, nr)) == 0.0:
            rn = np.sqrt(dot(ref, ref))
            nr = np.array([0.0, 0.0, 1.0]) if rn == 0.0 else ref / rn
        elif dot(nr, ref) < 0.0:
            nr = -nr
    return nr


def smallest_eigvec(cov):
    """eigenvector of the smallest eigenvalue of each covariance, the gap lambda_1 - lambda_0 and ||C|| (spectral): LAPACK's vector
    refined by two Rayleigh-quotient steps in long double (the adjugate of C - lambda I applied to the current vector)"""
    C = cov.reshape(-1, 3, 3)
    w, V = np.linalg.eigh(C)
    v = V[:, :, 0].astype(LD)
    CL = C.astype(LD)
    for _ in range(2):
        lam = np.einsum("mi,mij,mj->m", v, CL, v) / np.einsum("mi,mi->m", v, v)
        M = CL - lam[:, None, None] * np.eye(3, dtype=LD)
        adj = np.empty_like(M)
        for i in range(3):
            for j in range(3):
                r = [x for x in range(3) if x != j]; c = [x for x in range(3) if x != i]
                adj[:, i, j] = (-1) ** (i + j) * (M[:, r[0], c[0]] * M[:, r[1], c[1]] - M[:, r[0], c[1]] * M[:, r[1], c[0]])
        nv = np.einsum("mij,mj->mi", adj, v)
        nn = np.sqrt(np.einsum("mi,mi->m", nv, nv))
        ok = nn > 0
        v[ok] = nv[ok] / nn[ok, None]
        v[ok] *= np.where(np.einsum("mi,mi->m", v[ok], V[ok, :, 0].astype(LD)) < 0, -1, 1)[:, None]
    return v.astype(np.float64), w[:, 1] - w[:, 0], np.abs(w).max(axis=1)


def acos_condition(cov):
    """1 + 1 / sqrt(1 - h^2) where the solver's h = det(B) / (2 p^3) (fp64, as FastEigen3x3 forms it) is >= 0, else 1.  For h >= 0 the
    solver takes the smallest eigenvector from eval[1] (the cross product of the eigenvectors of eval[1] and eval[2]), and acos
    amplifies the rounding of h into eval[1] by 1 / sqrt(1 - h^2) as h -> 1.  For h < 0 it takes it from eval[0] = q + 2 p cos(acos(h) / 3
    + 2 pi / 3), which is insensitive to that rounding as h -> -1 (the derivative of the cosine vanishes there): a near-isotropic planar
    patch keeps the plain bound."""
    with np.errstate(all="ignore"):
        mc = cov.max(axis=1)
        A = cov / mc[:, None]
        norm = (A[:, 1] * A[:, 1] + A[:, 2] * A[:, 2]) + A[:, 5] * A[:, 5]
        q = ((A[:, 0] + A[:, 4]) + A[:, 8]) / 3
        b00, b11, b22 = A[:, 0] - q, A[:, 4] - q, A[:, 8] - q
        p = np.sqrt((((b00 * b00 + b11 * b11) + b22 * b22) + norm * 2) / 6)
        c00 = b11 * b22 - A[:, 5] * A[:, 5]
        c01 = A[:, 1] * b22 - A[:, 5] * A[:, 2]
        c02 = A[:, 1] * A[:, 5] - b11 * A[:, 2]
        h = np.clip((((b00 * c00 - A[:, 1] * c01) + A[:, 2] * c02) / (p * p * p)) * 0.5, -1.0, 1.0)
        return np.where(h >= 0, 1.0 + 1.0 / np.sqrt(np.maximum(1.0 - h * h, U)), 1.0)


def direction_metric(n, v, gap, norm, cov):
    """sin(angle between the lines of n and v) in units of u ||C|| acos_condition / gap"""
    s = np.linalg.norm(np.cross(n, v), axis=1)
    scale = U * norm * acos_condition(cov) / np.where(gap > 0, gap, np.nan)
    return s / scale, scale


def check_finish(rec, normals, qxyz, priors=None, K=None, diag_tie="strict"):
    """rec, normals, qxyz (and priors): rows of the checked queries.  Returns a dict: worst direction metric (units of u||C||/gap, must
    be <= K), rows whose exact branch or sign is wrong, and the branch / sign counts."""
    K = K_DIR if K is None else K
    cov = covariance(rec)
    kind, vec = solver_branch(cov, diag_tie)
    out = {"exact_bad": [], "sign_bad": [], "dir_worst": 0.0, "dir_row": -1, "n_exact": int((kind > 0).sum()), "n_sign": 0,
           "n_prior_sign": 0, "n_dir": 0, "sign_margin": np.inf}
    for i in np.nonzero(kind > 0)[0]:
        exp = finish_exact(vec[i], qxyz[i], None if priors is None else priors[i])
        if not np.array_equal(exp, normals[i]):
            out["exact_bad"].append(int(i))
    ev = np.nonzero(kind == 0)[0]
    if len(ev) == 0:
        return out
    v, gap, norm = smallest_eigvec(cov[ev])
    met, scale = direction_metric(normals[ev], v, gap, norm, cov[ev])
    finite = np.isfinite(met)
    bnd = K * scale
    if finite.any():
        j = int(np.nanargmax(np.where(finite, met, -1.0)))
        out["dir_worst"], out["dir_row"] = float(met[j]), int(ev[j])
    out["n_dir"] = int(finite.sum())
    out["dir_bad"] = [int(ev[j]) for j in np.nonzero(finite & (met > K))[0]]
    # signs
    q = qxyz[ev]
    qn = np.linalg.norm(q, axis=1)
    with np.errstate(all="ignore"):
        vq = np.abs(np.einsum("mi,mi->m", v, q)) / qn
    bnd = np.where(np.isfinite(bnd), bnd, np.inf)
    orient = (qn > 0) & (vq > bnd)
    nq = (normals[ev, 0] * q[:, 0] + normals[ev, 1] * q[:, 1]) + normals[ev, 2] * q[:, 2]
    out["n_sign"] = int(orient.sum())
    if orient.any():
        out["sign_margin"] = float(np.min((vq - bnd)[orient]))
    out["sign_bad"] += [int(ev[j]) for j in np.nonzero(orient & ~(nq < 0))[0]]
    if priors is not None:
        p = priors[ev]
        pn = np.linalg.norm(p, axis=1)
        with np.errstate(all="ignore"):
            vp = np.abs(np.einsum("mi,mi->m", v, p)) / pn
        tie = (nq == 0) & (pn > 0) & (vp > bnd)
        npd = (normals[ev, 0] * p[:, 0] + normals[ev, 1] * p[:, 1]) + normals[ev, 2] * p[:, 2]
        out["n_prior_sign"] = int(tie.sum())
        out["sign_bad"] += [int(ev[j]) for j in np.nonzero(tie & ~(npd > 0))[0]]
    return out


def check_all(xyz, knn, radius, rec, path, normals, priors=None, queries=None):
    """Every check on one device run (rec / path / normals over all points; queries: the flagged subset, or all).  Returns a summary dict;
    raises AssertionError naming the first failing stage and point."""
    n = len(xyz)
    queries = np.arange(n) if queries is None else np.asarray(queries)
    others = np.setdiff1d(np.arange(n), queries)
    assert np.isnan(rec[others]).all(), "[record] a point outside the query subset has a record"
    assert (path[others] == 0).all(), "[record] a point outside the query subset has a path code"
    assert (path[queries] > 0).all(), f"[record] queries without a path code: {np.nonzero(path[queries] == 0)[0][:10]}"
    _, sets = neighbour_sets(xyz, knn, radius, queries)
    S, A, cnt = cumulant_reference(xyz, sets)
    r = rec[queries]
    cw, cj, badc = check_cumulants(r, S, A, cnt)
    assert len(badc) == 0, (f"[count] neighbour count differs at {len(badc)} queries, first point {queries[badc[0]]} "
                            f"(path {path[queries[badc[0]]]}): device {r[badc[0], 9]:.0f}, reference {cnt[badc[0]]}")
    assert cw <= 1.0, f"[cumulant] cumulant off by {cw:.3g} x its bound at point {queries[cj]} (path {path[queries[cj]]})"
    f = check_finish(r, normals[queries], xyz[queries], None if priors is None else priors[queries])
    assert not f["exact_bad"], f"[exact] exact solver branch differs at points {queries[f['exact_bad'][:10]]}"
    assert not f.get("dir_bad"), f"[direction] direction off by {f['dir_worst']:.3g} u||C||/gap > K = {K_DIR} at point {queries[f['dir_row']]}"
    assert not f["sign_bad"], f"[sign] sign wrong at points {queries[f['sign_bad'][:10]]}"
    return {"cum": cw, "dir": f["dir_worst"] / K_DIR, "n": len(queries), "exact": f["n_exact"], "signs": f["n_sign"],
            "prior_signs": f["n_prior_sign"], "paths": np.bincount(path[queries], minlength=7)[1:]}


def assert_normals_close(got, ref, xyz, knn, radius, queries=None):
    """Gap-aware per-point comparison of two normal estimations of the same cloud xyz that may sum the cumulants in a different order
    (device and oracle, or two device runs).  got / ref: one row per query (queries: indices into xyz, default all).  Where the
    solver takes an exact branch (fewer than 3 neighbours, zero or diagonal covariance) both must be bit-identical.  Elsewhere the angle
    between them is bounded by both solves' direction bound (K_DIR u ||C|| acos_condition / gap) plus the covariance perturbation that
    reordering (k + 1)-term sums of magnitude (|p| + r)^2 causes, over the gap of the reference covariance; the sign must agree wherever
    the orientation decides it by more than that bound.  Returns the worst ratio to the bound."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float64)
    queries = np.arange(len(xyz)) if queries is None else np.asarray(queries)
    assert len(got) == len(ref) == len(queries)
    assert np.abs(np.linalg.norm(got, axis=1) - 1.0).max(initial=0.0) < 1e-12
    _, sets = neighbour_sets(xyz, knn, radius, queries)
    rec = restated_cumulants(xyz, sets)
    cov = covariance(rec)
    kind, _ = solver_branch(cov)
    ev = kind == 0
    assert np.array_equal(got[~ev], ref[~ev]), f"an exact solver branch differs at {np.nonzero(~ev)[0][:10]}"
    if not ev.any():
        return 0.0
    v, gap, norm = smallest_eigvec(cov[ev])
    q = xyz[queries[ev]]
    m = np.linalg.norm(q, axis=1) + radius
    k = rec[ev, 9]
    pert = 8 * (k + 1) * U * m * m   # |delta C| entrywise: both sums' bounds, divided by k, and the products of the means
    with np.errstate(all="ignore"):
        bound = (2 * K_DIR * U * norm * acos_condition(cov[ev]) + 3 * pert) / gap
    ang = np.linalg.norm(np.cross(got[ev], ref[ev]), axis=1)
    vacuous = ~np.isfinite(bound) | (bound >= 1.0)
    ratio = np.where(vacuous, 0.0, ang / np.where(vacuous, 1.0, bound))
    bad = np.nonzero(ratio > 1.0)[0]
    assert len(bad) == 0, (f"{len(bad)} normals off by more than their gap-aware bound; worst {ratio.max():.3g} x bound at query "
                           f"{queries[np.nonzero(ev)[0][bad[0]]]}")
    dots = (got[ev] * ref[ev]).sum(axis=1)
    with np.errstate(all="ignore"):
        decided = np.abs((v * q).sum(axis=1)) / np.linalg.norm(q, axis=1) > np.where(vacuous, np.inf, bound)
    assert (dots[decided] > 0).all(), "opposite orientation where the orientation rule decides the sign"
    return float(ratio.max())


def rows_in(sub, full):
    """index in full of every row of sub (rows bit-identical)"""
    at = {r.tobytes(): i for i, r in enumerate(np.ascontiguousarray(full, dtype=np.float64))}
    return np.array([at[r.tobytes()] for r in np.ascontiguousarray(sub, dtype=np.float64)], dtype=np.int64)


# ---- families -------------------------------------------------------------------------------------------------------------------
def lattice(n=7, h=0.25, offset=(0.0, 0.0, 0.0), planar=False):
    """an n^3 (or n^2 planar, z = 0) lattice of spacing h (a power of two: d2 exact, ties at every shell, d2 == r^2 for r = a multiple of h)"""
    g = np.arange(n) * h
    if planar:
        X, Y = np.meshgrid(g, g, indexing="ij")
        P = np.c_[X.ravel(), Y.ravel(), np.zeros(X.size)]
    else:
        X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
        P = np.c_[X.ravel(), Y.ravel(), Z.ravel()]
    return np.ascontiguousarray(P + np.asarray(offset))


def cluster_at_distance(seed=3, n_cluster=60, n_dup=6):
    """a query patch and, 1.03 m away, a tight cluster of 60 points (six of them duplicated): for knn > the patch size the k-th key falls
    in one histogram bin with more than 32 members, with exact ties among the duplicates (with r = 2 and lim2 = r^2, every d2 from the
    patch to the cluster lies in [1.0, 1.125), bin 8)"""
    rng = np.random.default_rng(seed)
    patch = np.c_[rng.uniform(-0.005, 0.005, (8, 2)), np.zeros(8)] + [5.0, 5.0, 1.0]
    cl = rng.normal(0.0, 0.004, (n_cluster, 3)) + [5.0, 6.03, 1.0]
    cl = np.vstack([cl, cl[:n_dup]])
    return np.ascontiguousarray(np.vstack([patch, cl]))


def coincident(offset=(3.0, -2.0, 1.0)):
    """a plane patch, three and more coincident points (zero covariance), a coincident pair (d2 = 0), an isolated point"""
    rng = np.random.default_rng(9)
    o = np.asarray(offset)
    plane = np.c_[rng.uniform(-1, 1, (200, 2)), 0.002 * rng.standard_normal(200)] + o
    trip = np.repeat([o + [4.0, 0.0, 0.0]], 4, axis=0)
    pair = np.repeat([o + [0.0, 4.0, 0.0]], 2, axis=0)
    lone = o + [[-4.0, -4.0, 0.0]]
    return np.ascontiguousarray(np.vstack([plane, trip, pair, lone]))


def plane_through_origin(n=400, seed=4):
    """points of the plane z = 0 around the origin: n . p == 0 exactly, so the orientation keeps the solver's (or the prior's) sign"""
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(np.c_[rng.uniform(-2, 2, (n, 2)), np.zeros(n)])


def radius_edge(h=0.25):
    """a planar lattice queried with r = 2 h: neighbours at d2 == r^2 exactly (excluded), and knn above the strict count"""
    return lattice(9, h, planar=True)
