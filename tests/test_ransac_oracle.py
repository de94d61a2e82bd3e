"""CPU: the C restatement of RegistrationRANSACBasedOnFeatureMatching (tests/oracle_ransac.c, DESIGN.md row K-ransac) against its
numpy twin -- feature correspondences with constructed ties, the mutual fallback at its threshold, small clouds with a known
transform, a run that the confidence stops -- and the first values of the hypothesis stream, pinned."""
import numpy as np
import pytest

import oracle_ransac as OR


def rot(yaw, pitch=0.0, roll=0.0):
    cy, sy, cp, sp, cr, sr = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    return np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]]) @ np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]]) @ np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])


def rigid(yaw, t, pitch=0.0, roll=0.0):
    T = np.eye(4)
    T[:3, :3] = rot(yaw, pitch, roll)
    T[:3, 3] = t
    return T


def pair(n, T, seed, noise=0.0, shuffle=True):
    """source points with random features, the target the source moved by T (permuted), its features the source's + noise"""
    rng = np.random.default_rng(seed)
    sx = rng.uniform(-10, 10, (n, 3))
    sf = rng.uniform(0, 100, (n, 33))
    perm = rng.permutation(n) if shuffle else np.arange(n)
    tx = (sx @ T[:3, :3].T + T[:3, 3])[perm]
    tf = sf[perm] + rng.normal(0, noise, (n, 33)) if noise else sf[perm].copy()
    return sx, sf, tx, tf


def test_stream_is_pinned():
    """idx(h, j) = mulhi64(splitmix64(seed + (h n + j + 1) 0x9E3779B97F4A7C15), size): the first values for seed 1, n = 3"""
    got = [OR.stream(1, h, 3, j, 1000) for h in range(3) for j in range(3)]
    assert got == [OR.np_stream(1, h, 3, j, 1000) for h in range(3) for j in range(3)]
    assert got == [566, 745, 971, 444, 444, 762, 877, 523, 285]
    # seed 0: the first splitmix64 output of the standard generator, 0xE220A8397B1DCDAF, scaled to 2^32
    assert OR.stream(0, 0, 3, 0, 1 << 32) == OR.np_stream(0, 0, 3, 0, 1 << 32) == 0xE220A839


@pytest.mark.parametrize("ns,nt", [(1, 1), (7, 50), (64, 63), (65, 129), (200, 90)])
def test_feature_corr_random(ns, nt):
    rng = np.random.default_rng(ns * 1000 + nt)
    fs, ft = rng.uniform(0, 50, (ns, 33)), rng.uniform(0, 50, (nt, 33))
    a, b = OR.feature_corr(fs, ft), OR.np_feature_corr(fs, ft)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_feature_corr_ties():
    """duplicate rows and zero rows: every tie goes to the lower index, both ways"""
    rng = np.random.default_rng(5)
    fs = rng.integers(0, 3, (40, 33)).astype(np.float64)
    fs[10] = fs[3]; fs[20:25] = 0.0
    ft = np.concatenate([fs[[3, 3, 20, 7]], np.zeros((3, 33)), rng.integers(0, 3, (30, 33)).astype(np.float64)])
    s2t, t2s = OR.feature_corr(fs, ft)
    n2 = OR.np_feature_corr(fs, ft)
    assert np.array_equal(s2t, n2[0]) and np.array_equal(t2s, n2[1])
    assert s2t[3] == 0 and s2t[10] == 0 and t2s[0] == 3 and t2s[1] == 3 and t2s[2] == 20 and s2t[20] == 2
    e = OR.feature_corr(fs, np.zeros((0, 33)))
    assert (e[0] == -1).all() and len(e[1]) == 0


def check_same(a, b):
    assert (a.hypotheses, a.validations, a.n_feature_corr, a.used_mutual, a.best_h, a.inliers) == \
           (b.hypotheses, b.validations, b.n_feature_corr, b.used_mutual, b.best_h, b.inliers)
    assert np.array_equal(a.T, b.T)
    assert a.sum_d2 == b.sum_d2 and a.rmse == b.rmse and a.fitness == b.fitness


@pytest.mark.parametrize("seed", [0, 1])
def test_known_transform(seed):
    """a permuted, moved copy with exact features: RANSAC recovers the transform; C and numpy agree bit for bit"""
    T = rigid(0.7, [3.0, -2.0, 0.5], 0.05, -0.03)
    sx, sf, tx, tf = pair(60, T, seed)
    p = OR.Params(seed=seed + 11)
    a, b = OR.ransac(sx, sf, tx, tf, p), OR.np_ransac(sx, sf, tx, tf, p)
    check_same(a, b)
    assert a.used_mutual and a.n_feature_corr == 60 and a.inliers == 60 and a.fitness == 1.0
    assert np.abs(a.T - T).max() < 1e-9
    assert a.hypotheses == a.best_h + 1   # fitness 1 -> k_d = 0: the loop stops right after the first perfect hypothesis


def test_confidence_stops_the_loop():
    """half the pairs are wrong: the first good hypothesis sets est_k from its fitness and the loop stops there"""
    T = rigid(-0.4, [1.0, 2.0, 0.0])
    sx, sf, tx, tf = pair(40, T, 3)
    rng = np.random.default_rng(9)
    sx[20:] = rng.uniform(-10, 10, (20, 3))          # these sources no longer match their targets' geometry
    p = OR.Params(seed=4, max_corr=0.3)
    a, b = OR.ransac(sx, sf, tx, tf, p), OR.np_ransac(sx, sf, tx, tf, p)
    check_same(a, b)
    assert 0 < a.inliers < 40 and a.hypotheses < p.max_iteration and a.hypotheses >= int(np.ceil(a.k_d))
    q = OR.ransac(sx, sf, tx, tf, OR.Params(seed=4, max_corr=0.3, max_iteration=5))
    assert q.hypotheses <= 5


@pytest.mark.parametrize("extra", [-1, 0])
def test_mutual_fallback_threshold(extra):
    """exactly 3 n - 1 mutual pairs fall back to the one-way set of all n_s pairs; 3 n pairs keep the mutual set"""
    n, ns = 3, 30
    rng = np.random.default_rng(2)
    sf = np.zeros((ns, 33)); ft = np.zeros((ns, 33))
    k = 3 * n + extra
    for i in range(ns):
        sf[i, i] = 100.0
    for j in range(ns):                                # target j < k is the mutual partner of source j; the rest all point at 0
        ft[j] = sf[j] if j < k else sf[0] + 0.5
    sx = rng.uniform(-5, 5, (ns, 3)); tx = sx + [1.0, 0, 0]
    p = OR.Params(ransac_n=n, max_iteration=50)
    a, b = OR.ransac(sx, sf, tx, ft, p), OR.np_ransac(sx, sf, tx, ft, p)
    check_same(a, b)
    assert a.used_mutual == (extra == 0)
    assert a.n_feature_corr == (k if extra == 0 else ns)


def test_empty_results():
    sx, sf, tx, tf = pair(10, np.eye(4), 1)
    for p in (OR.Params(ransac_n=2), OR.Params(max_corr=0.0)):
        r = OR.ransac(sx, sf, tx, tf, p)
        assert r.inliers == 0 and r.hypotheses == 0 and np.array_equal(r.T, np.eye(4))
    assert OR.ransac(sx[:2], sf[:2], tx, tf, OR.Params()).hypotheses == 0
    assert OR.ransac(sx, sf, tx[:0], tf[:0], OR.Params()).n_feature_corr == 0
    assert OR.ransac(sx, sf, tx, tf, OR.Params(max_iteration=0)).hypotheses == 0
