"""CPU: the C restatement of RegistrationRANSACBasedOnFeatureMatching (tests/oracle_ransac.c, DESIGN.md row K-ransac) against its
numpy twin at the settings test_ransac_oracle.py leaves out -- model sizes 4..8 with and without the mutual filter, the mutual
fallback of n = 8, one and two iterations, the extreme seeds, the extreme edge-length checkers -- and the inputs of the device
boundary tests (test_gpu_ransac_boundaries.py), each with the property it is chosen for asserted on the restatement: the seeds whose
best hypothesis is the last one of the first batch of 1024 or the first one of the second, and a pair the confidence never stops.
If the hypothesis stream or a construction changes, these tests fail instead of the device tests silently testing the wrong side."""
import numpy as np
import pytest

import oracle_ransac as OR
from test_ransac_oracle import check_same, pair, rigid


def shifted_seed(seed, n, shift):
    """The seed whose hypothesis h draws what `seed` draws at h + shift: idx(h, j) hashes seed + (h n + j + 1) G, so adding n G shift to
    the seed moves the whole stream by `shift` hypotheses (mod 2^64)."""
    return (seed + n * OR.GOLDEN * shift) % (1 << 64)


# ---- constructions shared with test_gpu_ransac_boundaries.py --------------------------------------------------------------
def model_pair(n, ns=300, seed=40):
    """A moved, permuted copy with a per-n share of the sources moved elsewhere (so several hypotheses validate and the confidence
    stops the loop after tens of them) and a tenth of the source features replaced (so the one-way and the mutual set differ)."""
    corrupt = {3: 0.5, 4: 0.4, 5: 0.3, 7: 0.2, 8: 0.15}[n]
    T = rigid(0.5, [2.0, -1.0, 0.5], -0.05, 0.03)
    sx, sf, tx, tf = pair(ns, T, seed + n)
    rng = np.random.default_rng(seed + 10 * n)
    k = int(round(corrupt * ns))
    sx[rng.permutation(ns)[:k]] = rng.uniform(-10, 10, (k, 3))
    fb = rng.permutation(ns)[:ns // 10]
    sf[fb] = rng.uniform(0, 100, (len(fb), 33))
    return sx, sf, tx, tf


def fallback_pair(n, extra, ns=30):
    """test_ransac_oracle.test_mutual_fallback_threshold's construction: exactly 3 n + extra mutual pairs, every other target is
    the source 0 feature moved by 0.5"""
    rng = np.random.default_rng(2)
    sf = np.zeros((ns, 33)); ft = np.zeros((ns, 33))
    k = 3 * n + extra
    for i in range(ns):
        sf[i, i] = 100.0
    for j in range(ns):
        ft[j] = sf[j] if j < k else sf[0] + 0.5
    sx = rng.uniform(-5, 5, (ns, 3))
    return sx, sf, sx + [1.0, 0, 0], ft


def stop_pair():
    """400 sources, all with exact geometry, but only 44 keep their features: the one-way set (mutual filter off) is about 11 %
    right, so about one hypothesis in 800 draws three right pairs.  Such a hypothesis has fitness 1 and stops the loop at once
    (k_d = 0), so the run's best hypothesis is the first all-right draw of the stream."""
    T = rigid(0.9, [4.0, -3.0, 1.0], 0.1, 0.05)
    sx, sf, tx, tf = pair(400, T, 21)
    rng = np.random.default_rng(22)
    bad = rng.permutation(400)[44:]
    sf[bad] = rng.uniform(0, 100, (len(bad), 33))
    return sx, sf, tx, tf


STOP_PARAMS = dict(mutual_filter=False, max_corr=0.3)
# seed 1 moved by these shifts puts the first all-right draw at h = 1023 (the last of the first default batch) and at h = 1024 (the
# first of the second); test_best_hypothesis_at_batch_edges pins them
BEST_AT = {1023: shifted_seed(1, 3, 1947), 1024: shifted_seed(1, 3, 1946)}


def noisy_pair():
    """300 sources, exact features, the target's geometry with 0.1 m of noise and a tenth of the sources moved elsewhere.  At a
    0.06 m validation radius no hypothesis reaches the fitness that would end the loop within 5000 hypotheses, most of them
    validate, and the best is replaced now and then."""
    T = rigid(-0.6, [1.5, 2.5, -0.5], 0.04, 0.02)
    sx, sf, tx, tf = pair(300, T, 31)
    rng = np.random.default_rng(32)
    tx = tx + rng.normal(0, 0.1, tx.shape)
    sx[rng.permutation(300)[:30]] = rng.uniform(-10, 10, (30, 3))
    return sx, sf, tx, tf


NOISY_PARAMS = dict(max_corr=0.06, seed=5)
NOISY_MAX = 5000


# ---- the restatement against its twin at the new settings ------------------------------------------------------------
def both(sx, sf, tx, tf, p):
    a, b = OR.ransac(sx, sf, tx, tf, p), OR.np_ransac(sx, sf, tx, tf, p)
    check_same(a, b)
    return a


@pytest.mark.parametrize("mutual", [True, False])
@pytest.mark.parametrize("n", [4, 5, 7, 8])
def test_model_size(n, mutual):
    a = both(*model_pair(n, ns=80), OR.Params(mutual_filter=mutual, ransac_n=n, max_corr=0.3, seed=7, max_iteration=2000))
    assert a.used_mutual == mutual and a.validations > 0 and a.inliers > 0


@pytest.mark.parametrize("extra", [-1, 0])
def test_mutual_fallback_n8(extra):
    """n = 8: 23 mutual pairs fall back to the one-way set, 24 keep the mutual set"""
    a = both(*fallback_pair(8, extra), OR.Params(ransac_n=8, max_iteration=50))
    assert a.used_mutual == (extra == 0) and a.n_feature_corr == (24 if extra == 0 else 30)


@pytest.mark.parametrize("max_iteration", [1, 2])
def test_one_and_two_iterations(max_iteration):
    sx, sf, tx, tf = model_pair(3, ns=60)
    for seed in range(4):
        a = both(sx, sf, tx, tf, OR.Params(max_corr=0.3, seed=seed, max_iteration=max_iteration))
        assert a.hypotheses <= max_iteration


@pytest.mark.parametrize("seed", [0, (1 << 64) - 1])
def test_extreme_seeds(seed):
    """seed + (h n + j + 1) G wraps around 2^64 from the first draw on"""
    a = both(*model_pair(4, ns=60), OR.Params(ransac_n=4, max_corr=0.3, seed=seed, max_iteration=500))
    assert a.validations > 0


@pytest.mark.parametrize("edge", [0.0, 1.0])
def test_edge_checker_extremes(edge):
    """0 passes every edge, 1 only edges of exactly equal length"""
    sx, sf, tx, tf = model_pair(3, ns=60)
    a = both(sx, sf, tx, tf, OR.Params(max_corr=0.3, checker_edge=edge, seed=3, max_iteration=300))
    if edge == 0.0:
        assert a.validations > 0


# ---- the properties the device tests rely on ----------------------------------------------------------------------------
def test_seed_shift_moves_the_stream():
    for seed, n, shift in ((1, 3, 1947), (5, 8, -3), ((1 << 64) - 1, 4, 10 ** 6)):
        s = shifted_seed(seed, n, shift)
        for h in (0, 1, 1023):
            for j in range(n):
                assert OR.np_stream(s, h, n, j, 1000) == OR.np_stream(seed, h + shift, n, j, 1000) == OR.stream(s, h, n, j, 1000)


@pytest.mark.parametrize("want", [1023, 1024])
def test_best_hypothesis_at_batch_edges(want):
    """the pinned seeds: the only update that sets best to fitness 1 happens at h = 1023 / 1024, and the loop stops right after"""
    sx, sf, tx, tf = stop_pair()
    a = both(sx, sf, tx, tf, OR.Params(seed=BEST_AT[want], **STOP_PARAMS))
    assert a.best_h == want and a.hypotheses == want + 1 and a.fitness == 1.0
    assert 1 < a.validations < 20


def test_confidence_never_stops_the_noisy_pair():
    sx, sf, tx, tf = noisy_pair()
    p = OR.Params(max_iteration=NOISY_MAX, **NOISY_PARAMS)
    a = OR.ransac(sx, sf, tx, tf, p)
    assert a.hypotheses == NOISY_MAX and a.k_d > NOISY_MAX and a.best_h > 2049
    assert NOISY_MAX // 2 < a.validations < NOISY_MAX
    # hypothesis 4096 validates: with 4097 hypotheses per batch it is the survivor in the second tile of the survivor scan
    v = [OR.ransac(sx, sf, tx, tf, OR.Params(max_iteration=k, **NOISY_PARAMS)).validations for k in (4096, 4097)]
    assert v[1] == v[0] + 1
    b = both(sx, sf, tx, tf, OR.Params(max_iteration=300, **NOISY_PARAMS))   # the twin on a prefix (it validates by brute force)
    assert b.validations > 200
