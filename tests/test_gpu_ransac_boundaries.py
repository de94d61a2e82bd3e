"""-m gpu: the loop-closure proposal (ransac.cu, features.cu, DESIGN.md rows K-ransac / K-fpfh) against the C restatements on both
sides of every tile, scan, batch and list boundary its kernels have.  RANSAC results are held to tests/oracle_ransac.c with the idiom
of test_gpu_place_recognition.check (counts, best h, set size and inliers equal, T bit-identical, fitness equal, rmse to 1e-12);
correspondences and FPFH rows are bit-identical.  Each input also asserts the side it was built for (the mutual-set size, the
oracle's best h, the oracle's neighbour counts), so that a changed launch constant fails here instead of testing one side twice.
Run with -s to see the sides reached.

  fm_tile_kernel / fm_merge_kernel  64-row source and target tiles; exact feature ties split across two tiles on either side
  mutual flags, survivor flags      batched look-back scan of 4096 items per tile: mutual sets below, at and above 4096, a batch
                                    of 4097 hypotheses whose survivor scan has a second tile
  rs_hyp_kernel                     ransac_n 3..8, the mutual fallback at 3 n - 1 / 3 n for n = 8
  rs_replay_kernel                  max_iteration and the best update at h = B - 1, B, B + 1 of the default batch of 1024
  op_ransac                         one source against targets of mixed sizes with an empty one in the middle
  rs_validate_kernel                a target grid coarsened far beyond the validation radius, sources moved outside its box
  fpfh_knn_kernel                   k-best list of 32-entry register rows: knn at and next to every row edge

Not tested: a non-finite feature row (s2t = -1, so the one-way set would index txyz[-1] on the device and in the restatement
alike; the input is undefined in every implementation)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_features as OF
import oracle_ransac as OR
from open3d_slam_b200 import engine as E
from test_fpfh_oracle import random_cloud
from test_gpu_fpfh import check as check_fpfh
from test_gpu_place_recognition import check, feat, same
from test_ransac_oracle import pair, rigid
from test_ransac_oracle_boundaries import (BEST_AT, NOISY_MAX, NOISY_PARAMS, STOP_PARAMS, fallback_pair, model_pair, noisy_pair,
                                           stop_pair)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CHILD = os.path.join(HERE, "ransac_boundary_child.py")
# the launch constants the inputs straddle (ransac.cu, runtime.cu, features.cu)
FM_TILE = 64          # feature rows per fm_tile_kernel tile, source and target
SCAN_TILE = 4096      # items per tile of scan_exclusive_i32_batch (SCAN_THREADS x SCAN_ITEMS)
DEFAULT_B = 1024      # hypotheses per batch without B2S_RANSAC_BATCH
FPFH_ROW = 32         # entries per register row of the fpfh_knn_kernel k-best list (B2S_FEATURE_MAX_KNN = 4 rows)
UPDATE = "update the boundary inputs in tests/test_gpu_ransac_boundaries.py to the new launch constants"


def run(eng, sx, sf, tx, tf, pr, mutual=True):
    got = E.registrationRANSACBasedOnFeatureMatching(eng, eng.cloud(sx), eng.cloud(tx), feat(eng, sf), feat(eng, tf), pr, mutual_filter=mutual)
    ref = OR.ransac(sx, sf, tx, tf, OR.Params.of(pr, mutual_filter=mutual))
    check(got, ref)
    return got, ref


def show(what, r):
    print(f"{what}: set {r.n_feature_corr} mutual {r.used_mutual} hypotheses {r.hypotheses} validations {r.validations} "
          f"best h {r.best_h} inliers {r.inliers}")


# ---- a. correspondences across tiles and ties ------------------------------------------------------------------------------
@pytest.mark.parametrize("ns,nt", [(4095, 4097), (4096, 4096), (4097, 130), (8193, 65)])
def test_correspondences_across_tiles_and_ties(engine_factory, ns, nt):
    """source rows 63 / 64, 127 / 128 and 4095 / 4096 are equal pairs in two source tiles, each copied into a target row, so that
    target row's nearest source is an exact tie merged across the tiles; target rows 63 / 64 are an equal pair in two target tiles,
    a copy of source row 10.  Every tie goes to the lower index."""
    eng = engine_factory()
    rng = np.random.default_rng(ns + 3 * nt)
    fs, ft = rng.uniform(0, 50, (ns, 33)), rng.uniform(0, 50, (nt, 33))
    ties = [a for a in (FM_TILE - 1, 2 * FM_TILE - 1, SCAN_TILE - 1) if a + 1 < ns]
    for k, a in enumerate(ties):
        fs[a + 1] = fs[a]
        ft[1 + k] = fs[a]
    ft[FM_TILE - 1] = ft[FM_TILE] = fs[10]
    s2t, t2s = E.featureCorrespondences(eng, feat(eng, fs), feat(eng, ft))
    r = OR.feature_corr(fs, ft)
    for k, a in enumerate(ties):   # the inputs sit on the intended sides
        assert a // FM_TILE != (a + 1) // FM_TILE and r[1][1 + k] == a and r[0][a] == r[0][a + 1] == 1 + k, (a, UPDATE)
    assert r[0][10] == FM_TILE - 1 and r[1][FM_TILE - 1] == r[1][FM_TILE] == 10
    assert np.array_equal(s2t, r[0]) and np.array_equal(t2s, r[1])
    print(f"ns {ns} nt {nt}: source tile ties at {ties}, target tie at {FM_TILE - 1}/{FM_TILE}")


# ---- b. a mutual set across the scan tile ----------------------------------------------------------------------------------
def corrupted_features(ns):
    """source rows whose features are replaced (each one drops out of the mutual set): an irregular subset, and for the sizes
    above one scan tile a contiguous run that straddles index 4096"""
    rng = np.random.default_rng(ns)
    if ns == SCAN_TILE + 1:
        return np.array([1000])                                     # the mutual set is exactly one tile; row 4096 is mutual
    idx = [rng.permutation(ns)[:ns // 40], np.arange(ns - 300, ns, 13)]
    if ns > SCAN_TILE + 200:
        idx += [np.arange(SCAN_TILE - 100, SCAN_TILE + 150), np.arange(6000, ns, 5)]
    return np.unique(np.concatenate(idx))


@pytest.mark.parametrize("ns", [SCAN_TILE - 1, SCAN_TILE, SCAN_TILE + 1, 2 * SCAN_TILE + 1])
def test_mutual_set_across_the_scan_tile(engine_factory, ns):
    eng = engine_factory()
    T = rigid(0.4, [2.0, 1.0, -0.5], 0.03, -0.02)
    sx, sf, tx, tf = pair(ns, T, 50 + ns)
    rng = np.random.default_rng(60 + ns)
    bad = corrupted_features(ns)
    sf[bad] = rng.uniform(0, 100, (len(bad), 33))
    geo = rng.permutation(ns)[:3 * ns // 10]                        # 30 % of the geometry wrong: several hypotheses validate
    sx[geo] = rng.uniform(-10, 10, (len(geo), 3))
    s2t, t2s = OR.feature_corr(sf, tf)
    mutual = np.flatnonzero(t2s[s2t] == np.arange(ns))
    want = {SCAN_TILE - 1: lambda m: m < SCAN_TILE, SCAN_TILE: lambda m: m < SCAN_TILE, SCAN_TILE + 1: lambda m: m == SCAN_TILE,
            2 * SCAN_TILE + 1: lambda m: m > SCAN_TILE}[ns]
    assert want(len(mutual)), (ns, len(mutual), UPDATE)
    if ns > SCAN_TILE:
        assert mutual[-1] >= SCAN_TILE                              # flags set in the second tile of the mutual scan
    pr = E.PlaceRecognitionParameters(ransacMaxCorrespondenceDistance=0.3, ransacSeed=4, ransacNumIter=3000)
    got, ref = run(eng, sx, sf, tx, tf, pr)
    assert ref.used_mutual and ref.n_feature_corr == len(mutual) and ref.validations > 1
    show(f"ns {ns}", ref)


# ---- c. model size -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mutual", [True, False])
@pytest.mark.parametrize("n", [3, 4, 5, 7, 8])
def test_model_size(engine_factory, n, mutual):
    eng = engine_factory()
    pr = E.PlaceRecognitionParameters(ransacModelSize=n, ransacMaxCorrespondenceDistance=0.3, ransacSeed=7, ransacNumIter=20000)
    got, ref = run(eng, *model_pair(n), pr, mutual=mutual)
    assert ref.used_mutual == mutual and 0 < ref.validations < ref.hypotheses
    show(f"n {n} mutual {mutual}", ref)


@pytest.mark.parametrize("extra", [-1, 0])
def test_mutual_fallback_threshold_n8(engine_factory, extra):
    """23 mutual pairs fall back to the one-way set, 24 keep the mutual set"""
    eng = engine_factory()
    pr = E.PlaceRecognitionParameters(ransacModelSize=8, ransacNumIter=50)
    got, ref = run(eng, *fallback_pair(8, extra), pr)
    assert ref.used_mutual == (extra == 0) and ref.n_feature_corr == (24 if extra == 0 else 30)


# ---- d. mixed batch ----------------------------------------------------------------------------------------------------------
def test_mixed_batch_with_an_empty_target(engine_factory):
    """one source against targets of 65, 0, 2, 4097 and 64 points (the first min(nt, 300) source points moved, plus random points
    with random features): each result is its single call's and the restatement's, the empty target's the empty result"""
    eng = engine_factory()
    sx, sf, _, _ = pair(300, np.eye(4), 70)
    rng = np.random.default_rng(71)
    targets = []
    for k, nt in enumerate((65, 0, 2, 4097, 64)):
        T = rigid(0.2 * k, [k, -1.0, 0.5])
        m = min(nt, len(sx))
        idx = rng.permutation(len(sx))[:m]
        tx = np.vstack([sx[idx] @ T[:3, :3].T + T[:3, 3], rng.uniform(-10, 10, (nt - m, 3))])
        tf = np.vstack([sf[idx], rng.uniform(0, 100, (nt - m, 33))])
        targets.append((tx, tf))
    pr = E.PlaceRecognitionParameters(ransacMaxCorrespondenceDistance=0.3, ransacSeed=2, ransacNumIter=3000)
    s, fs = eng.cloud(sx), feat(eng, sf)
    clouds, feats = [eng.cloud(tx) for tx, _ in targets], [feat(eng, tf) for _, tf in targets]
    batch = E.registrationRANSACBasedOnFeatureMatchingBatch(eng, s, clouds, fs, feats, pr)
    assert len(batch) == len(targets)
    for (tx, tf), c, f, got in zip(targets, clouds, feats, batch):
        assert same(got, E.registrationRANSACBasedOnFeatureMatching(eng, s, c, fs, f, pr))
        ref = OR.ransac(sx, sf, tx, tf, OR.Params.of(pr))
        check(got, ref)
        show(f"nt {len(tx)}", ref)
    e = batch[1]
    assert e.hypotheses == 0 and e.best_hypothesis == -1 and e.n_corr == 0 and e.n_feature_corr == 0 and np.array_equal(e.transformation_, np.eye(4))
    assert all(r.hypotheses > 0 for k, r in enumerate(batch) if k != 1)


# ---- e. replay at the batch edges -------------------------------------------------------------------------------------------
def noisy_params(max_iteration):
    return E.PlaceRecognitionParameters(ransacMaxCorrespondenceDistance=NOISY_PARAMS["max_corr"], ransacSeed=NOISY_PARAMS["seed"],
                                        ransacNumIter=max_iteration)


@pytest.mark.parametrize("max_iteration", [1, DEFAULT_B - 1, DEFAULT_B, DEFAULT_B + 1, 2 * DEFAULT_B + 1])
def test_max_iteration_at_the_batch_edges(engine_factory, max_iteration):
    eng = engine_factory()
    got, ref = run(eng, *noisy_pair(), noisy_params(max_iteration))
    assert ref.hypotheses == max_iteration, UPDATE                  # the confidence never ends the loop first
    show(f"max_iteration {max_iteration}", ref)


def test_a_run_that_ends_at_the_batch_edge_launches_no_further_batch(engine_factory):
    """max_iteration = B ends in one batch like B - 1; B + 1 needs a second one"""
    eng = engine_factory()
    sx, sf, tx, tf = noisy_pair()
    s, t, fs, ft = eng.cloud(sx), eng.cloud(tx), feat(eng, sf), feat(eng, tf)
    E.registrationRANSACBasedOnFeatureMatching(eng, s, t, fs, ft, noisy_params(DEFAULT_B))   # first call: scratch and grids
    launches = []
    for k in (DEFAULT_B - 1, DEFAULT_B, DEFAULT_B + 1):
        before = eng.launches
        E.registrationRANSACBasedOnFeatureMatching(eng, s, t, fs, ft, noisy_params(k))
        launches.append(eng.launches - before)
    print(f"launches for max_iteration B - 1, B, B + 1: {launches}")
    assert launches[0] == launches[1] < launches[2]


@pytest.mark.parametrize("want", [DEFAULT_B - 1, DEFAULT_B])
def test_best_update_at_the_batch_edge(engine_factory, want):
    """the seeds of test_ransac_oracle_boundaries.BEST_AT: the fitness-1 hypothesis that ends the loop is the last of the first
    batch (the stop is decided after its replay) or the first of the second"""
    eng = engine_factory()
    pr = E.PlaceRecognitionParameters(ransacMaxCorrespondenceDistance=STOP_PARAMS["max_corr"], ransacSeed=BEST_AT[want])
    got, ref = run(eng, *stop_pair(), pr, mutual=STOP_PARAMS["mutual_filter"])
    assert ref.best_h == want and got.best_hypothesis == want and got.hypotheses == want + 1, UPDATE
    show(f"best at {want}", ref)


def test_batches_of_4096_and_4097(tmp_path):
    """B2S_RANSAC_BATCH = 4096 and 4097 in child processes on the noisy pair (5000 hypotheses, hypothesis 4096 validates): with 4097
    the survivor scan of the first batch has a second tile holding that survivor.  Both equal the restatement."""
    outs = []
    for b in ("4096", "4097"):
        env = dict(os.environ)
        env["B2S_RANSAC_BATCH"] = b
        out = tmp_path / f"r{b}.json"
        subprocess.check_call([sys.executable, CHILD, str(out)], env=env)
        outs.append(json.loads(out.read_text()))
    assert outs[0] == outs[1]
    sx, sf, tx, tf = noisy_pair()
    ref = OR.ransac(sx, sf, tx, tf, OR.Params(max_iteration=NOISY_MAX, **NOISY_PARAMS))
    got = outs[0]
    assert (got["hypotheses"], got["validations"], got["best_hypothesis"], got["n_feature_corr"], got["used_mutual"], got["inliers"]) == \
           (ref.hypotheses, ref.validations, ref.best_h, ref.n_feature_corr, ref.used_mutual, ref.inliers)
    assert np.array_equal(np.array(got["T"]).reshape(4, 4), ref.T) and got["fitness"] == ref.fitness
    assert abs(got["rmse"] - ref.rmse) <= 1e-12 * max(ref.rmse, 1e-300)
    assert ref.hypotheses == NOISY_MAX > 4097 + 1
    show("B 4096 / 4097", ref)


# ---- f. validation grid -------------------------------------------------------------------------------------------------------
def grid_cell(points, cell):
    """grid_build's cell edge for a fresh cloud of these points: 8 cells per point (the allocation rounds the cloud up by at most a
    quarter), between 2^16 and 2^21 cells; the edge doubles until the box fits"""
    n_alloc = len(points) + len(points) // 4
    cap = min(max(n_alloc * 8 + 4096, 1 << 16), 1 << 21)
    assert cap == min(max(len(points) * 8 + 4096, 1 << 16), 1 << 21)   # the rounding does not change the budget
    ext = points.max(axis=0) - points.min(axis=0)
    while np.prod(np.floor(ext / cell) + 1.0) > cap:
        cell *= 2.0
    return cell


@pytest.mark.parametrize("mutual", [True, False])
def test_validation_grid_coarsened_beyond_the_radius(engine_factory, mutual):
    """a 40 m target validated at r = 0.05: the grid's cells are 32 times the radius, and the sources the target does not cover
    land outside its box"""
    eng = engine_factory()                                          # a fresh handle: grids only grow
    rng = np.random.default_rng(80)
    sx, sf = rng.uniform(-20, 20, (2000, 3)), rng.uniform(0, 100, (2000, 33))
    T = rigid(0.3, [1.0, -2.0, 0.5], 0.02, 0.01)
    keep = np.flatnonzero(sx[:, 0] < 8.0)
    perm = rng.permutation(len(keep))
    tx, tf = (sx[keep] @ T[:3, :3].T + T[:3, 3])[perm], sf[keep][perm]
    r = 0.05
    cell = grid_cell(tx, r)
    assert cell >= 16 * r, (cell, UPDATE)
    moved = sx @ T[:3, :3].T + T[:3, 3]
    outside = ((moved < tx.min(axis=0) - r) | (moved > tx.max(axis=0) + r)).any(axis=1)
    assert outside.sum() > 100
    pr = E.PlaceRecognitionParameters(ransacMaxCorrespondenceDistance=r, ransacSeed=6, ransacNumIter=3000)
    got, ref = run(eng, sx, sf, tx, tf, pr, mutual=mutual)
    assert ref.validations > 1 and ref.inliers == len(keep)
    print(f"grid cell {cell} m for r {r} m, {outside.sum()} sources outside the target box")
    show(f"grid mutual {mutual}", ref)


# ---- 3. FPFH k-best list at its register-row edges -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dense_cloud():
    return random_cloud(20000, 4, extent=1.0)                       # ~1300 points inside r = 0.5 of an interior query


@pytest.mark.parametrize("knn", [1, 2, FPFH_ROW - 1, FPFH_ROW, 2 * FPFH_ROW - 1, 2 * FPFH_ROW, 2 * FPFH_ROW + 1, 3 * FPFH_ROW,
                                 3 * FPFH_ROW + 1, 4 * FPFH_ROW - 1, 4 * FPFH_ROW])
def test_fpfh_knn_at_the_list_row_edges(engine_factory, dense_cloud, knn):
    """the k-th entry sits in lane (knn - 1) % 32 of row (knn - 1) // 32; every list is full, so every insert shifts across the rows"""
    eng = engine_factory()
    xyz, nrm = dense_cloud
    got, det = check_fpfh(eng, xyz, nrm, 0.5, knn)
    full = (det["nb_cnt"] == knn).mean()
    print(f"knn {knn}: row {(knn - 1) // FPFH_ROW} lane {(knn - 1) % FPFH_ROW}, {full:.4f} of the lists full")
    assert full == 1.0, (full, UPDATE)
    if knn == 1:
        assert not got.any()                                        # only the point itself: no pairs, all-zero rows
