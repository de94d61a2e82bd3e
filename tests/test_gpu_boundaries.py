"""-m gpu: the device path against the CPU oracle on both sides of every size switch the kernels make.

The kernels choose their code paths from the input size, from knn and from the SM count.  Each switch is crossed here by a pair of
inputs, one on either side, and both sides are held to the oracle with the idioms of test_gpu_parity.py (iterations and
correspondences equal, fitness to 1e-12, T to 1e-9, keyed bit-exact voxel means).  Where the library exposes which side a run took
(the ICP debug counters, the normals debug record), the test asserts it, so that a change of a launch constant makes these
tests fail instead of silently testing one side twice.  Run with -s to see the sides that were reached.

  ICP (csrc/icp.cu)        cluster size: doubles while size x threads < n (768 threads point-to-plane, 512 GICP), up to 8 or 16 CTAs
                           source tiles of 64 points: partial last tile, CTAs without tiles
                           source in shared memory while a CTA's chunk is at most ~4.9 k points, in global memory above
                           batches: cluster size of the largest source, shrunk while problems x size > 2 x SMs
                           certificates: runner-up ties, points crossing the d2 < r2 cut, large slacks far from the origin
  normals (csrc/normals.cu) knn 1..32 (33 refused), identity covariance below 3 neighbours, flagged (selected) queries,
                           every exit of the select kernel, coarsened grid cells
  voxel / sort             u32 keys up to 10 bits per axis, u64 up to 21, refused above; one-cluster sort up to 3 << 18 keys;
                           the wide grid from 2^19 points; results independent of the grid size (B2S_GRID_CAP, B2S_SORT)
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import normals_checks as NC
from oracle import oracle as O
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import synth
from open3d_slam_b200 import _lib as L

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CHILD = os.path.join(HERE, "boundary_child.py")
TILE = 64
UPDATE = "update the boundary sizes in tests/test_gpu_boundaries.py to the new launch constants"


def rel_rot(Ta, Tb):
    return np.linalg.norm(Ta[:3, :3] - Tb[:3, :3]) / np.linalg.norm(Tb[:3, :3])


def rel_trans(Ta, Tb):
    return np.linalg.norm(Ta[:3, 3] - Tb[:3, 3]) / max(np.linalg.norm(Tb[:3, 3]), 1.0)


def assert_matches_oracle(res, ref, what=""):
    assert res.iters == ref.iters and res.n_corr == ref.n_corr, (what, res.iters, ref.iters, res.n_corr, ref.n_corr)
    assert abs(res.fitness_ - ref.fitness) < 1e-12, (what, res.fitness_, ref.fitness)
    assert rel_rot(res.transformation_, ref.T) < 1e-9 and rel_trans(res.transformation_, ref.T) < 1e-9, (what, res.transformation_, ref.T)


def assert_same_registration(a, b, tol=1e-10, what=""):
    assert a.iters == b.iters and a.n_corr == b.n_corr, (what, a.iters, b.iters, a.n_corr, b.n_corr)
    assert np.abs(a.transformation_ - b.transformation_).max() < tol, what


def params(r=0.5, max_iter=30, ctas=0, reg_type="PointToPlaneIcp"):
    p = E.MapperParameters()
    p.icp.maxCorrespondenceDistance = r
    p.icp.maxNumIter = max_iter
    p.icpClusterCtas = ctas
    p.scanToMapRegType = reg_type
    return p


def room(n, rng, half=8.0, height=4.0, noise=0.02):
    """Floor and two walls of a room corner (the three planes constrain all six degrees of freedom)."""
    k = n // 3
    return np.vstack([np.c_[rng.uniform(-half, half, (n - 2 * k, 2)), noise * rng.standard_normal(n - 2 * k)],
                      np.c_[rng.uniform(-half, half, k), np.full(k, half) + noise * rng.standard_normal(k), rng.uniform(0, height, k)],
                      np.c_[np.full(k, -half) + noise * rng.standard_normal(k), rng.uniform(-half, half, k), rng.uniform(0, height, k)]])


def sample_source(tgt, n_src, rng, outliers=0.1):
    """Noisy target samples under the inverse of a known SE(3), plus a share of outliers 1.5-6 m above the room (beyond r of every
    target, and beyond the one-cell box of the first search).  Shuffled, so that the outliers are spread over every tile."""
    T_true = synth.se3(0.01, -0.015, 0.02, (0.06, -0.04, 0.03))
    pts = tgt[rng.integers(0, len(tgt), n_src)] + 0.01 * rng.standard_normal((n_src, 3))
    n_out = int(round(outliers * n_src))
    pts[:n_out] = np.c_[rng.uniform(-8, 8, (n_out, 2)), rng.uniform(5.5, 10.0, n_out)]
    src = (pts - T_true[:3, 3]) @ T_true[:3, :3]
    return np.ascontiguousarray(src[rng.permutation(n_src)])


def icp_pair(n_src, seed, n_tgt=20_000, outliers=0.1):
    """A room-corner target with oracle normals and a source sampled from it."""
    rng = np.random.default_rng(seed)
    tgt = room(n_tgt, rng)
    return sample_source(tgt, n_src, rng, outliers), tgt, O.estimate_normals(tgt, 10, 1.0)


# ----------------------------------------------------------------------------------------------------------------------
# what the ICP debug counters say about a launch
# ----------------------------------------------------------------------------------------------------------------------
def tile_counts(n, csize):
    """Points of CTA 0..7 when n source points are dealt out in 64-point tiles, tile t to CTA t % csize (icp_kernel)."""
    ntiles = -(-n // TILE)
    out = []
    for r in range(8):
        if r >= csize or r >= ntiles:
            out.append(0)
            continue
        mine = (ntiles - r + csize - 1) // csize
        last = (ntiles - 1) % csize == r
        out.append(mine * TILE - (ntiles * TILE - n if last else 0))
    return out


class Geometry:
    """Evaluation 0 of problem 0 as b2s_debug_icp_clocks recorded it: points and phase-2 queue length of CTA 0..7, and (point-to-
    plane) the points the whole cluster queued for phase 2.  The cluster sizes consistent with the point counts are kept as a
    set: below one tile every size deals the same."""

    def __init__(self, words, n, counted):
        w = np.asarray(words, dtype=np.int64)
        self.n = n
        self.counts = [int(w[256 + 4 * r + 3]) for r in range(8)]
        self.queues = [int(w[256 + 4 * r + 2]) for r in range(8)]
        self.queued = int(w[512 + 2]) if counted else sum(self.queues)
        self.sizes = {c for c in (1, 2, 4, 8, 16) if tile_counts(n, c) == self.counts}

    @property
    def shared(self):
        return self.queued > 0   # only the shared-memory path has a phase-2 queue (the sources carry outliers that need it)

    def __repr__(self):
        path = "shared memory" if self.shared else "no phase-2 queue (global memory)"
        return f"n={self.n}: cluster {sorted(self.sizes)} CTAs, {path}, phase-2 queue {self.queued}, points per CTA {self.counts}"


def traced(eng, call):
    """Run `call` with the ICP debug counters on (icp_kernel<3> for point-to-plane); returns (its result, the 1024 words)."""
    buf = (C.c_longlong * 1024)()
    L.check(L.lib().b2s_debug_icp_clocks(eng._h, 1, None))
    try:
        res = call()
        L.check(L.lib().b2s_debug_icp_clocks(eng._h, 1, buf))
    finally:
        L.check(L.lib().b2s_debug_icp_clocks(eng._h, 0, None))
    return res, list(buf)


def register_both_ways(engine_factory, n, seed, p, gicp=False, r=0.5):
    """Oracle, device (debug off), device (debug on): all three must agree; returns the launch geometry of the debug run."""
    src, tgt, nrm = icp_pair(n, seed)
    init = np.eye(4)
    eng = engine_factory(p)
    if gicp:
        snrm = O.estimate_normals(src, 10, 1.0)
        reg = E.cloudRegistrationFactory(eng, E.CloudRegistrationParameters(regType="GeneralizedIcp", icp=p.icp))
        ref = O.registration_gicp(src, snrm, tgt, nrm, r, init, max_iter=p.icp.maxNumIter)
        sc = eng.cloud(src, snrm)
    else:
        reg = E.cloudRegistrationFactory(eng, E.CloudRegistrationParameters(icp=p.icp))
        ref = O.registration_icp_p2plane(src, tgt, nrm, r, init, max_iter=p.icp.maxNumIter)
        sc = eng.cloud(src)
    tc = eng.cloud(tgt, nrm)
    res = reg.registerClouds(sc, tc, init)
    assert_matches_oracle(res, ref, f"n={n}")
    res_dbg, words = traced(eng, lambda: reg.registerClouds(sc, tc, init))
    assert_matches_oracle(res_dbg, ref, f"n={n} (debug counters on)")
    geo = Geometry(words, n, counted=not gicp)
    assert geo.sizes, f"n={n}: per-CTA point counts {geo.counts} match no cluster size of the 64-point tiling; {UPDATE}"
    return geo


def check_switch(kind, lo, hi):
    """lo and hi must lie on the two sides of one switch of the given kind."""
    msg = f"{lo} | {hi} no longer straddle the {kind} switch; {UPDATE}"
    if kind == "cluster":
        assert max(lo.sizes) < min(hi.sizes) and lo.shared and hi.shared, msg
    elif kind == "memory":
        assert lo.sizes == hi.sizes and lo.shared and not hi.shared, msg
    else:   # tiles: one CTA, every point in it
        assert lo.counts[0] == lo.n and hi.counts[0] == hi.n, msg


P2PLANE_GROUPS = [((1, 2), "tiles"), ((63, 64, 65), "tiles"), ((767, 768, 769), "cluster"), ((1536, 1537), "cluster"),
                  ((3072, 3073), "cluster"), ((39_424, 39_425), "memory")]
SIXTEEN_GROUPS = [((6144, 6145), "cluster"), ((78_848, 78_849), "memory")]
GICP_GROUPS = [((511, 512, 513), "cluster", 0), ((1024, 1025), "cluster", 0), ((2048, 2049), "cluster", 0),
               ((4096, 4097), "cluster", 16), ((39_424, 39_425), "memory", 0)]   # 8 -> 16 CTAs only when 16 are allowed


def _run_group(engine_factory, sizes, kind, p, gicp=False):
    geos = [register_both_ways(engine_factory, n, 100 + n % 997, p, gicp=gicp) for n in sizes]
    for g in geos:
        print(("GICP " if gicp else "point-to-plane ") + (f"[{p.icpClusterCtas} CTAs max] " if p.icpClusterCtas else "") + repr(g))
    if len(geos) == 3:   # the first pair stays on one side
        assert geos[0].sizes == geos[1].sizes and geos[0].shared == geos[1].shared, f"{geos[0]} | {geos[1]}: {UPDATE}"
    check_switch(kind, geos[-2], geos[-1])


@pytest.mark.parametrize("sizes,kind", P2PLANE_GROUPS, ids=[f"{k}-{s[-1]}" for s, k in P2PLANE_GROUPS])
def test_icp_point_to_plane_launch_boundaries(engine_factory, sizes, kind):
    _run_group(engine_factory, sizes, kind, params())


@pytest.mark.parametrize("sizes,kind", SIXTEEN_GROUPS, ids=[f"{k}-{s[-1]}" for s, k in SIXTEEN_GROUPS])
def test_icp_sixteen_cta_launch_boundaries(engine_factory, sizes, kind):
    _run_group(engine_factory, sizes, kind, params(ctas=16))


@pytest.mark.parametrize("sizes,kind,ctas", GICP_GROUPS, ids=[f"{k}-{s[-1]}" for s, k, _ in GICP_GROUPS])
def test_icp_gicp_launch_boundaries(engine_factory, sizes, kind, ctas):
    _run_group(engine_factory, sizes, kind, params(ctas=ctas, reg_type="GeneralizedIcp"), gicp=True)


# ----------------------------------------------------------------------------------------------------------------------
# batches
# ----------------------------------------------------------------------------------------------------------------------
def test_icp_ragged_batch(engine_factory):
    """One launch with an empty, a 1-point, a 65-point, a scan-sized and a global-memory source, four targets (one shared by two
    pairs).  The batch runs every problem with the cluster size of the largest source, CTAs without tiles included."""
    p = params()
    eng = engine_factory(p)
    reg = E.RegistrationIcpPointToPlane(eng)
    pairs = [icp_pair(40_000, 1), icp_pair(6000, 2), icp_pair(65, 3), icp_pair(1, 4), icp_pair(0, 5)]
    shared = pairs[1]
    pairs[2] = (pairs[2][0], shared[1], shared[2])          # the 65-point source against the scan-sized pair's target
    rng = np.random.default_rng(8)
    inits = [synth.se3(*rng.uniform(-0.01, 0.01, 3), rng.uniform(-0.03, 0.03, 3)) for _ in pairs]
    tclouds = {}
    for s, t, nr in pairs:
        if id(t) not in tclouds:
            tclouds[id(t)] = eng.cloud(t, nr)
    sclouds = [eng.cloud(s) for s, _, _ in pairs]
    targets = [tclouds[id(t)] for _, t, _ in pairs]
    assert len(tclouds) == 4
    batch = reg.registerCloudsBatch(sclouds, targets, inits)
    dbg, words = traced(eng, lambda: reg.registerCloudsBatch(sclouds, targets, inits))
    geo = Geometry(words, len(pairs[0][0]), counted=True)
    print("ragged batch, problem 0:", geo)
    assert geo.sizes == {8} and not geo.shared, f"{geo}: the 40 000-point source should run on 8 CTAs from global memory; {UPDATE}"
    for k, ((s, t, nr), init, b, d) in enumerate(zip(pairs, inits, batch, dbg)):
        ref = O.registration_icp_p2plane(s, t, nr, 0.5, init, max_iter=30)
        assert_matches_oracle(b, ref, f"batch problem {k} ({len(s)} points)")
        assert_matches_oracle(d, ref, f"batch problem {k} ({len(s)} points, debug counters on)")
        single = reg.registerClouds(sclouds[k], targets[k], init)
        assert_same_registration(b, single, what=f"batch problem {k} vs the same pair alone")


def test_icp_batch_shrink_threshold(engine_factory):
    """Batched clusters shrink while problems x cluster size > 2 x SMs.  Batches just below and just above each step (8 -> 4 and
    4 -> 2 CTAs) must equal every pair registered alone, and a seeded sample must equal the oracle."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = [(2 * sms) // 8, (2 * sms) // 8 + 1, (2 * sms) // 4, (2 * sms) // 4 + 1]
    expect = [8, 4, 4, 2]
    n_src = 6000                                  # 8 CTAs alone; 2 CTAs still hold a chunk in shared memory
    p = params()
    eng = engine_factory(p)
    reg = E.RegistrationIcpPointToPlane(eng)
    rng = np.random.default_rng(17)
    targets = [icp_pair(0, 40 + k) for k in range(3)]
    tclouds = [eng.cloud(t, nr) for _, t, nr in targets]
    srcs, tsel, inits = [], [], []
    for k in range(sizes[-1]):
        tsel.append(k % 3)
        srcs.append(sample_source(targets[k % 3][1], n_src, rng))
        inits.append(synth.se3(*rng.uniform(-0.01, 0.01, 3), rng.uniform(-0.03, 0.03, 3)))
    sclouds = [eng.cloud(s) for s in srcs]
    alone = [reg.registerClouds(sclouds[k], tclouds[tsel[k]], inits[k]) for k in range(len(srcs))]
    for m, want in zip(sizes, expect):
        args = (sclouds[:m], [tclouds[j] for j in tsel[:m]], inits[:m])
        _, words = traced(eng, lambda: reg.registerCloudsBatch(*args))
        geo = Geometry(words, n_src, counted=True)
        print(f"batch of {m} problems ({sms} SMs):", geo)
        assert geo.sizes == {want} and geo.shared, f"batch of {m}: {geo}, expected {want} CTAs; {UPDATE}"
        batch = reg.registerCloudsBatch(*args)
        for k in range(m):
            assert_same_registration(batch[k], alone[k], what=f"batch of {m}, problem {k}")
        for k in np.random.default_rng(m).choice(m, 2, replace=False):
            _, t, nr = targets[tsel[k]]
            assert_matches_oracle(batch[k], O.registration_icp_p2plane(srcs[k], t, nr, 0.5, inits[k], max_iter=30), f"batch of {m}, problem {k}")


# ----------------------------------------------------------------------------------------------------------------------
# certificates: multi-iteration cases on the shared-memory path, cluster sizes 2, 4, 8, 16
# ----------------------------------------------------------------------------------------------------------------------
CLUSTERS = [(2, 1400, 0), (4, 3000, 0), (8, 8000, 0), (16, 12_000, 16)]   # (cluster size, source points, icpClusterCtas)


def lattice_room(spacing=0.25, half=6.0, height=3.0):
    g = np.arange(-half, half + 1e-9, spacing)
    h = np.arange(0.0, height + 1e-9, spacing)
    floor = np.array([(x, y, 0.0) for x in g for y in g])
    wy = np.array([(x, half, z) for x in g for z in h[1:]])
    wx = np.array([(-half, y, z) for y in g for z in h[1:]])
    return np.vstack([floor, wy, wx])


def adversarial_source(tgt, n, rng, r, spacing=0.25, half=6.0):
    """Midpoints of lattice neighbours on all three planes: the runner-up gap of the certificate starts at ~0, and exact distance
    ties go to the lower index (some midpoints are nudged by up to 7.5e-8 m along the pair, either way).  Points at r (1 +- k 1e-4)
    above a floor lattice point, that the converging z motion carries across the strict d2 < r2 cut.  Outliers 0.5-3 m beyond r."""
    from scipy.spatial import cKDTree
    n_tie, n_cut = n // 2, n // 4
    n_out = n - n_tie - n_cut
    pairs = np.array(sorted(cKDTree(tgt).query_pairs(spacing * 1.0001)))
    a, b = tgt[pairs[:, 0]], tgt[pairs[:, 1]]
    pick = rng.integers(0, len(pairs), n_tie)
    tie = 0.5 * (a[pick] + b[pick]) + (b[pick] - a[pick]) * (1e-7 * rng.integers(-3, 4, n_tie))[:, None]
    j = rng.integers(-int(half / spacing) + 4, int(half / spacing) - 4, (n_cut, 2))
    k = rng.integers(-40, 41, n_cut)
    cut = np.c_[j * spacing, r * (1.0 + k * 1e-4)]
    out = np.c_[rng.uniform(-half, half, (n_out, 2)), 3.0 + r + rng.uniform(0.5, 3.0, n_out)]
    return np.ascontiguousarray(np.vstack([tie, cut, out])[rng.permutation(n)])


@pytest.mark.parametrize("csize,n,ctas", CLUSTERS, ids=[f"{c}cta" for c, _, _ in CLUSTERS])
def test_icp_certificates_ties_and_cut(engine_factory, csize, n, ctas):
    r = 0.3
    rng = np.random.default_rng(csize)
    tgt = lattice_room()
    nrm = O.estimate_normals(tgt, 10, 1.0)
    src = adversarial_source(tgt, n, rng, r)
    init = synth.se3(0.0, 0.0, np.deg2rad(0.3), (0.02, -0.015, 0.004))
    p = params(r=r, max_iter=50, ctas=ctas)
    eng = engine_factory(p)
    reg = E.RegistrationIcpPointToPlane(eng)
    sc, tc = eng.cloud(src), eng.cloud(tgt, nrm)
    ref = O.registration_icp_p2plane(src, tgt, nrm, r, init, max_iter=50)
    assert ref.iters >= 3
    assert_matches_oracle(reg.registerClouds(sc, tc, init), ref, f"{csize} CTAs")
    res, words = traced(eng, lambda: reg.registerClouds(sc, tc, init))
    assert_matches_oracle(res, ref, f"{csize} CTAs, debug counters on")
    geo = Geometry(words, n, counted=True)
    print(f"ties and cut, r={r}:", geo, f"iterations {ref.iters}")
    assert geo.sizes == {csize} and geo.shared, f"{geo}; expected {csize} CTAs from shared memory; {UPDATE}"


@pytest.mark.parametrize("csize,n,ctas", CLUSTERS, ids=[f"{c}cta" for c, _, _ in CLUSTERS])
def test_icp_certificates_far_from_origin(engine_factory, csize, n, ctas):
    """A few km from the origin, a rotation-dominated guess (points move decimetres per evaluation while the cloud converges) and
    outliers 5-20 m beyond r, whose large float slacks are worn down over many evaluations."""
    r = 1.0
    off = np.array([3000.0, -2000.0, 50.0])
    rng = np.random.default_rng(50 + csize)
    tgt = room(20_000, rng, noise=0.01)
    nrm = O.estimate_normals(tgt, 10, 1.0)
    pts = tgt[rng.integers(0, len(tgt), n)] + 0.005 * rng.standard_normal((n, 3))
    n_out = n // 5
    pts[:n_out] = np.c_[rng.uniform(-8, 8, (n_out, 2)), 4.0 + r + rng.uniform(5.0, 20.0, n_out)]
    src = pts[rng.permutation(n)] + off
    tgt = tgt + off
    centre = np.eye(4); centre[:3, 3] = off + np.array([0.0, 0.0, 1.0])
    init = centre @ synth.se3(np.deg2rad(0.5), np.deg2rad(-0.4), np.deg2rad(2.5), (0.05, -0.04, 0.02)) @ np.linalg.inv(centre)
    p = params(r=r, max_iter=60, ctas=ctas)
    eng = engine_factory(p)
    reg = E.RegistrationIcpPointToPlane(eng)
    sc, tc = eng.cloud(src), eng.cloud(tgt, nrm)
    ref = O.registration_icp_p2plane(src, tgt, nrm, r, init, max_iter=60)
    assert ref.iters >= 5
    assert_matches_oracle(reg.registerClouds(sc, tc, init), ref, f"{csize} CTAs")
    res, words = traced(eng, lambda: reg.registerClouds(sc, tc, init))
    assert_matches_oracle(res, ref, f"{csize} CTAs, debug counters on")
    geo = Geometry(words, n, counted=True)
    print("far from the origin:", geo, f"iterations {ref.iters}")
    assert geo.sizes == {csize} and geo.shared, f"{geo}; expected {csize} CTAs from shared memory; {UPDATE}"


@pytest.mark.parametrize("csize,n,ctas", CLUSTERS, ids=[f"{c}cta" for c, _, _ in CLUSTERS])
def test_icp_phase2_on_every_cta(engine_factory, csize, n, ctas):
    """Half the source are outliers spread over every tile: every CTA queues points for phase 2, drained through DSMEM."""
    src, tgt, nrm = icp_pair(n, 70 + csize, outliers=0.5)
    init = synth.se3(0.003, -0.002, 0.01, (0.03, 0.02, -0.01))
    p = params(ctas=ctas)
    eng = engine_factory(p)
    reg = E.RegistrationIcpPointToPlane(eng)
    sc, tc = eng.cloud(src), eng.cloud(tgt, nrm)
    ref = O.registration_icp_p2plane(src, tgt, nrm, 0.5, init, max_iter=30)
    assert_matches_oracle(reg.registerClouds(sc, tc, init), ref, f"{csize} CTAs")
    res, words = traced(eng, lambda: reg.registerClouds(sc, tc, init))
    assert_matches_oracle(res, ref, f"{csize} CTAs, debug counters on")
    geo = Geometry(words, n, counted=True)
    print("heavy outliers:", geo, "per-CTA queues", geo.queues)
    assert geo.sizes == {csize}, f"{geo}; expected {csize} CTAs; {UPDATE}"
    assert all(q > 0 for q in geo.queues[:min(csize, 8)]), f"phase 2 did not run on every CTA: {geo.queues}"


# ----------------------------------------------------------------------------------------------------------------------
# normals
# ----------------------------------------------------------------------------------------------------------------------
def assert_normals_match(got, ref, xyz, knn, radius, queries=None):
    """per point, within the gap-aware bound of tests/normals_checks.py (the two sides sum the cumulants in different orders); xyz is
    the cloud the neighbours come from, queries the rows of xyz that got / ref belong to (default: all)"""
    worst = NC.assert_normals_close(got, ref, xyz, knn, radius, queries)
    print(f"normals: worst {worst:.3g} of the gap-aware bound")


def _scan_voxels(eng):
    raw = synth.lidar_scan(synth.Scene(), synth.loop_trajectory(8)[0], seed=0).astype(np.float64)
    return E.voxelize(eng, eng.cloud(raw), 0.1)


@pytest.mark.parametrize("knn", [1, 2, 3, 4, 31, 32])
@pytest.mark.parametrize("cloud", ["scan", "config1"])
def test_normals_knn_edges(engine_factory, knn, cloud):
    """knn < 3 takes the identity-covariance branch; knn = 32 fills all 32 lanes of the phase-2 list."""
    eng = engine_factory(params())
    if cloud == "scan":
        cl, radius = _scan_voxels(eng), 3.0
    else:
        cl, radius = eng.cloud(synth.planar_cloud_config1(noise=0.01)[1]), 1.0
    xyz, _ = cl.download()
    L.check(L.lib().b2s_estimate_normals(eng._h, cl._c, knn, C.c_double(radius)))
    _x, got = cl.download()
    assert np.array_equal(_x, xyz)
    assert_normals_match(got, O.estimate_normals(xyz, knn, radius), xyz, knn, radius)


def test_normals_knn_33_is_refused(engine_factory):
    eng = engine_factory(params())
    cl = eng.cloud(synth.planar_cloud_config1()[1])
    assert L.lib().b2s_estimate_normals(eng._h, cl._c, 33, C.c_double(1.0)) == L.E_UNSUPPORTED
    L.check(L.lib().b2s_estimate_normals(eng._h, cl._c, 32, C.c_double(1.0)))


def _oracle_cropper(c):
    return O.cropper(c.cropperName, c.croppingMinRadius, c.croppingMaxRadius, c.croppingMinZ, c.croppingMaxZ)


def _process_scan_matches(engine_factory, raw, p):
    eng = engine_factory(p)
    s2m = E.scanToMapRegistrationFactory(eng, p)
    ps = s2m.processForScanMatchingAndMerging(eng.cloud(raw))
    (mx, mn), (ax, an) = O.process_scan(raw.astype(np.float64), _oracle_cropper(p.mapBuilder.cropper), _oracle_cropper(p.scanProcessing.cropper),
                                        p.scanProcessing.voxelSize, p.icp.knn, p.icp.maxDistanceKnn, p.scanProcessing.downSamplingRatio, p.seed)
    gx, gn = ps.merge_.download()
    # the voxel cloud the normals were estimated on (merge_ is its selected subset), in the device's order: the map builder's cropper
    # in the sensor frame, then the voxel down-sample; the oracle runs on that same cloud (equal d2 go to the lower index)
    t0, _ = E.voxelize(eng, E.crop(eng, eng.cloud(raw), p.mapBuilder.cropper.to_c(center=(0.0, 0.0, 0.0))), p.scanProcessing.voxelSize).download()
    idx = NC.rows_in(gx, t0)
    hx, _ = ps.match_.download()
    from scipy.spatial import cKDTree
    assert len(gx) == len(mx) and len(hx) == len(ax)
    d, j = cKDTree(mx).query(gx)
    assert d.max() == 0.0 and len(np.unique(j)) == len(mx)      # identical point sets (bit-exact voxel means)
    assert_normals_match(gn, O.estimate_normals(t0, p.icp.knn, p.icp.maxDistanceKnn)[idx], t0, p.icp.knn, p.icp.maxDistanceKnn, idx)
    d, j = cKDTree(ax).query(hx)
    assert d.max() == 0.0 and len(np.unique(j)) == len(ax)


@pytest.mark.parametrize("knn", [3, 32])
def test_process_scan_flagged_normals_knn(engine_factory, knn):
    """downsampling ratio < 1: normals only for the selected points (the flagged query list), neighbours from the full cloud."""
    raw = synth.lidar_scan(synth.Scene(), synth.loop_trajectory(4)[1], seed=11)
    p = E.MapperParameters(seed=5)
    p.scanProcessing.downSamplingRatio = 0.3
    p.scanProcessing.cropper = E.ScanCroppingParameters("MinMaxRadius", 2.0, 25.0)
    p.icp.knn = knn
    _process_scan_matches(engine_factory, raw, p)


def run_child(args, env_extra, timeout=600):
    env = dict(os.environ)
    env.update(env_extra)
    proc = subprocess.run([sys.executable, "-s", CHILD] + args, env=env, capture_output=True, text=True, timeout=timeout, cwd=os.path.dirname(HERE))
    assert proc.returncode == 0, f"child {args} {env_extra} exited with {proc.returncode}:\n{proc.stdout}\n{proc.stderr}"
    return proc


def test_normals_select_exits_and_coarse_grid_from_the_record(engine_factory):
    """Every exit of the select kernel -- R = 1, R = 2, R = 3 (path codes 1-3), more candidates than its buffer (5), unresolved after
    the last block (6) -- is taken on the cloud processForScanMatchingAndMerging estimates: exits_scan cropped and voxelized, at the
    0.4 m process-scan cell.  b2s_debug_estimate_normals records the path of every query on that cloud (held to tests/normals_checks.py)
    and the production merge_ normals agree with its record; then the same clouds match the oracle.

    The two-patch cloud's index cell must have been coarsened from radius / 4 = 0.25 m to at least 1 m.  Shown from the selection
    record rather than the grid header, because the record is what the normals kernels saw: a query resolved at R = 1 sits in the
    middle cell of a block three cells wide, so every bounded block face lies at most 2 cells from it and its certified ball has
    lim2 < (2 cell)^2.  lim2 == r^2 at every such query therefore needs 2 cell > r = 1 m (or a block without a bounded face, which over
    the kilometres-wide box needs far larger cells), and the header only ever doubles the cell, 0.25 m x 2^j, so cell >= 1 m.  With the
    0.25 m cell, lim2 < 0.25 at R = 1."""
    sys.path.insert(0, HERE)
    try:
        import boundary_child as BC
        from test_gpu_normals_kernels import run_and_check
    finally:
        sys.path.remove(HERE)
    p = BC.exits_params()
    es = engine_factory(p)
    raw = BC.exits_scan()
    ps = E.scanToMapRegistrationFactory(es, p).processForScanMatchingAndMerging(es.cloud(raw))
    gx, gn = ps.merge_.download()
    # the voxel cloud the estimation ran on, in the device's order: the map builder's cropper (sensor frame), then the voxel down-sample
    cropped = E.crop(es, es.cloud(raw), p.mapBuilder.cropper.to_c(center=(0.0, 0.0, 0.0)))
    t0, _ = E.voxelize(es, cropped, p.scanProcessing.voxelSize).download()
    knn, radius, cell = p.icp.knn, p.icp.maxDistanceKnn, 4 * p.scanProcessing.voxelSize
    _, path, dbg = run_and_check(es, f"exits_scan process-scan cell {cell:g}", t0, knn, radius, cell_hint=cell, full=True)[:3]
    counts = np.bincount(path, minlength=7)
    print(f"select exits: R=1 {counts[1]}, R=2 {counts[2]}, R=3 {counts[3]}, full-radius block {counts[4]}, over capacity {counts[5]}, "
          f"unresolved {counts[6]}")
    assert all(counts[c] > 0 for c in (1, 2, 3, 5, 6)), f"not every exit of the select kernel was taken: {counts.tolist()}"
    idx = NC.rows_in(gx, t0)
    worst = NC.assert_normals_close(gn, dbg[idx], t0, knn, radius, queries=idx)
    print(f"processForScanMatchingAndMerging merge_ vs the debug entry: worst {worst:.3g} of the gap-aware bound ({len(idx)} of {len(t0)})")

    eng = engine_factory(params())
    _, path, _, sel = run_and_check(eng, "two_patches", BC.two_patches(), 10, 1.0, full=True)
    r1 = path == 1
    print(f"two-patch cloud: {r1.sum()} queries resolved at R = 1, lim2 {np.unique(sel[r1, 3])}")
    assert r1.any() and (sel[r1, 3] == 1.0).all(), "the two-patch index cell was not coarsened to at least 4 x radius / 4"

    _process_scan_matches(engine_factory, BC.exits_scan(), BC.exits_params())

    xyz = BC.two_patches()
    cl = eng.cloud(xyz)
    L.check(L.lib().b2s_estimate_normals(eng._h, cl._c, 10, C.c_double(1.0)))
    _x, got = cl.download()
    nrm = O.estimate_normals(xyz, 10, 1.0)
    assert_normals_match(got, nrm, xyz, 10, 1.0)
    # ICP against the two-patch target (its grid coarsens as well)
    rng = np.random.default_rng(3)
    src = xyz[rng.integers(0, len(xyz) // 2, 2500)] + 0.005 * rng.standard_normal((2500, 3))
    init = synth.se3(0.004, -0.003, 0.01, (0.03, -0.02, 0.01))
    reg = E.cloudRegistrationFactory(eng, E.CloudRegistrationParameters(icp=params().icp))
    res = reg.registerClouds(eng.cloud(src), eng.cloud(xyz, nrm), init)
    assert_matches_oracle(res, O.registration_icp_p2plane(src, xyz, nrm, 0.5, init, max_iter=30), "two-patch target")


# ----------------------------------------------------------------------------------------------------------------------
# voxel down-sample, sort, grid size
# ----------------------------------------------------------------------------------------------------------------------
def box_cloud(n, cells_x, voxel, seed):
    """n points whose largest extent gives floor(extent / voxel) + 3 == cells_x (the key-width rule of op_voxel_down_sample)."""
    rng = np.random.default_rng(seed)
    ext = (cells_x - 3) * voxel + 0.4 * voxel
    xyz = np.c_[rng.uniform(0.0, ext, n), rng.uniform(0.0, 20.0, n), rng.uniform(0.0, 3.0, n)]
    xyz[0] = (0.0, 0.0, 0.0); xyz[1] = (ext, 20.0, 3.0)
    return xyz


def assert_voxels_bit_exact(eng, xyz, voxel):
    gx, _ = E.voxelize(eng, eng.cloud(xyz), voxel).download()
    ox, _ = O.voxel_down_sample(xyz, voxel)
    assert gx.shape == ox.shape
    assert np.array_equal(ox[np.lexsort(ox.T[::-1])], gx[np.lexsort(gx.T[::-1])])
    return gx


@pytest.mark.parametrize("n", [786_432, 786_433], ids=["cluster-sort", "multi-kernel-sort"])
@pytest.mark.parametrize("cells", [1024, 1025], ids=["u32", "u64"])
def test_voxel_key_width_and_sort(engine_factory, cells, n):
    eng = engine_factory(params())
    assert_voxels_bit_exact(eng, box_cloud(n, cells, 0.25, cells + n), 0.25)


def test_voxel_21_bit_limit(engine_factory):
    eng = engine_factory(params())
    xyz = box_cloud(5000, 1 << 21, 0.25, 3)
    assert_voxels_bit_exact(eng, xyz, 0.25)
    beyond = box_cloud(5000, (1 << 21) + 1, 0.25, 3)
    assert L.lib().b2s_voxel_down_sample(eng._h, eng.cloud(beyond)._c, C.c_double(0.25), E.Cloud(eng)._c) == L.E_INVALID


@pytest.mark.parametrize("n", [(1 << 19) - 1, 1 << 19])
def test_wide_grid_switch_voxel_and_normals(engine_factory, n):
    eng = engine_factory(params())
    rng = np.random.default_rng(n)
    xyz = room(n, rng, half=30.0, height=6.0)
    assert_voxels_bit_exact(eng, xyz, 0.1)
    cl = eng.cloud(xyz)
    L.check(L.lib().b2s_estimate_normals(eng._h, cl._c, 10, C.c_double(0.5)))
    _x, got = cl.download()
    assert_normals_match(got, O.estimate_normals(xyz, 10, 0.5), xyz, 10, 0.5)


def test_results_independent_of_grid_size(tmp_path):
    """The same operations under the default grid, B2S_GRID_CAP = 1 and 7 and the multi-kernel sort.  Crop, voxel means and
    selections must be bit-identical.  The order of the points inside one cell of a neighbour grid comes from atomics, and with it
    the order in which normals sum their covariance terms and ICP drains its phase-2 queue: normals are held to the oracle's
    criteria, registrations to equal iterations and correspondences and 1e-10."""
    runs = {}
    for name, env in (("default", {}), ("cap1", {"B2S_GRID_CAP": "1"}), ("cap7", {"B2S_GRID_CAP": "7"}), ("multi", {"B2S_SORT": "multi"})):
        out = tmp_path / f"{name}.npz"
        run_child(["ops", str(out)], env)
        runs[name] = dict(np.load(out))
    base = runs.pop("default")
    # the clouds the three normal estimations of run_ops take their neighbours from, and their knn / radius
    p = E.MapperParameters(seed=9)
    p.scanProcessing.downSamplingRatio = 0.5
    sc = p.mapBuilder.cropper
    raw = synth.lidar_scan(synth.Scene(), synth.loop_trajectory(8)[0], seed=70).astype(np.float64)
    t0, _ = O.voxel_down_sample(O.crop(O.cropper(sc.cropperName, sc.croppingMinRadius, sc.croppingMaxRadius, sc.croppingMinZ,
                                               sc.croppingMaxZ), raw)[0], p.scanProcessing.voxelSize)
    nbh = {"normals": (base["normals_xyz"], 20, 3.0, None), "merge_nrm": (t0, p.icp.knn, p.icp.maxDistanceKnn, NC.rows_in(base["merge_xyz"], t0)),
           "match_nrm": (t0, p.icp.knn, p.icp.maxDistanceKnn, NC.rows_in(base["match_xyz"], t0))}
    for name, got in runs.items():
        assert set(got) == set(base)
        for k in ("crop", "voxel", "normals_xyz", "merge_xyz", "match_xyz", "carved"):
            assert got[k].shape == base[k].shape and np.array_equal(got[k], base[k]), f"{name}: {k} differs from the default grid"
        for k in ("normals", "merge_nrm", "match_nrm"):
            print(f"{name}: {k} max |difference| {np.abs(got[k] - base[k]).max():.3g}")
            assert_normals_match(got[k], base[k], *nbh[k])
        for k in ("reg", "step1", "step2", "step3"):
            assert np.array_equal(got[k][-2:], base[k][-2:]), f"{name}: {k} iterations / correspondences differ"
            assert np.abs(got[k][:-2] - base[k][:-2]).max() < 1e-10, f"{name}: {k} differs"
        for k in ("map_xyz", "mapper_map"):
            a, b = got[k], base[k]
            assert a.shape == b.shape, f"{name}: {k} size differs"
            assert np.abs(a[np.lexsort(a.T[::-1])] - b[np.lexsort(b.T[::-1])]).max() < 1e-9, f"{name}: {k} differs"
