"""GPU: b2s_submap_odometry_constraints (buildOdometryConstraint, core/src/constraint_builders.cpp:33-118), batched over (parent, child)
pairs and read from the resident submaps -- parity with the oracle on the closed lap, equality with the composition of the existing
entry points (b2s_submap_to_cloud x 2 + b2s_overlap + b2s_information_matrix), batching and run-to-run determinism, the states a
resident map can be in (tombstones, carving, b2s_submap_transform, a point-to-point map), and the boundaries of the new kernels
(K-info-wide's tile and grid-stride sizes, d = r, distance ties, empty overlaps, errors)."""
import copy

import numpy as np
import pytest

from oracle import oracle as O
from oracle_backend import OracleBackend
from oracle_backend_constraints import ConstraintOracleBackend, odometry_constraint
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W

pytestmark = pytest.mark.gpu

TILE = 1024   # WI_TILE of constraints.cu


def rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    s = np.abs(b).max()
    return np.abs(a - b).max() / (s if s > 0 else 1.0)


def keyed(xyz):
    """the rows sorted by (voxel key, x, y, z): the overlap clouds as keyed sets"""
    k = np.floor(xyz / 0.1).astype(np.int64)
    return xyz[np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0], k[:, 2], k[:, 1], k[:, 0]))]


@pytest.fixture(scope="module")
def lap():
    """the config-5 segment of the closed lap through SegmentMapper on both backends (carving, dense map, 10 m submaps)"""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    sp = S.SubmapParameters(radius=10.0)
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=True)
    ora = ConstraintOracleBackend(copy.deepcopy(p), carving=True, dense=True)
    md, mo = S.SegmentMapper(dev, sp), S.SegmentMapper(ora, sp)
    for k in range(208):
        raw, d = lp.scan(k, seed=k), lp.delta(k)
        md.addRangeMeasurement(raw, d)
        mo.addRangeMeasurement(raw, d)
    assert len(md.submaps.submaps) == len(mo.submaps.submaps) >= 3
    yield dev, ora, md, mo
    dev.close()


def lap_pairs(md):
    sc = md.submaps
    return [(sc.submaps[t].parent, t) for t in range(1, len(sc.submaps))]


def test_closed_lap_parity(lap):
    dev, ora, md, mo = lap
    eng = dev.eng
    pairs = lap_pairs(md)
    for refine in (False, True):
        prm = E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=refine)
        cd, co = [], []
        S.computeOdometryConstraints(dev, md.submaps, cd, finishedIds=list(range(len(md.submaps.submaps))), params=prm)
        S.computeOdometryConstraints(ora, mo.submaps, co, finishedIds=list(range(len(mo.submaps.submaps))), params=prm)
        assert [(c.sourceSubmapIdx, c.targetSubmapIdx) for c in cd] == [(c.sourceSubmapIdx, c.targetSubmapIdx) for c in co] == pairs
        so = [E.Cloud(eng) for _ in pairs]; to = [E.Cloud(eng) for _ in pairs]
        got = E.buildOdometryConstraintsBatch(eng, [md.submaps.submaps[s].handle for s, _ in pairs], [md.submaps.submaps[t].handle for _, t in pairs],
                                              prm, so, to)
        for (s, t), g, a, b, c_dev, c_ora in zip(pairs, got, so, to, cd, co):
            # the oracle on the device's own maps (getMapPointCloudCopy): the bars of DESIGN section 3
            (px, pn), (cx, cn) = dev.map_cloud(md.submaps.submaps[s].handle), dev.map_cloud(md.submaps.submaps[t].handle)
            ref, (rsx, _), (rtx, _) = odometry_constraint(px, pn, cx, cn, prm)
            assert (g.nSourceOverlap, g.nTargetOverlap) == (ref.nSourceOverlap, ref.nTargetOverlap) and g.nSourceOverlap > 1000
            ax, _ = a.download(); bx, _ = b.download()
            assert np.array_equal(keyed(ax), keyed(rsx)) and np.array_equal(keyed(bx), keyed(rtx))
            assert rel(g.informationMatrix_, ref.informationMatrix_) < 1e-9
            if refine:
                assert g.icp.iters == ref.icp.iters and g.icp.n_corr == ref.icp.n_corr
                assert np.abs(g.sourceToTarget_ - ref.sourceToTarget_).max() < 1e-8 and abs(g.icp.fitness_ - ref.icp.fitness_) < 1e-12
            else:
                assert np.array_equal(g.sourceToTarget_, np.eye(4)) and g.icp is None
            # and the device constraint against the oracle backend's own run (its maps agree to ~1e-7 after 200 chained scans)
            assert np.array_equal(c_dev.informationMatrix, g.informationMatrix_)
            assert rel(c_dev.informationMatrix, c_ora.informationMatrix) < 1e-6 and np.abs(c_dev.sourceToTarget - c_ora.sourceToTarget).max() < 1e-6
            assert c_dev.isOdometryConstraint and c_dev.isInformationMatrixValid


def composed(eng, parent, child, prm, T=None):
    """b2s_submap_to_cloud x 2, b2s_overlap at the identity, b2s_information_matrix: the composition the new call replaces"""
    v = E.getMapVoxelSize(prm.mapVoxelSize, prm.voxelSizeIfMapVoxelSizeIsZero)
    sc, tc = parent.toCloud(), child.toCloud()
    so, to = E.computeOverlappingClouds(eng, sc, tc, np.eye(4), prm.voxelExpansionFactorOverlapComputation * v, prm.minNumPointsPerVoxel)
    info = E.getInformationMatrixFromPointClouds(eng, so, to, prm.voxelExpansionFactorIcpCorrespondenceDistance * v, np.eye(4) if T is None else T)
    return so, to, info


def check_against_composition(eng, parent, child, prm=None):
    prm = prm or E.OdometryConstraintParameters()
    a, b = E.Cloud(eng), E.Cloud(eng)
    (g,) = E.buildOdometryConstraintsBatch(eng, [parent], [child], prm, [a], [b])
    so, to, info = composed(eng, parent, child, prm, g.sourceToTarget_)
    for x, y in ((a, so), (b, to)):
        (xx, xn), (yx, yn) = x.download(), y.download()
        assert np.array_equal(xx, yx) and np.array_equal(xn, yn, equal_nan=True)   # bit-identical, in order
    assert (g.nSourceOverlap, g.nTargetOverlap) == (len(so), len(to))
    assert rel(g.informationMatrix_, info) < 1e-12                                # only the summation order differs
    return g


def test_against_existing_entry_points(lap):
    dev, _ora, md, _mo = lap
    for s, t in lap_pairs(md):
        for refine in (False, True):
            check_against_composition(dev.eng, md.submaps.submaps[s].handle, md.submaps.submaps[t].handle,
                                      E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=refine))


def fields(r):
    return (r.sourceToTarget_.tobytes(), r.informationMatrix_.tobytes(), r.nSourceOverlap, r.nTargetOverlap,
            None if r.icp is None else (r.icp.transformation_.tobytes(), r.icp.fitness_, r.icp.inlier_rmse_, r.icp.n_corr, r.icp.iters))


def test_batching_and_determinism(lap):
    dev, _ora, md, _mo = lap
    eng = dev.eng
    pairs = lap_pairs(md)
    srcs, tgts = [md.submaps.submaps[s].handle for s, _ in pairs], [md.submaps.submaps[t].handle for _, t in pairs]
    for refine in (False, True):
        prm = E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=refine)
        batch = E.buildOdometryConstraintsBatch(eng, srcs, tgts, prm)
        again = E.buildOdometryConstraintsBatch(eng, srcs, tgts, prm)
        singles = [E.buildOdometryConstraint(eng, s, t, prm) for s, t in zip(srcs, tgts)]
        assert [fields(r) for r in batch] == [fields(r) for r in again] == [fields(r) for r in singles]
        # a pair twice and in the reverse order: the same records
        rev = E.buildOdometryConstraintsBatch(eng, srcs[::-1] + srcs[:1], tgts[::-1] + tgts[:1], prm)
        assert [fields(r) for r in rev] == [fields(r) for r in batch[::-1] + batch[:1]]


# ---- constructed submaps ---------------------------------------------------------------------------------------------------------
def submap(eng, xyz, nrm=None, cap=None):
    sm = E.Submap(eng, cap or max(2 * len(xyz), 1024))
    sm.setMapPointCloud(eng.cloud(np.asarray(xyz, dtype=np.float64).reshape(-1, 3), nrm))
    return sm


def plane_points(n, seed, lo=0.05, hi=2.3, z=1.0):
    rng = np.random.default_rng(seed)
    xyz = np.c_[rng.uniform(lo, hi, (n, 2)), np.full(n, z) + rng.uniform(-0.02, 0.02, n)]
    return xyz, np.tile([0.0, 0.0, 1.0], (n, 1))


def brute_info(src, tgt, r, T=None):
    """fp64 restatement: exact 1-NN with d2 < r2 (d2 = (dx dx + dy dy) + dz dz), ties to the lower index, moments of the matched
    target points -> [O3D]'s 6x6; and the correspondence count"""
    src = np.asarray(src, dtype=np.float64)
    if T is not None and not np.array_equal(T, np.eye(4)):
        src = src @ T[:3, :3].T + T[:3, 3]
    G = np.zeros((6, 6))
    if len(src) == 0 or len(tgt) == 0:
        return G, 0
    d = src[:, None, :] - tgt[None, :, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    d2 = np.where(d2 < r * r, d2, np.inf)
    j = np.argmin(d2, axis=1)            # first minimum: the lower index
    ok = np.isfinite(d2[np.arange(len(src)), j])
    for x, y, z in tgt[j[ok]]:
        J = np.array([[0, z, -y, 1, 0, 0], [-z, 0, x, 0, 1, 0], [y, -x, 0, 0, 0, 1]], dtype=np.float64)
        G += J.T @ J
    return G, int(ok.sum())


P125 = E.OdometryConstraintParameters(mapVoxelSize=0.125)   # r = 1.5 x 0.125 = 0.1875 and its square are exact in binary


@pytest.mark.parametrize("ns", [0, 1, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1])
def test_source_sizes_around_the_tile(engine_factory, ns):
    eng = engine_factory()
    sx, sn = plane_points(max(ns, 1), 1)
    tx, tn = plane_points(700, 2)
    parent = submap(eng, sx[:ns], sn[:ns], cap=4096)
    child = submap(eng, tx, tn)
    g = check_against_composition(eng, parent, child, P125)
    G, n = brute_info(sx[:ns], tx, 0.1875)
    assert g.nSourceOverlap == ns and g.informationMatrix_[3, 3] == n and rel(g.informationMatrix_, G) < 1e-12


def test_grid_stride_over_a_batch(engine_factory):
    """more tiles than K-info-wide's grid (4 CTAs per SM): the grid-stride loop walks the tiles of several pairs"""
    eng = engine_factory()
    parents, children = [], []
    for k in range(6):
        sx, sn = plane_points(110_000 + 37 * k, 10 + k, z=1.0 + 3.0 * k)   # each pair in its own overlap voxel
        tx, tn = plane_points(90_000, 20 + k, z=1.0 + 3.0 * k)
        parents.append(submap(eng, sx, sn)); children.append(submap(eng, tx, tn))
    prm = E.OdometryConstraintParameters()
    batch = E.buildOdometryConstraintsBatch(eng, parents, children, prm)
    assert sum((r.nSourceOverlap + TILE - 1) // TILE for r in batch) > 4 * 132
    for p, c, r in zip(parents, children, batch):
        so, to, info = composed(eng, p, c, prm)
        assert rel(r.informationMatrix_, info) < 1e-12 and r.nSourceOverlap == len(so)
    assert [fields(r) for r in batch] == [fields(r) for r in E.buildOdometryConstraintsBatch(eng, parents, children, prm)]


def test_distance_exactly_r_and_ties(engine_factory):
    eng = engine_factory()
    r = 0.1875
    s = np.array([[1.0, 1.0, 1.0], [1.5, 1.0, 1.0], [2.0, 1.0, 1.0], [1.0, 2.0, 1.0]])
    t = np.array([[1.0 + r, 1.0, 1.0],                        # source 0: exactly at r -> no correspondence
                  [1.5, 1.0 + 0.0625, 1.0], [1.5, 1.0 - 0.0625, 1.0],   # source 1: a tie -> the lower index (1)
                  [2.0 - 0.125, 1.0, 1.0], [2.0, 1.0, 1.0 + 0.125],     # source 2: a tie at 0.125
                  [1.0, 2.0 + r - 2.0 ** -20, 1.0]])          # source 3: just inside r
    nrm = np.tile([0.0, 0.0, 1.0], (len(t), 1))
    parent, child = submap(eng, s, nrm[:4]), submap(eng, t, nrm)
    g = check_against_composition(eng, parent, child, P125)
    G, n = brute_info(s, t, r)
    assert n == 3 and g.informationMatrix_[3, 3] == 3 and rel(g.informationMatrix_, G) < 1e-12
    # the tie partners differ: the lower index decides which moments are summed
    assert G[0, 4] != brute_info(s, t[[0, 2, 1, 4, 3, 5]], r)[0][0, 4]


def test_disjoint_and_mixed_batch(engine_factory):
    eng = engine_factory()
    sx, sn = plane_points(3000, 1); tx, tn = plane_points(2500, 2)
    far = tx + [50.0, 0.0, 0.0]
    a, b, c = submap(eng, sx, sn), submap(eng, tx, tn), submap(eng, far, tn)
    prm = E.OdometryConstraintParameters()
    empty = check_against_composition(eng, a, c, prm)
    assert (empty.nSourceOverlap, empty.nTargetOverlap) == (0, 0) and not empty.informationMatrix_.any()
    src, tgt = [a, a, a, b], [b, c, b, a]
    for refine in (False, True):
        prm = E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=refine)
        batch = E.buildOdometryConstraintsBatch(eng, src, tgt, prm)
        assert [fields(r) for r in batch] == [fields(E.buildOdometryConstraint(eng, s, t, prm)) for s, t in zip(src, tgt)]
        assert batch[1].nSourceOverlap == 0 and batch[0].nSourceOverlap == 3000


def test_resident_map_states(engine_factory):
    """tombstones and carving come with the closed lap (test_against_existing_entry_points); here: after b2s_submap_transform, after
    more fusion, and a point-to-point map whose normals are NaN"""
    eng = engine_factory()
    sx, sn = plane_points(4000, 1); tx, tn = plane_points(3000, 2)
    parent, child = submap(eng, sx, sn), submap(eng, tx, tn)
    child.transform(np.array([[1, 0, 0, 0.03], [0, 1, 0, -0.02], [0, 0, 1, 0.01], [0, 0, 0, 1.0]]))
    for refine in (False, True):
        check_against_composition(eng, parent, child, E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=refine))
    # fusion into a resident map: scans that land on map voxels leave tombstones behind
    scan = eng.cloud(*plane_points(2000, 7))
    child.insertScan(None, scan, np.eye(4))
    child.insertScan(None, scan, np.array([[1, 0, 0, 0.01], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]]))
    check_against_composition(eng, parent, child)
    # a point-to-point map: no normals (NaN) -> the unrefined constraint works, the refinement refuses
    p2p = engine_factory(E.MapperParameters(scanToMapRegType="PointToPointIcp"))
    pa, ch = submap(p2p, sx, sn), E.Submap(p2p, 8192)
    ch.setMapPointCloud(p2p.cloud(tx))
    check_against_composition(p2p, pa, ch)
    with pytest.raises(L.B2SError) as e:
        E.buildOdometryConstraint(p2p, pa, ch, E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=True))
    assert e.value.code == L.E_NO_NORMALS
    E.buildOdometryConstraint(p2p, ch, pa, E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=True))   # parent may lack them


def test_errors(engine_factory):
    e1, e2 = engine_factory(), engine_factory()
    sx, sn = plane_points(500, 1)
    a, b, other = submap(e1, sx, sn), submap(e1, sx, sn), submap(e2, sx, sn)
    assert E.buildOdometryConstraintsBatch(e1, [], []) == []
    for s, t in ((a, other), (other, a)):
        with pytest.raises(L.B2SError) as e:
            E.buildOdometryConstraint(e1, s, t)
        assert e.value.code == L.E_INVALID
    for prm in (E.OdometryConstraintParameters(mapVoxelSize=-0.2), E.OdometryConstraintParameters(mapVoxelSize=0.0, voxelSizeIfMapVoxelSizeIsZero=0.0),
                E.OdometryConstraintParameters(minNumPointsPerVoxel=0)):
        with pytest.raises(L.B2SError) as e:
            E.buildOdometryConstraint(e1, a, b, prm)
        assert e.value.code == L.E_INVALID
    with pytest.raises(L.B2SError):
        E.buildOdometryConstraintsBatch(e1, [a], [b], None, [E.Cloud(e2)], [E.Cloud(e1)])
    # |v| <= 1e-3 -> 0.04: the same constraint as an explicit 0.04
    z = E.buildOdometryConstraint(e1, a, b, E.OdometryConstraintParameters(mapVoxelSize=0.0))
    assert fields(z) == fields(E.buildOdometryConstraint(e1, a, b, E.OdometryConstraintParameters(mapVoxelSize=0.04)))
