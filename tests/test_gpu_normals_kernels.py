"""GPU tests of the normal estimation's kernels one by one (normals.cu: normals_select2_kernel, normals_finish_kernel,
normals_phase2_kernel) through b2s_debug_estimate_normals, which runs the production launches and records, per point, the cumulants and
neighbour count the eigen-solver received and the path that resolved the query.  Every record is held to tests/normals_checks.py:
the exact neighbour count, the cumulants within their summation bound, the solver's exact branches bit for bit, the direction within
the gap-aware bound and the sign by the orientation and prior rules.  The clouds are built so that the recorded path codes prove each exit
of the block gather was taken (asserted, not printed), and the selection record (candidates in the certified ball, the histogram bin of
the k-th key and its member count, lim2) proves the constructed edge cases -- nc around knn, the clamp into bin 31, more than 32 members
in the boundary bin, 256 / 257 candidates -- were reached.  The production entries that pass flags (processForScanMatchingAndMerging
with ratio < 1) and priors (computeFeatures) are compared with the debug entry on the same clouds.  The worst cumulant and direction
metric per family is printed as a fraction of its bound."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import normals_checks as NC
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import boundary_child as BC  # noqa: E402
from test_features_front_end import lidar_map  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng(engine_factory):
    return engine_factory(E.MapperParameters())


def debug_normals(eng, xyz, knn, radius, cell_hint=0.0, flags=None, priors=None):
    xyz = np.ascontiguousarray(xyz, dtype=np.float64)
    n = len(xyz)
    cl = eng.cloud(xyz, priors)
    rec = np.empty((n, 10)); path = np.empty(n, dtype=np.int32); sel = np.empty((n, 4))
    fl = None if flags is None else np.ascontiguousarray(flags, dtype=np.int32)
    L.check(L.lib().b2s_debug_estimate_normals(eng._h, cl._c, C.c_int32(knn), C.c_double(radius), C.c_double(cell_hint),
                                               None if fl is None else fl.ctypes.data_as(C.POINTER(C.c_int32)),
                                               C.c_int32(priors is not None), rec.ctypes.data_as(C.POINTER(C.c_double)),
                                               path.ctypes.data_as(C.POINTER(C.c_int32)), sel.ctypes.data_as(C.POINTER(C.c_double))))
    x, nrm = cl.download()
    assert np.array_equal(x, xyz)
    return rec, path, nrm, sel


def run_and_check(eng, name, xyz, knn, radius, cell_hint=0.0, flags=None, priors=None, full=False):
    rec, path, nrm, sel = debug_normals(eng, xyz, knn, radius, cell_hint, flags, priors)
    queries = None if flags is None else np.nonzero(flags)[0]
    s = NC.check_all(xyz, knn, radius, rec, path, nrm, priors, queries)
    print(f"{name:28s} n {s['n']:6d} knn {knn:2d}: cumulants {s['cum']:.3g}, direction {s['dir']:.3g} of bound; exact branches "
          f"{s['exact']}, signs {s['signs']} (+{s['prior_signs']} prior); paths 1..6 {s['paths'].tolist()}")
    return (rec, path, nrm, sel) if full else (path, nrm)


def _scan_voxels(offset=(0.0, 0.0, 0.0), n_max=None):
    raw = synth.lidar_scan(synth.Scene(), synth.loop_trajectory(8)[0], seed=0).astype(np.float64)
    from oracle import oracle as O
    vx, _ = O.voxel_down_sample(raw, 0.1)
    if n_max:
        vx = vx[np.random.default_rng(0).permutation(len(vx))[:n_max]]
    return np.ascontiguousarray(vx + np.asarray(offset))


def test_every_exit_of_the_block_gather(eng):
    """exits_scan at the 0.4 m cell of process_scan (R = 1, 2, 3, over capacity, not certified: the radius does not fit the row
    table) and at the default radius / 4 cell (the full-radius block, and fewer than k inside the radius)"""
    xyz = BC.exits_scan()
    rec1, p1, _, _ = run_and_check(eng, "exits_scan cell 0.4", xyz, 20, 4.0, cell_hint=0.4, full=True)
    for code in (1, 2, 3, 5, 6):
        assert (p1 == code).any(), f"path {code} not reached: {np.bincount(p1, minlength=7)}"
    rec, p2, _, _ = run_and_check(eng, "exits_scan cell r/4", xyz, 20, 4.0, full=True)
    assert (p2 == 4).any(), f"the full-radius block was not reached: {np.bincount(p2, minlength=7)}"
    assert ((p2 == 4) & (rec[:, 9] < 20)).any(), "no query finished by the full-radius block with fewer than k inside the radius"
    assert ((p1 == 6) & (rec1[:, 9] < 20)).any(), "no phase-2 query with fewer than k inside the radius"
    run_and_check(eng, "two_patches", BC.two_patches(), 10, 1.0)


@pytest.mark.parametrize("knn", [1, 2, 3, 4, 5, 10, 20, 31, 32])
def test_knn_sweep(eng, knn):
    run_and_check(eng, "lattice", NC.lattice(9, 0.25), knn, 0.9)
    run_and_check(eng, "scan voxels", _scan_voxels(n_max=20000), knn, 3.0, cell_hint=0.4)


def _clusters(sizes, radius, seed):
    """one tight cluster per size (every point within radius of every other of its cluster), clusters 10 radii apart"""
    rng = np.random.default_rng(seed)
    parts = [rng.uniform(-0.25, 0.25, (m, 3)) * radius + [10.0 * radius * j, 0.0, 1.0] for j, m in enumerate(sizes)]
    return np.ascontiguousarray(np.vstack(parts)), np.repeat(np.arange(len(sizes)), sizes)


@pytest.mark.parametrize("knn", [1, 2, 3, 4, 5, 10, 20, 31, 32])
def test_certified_count_around_knn(eng, knn):
    """clusters of knn - 1, knn and knn + 1 points with a cell of 2 r: the certified ball is the search ball (lim2 = r^2), so every
    query of a cluster of m points has exactly nc = m candidates -- fewer than k (final because the block covers the radius), k, and
    one more than k (the histogram selection)"""
    r = 0.5
    sizes = [m for m in (knn - 1, knn, knn + 1) if m > 0]
    xyz, lab = _clusters(sizes, r, knn)
    rec, path, _, sel = run_and_check(eng, f"clusters around knn {knn}", xyz, knn, r, cell_hint=2 * r, full=True)
    assert np.isin(path, (1, 2)).all(), np.bincount(path, minlength=7)
    assert (sel[:, 3] == r * r).all(), "the certified ball is not the search ball"
    m = np.asarray(sizes)[lab]
    assert np.array_equal(sel[:, 0], m) and np.array_equal(rec[:, 9], np.minimum(m, knn))
    assert np.array_equal(sel[:, 1] >= 0, m > knn)   # the histogram runs exactly when nc > knn


def test_kth_key_clamped_into_bin_31(eng):
    """a query, 6 close points and two mirrored points +-p with d2 just below r^2 (a tie): with knn = 8 the k-th key is one of
    the two, its d2 * 32 / lim2 rounds to 32 and the clamp puts it in bin 31; the lower index must win the tie"""
    rng = np.random.default_rng(0)
    far = None
    for r in np.arange(0.3, 0.9, 0.0007):   # a radius whose 32 / r^2 rounds up, then a point at d2 < r^2 with d2 * 32 / r^2 >= 32
        r2, sc = r * r, 32.0 / (r * r)
        if not np.nextafter(r2, 0.0) * sc >= 32.0:
            continue
        D = rng.normal(size=(4000, 3))
        D /= np.linalg.norm(D, axis=1)[:, None]
        for jj in range(1, 6):
            P = D * (r * (1 - jj * 2.0 ** -53))
            d = (P[:, 0] * P[:, 0] + P[:, 1] * P[:, 1]) + P[:, 2] * P[:, 2]
            ok = (d < r2) & (d * sc >= 32.0)
            if ok.any():
                far = P[np.argmax(ok)]
                break
        if far is not None:
            break
    assert far is not None, "no radius puts a d2 below r^2 at d2 * 32 / r^2 >= 32"
    rng = np.random.default_rng(4)
    close = rng.uniform(-0.2, 0.2, (6, 3)) * r
    xyz = np.vstack([[[0.0, 0.0, 0.0]], close, [far, -far]])
    rec, path, _, sel = run_and_check(eng, f"bin-31 clamp, r = {r:.3f}", xyz, 8, r, cell_hint=2 * r, full=True)
    assert path[0] in (1, 2) and sel[0, 3] == r2 and sel[0, 0] == 9 and sel[0, 1] == 31, sel[0]
    # the set itself (the lower index 7 wins the tie) is held by check_all


def test_histogram_edges(eng):
    """more than 32 members in the k-th key's bin (the rank loop's second pass), ties at every lattice shell, d2 == r^2 excluded"""
    rec, path, _, sel = run_and_check(eng, "cluster at 1.03 m", NC.cluster_at_distance(), 20, 2.0, cell_hint=4.0, full=True)
    assert (sel[:8, 2] > 32).all() and (sel[:8, 3] == 4.0).all(), sel[:8]
    for knn in (8, 9, 10, 20):   # 9 points strictly inside r = 2 h, 4 more at d2 == r^2
        rec, _, _, _ = run_and_check(eng, f"radius edge knn {knn}", NC.radius_edge(), knn, 0.5, full=True)
        assert rec[40, 9] == min(knn, 9)   # the centre of the 9 x 9 lattice
    run_and_check(eng, "lattice 3D, r = 2 h", NC.lattice(9, 0.25), 32, 0.5)


def test_block_of_256_and_257_candidates(eng):
    """a cluster of 256 (257) mutually close points with a cell of 2 r: every query has nc = 256 -- the buffer is exactly full -- (257:
    over capacity, phase 2)"""
    r = 0.5
    for m, paths in ((256, (1, 2)), (257, (5,))):
        xyz, _ = _clusters([m], r, m)
        _, path, _, sel = run_and_check(eng, f"{m} candidates in the block", xyz, 20, r, cell_hint=2 * r, full=True)
        assert np.isin(path, paths).all() and (sel[:, 0] == m).all(), (np.bincount(path, minlength=7), sel[:3])


def test_grid_faces(eng):
    """queries at the two corners of the bounding box lie in the first and the last grid cell on every axis (the grid's origin is the
    box's minimum), where the block's faces towards the outside are unbounded"""
    rng = np.random.default_rng(3)
    for m in (100, 200):
        blob = rng.uniform(-0.3, 0.3, (m, 3))
        xyz = np.vstack([[[0.0, 0.0, 0.0]], blob + 0.3, [[20.0, 20.0, 20.0]], 19.7 + blob])
        run_and_check(eng, f"grid corners, {m} per corner", xyz, 20, 1.0, cell_hint=0.25)


def test_coincident_points_and_priors(eng):
    """zero covariances (three and more coincident points), d2 = 0, isolated points; without and with priors, and the plane through
    the origin where the prior decides the sign"""
    xyz = NC.coincident()
    rng = np.random.default_rng(1)
    pri = rng.normal(size=xyz.shape)
    for knn in (2, 3, 4, 5, 10):
        run_and_check(eng, f"coincident knn {knn}", xyz, knn, 0.3)
        run_and_check(eng, f"coincident knn {knn} prior", xyz, knn, 0.3, priors=pri)
    pl = np.vstack([NC.plane_through_origin(), [[5.0, 5.0, 0.0], [-5.0, 6.0, 0.0]]])
    for s in (1.0, -1.0):
        run_and_check(eng, f"plane z = 0, prior z {s:+.0f}", pl, 10, 0.5, priors=np.tile([0.0, 0.0, s], (len(pl), 1)))


@pytest.mark.parametrize("offset", [0.0, 1e2, 1e3, 1e4])
def test_offsets(eng, offset):
    run_and_check(eng, f"scan voxels + {offset:g}", _scan_voxels((offset, -offset, 0.1 * offset), 20000), 20, 3.0, cell_hint=0.4)
    run_and_check(eng, f"lattice + {offset:g}", NC.lattice(8, 0.25, (offset, offset, offset)), 20, 0.6)


def test_query_subset_and_cell_rules(eng):
    xyz = _scan_voxels(n_max=20000)
    flags = (np.random.default_rng(2).random(len(xyz)) < 0.3).astype(np.int32)
    run_and_check(eng, "flagged 30 %", xyz, 20, 3.0, cell_hint=0.4, flags=flags)
    run_and_check(eng, "default cell r/4", xyz, 20, 3.0)
    run_and_check(eng, "cell clamp r/16", xyz, 20, 3.0, cell_hint=1e-3)
    run_and_check(eng, "config1", synth.planar_cloud_config1(noise=0.01)[1].astype(np.float64), 10, 1.0)


def test_grid_faces(eng):
    """a box of 256 / 257 points around a query at each corner cell of the grid (unbounded faces) and 256 / 257 block candidates"""
    rng = np.random.default_rng(3)
    for m in (255, 256):
        blob = rng.uniform(-0.3, 0.3, (m, 3))
        xyz = np.vstack([[[0.0, 0.0, 0.0]], blob, [[20.0, 20.0, 20.0]], blob + 20.0])
        run_and_check(eng, f"faces, {m + 1} in the block", xyz, 20, 1.0, cell_hint=0.25)


def test_production_entry_matches_the_record(eng):
    """b2s_estimate_normals on the same cloud: per-point within the gap-aware bound of the debug entry's normals (the grid's atomic
    cell fill may reorder the butterfly's inputs, so bit equality is not required)"""
    xyz = _scan_voxels(n_max=20000)
    vs = E.MapperParameters().scanProcessing.voxelSize
    _, _, dbg, _ = debug_normals(eng, xyz, 20, 3.0, cell_hint=4 * vs if vs > 0 else 0.0)
    cl = eng.cloud(xyz)
    L.check(L.lib().b2s_estimate_normals(eng._h, cl._c, 20, C.c_double(3.0)))
    _, got = cl.download()
    worst = NC.assert_normals_close(got, dbg, xyz, 20, 3.0)
    print(f"b2s_estimate_normals vs the debug entry: worst {worst:.3g} of the gap-aware bound")


def test_process_scan_flagged_matches_the_record(engine_factory, eng):
    """processForScanMatchingAndMerging with downSamplingRatio < 1 estimates normals for the selected points only (the query list from
    the selection flags), neighbours from the whole voxel cloud, and merge_ is the selected points: its normals against the debug entry
    run on the same voxel cloud with the same flags and cell"""
    p = E.MapperParameters(seed=5)
    p.scanProcessing.downSamplingRatio = 0.3
    p.scanProcessing.cropper = E.ScanCroppingParameters("MinMaxRadius", 2.0, 25.0)
    raw = synth.lidar_scan(synth.Scene(), synth.loop_trajectory(4)[1], seed=11).astype(np.float64)
    e2 = engine_factory(p)
    ps = E.scanToMapRegistrationFactory(e2, p).processForScanMatchingAndMerging(e2.cloud(raw))
    hx, hn = ps.merge_.download()
    # the voxel cloud the flagged estimation ran on, in the device's order (equal d2 go to the lower index, so the order matters):
    # the map builder's cropper (sensor frame) and the voxel down-sample, as the pre-processing runs them
    cropped = E.crop(e2, e2.cloud(raw), p.mapBuilder.cropper.to_c(center=(0.0, 0.0, 0.0)))
    t0, _ = E.voxelize(e2, cropped, p.scanProcessing.voxelSize).download()
    idx = NC.rows_in(hx, t0)
    flags = np.zeros(len(t0), dtype=np.int32)
    flags[idx] = 1
    knn, radius = p.icp.knn, p.icp.maxDistanceKnn
    _, _, dbg = run_and_check(eng, "process_scan flagged", t0, knn, radius, cell_hint=4 * p.scanProcessing.voxelSize, flags=flags,
                              full=True)[:3]
    worst = NC.assert_normals_close(hn, dbg[idx], t0, knn, radius, queries=idx)
    print(f"processForScanMatchingAndMerging merge_ vs the debug entry: worst {worst:.3g} of the gap-aware bound ({len(idx)} of {len(t0)})")


def test_compute_features_matches_the_record(eng):
    """Submap::computeFeatures estimates the sparse cloud's normals with the voxel-mean normals as priors: its normals against the
    debug entry run with the same priors on the same sparse cloud"""
    P = E.PlaceRecognitionParameters()
    xyz, nrm = lidar_map(1)
    sm = E.Submap(eng, 100_000)
    sm.setMapPointCloud(eng.cloud(xyz, nrm))
    sm.computeFeatures(P)
    dx, dn = sm.getSparseMapPointCloud().download()
    vx, vn = E.voxelize(eng, sm.toCloud(), P.featureVoxelSize).download()
    idx = NC.rows_in(dx, vx)
    assert len(idx) == len(vx)
    _, _, dbg = run_and_check(eng, "computeFeatures sparse cloud", vx, P.normalKnn, P.normalEstimationRadius, priors=vn, full=True)[:3]
    worst = NC.assert_normals_close(dn, dbg[idx], vx, P.normalKnn, P.normalEstimationRadius, queries=idx)
    print(f"computeFeatures vs the debug entry: worst {worst:.3g} of the gap-aware bound")
