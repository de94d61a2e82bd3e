"""-m gpu: map fusion and the map-side voxel hashes against the CPU oracle at voxel faces, key limits, probe wrap-around and capacities.

The parity tests feed the map side random scans, on which no point lies near a voxel face, no key comes near the key limit, no
probe run wraps past the end of a table and no capacity is reached.  Each edge is crossed here and held to the oracle with the
idioms of test_gpu_boundaries.py: keyed bit-exact positions, normals to 1e-12, dense sums to 1e-12.  The table rules the inputs are
built from live in tests/voxel_hash.py, which test_voxel_hash_rules.py checks against the CUDA sources.

  voxel faces (K-fuse)   the mean of three members rounds below the lower face / above the upper face of its voxel, on x, y and
                         z, for positive and negative coordinates, at the identity and at an exact translation; the next scan
                         touches the new voxel or only the old one; with and without a (no-op) carve, i.e. a rehash, in between
  key limit              |floor(p / v)| = 2^20 - 2 is kept and equals the oracle; 2^20 - 1 is refused with B2S_E_INVALID by the
                         fusion, the dense map, sparse carving, the overlap and the voxel map, and reported absent by queries
  far rays (C1, C2)      one or two scan points beyond the key limit still cast their rays through the voxels near the sensor
  probe wrap-around      keys homed at the last slot and at slot 0 of the dense map, the fusion hash, the voxel map, the overlap
                         and the dense-carve ray table form one run of occupied slots across the end of the table
  capacities             submap capacity, FUSE_DUP_CAP, the 7/8-full dense map and voxel map: at the limit equal to the oracle,
                         one past it B2S_E_CAPACITY, after which a new submap on the same engine behaves like one on a fresh engine
"""
import numpy as np
import pytest

import voxel_hash as VH
from oracle import oracle as O
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import synth
from open3d_slam_b200 import _lib as L

pytestmark = pytest.mark.gpu

V = 0.1                          # map voxel
INV = 1.0 / V
DV = 0.05                        # dense voxel
NORMAL = np.array([0.0, 0.0, 1.0])
LIMIT = VH.KEY_LIMIT - 1         # the largest accepted key index


def keyed(xyz, nrm, voxel=V):
    k = np.floor(xyz * (1.0 / voxel)).astype(np.int64)
    order = np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0], k[:, 2], k[:, 1], k[:, 0]))
    return xyz[order], nrm[order]


def assert_map_equal(sm, ref_x, ref_n, what=""):
    gx, gn = sm.getMapPointCloud()
    assert len(gx) == len(ref_x), (what, len(gx), len(ref_x))
    a, an = keyed(gx, gn); b, bn = keyed(ref_x, ref_n)
    assert np.array_equal(a, b), (what, a[np.any(a != b, axis=1)][:4], b[np.any(a != b, axis=1)][:4])
    assert np.abs(an - bn).max() < 1e-12, what


def assert_dense_equal(sm, dm, what=""):
    gx, gk = sm.getDenseMap(); rx, _rn, rk = dm.to_cloud()
    assert len(gx) == len(rx), (what, len(gx), len(rx))
    o1 = np.lexsort((gk[:, 2], gk[:, 1], gk[:, 0])); o2 = np.lexsort((rk[:, 2], rk[:, 1], rk[:, 0]))
    assert np.array_equal(gk[o1], rk[o2]), what
    assert np.abs(gx[o1] - rx[o2]).max() < 1e-12, what


def raises(code, *calls):
    with pytest.raises(L.B2SError) as ei:
        for c in calls:
            c()
    assert ei.value.code == code, (ei.value.code, code)


def params(cropper=("MinMaxRadius", 0.0, 30.0)):
    p = E.MapperParameters()
    p.mapBuilder.cropper = E.ScanCroppingParameters(*cropper)
    p.denseMapVoxelSize = DV
    return p


def ocrop(cropper=("MinMaxRadius", 0.0, 30.0)):
    return O.cropper(*cropper)


def nrms(n):
    return np.tile(NORMAL, (n, 1))


def translation(t):
    T = np.eye(4); T[:3, 3] = t
    return T


# ----------------------------------------------------------------------------------------------------------------------
# A. voxel faces in fusion
# ----------------------------------------------------------------------------------------------------------------------
def face_side(k, side, n=10):
    """The n doubles closest to the lower (side -1) or upper (side +1) face of voxel k under floor(x * (1/v))."""
    x = (k if side < 0 else k + 1) * V
    while VH.key_of([x], V)[0] >= k + (0 if side < 0 else 1):
        x = np.nextafter(x, -np.inf)
    while VH.key_of([x], V)[0] < k:
        x = np.nextafter(x, np.inf)
    out = []
    while len(out) < n:
        if VH.key_of([x], V)[0] == k:
            out.append(float(x))
        x = np.nextafter(x, np.inf if side < 0 else -np.inf)
    return out


def crossing(k, side, t):
    """Members (a, b, c) of voxel k: a first fused alone (map point a), then b and c (scan points b - t, c - t under the
    translation t) or b twice (t = None: the identity insertion stages every scan point twice), so that ((a + b) + c) / 3
    rounds out of voxel k.  None when no such triple lies within a few ulps of the face."""
    cand = face_side(k, side)
    for a in cand:
        for b in cand:
            for c in ([b] if t is None else cand):
                m = ((a + b) + c) / 3.0
                if VH.key_of([m], V)[0] == k:
                    continue
                if t is not None and not ((b - t) + t == b and (c - t) + t == c):
                    continue
                return a, b, c, m
    return None


T_EXACT = np.array([0.5, -0.25, 0.125])


def face_groups(exact):
    """12 voxels, one per (axis, sign, face), each with a crossing; the other two coordinates are dyadic, so they stay put."""
    groups = []
    t = T_EXACT if exact else np.zeros(3)
    found = {}
    for sign in (1, -1):
        for side in (-1, 1):
            ks = iter(range(sign * 50, sign * 200, sign))
            for axis in range(3):      # the next voxel from 5 m out with a crossing, a different one per axis
                found[(axis, sign, side)] = next(h for h in (crossing(k, side, t[axis] if exact else None) for k in ks) if h)
    for g, (axis, sign, side) in enumerate((a, s, f) for a in range(3) for s in (1, -1) for f in (-1, 1)):
        a, b, c, m = found[(axis, sign, side)]
        other = [-11.25 + 2.0 * g, 3.75 + 0.5 * axis]
        pts = []
        for x in (a, b, c, m):
            p = np.empty(3); p[axis] = x; p[[i for i in range(3) if i != axis]] = other
            pts.append(p)
        pa, pb, pc, pm = pts
        key_old = VH.key_of(pa, V); key_new = VH.key_of(pm, V)
        assert key_old != key_new
        groups.append(dict(a=pa, b=pb, c=pc, old=key_old, new=key_new))
    keys = [g["old"] for g in groups] + [g["new"] for g in groups]
    assert len(set(keys)) == len(keys)
    return groups


@pytest.mark.parametrize("exact", [False, True], ids=["identity", "translation"])
@pytest.mark.parametrize("follow", ["new_voxel", "old_voxel"])
@pytest.mark.parametrize("carve", [False, True], ids=["incremental", "rehash"])
def test_fused_mean_crossing_a_voxel_face(engine_factory, exact, follow, carve):
    groups = face_groups(exact)
    p = params()
    eng = engine_factory(p)
    sm = E.Submap(eng, 10_000)
    T = translation(T_EXACT) if exact else np.eye(4)
    crop = ocrop()
    mx = np.zeros((0, 3)); mn = np.zeros((0, 3))

    def insert(scan, Ti, what):
        nonlocal mx, mn
        sm.insertScan(None, eng.cloud(scan, nrms(len(scan))), Ti)
        mx, mn = O.submap_insert_scan(mx, mn, scan, nrms(len(scan)), Ti, V, crop)
        assert_map_equal(sm, mx, mn, what)

    insert(np.array([g["a"] for g in groups]), np.eye(4), "first insertion")
    second = [g["b"] for g in groups] if not exact else [q for g in groups for q in (g["b"] - T_EXACT, g["c"] - T_EXACT)]
    insert(np.array(second), T, "the crossing insertion")
    moved = {VH.key_of(x, V) for x in mx}
    assert all(g["new"] in moved and g["old"] not in moved for g in groups)      # the oracle moved every mean
    if carve:      # a ray straight up from the sensor, far from every group: nothing is carved, the fusion hash is rebuilt
        raw = np.array([[0.0, 0.0, 1.0]])
        prm = E.SpaceCarvingParameters()
        assert sm.carve(eng.cloud(raw), T, prm, force=True) == 0
        assert not O.carve(mx, mn, O.transform(T, raw)[0], T[:3, 3], O.cropper("MinMaxRadius", 0.0, 30.0, center=T[:3, 3])).any()
    third = np.array([VH.point_in(g[follow.split("_")[0]], V) for g in groups])
    insert(third - T[:3, 3] if exact else third, T, f"a scan touching the {follow.replace('_', ' ')}")
    assert len(mx) == (len(groups) if follow == "new_voxel" else 2 * len(groups))
    insert(third - T[:3, 3] if exact else third, T, "once more")


def test_relinked_mean_merges_with_a_map_point_of_its_new_voxel(engine_factory):
    """A mean that moves into a voxel that already holds a map point (here one outside the cropper at the time) is queued as a
    duplicate: the two merge at the next insertion in which both are inside the cropper, as the reference's re-bucketing does."""
    groups = face_groups(False)
    p = params(("MaxRadius", 0.0, 30.0))
    eng = engine_factory(p)
    sm = E.Submap(eng, 10_000)
    mx = np.zeros((0, 3)); mn = np.zeros((0, 3))
    far = translation([40.0, 0.0, 0.0])

    def insert(scan, Ti, what):
        nonlocal mx, mn
        sm.insertScan(None, eng.cloud(scan, nrms(len(scan))), Ti)
        mx, mn = O.submap_insert_scan(mx, mn, scan, nrms(len(scan)), Ti, V, O.cropper("MaxRadius", 0.0, 30.0))
        assert_map_equal(sm, mx, mn, what)

    # points of the new voxels, fused while the sensor sits 40 m away: most are outside the cropper and pass through
    insert(np.array([VH.point_in(g["new"], V) for g in groups]) - far[:3, 3], far, "new voxels seen from afar")
    insert(np.array([g["a"] for g in groups]), np.eye(4), "first insertion")
    insert(np.array([g["b"] for g in groups]), np.eye(4), "the crossing insertion")
    insert(np.array([[0.05, 0.05, 25.05]]), np.eye(4), "an unrelated scan: the queued duplicates merge")
    insert(np.array([[0.05, 0.05, 25.05]]), np.eye(4), "once more")


# ----------------------------------------------------------------------------------------------------------------------
# B. key limit and far rays
# ----------------------------------------------------------------------------------------------------------------------
def limit_points(k, voxel):
    """One point per (axis, sign) whose key index on that axis is +-k (and 3 on the others)."""
    out = []
    for axis in range(3):
        for sign in (1, -1):
            key = [3, 3, 3]; key[axis] = sign * k
            out.append(VH.point_in(key, voxel))
    return np.array(out)


def test_key_limit_fusion_and_dense_map(engine_factory):
    eng = engine_factory(params(("None",)))
    inside = np.vstack([limit_points(LIMIT, V), [[0.05, 0.05, 0.05]]])
    sm = E.Submap(eng, 1000)
    mx = np.zeros((0, 3)); mn = np.zeros((0, 3))
    for T in (np.eye(4), translation([0.01, -0.01, 0.01])):      # the translation keeps every point in its voxel
        sm.insertScan(None, eng.cloud(inside, nrms(len(inside))), T)
        mx, mn = O.submap_insert_scan(mx, mn, inside, nrms(len(inside)), T, V, ocrop(("None",)))
        assert_map_equal(sm, mx, mn, "fusion at the key limit")
    for q in limit_points(LIMIT + 1, V):
        bad = E.Submap(eng, 1000)
        raises(L.E_INVALID, lambda: bad.insertScan(None, eng.cloud(q[None], nrms(1)), np.eye(4)), bad.size)
    # dense map: insert, query, remove
    dinside = np.vstack([limit_points(LIMIT, DV), [[0.025, 0.025, 0.025]]])
    douter = limit_points(LIMIT + 1, DV)
    sm = E.Submap(eng, 1000)
    dm = O.DenseMap(DV, 1 << 10)
    sm.insertScanDenseMap(eng.cloud(dinside), np.eye(4), None)
    dm.insert(O.transform(np.eye(4), dinside)[0])
    assert_dense_equal(sm, dm, "dense map at the key limit")
    counts, means = sm.denseQuery(eng.cloud(np.vstack([dinside, douter])))
    assert np.array_equal(counts, [2] * len(dinside) + [0] * len(douter))         # the identity insertion stages every point twice
    assert np.array_equal(means[:len(dinside)], dinside)
    sm.denseRemove(eng.cloud(np.vstack([dinside[:3], douter])))
    assert sm.denseSize() == len(dinside) - 3
    counts, _ = sm.denseQuery(eng.cloud(dinside), with_means=False)
    assert np.array_equal(counts > 0, np.arange(len(dinside)) >= 3)
    for q in douter:
        bad = E.Submap(eng, 1000)
        raises(L.E_INVALID, lambda: bad.insertScanDenseMap(eng.cloud(q[None]), np.eye(4), None), bad.denseSize)


def test_key_limit_overlap_and_voxel_map(engine_factory):
    eng = engine_factory(params())
    pts = np.vstack([limit_points(LIMIT, V), [[0.05, 0.05, 0.05]]])
    tgt = np.vstack([pts[::2], [[7.05, 0.05, 0.05]]])
    so, to = E.computeOverlappingClouds(eng, eng.cloud(pts, nrms(len(pts))), eng.cloud(tgt, nrms(len(tgt))), np.eye(4), V, 1)
    fs, ft = O.overlap_flags(pts, tgt, np.eye(4), V, 1)
    assert 0 < fs.sum() < len(pts) and 0 < ft.sum() < len(tgt)
    assert np.array_equal(so.download()[0], pts[fs]) and np.array_equal(to.download()[0], tgt[ft])
    for q in limit_points(LIMIT + 1, V):
        raises(L.E_INVALID, lambda: E.computeOverlappingClouds(eng, eng.cloud(q[None], nrms(1)), eng.cloud(tgt, nrms(len(tgt))), np.eye(4), V, 1),
               eng.synchronize)
    vv = 0.25
    vm = E.VoxelMap(eng, vv, 64)
    vin = np.vstack([limit_points(LIMIT, vv), [[0.1, 0.1, 0.1]]])
    vout = limit_points(LIMIT + 1, vv)
    vm.insertCloud("map", eng.cloud(vin))
    assert vm.size() == len(vin)
    flags, hits = vm.hasVoxelContainingPoint(eng.cloud(np.vstack([vin, vout])))
    assert hits == len(vin) and np.array_equal(flags, np.arange(len(vin) + len(vout)) < len(vin))
    idx = vm.getIndicesInVoxel("map", eng.cloud(np.vstack([vin, vout])))
    assert [list(i) for i in idx] == [[j] for j in range(len(vin))] + [[]] * len(vout)
    for q in vout:
        bad = E.VoxelMap(eng, vv, 64)
        raises(L.E_INVALID, lambda: bad.insertCloud("map", eng.cloud(q[None])), bad.size)


@pytest.mark.parametrize("sign", [1, -1])
def test_key_limit_sparse_carving(engine_factory, sign):
    """C1 keys the map points inside the cropper: one at +-(2^20 - 2) voxels is carved like the oracle carves it, one voxel
    further is refused."""
    p = params(("MaxRadius", 0.0, 20.0))
    eng = engine_factory(p)
    key = [sign * LIMIT, 0, 0]
    P = VH.point_in(key, V)
    T = translation([P[0] - sign * 7.0, 0.05, 0.05])
    mx = np.array([P, P + [0.0, 0.1, 0.0], P + [0.0, 3.0, 0.0], P - [sign * 2.0, 0.0, 0.0]])
    mn = np.array([[1.0, 0.0, 0.0]] * 4)
    raw = np.array([[sign * 7.5, 0.0, 0.0], [sign * 7.5, 0.1, 0.0]])
    prm = E.SpaceCarvingParameters(voxelSize=V, maxRaytracingLength=20.0, truncationDistance=0.1, minDotProductWithNormal=0.5)
    sm = E.Submap(eng, 1000)
    sm.setMapPointCloud(eng.cloud(mx, mn)); sm._cropperPose = T
    n = sm.carve(eng.cloud(raw), T, prm, force=True)
    rem = O.carve(mx, mn, O.transform(T, raw)[0], T[:3, 3], O.cropper("MaxRadius", 0.0, 20.0, center=T[:3, 3]), V, 20.0, 0.1, 0.5)
    assert 0 < rem.sum() < len(mx) and n == int(rem.sum())
    gx, gn = sm.getMapPointCloud()
    assert np.array_equal(gx, mx[~rem]) and np.array_equal(gn, mn[~rem])
    bad = E.Submap(eng, 1000)
    bad.setMapPointCloud(eng.cloud(np.vstack([mx, VH.point_in([sign * (LIMIT + 1), 0, 0], V)]), np.vstack([mn, [1.0, 0.0, 0.0]])))
    bad._cropperPose = T
    raises(L.E_INVALID, lambda: bad.carve(eng.cloud(raw), T, prm, force=True))


def near_map(rng, n=4000):
    """Dense-map content around a sensor at the origin: a shell of points 1-19 m out in every direction."""
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d * rng.uniform(1.0, 19.0, (n, 1))


FAR = 200_000.0     # 2 million map voxels along two axes of each direction below: beyond the 21-bit fields


@pytest.mark.parametrize("case", ["one", "same_voxel", "two_voxels"])
def test_far_rays_carve_the_dense_map(engine_factory, case):
    """C2: a return beyond the key limit is still a ray: it carves up to maxRaytracingLength, like the reference's int32 keys."""
    rng = np.random.default_rng(3)
    d1 = np.array([0.6, 0.64, 0.48]); d2 = np.array([-0.48, 0.6, -0.64])
    pts = near_map(rng)
    along = np.vstack([np.outer(np.arange(1.0, 19.0, 0.5), d) for d in (d1, d2)])     # voxels on both rays
    content = np.vstack([pts, along])
    far = {"one": [FAR * d1], "same_voxel": [FAR * d1, FAR * d1 + 0.01], "two_voxels": [FAR * d1, FAR * d2]}[case]
    scan = np.vstack([pts[:200], far, pts[200:400]])
    eng = engine_factory(params())
    sm = E.Submap(eng, 1000)
    sm.insertScanDenseMap(eng.cloud(content), translation([1.0, 0.0, 0.0]), None)
    dm = O.DenseMap(DV, 1 << 16); dm.insert(O.transform(translation([1.0, 0.0, 0.0]), content)[0])
    prm = E.SpaceCarvingParameters(maxRaytracingLength=20.0, truncationDistance=0.1, neighborhoodRadiusDenseMap=0.1)
    sensor = np.array([1.0, 0.0, 0.0])
    n = sm.carveDenseMap(eng.cloud(scan), sensor, prm)
    ref = dm.carve(scan, sensor, DV, 0.1, 0.1, 20.0)
    near_only = O.DenseMap(DV, 1 << 16); near_only.insert(O.transform(translation([1.0, 0.0, 0.0]), content)[0])
    assert ref > near_only.carve(np.vstack([pts[:200], pts[200:400]]), sensor, DV, 0.1, 0.1, 20.0)      # the far rays matter
    assert n == ref
    assert_dense_equal(sm, dm, "after carving with far rays")


def test_far_ray_carves_the_sparse_map(engine_factory):
    """C1: a scan point beyond the key limit marches up to maxRaytracingLength through the map points near the sensor."""
    rng = np.random.default_rng(4)
    d = np.array([0.6, 0.64, 0.48])
    mx = np.vstack([near_map(rng, 2000), np.outer(np.arange(1.0, 19.0, 0.25), d)])
    mn = np.tile(d, (len(mx), 1))
    raw = np.array([FAR * d, [3.0, 0.0, 0.0]])
    p = params(("MaxRadius", 0.0, 20.0))
    eng = engine_factory(p)
    prm = E.SpaceCarvingParameters(voxelSize=V, maxRaytracingLength=20.0, truncationDistance=0.1, minDotProductWithNormal=0.5)
    sm = E.Submap(eng, 10_000)
    sm.setMapPointCloud(eng.cloud(mx, mn))
    n = sm.carve(eng.cloud(raw), np.eye(4), prm, force=True)
    rem = O.carve(mx, mn, raw, np.zeros(3), O.cropper("MaxRadius", 0.0, 20.0), V, 20.0, 0.1, 0.5)
    assert rem.sum() > 20 and n == int(rem.sum())
    assert np.array_equal(sm.getMapPointCloud()[0], mx[~rem])


# ----------------------------------------------------------------------------------------------------------------------
# C. probe runs across the end of a table
# ----------------------------------------------------------------------------------------------------------------------
def wrap_keys(slots, n_each, seed):
    """Members: keys homed at the last slot and at slot 0 (one run of occupied slots across the end).  Absent: keys homed at
    slots inside that run."""
    b = VH.KEY_LIMIT - 16      # room for the small translations below
    members = VH.keys_homed_at(slots - 1, slots, n_each, seed, b) + VH.keys_homed_at(0, slots, n_each, seed + 1, b)
    absent = [k for s in (slots - 1, 0, 1, n_each) for k in VH.keys_homed_at(s, slots, 2, seed + 2 + s, b) if k not in members]
    return members, absent


def test_dense_map_probe_run_wraps(engine_factory):
    members, absent = wrap_keys(VH.DENSE_SLOTS, 6, 10)
    pts = np.array([VH.point_in(k, DV) for k in members]); q_abs = np.array([VH.point_in(k, DV) for k in absent])
    eng = engine_factory(params())
    sm = E.Submap(eng, 1000)
    T = translation([0.0, 0.0, 0.0])
    sm.insertScanDenseMap(eng.cloud(pts), T, None)
    dm = O.DenseMap(DV, 1 << 10); dm.insert(O.transform(T, pts)[0])
    assert_dense_equal(sm, dm, "dense keys around the end of the table")
    counts, means = sm.denseQuery(eng.cloud(np.vstack([pts, q_abs])))
    assert np.array_equal(counts, [2] * len(pts) + [0] * len(q_abs)) and np.array_equal(means[:len(pts)], pts)
    sm.denseRemove(eng.cloud(pts[[1, 6]]))          # the middle of the run on both sides of the end
    counts, _ = sm.denseQuery(eng.cloud(np.vstack([pts, q_abs])), with_means=False)
    assert np.array_equal(counts > 0, [i not in (1, 6) for i in range(len(pts))] + [False] * len(q_abs))
    sm.insertScanDenseMap(eng.cloud(q_abs), T, None)     # absent keys take the slots after the run
    dm2 = O.DenseMap(DV, 1 << 10); dm2.insert(O.transform(T, np.vstack([pts[[i for i in range(len(pts)) if i not in (1, 6)]], q_abs]))[0])
    assert_dense_equal(sm, dm2, "after removal and re-insertion")


def test_fusion_hash_probe_run_wraps(engine_factory):
    capacity = 2000
    slots = VH.fusion_slots(capacity)
    members, absent = wrap_keys(slots, 6, 20)
    eng = engine_factory(params(("None",)))
    sm = E.Submap(eng, capacity)
    mx = np.zeros((0, 3)); mn = np.zeros((0, 3))
    T = translation([0.5, 0.0, 0.0])
    for scan in (np.array([VH.point_in(k, V) for k in members]) - T[:3, 3],
                 np.array([VH.point_in(k, V) for k in members[::2] + absent]) - T[:3, 3]):
        sm.insertScan(None, eng.cloud(scan, nrms(len(scan))), T)
        mx, mn = O.submap_insert_scan(mx, mn, scan, nrms(len(scan)), T, V, ocrop(("None",)))
        assert_map_equal(sm, mx, mn, "fusion keys around the end of the table")
    assert len(mx) == len(members) + len(absent)


def test_voxel_map_and_overlap_probe_runs_wrap(engine_factory):
    eng = engine_factory(params())
    vv = 0.25
    vm = E.VoxelMap(eng, vv, 512)
    slots = VH.grown(VH.SCRATCH_TABLE_MIN, 512)
    members, absent = wrap_keys(slots, 6, 30)
    pts = np.array([VH.point_in(k, vv) for k in members]); q_abs = np.array([VH.point_in(k, vv) for k in absent])
    vm.insertCloud("map", eng.cloud(np.vstack([pts, pts[:3]])))
    assert vm.size() == len(pts)
    flags, hits = vm.hasVoxelContainingPoint(eng.cloud(np.vstack([pts, q_abs])))
    assert hits == len(pts) and np.array_equal(flags, np.arange(len(pts) + len(q_abs)) < len(pts))
    idx = vm.getIndicesInVoxel("map", eng.cloud(np.vstack([pts, q_abs])))
    want = [[i, len(pts) + i] if i < 3 else [i] for i in range(len(pts))] + [[]] * len(q_abs)
    assert [list(i) for i in idx] == want
    # overlap: fewer than 512 points in all, so its table has 1024 slots as well
    ov_slots = VH.grown(VH.SCRATCH_TABLE_MIN, 40)
    members, absent = wrap_keys(ov_slots, 6, 40)
    src = np.array([VH.point_in(k, V) for k in members + absent[:3]])
    tgt = np.array([VH.point_in(k, V) for k in members[::2] + absent[3:]])
    so, to = E.computeOverlappingClouds(eng, eng.cloud(src, nrms(len(src))), eng.cloud(tgt, nrms(len(tgt))), np.eye(4), V, 1)
    fs, ft = O.overlap_flags(src, tgt, np.eye(4), V, 1)
    assert fs.sum() == len(members[::2]) and np.array_equal(so.download()[0], src[fs]) and np.array_equal(to.download()[0], tgt[ft])


def test_dense_carve_ray_table_probe_run_wraps(engine_factory):
    """The ray set of C2 is the first scan point of every voxel: scan voxels homed at both ends of the 1024-slot ray table, each
    with two points, so the rays of the second points are dropped across the end of the table."""
    members, _ = wrap_keys(VH.grown(VH.SCRATCH_TABLE_MIN, 20), 5, 50)
    first = np.array([VH.point_in(k, DV) for k in members])
    scan = np.vstack([first, first + DV * 0.25])           # the second point of each voxel
    rng = np.random.default_rng(5)
    content = near_map(rng, 6000)
    eng = engine_factory(params())
    sm = E.Submap(eng, 1000)
    T = translation([0.0, 0.0, 0.0])
    sm.insertScanDenseMap(eng.cloud(content), T, None)
    dm = O.DenseMap(DV, 1 << 16); dm.insert(O.transform(T, content)[0])
    prm = E.SpaceCarvingParameters(maxRaytracingLength=20.0, truncationDistance=0.1, neighborhoodRadiusDenseMap=0.1)
    n = sm.carveDenseMap(eng.cloud(scan), np.zeros(3), prm)
    assert n == dm.carve(scan, np.zeros(3), DV, 0.1, 0.1, 20.0) > 0
    assert_dense_equal(sm, dm, "after carving with rays keyed around the end of the table")


# ----------------------------------------------------------------------------------------------------------------------
# D. capacities: at the limit and one past it
# ----------------------------------------------------------------------------------------------------------------------
def grid(n, voxel, origin, width=200):
    """n points at the centres of n distinct voxels, in a block starting at the voxel `origin`."""
    i = np.arange(n)
    k = np.c_[i % width, (i // width) % width, i // (width * width)] + np.asarray(origin)
    p = (k + 0.5) * voxel
    assert np.array_equal(np.floor(p * (1.0 / voxel)).astype(np.int64), k)
    return p


def assert_engine_recovers(eng, engine_factory, p):
    """A new submap on `eng` fuses two scans and registers a third against the map exactly like one on a fresh engine."""
    sc = synth.Scene(); poses = synth.loop_trajectory(4)
    out = []
    for e in (eng, engine_factory(p)):
        s2m = E.ScanToMapIcp(e)
        sm = E.Submap(e, 300_000)
        for k in range(2):
            ps = s2m.processForScanMatchingAndMerging(e.cloud(synth.lidar_scan(sc, poses[k], seed=k).astype(np.float64)))
            sm.insertScan(None, ps.merge_, np.linalg.inv(poses[0]) @ poses[k])
        ps = s2m.processForScanMatchingAndMerging(e.cloud(synth.lidar_scan(sc, poses[2], seed=2).astype(np.float64)))
        res = E.RegistrationIcpPointToPlane(e).registerClouds(ps.match_, sm.toCloud(), np.linalg.inv(poses[0]) @ poses[1])
        out.append((sm.getMapPointCloud(), res))
    (ax, an), ra = out[0]; (bx, bn), rb = out[1]
    assert len(ax) == len(bx) and np.array_equal(keyed(ax, an)[0], keyed(bx, bn)[0])
    assert ra.iters == rb.iters and ra.n_corr == rb.n_corr and np.abs(ra.transformation_ - rb.transformation_).max() < 1e-10


def test_submap_capacity(engine_factory):
    p = params()
    eng = engine_factory(p)
    cap = 3000
    pts = grid(cap + 1, V, (20, 20, 0), width=20)
    sm = E.Submap(eng, cap)
    sm.insertScan(None, eng.cloud(pts[:cap], nrms(cap)), np.eye(4))
    mx, mn = O.submap_insert_scan(np.zeros((0, 3)), np.zeros((0, 3)), pts[:cap], nrms(cap), np.eye(4), V, ocrop())
    assert len(mx) == cap
    assert_map_equal(sm, mx, mn, "a submap filled exactly")
    full = E.Submap(eng, cap)
    raises(L.E_CAPACITY, lambda: full.insertScan(None, eng.cloud(pts, nrms(cap + 1)), np.eye(4)), full.size)
    assert_engine_recovers(eng, engine_factory, p)


def test_fusion_duplicate_list_capacity(engine_factory):
    """Every voxel holding two pass-through points (an identity insertion outside the cropper) is queued as a duplicate."""
    p = params()
    eng = engine_factory(p)
    n = VH.FUSE_DUP_CAP
    pts = grid(n + 1, V, (400, 0, 0), width=64)            # 40 m and more from the sensor: outside the 30 m cropper
    sm = E.Submap(eng, 2 * n + 4)
    sm.insertScan(None, eng.cloud(pts[:n], nrms(n)), np.eye(4))
    mx, mn = O.submap_insert_scan(np.zeros((0, 3)), np.zeros((0, 3)), pts[:n], nrms(n), np.eye(4), V, ocrop())
    assert len(mx) == 2 * n
    assert_map_equal(sm, mx, mn, "FUSE_DUP_CAP voxels of two points")
    over = E.Submap(eng, 2 * n + 4)
    raises(L.E_CAPACITY, lambda: over.insertScan(None, eng.cloud(pts, nrms(n + 1)), np.eye(4)), over.size)
    assert_engine_recovers(eng, engine_factory, p)


def test_dense_map_capacity(engine_factory):
    p = params()
    eng = engine_factory(p)
    n = VH.dense_fill_limit()
    pts = grid(n + 1, DV, (-100, -100, -40), width=200)
    T = translation([1.0, 0.0, 0.0])
    sm = E.Submap(eng, 1000)
    sm.insertScanDenseMap(eng.cloud(pts[:n]), T, None)
    assert sm.denseSize() == n
    dm = O.DenseMap(DV, VH.DENSE_SLOTS); dm.insert(O.transform(T, pts[:n])[0])
    assert_dense_equal(sm, dm, "a dense map filled to 7/8")
    over = E.Submap(eng, 1000)
    raises(L.E_CAPACITY, lambda: over.insertScanDenseMap(eng.cloud(pts), T, None), over.denseSize)
    assert_engine_recovers(eng, engine_factory, p)


def test_voxel_map_capacity(engine_factory):
    p = params()
    eng = engine_factory(p)
    vv, capacity = 0.25, 1000
    n = VH.dense_fill_limit(VH.grown(VH.SCRATCH_TABLE_MIN, capacity))
    assert n >= capacity
    pts = grid(n + 1, vv, (-10, -10, -10), width=20)
    vm = E.VoxelMap(eng, vv, capacity)
    vm.insertCloud("map", eng.cloud(pts[:n]))
    assert vm.size() == n
    flags, hits = vm.hasVoxelContainingPoint(eng.cloud(pts))
    assert hits == n and flags[:n].all() and not flags[n]
    idx = vm.getIndicesInVoxel("map", eng.cloud(pts[:n]))
    assert all(list(i) == [j] for j, i in enumerate(idx))
    over = E.VoxelMap(eng, vv, capacity)
    raises(L.E_CAPACITY, lambda: over.insertCloud("map", eng.cloud(pts)), over.size)
    assert_engine_recovers(eng, engine_factory, p)
