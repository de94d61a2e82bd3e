"""GPU: b2s_assemble_map / b2s_assemble_colored_map (Mapper::getAssembledMapPointCloud, assembleColoredPointCloud, voxelize; DESIGN.md
row A1) -- bit-identical to concatenating b2s_submap_to_cloud on the closed lap before and after a loop-closure correction, the voxel
path against the oracle (also 5 km from the origin), the colours against the in-order restatement, the normals rule, empty and error
cases, the launch geometry of K-assemble and the batched scan, a map of more than 2^24 points, and no side effects: the submaps are
unchanged, a repeated call is bit-identical, and graph-replayed mapper steps neither re-capture nor change when assemblies run between them."""
import copy
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from oracle_backend_assembly import PALETTE, colored
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W

pytestmark = pytest.mark.gpu

SCAN_TILE = 4096      # SCAN_TILE of runtime.cu (the batched scan)
AS_THREADS = 256      # K-assemble's CTA
BASE_TILE = 1024      # AS_BASE_THREADS: the per-submap totals are scanned 1024 at a time


def bits(a):
    return None if a is None else np.ascontiguousarray(a).view(np.uint64)


def same(a, b):
    return (a is None and b is None) or (a is not None and b is not None and a.shape == b.shape and np.array_equal(bits(a), bits(b)))


def composition(sms):
    """b2s_submap_to_cloud of every submap, concatenated in order (normals as stored, NaN for a map without)"""
    xs, ns = [], []
    for s in sms:
        c = s.toCloud()
        x, n = c.download()
        xs.append(x); ns.append(n)
        c.free()
    return np.concatenate(xs) if xs else np.zeros((0, 3)), (np.concatenate(ns) if ns else np.zeros((0, 3))), xs


def keyed(x, *cols):
    o = np.lexsort(x.T[::-1])
    return (x[o],) + tuple(None if c is None else c[o] for c in cols)


def submap_from(eng, xyz, nrm=None, capacity=None):
    sm = E.Submap(eng, capacity or max(len(xyz), 16))
    c = eng.cloud(xyz, nrm)
    sm.setMapPointCloud(c)
    c.free()
    return sm


@pytest.fixture(scope="module")
def lap():
    """the closed lap through SegmentMapper on the device: carving on (tombstones from fusion, carved points), 2 m submaps so that the
    palette wraps (at least 13 submaps)"""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=False, graph=True)
    md = S.SegmentMapper(dev, S.SubmapParameters(radius=2.0))
    for k in range(140):
        md.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    assert len(md.submaps.submaps) >= 13
    assert sum(dev.counters(s.handle)["carved_points_total"] for s in md.submaps.submaps) > 0
    yield dev, md
    dev.close()


def check_parity(dev, sms):
    cx, cn, _ = composition(sms)
    c = E.getAssembledMapPointCloud(dev.eng, sms)
    x, n = c.download()
    assert same(x, cx) and same(n, cn) and len(x) > 100_000
    return cx, cn


def test_parity_with_the_composition_before_and_after_a_loop_closure(lap):
    dev, md = lap
    sms = [s.handle for s in md.submaps.submaps]
    before, _ = check_parity(dev, sms)
    assert md.getAssembledMapPointCloud().size()[0] == len(before) == md.submaps.getTotalNumPoints()
    sc = md.submaps
    src = max(sc.finishedSubmapsIdxs)
    T = np.eye(4); T[:3, 3] = [0.05, -0.03, 0.0]
    lc = S.Constraint(T, src, 0, np.eye(6) * 1e3)
    S.loopClosureCycle(dev, md, S.OptimizationProblem(dev), [lc])
    after, _ = check_parity(dev, sms)
    assert len(after) == len(before) and not np.array_equal(after, before)


def oracle_check(eng, sms, voxel):
    cx, cn, _ = composition(sms)
    g = E.getAssembledMapPointCloud(eng, sms, voxel)
    gx, gn = g.download()
    ox, on = O.voxel_down_sample(cx, voxel, cn)
    assert gx.shape == ox.shape and g.HasNormals()
    a, an = keyed(gx, gn)
    b, bn = keyed(ox, on)
    assert np.array_equal(a, b) and np.array_equal(an, bn)   # the same voxels, members summed in the same order: bit-identical


@pytest.mark.parametrize("voxel", [0.1, 0.25, 1.0])
def test_voxelized_against_the_oracle(lap, voxel):
    dev, md = lap
    oracle_check(dev.eng, [s.handle for s in md.submaps.submaps], voxel)


def test_voxelized_5_km_from_the_origin(lap):
    dev, md = lap
    eng = dev.eng
    far = []
    for s in md.submaps.submaps[:6]:
        x, n = s.handle.getMapPointCloud()
        far.append(submap_from(eng, x + np.array([5000.0, -3000.0, 40.0]), n))
    for v in (0.1, 1.0):
        oracle_check(eng, far, v)


@pytest.mark.parametrize("voxel", [0.0, 0.25, 1.0])
def test_coloured_map(lap, voxel):
    dev, md = lap
    sms = [s.handle for s in md.submaps.submaps]
    assert len(sms) >= 13
    _cx, _cn, parts = composition(sms)
    c, rgb = md.assembleColoredPointCloud(voxel)
    x, n = c.download()
    assert n is None and not c.HasNormals() and len(rgb) == len(x)
    rx, rrgb = colored([(p, None) for p in parts], voxel)
    if voxel <= 0.0:
        assert same(x, rx) and same(rgb, rrgb)
        return
    a, argb = keyed(x, rgb)
    b, brgb = keyed(rx, rrgb)
    assert np.array_equal(a, b) and np.array_equal(argb, brgb)
    assert (np.unique(rrgb, axis=0).shape[0] > 11)              # voxels shared by submaps of different colours


@pytest.fixture(scope="module")
def p2p():
    eng = E.Engine(E.MapperParameters(scanToMapRegType="PointToPointIcp"))
    rng = np.random.default_rng(7)
    mk = lambda n, off, normals=True: submap_from(eng, rng.uniform(-3, 3, (n, 3)) + off,
                                                  (lambda v: v / np.linalg.norm(v, axis=1, keepdims=True))(rng.normal(size=(n, 3))) if normals else None)
    subs = {"a": mk(3000, 0.0), "b": mk(2000, 2.0), "p": mk(1500, 1.0, normals=False), "e": mk(0, 0.0), "ep": mk(0, 0.0, normals=False)}
    yield eng, subs
    eng.close()


def test_normals_rule(p2p):
    eng, s = p2p
    assert E.getAssembledMapPointCloud(eng, [s["a"], s["b"]]).HasNormals()
    assert E.getAssembledMapPointCloud(eng, [s["a"], s["ep"], s["b"]]).HasNormals()   # an empty map without normals contributes nothing
    for sms in ([s["a"], s["p"], s["b"]], [s["p"]], [s["p"], s["ep"]]):
        for v in (0.0, 0.5):
            c = E.getAssembledMapPointCloud(eng, sms, v)
            x, n = c.download()
            assert n is None and len(x) > 0
    mixed = E.getAssembledMapPointCloud(eng, [s["a"], s["p"], s["b"]])
    cx, _cn, _ = composition([s["a"], s["p"], s["b"]])
    assert same(mixed.download()[0], cx)
    v = E.getAssembledMapPointCloud(eng, [s["a"], s["p"], s["b"]], 0.5).download()[0]
    assert same(keyed(v)[0], keyed(O.voxel_down_sample(cx, 0.5)[0])[0])


def test_empty_inputs_and_voxel_at_or_below_zero(p2p):
    eng, s = p2p
    for sms in ([], [s["e"]], [s["e"], s["ep"]]):
        for v in (0.0, 0.25):
            c = E.getAssembledMapPointCloud(eng, sms, v)
            assert c.size() == (0, False)
            cc, rgb = E.assembleColoredPointCloud(eng, sms, v)
            assert cc.size() == (0, False) and rgb.shape == (0, 3)
    sms = [s["e"], s["a"], s["e"], s["ep"], s["b"], s["e"]]   # empty maps interleaved with full ones
    cx, cn, _ = composition(sms)
    for v in (0.0, -1.0):
        x, n = E.getAssembledMapPointCloud(eng, sms, v).download()
        assert same(x, cx) and same(n, cn)
    one = E.getAssembledMapPointCloud(eng, [s["a"]]).download()
    assert same(one[0], composition([s["a"]])[0])
    oracle_check(eng, sms, 0.25)


def test_errors(p2p):
    eng, s = p2p
    lib = L.lib()
    out = E.Cloud(eng)
    arr = (C.c_void_p * 2)(s["a"]._s, None)
    assert lib.b2s_assemble_map(eng._h, C.c_int32(-1), arr, C.c_double(0.0), out._c) == L.E_INVALID
    assert lib.b2s_assemble_map(eng._h, C.c_int32(2), arr, C.c_double(0.0), out._c) == L.E_INVALID    # null entry
    other = E.Engine(E.MapperParameters(scanToMapRegType="PointToPointIcp"))
    foreign = submap_from(other, np.zeros((4, 3)))
    with pytest.raises(L.B2SError) as e:
        E.getAssembledMapPointCloud(eng, [s["a"], foreign])
    assert e.value.code == L.E_INVALID
    m = E.Mapper(eng, 1024)
    staging = m.enableGraph(1024)
    one = (C.c_void_p * 1)(s["a"]._s)
    assert lib.b2s_assemble_map(eng._h, C.c_int32(1), one, C.c_double(0.0), staging._c) == L.E_INVALID
    assert lib.b2s_assemble_colored_map(eng._h, C.c_int32(1), one, C.c_double(0.0), staging._c, None, C.c_size_t(0), None) == L.E_INVALID
    many = (C.c_void_p * (L.ASSEMBLY_MAX_SUBMAPS + 1))(*([s["e"]._s] * (L.ASSEMBLY_MAX_SUBMAPS + 1)))
    assert lib.b2s_assemble_map(eng._h, C.c_int32(L.ASSEMBLY_MAX_SUBMAPS + 1), many, C.c_double(0.0), out._c) == L.E_UNSUPPORTED
    # a colour buffer smaller than the output
    n = C.c_size_t()
    rgb = np.empty((10, 3))
    assert lib.b2s_assemble_colored_map(eng._h, C.c_int32(1), one, C.c_double(0.0), out._c, E._pd(rgb), C.c_size_t(10), C.byref(n)) == L.E_CAPACITY
    assert n.value == 3000
    # the 21-bit key limit: 2 points 100 km apart (inside the map-side key range) are 2.5 M voxels of 0.04 m, 10^5 voxels of 1 m
    wide = submap_from(eng, np.array([[0.0, 0.0, 0.0], [1.0e5, 0.0, 0.0]]), np.array([[0.0, 0.0, 1.0]] * 2))
    with pytest.raises(L.B2SError) as e:
        E.getAssembledMapPointCloud(eng, [wide], 0.04)
    assert e.value.code == L.E_INVALID
    assert E.getAssembledMapPointCloud(eng, [wide], 1.0).size()[0] == 2
    # the submaps are untouched by the failures and the handle goes on
    assert same(E.getAssembledMapPointCloud(eng, [s["a"]]).download()[0], composition([s["a"]])[0])
    other.close()


@pytest.fixture(scope="module")
def sizes():
    eng = E.Engine()
    rng = np.random.default_rng(11)
    made = {}
    for m in (0, 1, AS_THREADS - 1, AS_THREADS, AS_THREADS + 1, SCAN_TILE - 1, SCAN_TILE, SCAN_TILE + 1):
        made[m] = submap_from(eng, rng.uniform(-5, 5, (m, 3)), rng.normal(size=(m, 3)))
    yield eng, made
    eng.close()


@pytest.mark.parametrize("m", [0, 1, AS_THREADS - 1, AS_THREADS, AS_THREADS + 1, SCAN_TILE - 1, SCAN_TILE, SCAN_TILE + 1])
def test_map_sizes(sizes, m):
    eng, made = sizes
    sms = [made[m], made[1], made[m]]
    cx, cn, _ = composition(sms)
    x, n = E.getAssembledMapPointCloud(eng, sms).download()
    assert same(x, cx) and same(n, cn) and len(x) == 2 * m + 1


@pytest.mark.parametrize("count", [1, 2, BASE_TILE - 1, BASE_TILE, BASE_TILE + 1, 2 * BASE_TILE + 1, L.ASSEMBLY_MAX_SUBMAPS])
def test_submap_counts(sizes, count):
    eng, made = sizes
    cycle = [made[0], made[1], made[AS_THREADS + 1]]
    sms = [cycle[k % 3] for k in range(count)]
    parts = [composition([c])[0] for c in cycle]
    ref = np.concatenate([parts[k % 3] for k in range(count)])
    x, n = E.getAssembledMapPointCloud(eng, sms).download()
    assert same(x, ref)
    c, rgb = E.assembleColoredPointCloud(eng, sms)
    lab = np.concatenate([np.full(len(parts[k % 3]), k % 11) for k in range(count)])
    assert same(c.download()[0], ref) and same(rgb, PALETTE[lab])


def test_more_than_2_24_points(sizes):
    eng, _ = sizes
    rng = np.random.default_rng(5)
    m = 5_700_000
    big = submap_from(eng, rng.uniform(-100, 100, (m, 3)), rng.normal(size=(m, 3)))
    sms = [big, big, big]                                          # 17.1 M > 2^24 points
    part = composition([big])[0]
    x, _n = E.getAssembledMapPointCloud(eng, sms).download()
    assert len(x) == 3 * m > (1 << 24) and same(x, np.concatenate([part] * 3))
    del x
    gx, gn = E.getAssembledMapPointCloud(eng, sms, 0.5).download()
    cx, cn, _ = composition(sms)
    ox, on = O.voxel_down_sample(cx, 0.5, cn)
    a, an = keyed(gx, gn); b, bn = keyed(ox, on)
    assert np.array_equal(a, b) and np.array_equal(an, bn)


def test_no_side_effects_and_repeatable(lap):
    dev, md = lap
    sms = [s.handle for s in md.submaps.submaps]
    before = [s.getMapPointCloud() for s in sms]
    r1 = E.getAssembledMapPointCloud(dev.eng, sms, 0.1).download()
    c1, rgb1 = E.assembleColoredPointCloud(dev.eng, sms, 0.1)
    r2 = E.getAssembledMapPointCloud(dev.eng, sms, 0.1).download()
    c2, rgb2 = E.assembleColoredPointCloud(dev.eng, sms, 0.1)
    assert same(r1[0], r2[0]) and same(r1[1], r2[1]) and same(c1.download()[0], c2.download()[0]) and same(rgb1, rgb2)
    after = [s.getMapPointCloud() for s in sms]
    for (a, an), (b, bn) in zip(before, after):
        assert same(a, b) and same(an, bn)


def test_graph_replayed_steps_do_not_recapture():
    """mapper steps replayed from their CUDA graph, with an assembly of the growing map after every step: no capture beyond the run
    without assemblies, and the same step results"""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    runs = []
    for with_assembly in (False, True):
        dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=True)
        md = S.SegmentMapper(dev, S.SubmapParameters(radius=1000.0))
        caps, res = [], []
        for k in range(40):
            r = md.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
            if with_assembly:
                sms = [s.handle for s in md.submaps.submaps]
                E.getAssembledMapPointCloud(dev.eng, sms, 0.1)
                E.assembleColoredPointCloud(dev.eng, sms, 0.1)
                E.getAssembledMapPointCloud(dev.eng, sms)
            caps.append(dev.eng.graphCaptures)
            res.append(None if r is None else (np.array(r.transformation_), r.fitness_, r.inlier_rmse_))
        runs.append((caps, res))
        dev.close()
    (c0, r0), (c1, r1) = runs
    assert c1 == c0 and c1[-1] >= 1
    # two runs of the chain agree to the last bits only up to the ICP's run-to-run freedom (which CTA drains which phase-2 entry)
    for a, b in zip(r0, r1):
        assert (a is None and b is None) or (np.abs(a[0] - b[0]).max() <= 1e-9 and abs(a[1] - b[1]) <= 1e-9 and abs(a[2] - b[2]) <= 1e-9)
