"""GPU: b2s_assemble_dense_maps (VoxelizedPointCloud::toPointCloud of every submap's dense map: SubmapCollection::dumpToFile(.., true),
publishDenseMap; DESIGN.md row A2) -- bit-identical to concatenating b2s_submap_dense_download on the closed lap with dense carving, after
denseRemove / denseClear and after a loop-closure correction, and in agreement with the oracle's dense maps; slot order at the count and
gather kernels' tile edges and across the end of the table; the job-count edges of the batched scan and the job-total scan; the capacity
limit and a total above 2^24; the errors; and no side effects: the dense maps are unchanged, a repeated call is bit-identical, and
graph-replayed mapper steps neither re-capture nor change when exports run between them."""
import copy
import ctypes as C

import numpy as np
import pytest

import voxel_hash as VH
from oracle_backend_dense_export import DenseExportOracleBackend, dense_cloud
from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W

pytestmark = pytest.mark.gpu

DX_TILE = 2048        # slots per CTA of the count and gather kernels (AS_THREADS x DX_ITEMS, assemble.cu)
DX_ITEMS = 8          # consecutive slots per thread
BASE_TILE = 1024      # AS_BASE_THREADS: the per-entry totals are scanned 1024 at a time
DV = 0.05             # the default dense voxel (denseMapVoxelSize)
SLOTS = VH.DENSE_SLOTS
MAX_POINTS = 0x7FFFFFFF // 3


def bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def same(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def translation(t):
    T = np.eye(4); T[:3, 3] = t
    return T


T_INS = translation([0.5, -0.25, 0.125])   # not near identity: every point lands once (no duplication quirk)


def export(eng, sms, out=None):
    c, off = E.assembleDenseMaps(eng, sms, out)
    x, n = c.download()
    assert n is None and not c.HasNormals()
    return x, off


def check_export(eng, sms):
    """the export equals the concatenated dense downloads bit for bit, and its offsets are their cumulative sizes"""
    parts = [s.getDenseMap() for s in sms]
    x, off = export(eng, sms)
    ref = np.concatenate([p[0] for p in parts]) if parts else np.zeros((0, 3))
    assert same(x, ref)
    assert np.array_equal(off, np.r_[0, np.cumsum([len(p[0]) for p in parts])].astype(np.int64))
    return x, off, parts


def dense_submap(eng, xyz, T=T_INS):
    """a submap whose dense map holds the map-frame points xyz, inserted as raw points at the pose T"""
    sm = E.Submap(eng, 1000)
    raw = (np.asarray(xyz) - T[:3, 3]) @ T[:3, :3]
    c = eng.cloud(raw)
    sm.insertScanDenseMap(c, T, None)
    c.free()
    return sm


def grid(n, origin, width=100):
    """n points at the centres of n distinct dense voxels"""
    i = np.arange(n)
    k = np.c_[i % width, (i // width) % width, i // (width * width)] + np.asarray(origin)
    return (k + 0.5) * DV


# ----------------------------------------------------------------------------------------------------------------------
# the closed lap
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lap():
    """the closed lap through SegmentMapper on the device and on the oracle: dense map and carving on, 2 m submaps (at least 13)"""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=True)
    ora = DenseExportOracleBackend(copy.deepcopy(p), carving=True, dense=True)
    md, mo = S.SegmentMapper(dev, S.SubmapParameters(radius=2.0)), S.SegmentMapper(ora, S.SubmapParameters(radius=2.0))
    for k in range(140):
        md.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
        mo.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    assert len(md.submaps.submaps) >= 13
    cs = [dev.counters(s.handle) for s in md.submaps.submaps]
    assert sum(c["dense_carve_runs"] for c in cs) > 0 and sum(c["carved_voxels_total"] for c in cs) > 0
    yield dev, md, ora, mo
    dev.close()


def test_parity_on_the_closed_lap(lap):
    dev, md, ora, mo = lap
    eng = dev.eng
    sms = [s.handle for s in md.submaps.submaps]
    x0, off0, parts = check_export(eng, sms)
    assert len(x0) > 1_000_000
    # the SegmentMapper and Submap entry points are the same call
    per = md.getDenseSubmapPointClouds()
    assert len(per) == len(sms) and all(same(a, p[0]) for a, p in zip(per, parts))
    assert same(md.getActiveDenseMapPointCloud(), parts[md.submaps.activeSubmapIdx][0])
    assert same(sms[3].getDenseMapPointCloud().download()[0], parts[3][0])

    # the oracle's dense maps, keyed by the keys the dense download returns
    assert len(mo.submaps.submaps) == len(sms)
    for k, (xo, (_x, gk)) in enumerate(zip(mo.getDenseSubmapPointClouds(), parts)):
        _ox, _on, ok = mo.submaps.submaps[k].handle.dense.to_cloud()
        gx = x0[off0[k]:off0[k + 1]]
        assert len(gx) == len(xo) == len(ok)
        q1 = np.lexsort(gk.T[::-1]); q2 = np.lexsort(ok.T[::-1])
        assert np.array_equal(gk[q1], ok[q2]) and np.abs(gx[q1] - xo[q2]).max() < 1e-8

    # voxels emptied by denseRemove and denseClear are skipped
    a, b = sms[0], sms[1]
    na = a.denseSize()
    a.denseRemove(eng.cloud(parts[0][0][:500]))
    b.denseClear()
    assert 0 < na - a.denseSize() <= 500 and b.denseSize() == 0
    x1, off1, parts1 = check_export(eng, sms)
    assert len(parts1[0][0]) == a.denseSize() and off1[2] - off1[1] == 0 and len(x1) < len(x0)

    # a loop-closure correction moves the sums (VoxelizedPointCloud::transform)
    sc = md.submaps
    T = np.eye(4); T[:3, 3] = [0.05, -0.03, 0.0]
    S.loopClosureCycle(dev, md, S.OptimizationProblem(dev), [S.Constraint(T, max(sc.finishedSubmapsIdxs), 0, np.eye(6) * 1e3)])
    x2, off2, _ = check_export(eng, sms)
    assert np.array_equal(off2, off1) and not np.array_equal(x2, x1)


def test_no_side_effects_and_repeatable(lap):
    dev, md, _ora, _mo = lap
    sms = [s.handle for s in md.submaps.submaps]
    before = [s.getDenseMap() for s in sms]
    x1, off1 = export(dev.eng, sms)
    x2, off2 = export(dev.eng, sms)
    assert same(x1, x2) and np.array_equal(off1, off2)
    for (a, ak), (b, bk) in zip(before, [s.getDenseMap() for s in sms]):
        assert same(a, b) and np.array_equal(ak, bk)


# ----------------------------------------------------------------------------------------------------------------------
# table edges: home slots at the tile boundaries of the count and gather kernels, and a probe run across the end of the table
# ----------------------------------------------------------------------------------------------------------------------
EDGE_SLOTS = sorted({0, 1, DX_ITEMS - 1, DX_ITEMS, 255, 256, DX_TILE - 1, DX_TILE, DX_TILE + 1, 2 * DX_TILE - 1, 2 * DX_TILE,
                     SLOTS - DX_TILE - 1, SLOTS - DX_TILE, SLOTS - DX_TILE + 1, SLOTS - 2, SLOTS - 1})


def two_points_each(keys):
    """two points inside every voxel (counts of 2, means that are not the points)"""
    c = np.array([VH.point_in(k, DV) for k in keys])
    return np.vstack([c - 0.011, c + 0.007])


@pytest.fixture(scope="module")
def edges():
    eng = E.Engine()
    edge_keys = [VH.keys_homed_at(s, SLOTS, 1, seed=s)[0] for s in EDGE_SLOTS]
    wrap_keys = VH.keys_homed_at(SLOTS - 1, SLOTS, 3, seed=1) + VH.keys_homed_at(2, SLOTS, 1, seed=2)
    subs = {"edge": dense_submap(eng, two_points_each(edge_keys)), "wrap": dense_submap(eng, two_points_each(wrap_keys)),
            "none": E.Submap(eng, 16), "small": dense_submap(eng, grid(300, (-40, 20, 3)))}
    yield eng, subs, edge_keys, wrap_keys
    eng.close()


def homes(keys):
    return [VH.home(tuple(int(v) for v in k), SLOTS) for k in keys]


def test_slot_order_at_the_tile_edges_and_across_the_end(edges):
    eng, s, edge_keys, wrap_keys = edges
    x, off, parts = check_export(eng, [s["edge"], s["wrap"], s["none"], s["edge"]])
    ex, ek = parts[0]
    assert len(ex) == len(EDGE_SLOTS) and homes(ek) == EDGE_SLOTS          # one voxel per chosen slot, in slot order
    wx, wk = parts[1]
    # three keys homed at the last slot take it and wrap to slots 0 and 1; the key homed at slot 2 follows them
    assert homes(wk) == [SLOTS - 1, SLOTS - 1, 2, SLOTS - 1]
    assert tuple(wk[2]) == tuple(wrap_keys[3]) and {tuple(k) for k in wk} == {tuple(k) for k in wrap_keys}
    counts, means = s["edge"].denseQuery(eng.cloud(ex))
    assert np.array_equal(counts, [2] * len(ex)) and same(means, ex)
    assert same(x[off[3]:off[4]], ex) and off[3] - off[2] == 0


# ----------------------------------------------------------------------------------------------------------------------
# job counts: the batched scan and the job-total scan over many entries
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count", [1, BASE_TILE, BASE_TILE + 1, 2 * BASE_TILE + 1])
def test_entry_counts(edges, count):
    eng, s, _, _ = edges
    small, none = s["small"], s["none"]
    part = small.getDenseMap()[0]
    x, off = export(eng, [small] * count)
    assert same(x, np.tile(part, (count, 1))) and np.array_equal(off, np.arange(count + 1) * len(part))
    mixed = [small if k % 3 != 1 else none for k in range(count)]
    x, off = export(eng, mixed)
    sizes = [len(part) if m is small else 0 for m in mixed]
    assert same(x, np.tile(part, (sum(m is small for m in mixed), 1))) and np.array_equal(off, np.r_[0, np.cumsum(sizes)])


def test_entry_limit(edges):
    eng, s, _, _ = edges
    small, none = s["small"], s["none"]
    part = small.getDenseMap()[0]
    n = L.ASSEMBLY_MAX_SUBMAPS
    sms = [small if k % 4096 == 7 or k == n - 1 else none for k in range(n)]
    x, off = export(eng, sms)
    m = sum(sm is small for sm in sms)
    assert same(x, np.tile(part, (m, 1)))
    assert np.array_equal(off, np.r_[0, np.cumsum([len(part) if sm is small else 0 for sm in sms])])
    with pytest.raises(L.B2SError) as e:
        E.assembleDenseMaps(eng, sms + [none])
    assert e.value.code == L.E_UNSUPPORTED


# ----------------------------------------------------------------------------------------------------------------------
# capacity: more than (2^31 - 1) / 3 points in total, and a total above 2^24
# ----------------------------------------------------------------------------------------------------------------------
def test_capacity(edges):
    eng, s, _, _ = edges
    big = dense_submap(eng, grid(1_000_000, (-50, -50, -20)))
    assert big.denseSize() == 1_000_000 and 716 * 1_000_000 > MAX_POINTS >= 715 * 1_000_000
    part = big.getDenseMap()[0]
    out = eng.cloud(np.arange(12.0).reshape(4, 3))
    offsets = np.full(717, -7, dtype=np.int64)
    arr = (C.c_void_p * 716)(*([big._s] * 716))
    assert L.lib().b2s_assemble_dense_maps(eng._h, C.c_int32(716), arr, out._c, offsets.ctypes.data_as(C.POINTER(C.c_int64))) == L.E_CAPACITY
    assert same(out.download()[0], np.arange(12.0).reshape(4, 3)) and np.all(offsets == -7)   # nothing written
    x, off = export(eng, [big] * 17, out)                                                    # 17 M > 2^24 points
    assert len(x) == 17_000_000 > (1 << 24) and np.array_equal(off, np.arange(18) * 1_000_000)
    assert all(same(x[k * 1_000_000:(k + 1) * 1_000_000], part) for k in (0, 8, 16))
    del x
    big.free()


# ----------------------------------------------------------------------------------------------------------------------
# errors
# ----------------------------------------------------------------------------------------------------------------------
def test_errors_and_empty_input(edges):
    eng, s, _, _ = edges
    lib = L.lib()
    out = E.Cloud(eng)
    offsets = np.full(3, -7, dtype=np.int64)
    po = offsets.ctypes.data_as(C.POINTER(C.c_int64))
    arr = (C.c_void_p * 2)(s["small"]._s, None)
    assert lib.b2s_assemble_dense_maps(eng._h, C.c_int32(-1), arr, out._c, po) == L.E_INVALID
    assert lib.b2s_assemble_dense_maps(eng._h, C.c_int32(2), arr, out._c, po) == L.E_INVALID      # null entry
    other = E.Engine()
    foreign = dense_submap(other, grid(10, (0, 0, 0)))
    with pytest.raises(L.B2SError) as e:
        E.assembleDenseMaps(eng, [s["small"], foreign])
    assert e.value.code == L.E_INVALID
    with pytest.raises(L.B2SError) as e:
        E.assembleDenseMaps(eng, [s["small"]], E.Cloud(other))                                     # output of another handle
    assert e.value.code == L.E_INVALID
    m = E.Mapper(eng, 1024)
    staging = m.enableGraph(1024)
    one = (C.c_void_p * 1)(s["small"]._s)
    assert lib.b2s_assemble_dense_maps(eng._h, C.c_int32(1), one, staging._c, po) == L.E_INVALID
    many = (C.c_void_p * (L.ASSEMBLY_MAX_SUBMAPS + 1))(*([s["none"]._s] * (L.ASSEMBLY_MAX_SUBMAPS + 1)))
    assert lib.b2s_assemble_dense_maps(eng._h, C.c_int32(L.ASSEMBLY_MAX_SUBMAPS + 1), many, out._c, po) == L.E_UNSUPPORTED
    assert np.all(offsets == -7)
    # empty inputs: no entries, or only entries without a dense map; NULL offsets
    for sms in ([], [s["none"]], [s["none"]] * 3):
        c, off = E.assembleDenseMaps(eng, sms)
        assert c.size() == (0, False) and np.array_equal(off, np.zeros(len(sms) + 1, dtype=np.int64))
    assert lib.b2s_assemble_dense_maps(eng._h, C.c_int32(1), one, out._c, None) == L.OK
    assert same(out.download()[0], s["small"].getDenseMap()[0])
    other.close()


# ----------------------------------------------------------------------------------------------------------------------
# exports between graph-replayed mapper steps
# ----------------------------------------------------------------------------------------------------------------------
def test_graph_replayed_steps_do_not_recapture():
    """mapper steps replayed from their CUDA graph with the dense map on, with an export of the growing dense maps after every step:
    no capture beyond the run without exports, and the same step results"""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    runs = []
    for with_export in (False, True):
        dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=True)
        md = S.SegmentMapper(dev, S.SubmapParameters(radius=1000.0))
        caps, res, sizes = [], [], []
        for k in range(40):
            r = md.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
            if with_export:
                sizes.append(sum(len(a) for a in md.getDenseSubmapPointClouds()))
                md.getActiveDenseMapPointCloud()
            caps.append(dev.eng.graphCaptures)
            res.append(None if r is None else (np.array(r.transformation_), r.fitness_, r.inlier_rmse_))
        runs.append((caps, res))
        if with_export:
            assert sizes[-1] > max(sizes[:5]) and sizes[-1] > 0     # the first scan feeds no dense map; later ones grow it
        dev.close()
    (c0, r0), (c1, r1) = runs
    assert c1 == c0 and c1[-1] >= 1
    # two runs of the chain agree to the last bits only up to the ICP's run-to-run freedom (which CTA drains which phase-2 entry)
    for a, b in zip(r0, r1):
        assert (a is None and b is None) or (np.abs(a[0] - b[0]).max() <= 1e-9 and abs(a[1] - b[1]) <= 1e-9 and abs(a[2] - b[2]) <= 1e-9)
