"""GPU: session state (b2s_submaps_export_state / b2s_submap_import_state / b2s_odometry_*_state, DESIGN.md row A3).  On the closed lap
with sparse and dense carving, plus a loop-closure-corrected submap, submaps after denseRemove / denseClear, one never fed a dense scan,
an empty one, a point-to-point map and a merge-off localisation map: an import on a fresh handle and on a second handle downloads,
assembles (A1, A2), counts and boxes exactly like the original, and re-exports to the same bytes.  The same for an odometry object.
The same host-driven insert / carve / dense insert / dense carve sequence continues the original and the import alike, and so do 20
more mapper and slam steps, eager and graph-replayed, with one capture after the import.  Every validation rule refuses its blob with
B2S_E_INVALID and leaves the handle usable, and exports between graph-replayed steps capture nothing."""
import copy
import ctypes as C

import numpy as np
import pytest

from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W

pytestmark = pytest.mark.gpu

MS_NINS, MS_DUPSEL, MS_NDUP, MS_NTOUCHED, MS_WSEL, MS_NW = 5, 19, 20, 18, 24, 25


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def same(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def bbox(eng, sm):
    box = np.zeros(6)
    L.check(L.lib().b2s_debug_submap_bbox(eng._h, sm._s, box.ctypes.data_as(C.POINTER(C.c_double))))
    return box


def snapshot(eng, sm):
    """everything a later reader sees of a submap"""
    xyz, nrm = sm.getMapPointCloud()
    dx, dk = sm.getDenseMap()
    return dict(xyz=xyz, nrm=nrm, dx=dx, dk=dk, pose=sm.getPose(), counters=sm.mapperCounters(), box=bbox(eng, sm), size=sm.size(),
                dsize=sm.denseSize())


def assert_same_snapshot(a, b):
    for k in ("xyz", "nrm", "dx", "dk", "pose", "box"):
        assert same(a[k], b[k]), k
    assert a["counters"] == b["counters"] and a["size"] == b["size"] and a["dsize"] == b["dsize"]


def translation(t):
    T = np.eye(4); T[:3, 3] = t
    return T


def rot_z(a, t=(0.0, 0.0, 0.0)):
    T = translation(t); c, s = np.cos(a), np.sin(a)
    T[:2, :2] = [[c, -s], [s, c]]
    return T


@pytest.fixture(scope="module")
def lap():
    """the closed lap through SegmentMapper on the device (sparse and dense carving, graph replay, 2 m submaps) and the special submaps"""
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=True)
    md = S.SegmentMapper(dev, S.SubmapParameters(radius=2.0))
    for k in range(100):
        md.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    sms = [s.handle for s in md.submaps.submaps]
    assert len(sms) >= 8
    eng = dev.eng
    sms[1].transform(rot_z(0.05, (0.3, -0.2, 0.01)))                       # a loop-closure correction
    probe = eng.cloud(sms[2].getDenseMap()[0][::3])
    sms[2].denseRemove(probe)                                              # count-0 keys left behind
    sms[3].denseClear()
    sparse_only = E.Submap(eng, 50_000)                                    # never fed a dense scan
    raw = eng.cloud(np.ascontiguousarray(lp.scan(5, seed=5), dtype=np.float32))
    ps = dev.mapper.scan2MapReg_.processForScanMatchingAndMerging(raw)
    sparse_only.insertScan(raw, ps.merge_, translation([0.2, 0.1, 0.0]))
    empty = E.Submap(eng, 1000)
    loc = E.Submap(eng, 400_000)                                           # a merge-off localisation map from setInitialMap
    xyz, nrm = sms[0].getMapPointCloud()
    loc.setInitialMap(eng.cloud(xyz, nrm), 0.1)
    loc.setMergeScans(False)
    # a point-to-point map (no normals) on a handle of the same map voxel size
    p2p = E.Engine(E.MapperParameters(seed=3, scanToMapRegType="PointToPointIcp"))
    nn = E.Submap(p2p, 100_000)
    nn.setMapPointCloud(p2p.cloud(xyz[::2]))
    nn.insertScan(None, p2p.cloud(lp.scan(6, seed=6).astype(np.float64)[:4000]), translation([0.1, 0.0, 0.0]))
    yield dict(dev=dev, md=md, lp=lp, eng=eng, sms=sms, extra=[sparse_only, empty, loc], p2p=p2p, nn=nn)
    dev.close()


def test_round_trip_bit_for_bit(lap):
    eng, sms, extra = lap["eng"], lap["sms"], lap["extra"]
    listed = sms + extra
    before = [snapshot(eng, s) for s in listed]
    caps = eng.graphCaptures
    blobs = E.exportSubmapStates(eng, listed)
    assert E.exportSubmapStates(eng, listed) == blobs                      # export only reads: byte-identical, nothing re-captured
    assert eng.graphCaptures == caps
    for s, b in zip(listed, before):
        assert_same_snapshot(snapshot(eng, s), b)
    hdr = [E.parseStateHeader(b) for b in blobs]
    assert all(h.kind == "submap" and h.total_bytes == len(b) for h, b in zip(hdr, blobs))
    assert hdr[-3].params["dense_cap"] == 0 and hdr[-2].params["vcap"] == 0 and hdr[-1].params["flags"] & L.STATE_F_MERGE_SCANS == 0
    assert hdr[2].section(blobs[2], "dense", "dense")["count"].min() == 0   # the keys denseRemove emptied travel with the blob
    a1 = E.getAssembledMapPointCloud(eng, listed).download()
    a2x, a2o = E.assembleDenseMaps(eng, listed)
    a2 = a2x.download()[0]
    for other in (E.Engine(E.MapperParameters(seed=3)), E.Engine(E.MapperParameters(seed=9))):
        imp = [E.importSubmapState(other, b) for b in blobs]
        for s, b in zip(imp, before):
            assert_same_snapshot(snapshot(other, s), b)
        assert E.exportSubmapStates(other, imp) == blobs
        b1 = E.getAssembledMapPointCloud(other, imp).download()
        assert same(b1[0], a1[0]) and a1[1] is not None and same(b1[1], a1[1])
        bx, bo = E.assembleDenseMaps(other, imp)
        assert same(bx.download()[0], a2) and np.array_equal(bo, a2o)
        assert [s.nScansInsertedMap_ for s in imp] == [s.mapperCounters()["inserted_map"] for s in listed]
    # the point-to-point map, on its own handle
    p2p, nn = lap["p2p"], lap["nn"]
    ref = snapshot(p2p, nn)
    blob = E.exportSubmapStates(p2p, [nn])[0]
    assert E.parseStateHeader(blob).params["flags"] & L.STATE_F_NO_NORMALS
    back = E.importSubmapState(E.Engine(E.MapperParameters(seed=3, scanToMapRegType="PointToPointIcp")), blob)
    assert_same_snapshot(snapshot(back.eng, back), ref)


def test_odometry_round_trip(lap):
    lp = lap["lp"]
    dev = S.DeviceBackend(E.MapperParameters(seed=3), carving=True, dense=True, graph=False)
    sm = dev.new_submap()
    dev.first_scan_with_odometry(sm, lp.scan(0, seed=0), 0)
    for k in range(1, 12):
        dev.step_with_odometry(sm, lp.scan(k, seed=k), k * 1_000_000)
    od = dev.odometry()
    blob = od.exportState()
    assert od.exportState() == blob
    for eng in (E.Engine(E.MapperParameters(seed=3)), E.Engine(E.MapperParameters(seed=5))):
        back = E.DeviceLidarOdometry.importState(eng, blob)
        assert back.exportState() == blob
        for t in (0, 3_500_000, 11_000_000, 20_000_000):
            assert same(back._lookup(t)[0], od._lookup(t)[0]) and back._lookup(t)[1] == od._lookup(t)[1]
            assert same(back._map_lookup(t)[0], od._map_lookup(t)[0]) and back._map_lookup(t)[1] == od._map_lookup(t)[1]
        assert same(back.getPreProcessedCloud().download()[0], od.getPreProcessedCloud().download()[0])
    dev.close()


def test_deterministic_continuation(lap):
    """the same host-driven F1 / C1 / F3 / C2 sequence at fixed poses on the original and on the import.  Fusion assigns the slots of
    new voxels in arrival order, so the maps are compared as sets of rows (bit for bit); the dense sums are atomics in arrival order, so
    the dense means agree to rounding and the keys and counts exactly."""
    eng, dev, lp, sms = lap["eng"], lap["dev"], lap["lp"], lap["sms"]
    other = E.Engine(E.MapperParameters(seed=3))
    prm = eng.params.mapBuilder.carving
    raw_xyz = np.ascontiguousarray(lp.scan(40, seed=40), dtype=np.float32)
    merge = E.ScanToMapIcp(other).processForScanMatchingAndMerging(other.cloud(raw_xyz)).merge_.download()   # one pre-processed scan for both
    for src in (sms[1], sms[-1]):
        blob = E.exportSubmapStates(eng, [src])[0]
        orig = E.importSubmapState(eng, blob)                              # a twin on the same handle, so the lap itself stays as it is
        imp = E.importSubmapState(other, blob)
        T = src.getPose() @ rot_z(0.02, (0.15, 0.05, 0.0))
        for sm, e in ((orig, eng), (imp, other)):
            raw = e.cloud(raw_xyz)
            sm.carve(raw, T, prm, force=True)
            sm.insertScan(raw, e.cloud(*merge), T)
            sm.insertScanDenseMap(raw, T, None)
            sm.carveDenseMap(raw, T[:3, 3], prm)
        a, b = snapshot(eng, orig), snapshot(other, imp)
        ra = np.c_[bits(a["xyz"]), bits(a["nrm"])]; rb = np.c_[bits(b["xyz"]), bits(b["nrm"])]
        ra, rb = ra[np.lexsort(ra.T[::-1])], rb[np.lexsort(rb.T[::-1])]
        assert ra.shape == rb.shape and np.array_equal(ra, rb), (ra.shape, rb.shape, int((ra != rb).any(axis=1).sum()) if ra.shape == rb.shape else -1)
        qa, qb = np.lexsort(a["dk"].T[::-1]), np.lexsort(b["dk"].T[::-1])
        assert np.array_equal(a["dk"][qa], b["dk"][qb]) and np.abs(a["dx"][qa] - b["dx"][qb]).max() < 1e-9
        assert a["counters"] == b["counters"] and same(a["pose"], b["pose"]) and a["size"] == b["size"]


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("chain", ["mapper", "slam"])
def test_chain_continuation(lap, chain, graph):
    """20 more scans through b2s_mapper_step_* / b2s_slam_step_* on the original and on the import: the same decisions and iteration
    counts, transforms within the ICP's launch-to-launch last-bit variation (1e-8); after the import the chain captures once"""
    lp = lap["lp"]
    p = E.MapperParameters(seed=3)

    def run(be, sm, ks):
        out = []
        for k in ks:
            if chain == "slam":
                r, acc = be.step_with_odometry(sm, lp.scan(k, seed=k), k * 1_000_000)
            else:
                r, acc = be.step(sm, lp.scan(k, seed=k), lp.delta(k))
            out.append((acc, r.iters, r.transformation_.copy(), r.fitness_))
        return out

    a = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=graph)
    sm = a.new_submap()
    if chain == "slam":
        a.first_scan_with_odometry(sm, lp.scan(0, seed=0), 0)
    else:
        a.first_scan(sm, lp.scan(0, seed=0))
    run(a, sm, range(1, 10))
    caps_a = a.eng.graphCaptures
    blob = a.export_submaps([sm])[0]
    oblob = a.export_odometry() if chain == "slam" else None
    b = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=graph)
    sm2 = b.import_submap(blob)
    if oblob is not None:
        b.import_odometry(oblob)
    caps_b = b.eng.graphCaptures
    ra, rb = run(a, sm, range(10, 30)), run(b, sm2, range(10, 30))
    for (acc1, it1, T1, f1), (acc2, it2, T2, f2) in zip(ra, rb):
        assert acc1 == acc2 and it1 == it2
        assert np.abs(T1 - T2).max() < 1e-8 and abs(f1 - f2) < 1e-8
    if graph:
        assert a.eng.graphCaptures == caps_a                               # the export dropped nothing
        assert b.eng.graphCaptures == caps_b + 1                           # the import's first graph step captured once
    assert sm.mapperCounters() == sm2.mapperCounters()
    a.close(); b.close()


def test_exports_between_graph_steps_capture_nothing(lap):
    lp = lap["lp"]
    be = S.DeviceBackend(E.MapperParameters(seed=3), carving=True, dense=True, graph=True)
    sm = be.new_submap()
    be.first_scan_with_odometry(sm, lp.scan(0, seed=0), 0)
    for k in range(1, 6):
        be.step_with_odometry(sm, lp.scan(k, seed=k), k * 1_000_000)
    caps = be.eng.graphCaptures
    for k in range(6, 12):
        be.export_submaps([sm]); be.export_odometry()
        be.step_with_odometry(sm, lp.scan(k, seed=k), k * 1_000_000)
    assert be.eng.graphCaptures == caps
    be.close()


# ---- refusals ---------------------------------------------------------------------------------------------------------------------------
def refuse(eng, blob, what, odometry=False):
    out = C.c_void_p()
    fn = L.lib().b2s_odometry_import_state if odometry else L.lib().b2s_submap_import_state
    rc = fn(eng._h, bytes(blob), C.c_size_t(len(blob)), C.byref(out))
    assert rc == L.E_INVALID and not out.value, (what, rc, L.lib().b2s_last_error())
    # the handle stays usable: a registration still succeeds
    src = np.random.default_rng(0).uniform(-1, 1, (500, 3))
    tgt = eng.cloud(src, np.tile([0.0, 0.0, 1.0], (500, 1)))
    r = E.RegistrationIcpPointToPlane(eng).registerClouds(eng.cloud(src), tgt, np.eye(4))
    assert r.fitness_ > 0.99


def patched(blob, name, index, value, dtype="<i4", field=None):
    b = bytearray(blob)
    h = E.parseStateHeader(bytes(b))
    a = h.section(b, name, dtype)
    if field is None:
        a[index] = value
    else:
        a[field][index] = value
    return bytes(b)


def word(blob, k, value):
    b = bytearray(blob)
    np.frombuffer(b, dtype="<u8", count=32)[k] = value
    return bytes(b)


def test_refusals(lap):
    eng, sms = lap["eng"], lap["sms"]
    blob = E.exportSubmapStates(eng, [sms[-1]])[0]
    h = E.parseStateHeader(blob)
    p = h.params
    other = E.Engine(E.MapperParameters(seed=3))
    assert E.exportSubmapStates(other, [E.importSubmapState(other, blob)])[0] == blob
    vr = h.section(blob, "voxels", "voxels")
    live = np.flatnonzero(vr["head"] >= 0)
    cases = {
        "truncated": blob[:-8],
        "short header": blob[:100],
        "magic": word(blob, L.STATE_W_MAGIC, L.STATE_MAGIC_ODOMETRY),
        "version": word(blob, L.STATE_W_VERSION, 2),
        "byte order": word(blob, L.STATE_W_BYTE_ORDER, 0x0807060504030201),
        "total": word(blob, L.STATE_W_TOTAL_BYTES, len(blob) + 8) + bytes(8),
        "section length": word(blob, L.STATE_W_SECTIONS + 4, h.sections["map_xyz"][1] + 24),
        "dn above capacity": word(blob, L.STATE_W_PARAMS + 6, p["capacity"] + 1),
        "table size": word(blob, L.STATE_W_PARAMS + 1, p["vcap"] * 2),
        "record slot": patched(blob, "voxels", 0, p["vcap"], "voxels", "slot"),
        "negative slot": patched(blob, "voxels", 1, -5, "voxels", "slot"),
        "two records of a slot": patched(blob, "voxels", 1, int(vr["slot"][0]), "voxels", "slot"),
        "EMPTY key": patched(blob, "voxels", 2, 0xFFFFFFFFFFFFFFFF, "voxels", "key"),
        "dense slot": patched(blob, "dense", 0, p["dense_cap"], "dense", "slot"),
        "two dense records of a slot": patched(blob, "dense", 1, int(h.section(blob, "dense", "dense")["slot"][0]), "dense", "slot"),
        "chain head": patched(blob, "voxels", int(live[0]), p["dn"], "voxels", "head"),
        "chain link": patched(blob, "vnext", 0, p["dn"] + 3),
        "cycle": patched(blob, "vnext", int(vr["head"][live[0]]), int(vr["head"][live[0]])),
        "merged chains": patched(blob, "voxels", int(live[1]), int(vr["head"][live[0]]), "voxels", "head"),
        "worklist entry": patched(blob, "wlist", 0, -2) if p["n_wlist"] else patched(blob, "wflag", 0, 7),
        "worklist flag": patched(blob, "wflag", 0, 2),
        "mapper words": patched(blob, "mstate", MS_NTOUCHED, 5),
        "map voxel size": word(blob, L.STATE_W_MAP_VOXEL, int(np.array([0.2]).view("<u8")[0])),
    }
    if p["n_dups"]:
        cases["duplicate entry"] = patched(blob, "dups", 0, p["vcap"])
    for name, bad in cases.items():
        refuse(other, bad, name)
    # a config mismatch: the same blob on a handle of another map voxel size
    mp = E.MapperParameters(seed=3); mp.mapBuilder.mapVoxelSize = 0.2
    refuse(E.Engine(mp), blob, "config mismatch")
    # odometry blobs
    lp = lap["lp"]
    be = S.DeviceBackend(E.MapperParameters(seed=3), carving=True, dense=True, graph=False)
    sm = be.new_submap()
    be.first_scan_with_odometry(sm, lp.scan(0, seed=0), 0)
    be.step_with_odometry(sm, lp.scan(1, seed=1), 1_000_000)
    ob = be.export_odometry()
    oh = E.parseStateHeader(ob)
    o, n = oh.sections["state"]
    for what, bad in (("truncated", ob[:-8]), ("magic", word(ob, L.STATE_W_MAGIC, L.STATE_MAGIC_SUBMAP)),
                      ("previous points", word(ob, L.STATE_W_PARAMS + 2, oh.params["capacity"] + 1)), ("version", word(ob, L.STATE_W_VERSION, 7))):
        refuse(other, bad, what, odometry=True)
    st = bytearray(ob)
    np.frombuffer(st, dtype="<i4", count=n // 4, offset=o)[288 // 4] = 1 << 20   # the odometry buffer's head, far past the buffer
    refuse(other, bytes(st), "buffer position", odometry=True)
    be.close()


def test_argument_errors(lap):
    eng, sms = lap["eng"], lap["sms"]
    lib = L.lib()
    offs = (C.c_size_t * 4)()
    arr = (C.c_void_p * 2)(sms[0]._s, None)
    assert lib.b2s_submaps_export_state(eng._h, C.c_int32(-1), arr, None, C.c_size_t(0), offs) == L.E_INVALID
    assert lib.b2s_submaps_export_state(eng._h, C.c_int32(2), arr, None, C.c_size_t(0), offs) == L.E_INVALID
    other = E.Engine(E.MapperParameters(seed=3))
    arr1 = (C.c_void_p * 1)(sms[0]._s)
    assert lib.b2s_submaps_export_state(other._h, C.c_int32(1), arr1, None, C.c_size_t(0), offs) == L.E_INVALID
    big = (C.c_void_p * 65536)(*([sms[0]._s] * 65536))
    assert lib.b2s_submaps_export_state(eng._h, C.c_int32(65536), big, None, C.c_size_t(0), offs) == L.E_UNSUPPORTED
    # a buffer smaller than the blobs (a submap that grew since the size call): nothing past capacity is written
    assert lib.b2s_submaps_export_state(eng._h, C.c_int32(1), arr1, None, C.c_size_t(0), offs) == L.OK
    need = int(offs[1])
    buf = np.full(need + 64, 0xAB, dtype=np.uint8)
    assert lib.b2s_submaps_export_state(eng._h, C.c_int32(1), arr1, buf.ctypes.data_as(C.c_void_p), C.c_size_t(need - 8), offs) == L.E_CAPACITY
    assert (buf == 0xAB).all()
    assert lib.b2s_submaps_export_state(eng._h, C.c_int32(0), arr1, None, C.c_size_t(0), offs) == L.OK and offs[0] == 0


# ---- SegmentMapper sessions ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("entry", ["addRangeMeasurement", "addRangeScan"])
def test_session_save_and_load(lap, tmp_path, entry):
    """SegmentMapper over the lap with hand-overs, dense map and carving, graph replay: saved at scan K, loaded into a new DeviceBackend
    and finished.  Saving only reads, so the saved mapper finishing the lap is the uninterrupted run: the loaded one logs the same
    events and its poses agree within the ICP's last-bit variation"""
    lp = lap["lp"]
    p = E.MapperParameters(seed=3)

    def run(m, ks):
        for k in ks:
            if entry == "addRangeScan":
                m.addRangeScan(lp.scan(k, seed=k), k * 1_000_000)
            else:
                m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))

    N, K = 70, 40
    a = S.SegmentMapper(S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=True), S.SubmapParameters(radius=2.0))
    run(a, range(K))
    n_events = len(a.submaps.events)
    assert any(e[0] == "active_submap_changed" for e in a.submaps.events)
    path = str(tmp_path / "session.npz")
    a.saveSession(path)
    be = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=True)
    b = S.SegmentMapper.loadSession(path, be)
    assert len(b.submaps.submaps) == len(a.submaps.submaps) and b._k == K and b.results == []
    for x, y in zip(a.submaps.submaps, b.submaps.submaps):
        assert_same_snapshot(snapshot(a.backend.eng, x.handle), snapshot(be.eng, y.handle))
    run(a, range(K, N))
    run(b, range(K, N))
    ea, eb = a.submaps.events[n_events:], b.submaps.events
    assert any(e[0] == "active_submap_changed" for e in eb) and ea == eb
    assert len(b.poses) == N and max(np.abs(x - y).max() for x, y in zip(a.poses, b.poses)) < 1e-8
    a.backend.close(); be.close()
