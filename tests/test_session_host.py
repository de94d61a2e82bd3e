"""CPU: the session-state blob layout (include/b2s.h "session state", DESIGN.md row A3) restated in Python -- open3d_slam_b200/_lib.py's
constants, section orders and record layouts, and the section lengths engine.parseStateHeader reads -- checked against the header and the
CUDA source, so a changed layout fails here, naming the constant, before any blob is read with the wrong offsets.  No GPU needed."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header():
    with open(os.path.join(ROOT, "include", "b2s.h")) as f:
        return re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)


def defines():
    return {m.group(1): int(m.group(2).rstrip("uUlL"), 0) for m in re.finditer(r"#define\s+(B2S_STATE_\w+)\s+(0x[0-9a-fA-F]+\w*|\d+)", header())}


def enum_values(prefix):
    out = {}
    for body in re.findall(r"enum\s*\{(.*?)\}", header(), flags=re.S):
        for name, value in re.findall(r"(" + prefix + r"\w+)\s*=\s*(\d+)", body):
            out[name] = int(value)
    return out


def test_header_constants():
    d = defines()
    assert d["B2S_STATE_VERSION"] == L.STATE_VERSION and d["B2S_STATE_BYTE_ORDER"] == L.STATE_BYTE_ORDER
    assert d["B2S_STATE_MAGIC_SUBMAP"] == L.STATE_MAGIC_SUBMAP and d["B2S_STATE_MAGIC_ODOMETRY"] == L.STATE_MAGIC_ODOMETRY
    assert struct.pack("<Q", L.STATE_MAGIC_SUBMAP) == b"B2SSUBM1" and struct.pack("<Q", L.STATE_MAGIC_ODOMETRY) == b"B2SODOM1"
    assert d["B2S_STATE_HEADER_BYTES"] == L.STATE_HEADER_BYTES == 256
    assert d["B2S_STATE_MSTATE_WORDS"] == L.STATE_MSTATE_WORDS and d["B2S_STATE_POSE_SLOTS"] == L.STATE_POSE_SLOTS
    w = enum_values("B2S_STATE_W_")
    assert (w["B2S_STATE_W_MAGIC"], w["B2S_STATE_W_VERSION"], w["B2S_STATE_W_BYTE_ORDER"], w["B2S_STATE_W_TOTAL_BYTES"],
            w["B2S_STATE_W_MAP_VOXEL"], w["B2S_STATE_W_N_SECTIONS"], w["B2S_STATE_W_SECTIONS"], w["B2S_STATE_W_PARAMS"]) == \
        (L.STATE_W_MAGIC, L.STATE_W_VERSION, L.STATE_W_BYTE_ORDER, L.STATE_W_TOTAL_BYTES, L.STATE_W_MAP_VOXEL, L.STATE_W_N_SECTIONS,
         L.STATE_W_SECTIONS, L.STATE_W_PARAMS)
    f = enum_values("B2S_STATE_F_")
    assert (f["B2S_STATE_F_HAS_NORMALS"], f["B2S_STATE_F_NO_NORMALS"], f["B2S_STATE_F_MERGE_SCANS"], f["B2S_STATE_F_DENSE_HAS_NORMALS"]) == \
        (L.STATE_F_HAS_NORMALS, L.STATE_F_NO_NORMALS, L.STATE_F_MERGE_SCANS, L.STATE_F_DENSE_HAS_NORMALS)


@pytest.mark.parametrize("prefix, names, count", [("B2S_SS_", L.STATE_SUBMAP_SECTIONS, "B2S_SS_COUNT"),
                                                  ("B2S_OS_", L.STATE_ODOMETRY_SECTIONS, "B2S_OS_COUNT")])
def test_section_order(prefix, names, count):
    e = enum_values(prefix)
    n = e.pop(count)
    assert n == len(names) and sorted(e.values()) == list(range(n))
    # the header's names in value order, lower-cased without the prefix, are the Python names
    assert [k[len(prefix):].lower() for k, _v in sorted(e.items(), key=lambda kv: kv[1])] == names
    # every section length fits between the section words and the parameter words
    assert L.STATE_W_SECTIONS + n <= L.STATE_W_PARAMS


@pytest.mark.parametrize("prefix, names", [("B2S_SP_", L.STATE_SUBMAP_PARAMS), ("B2S_OP_", L.STATE_ODOMETRY_PARAMS)])
def test_parameter_words(prefix, names):
    e = enum_values(prefix)
    assert [k[len(prefix):].lower() for k, _v in sorted(e.items(), key=lambda kv: kv[1])] == names
    assert sorted(e.values()) == list(range(L.STATE_W_PARAMS, L.STATE_W_PARAMS + len(names)))
    assert L.STATE_W_PARAMS + len(names) <= L.STATE_HEADER_BYTES // 8


def test_record_layouts():
    assert C.sizeof(L.StateVoxelRecord) == 24 and C.sizeof(L.StateDenseRecord) == 64
    assert E._VOXEL_REC.itemsize == 24 and E._DENSE_REC.itemsize == 64
    for st, dt in ((L.StateVoxelRecord, E._VOXEL_REC), (L.StateDenseRecord, E._DENSE_REC)):
        for name, _t in st._fields_:
            assert getattr(st, name).offset == dt.fields[name][1], name
    h = header()
    assert re.search(r"uint64_t key;\s*int32_t slot, head, stamp, reserved_;\s*\}\s*b2s_state_voxel_record", h)
    assert re.search(r"uint64_t key;\s*double sum\[6\];\s*int32_t slot, count;\s*\}\s*b2s_state_dense_record", h)


# the submap blob's section lengths from its counters, as state.cu's submap_sections computes them
def submap_sections(dn, nv, ndup, nw, nd, fused, dense):
    pad8 = lambda b: (b + 7) & ~7   # noqa: E731
    opts = C.sizeof(L.MapperOptions)
    return [L.STATE_POSE_SLOTS * 128, pad8(opts), L.STATE_MSTATE_WORDS * 4, 48, 24 * dn, 24 * dn] + \
        [pad8(4 * dn) if fused else 0] * 3 + [pad8(4 * ndup), pad8(4 * nw), 24 * nv, 8 if dense else 0, 64 * nd]


def test_submap_section_lengths_match_the_source():
    src = open(os.path.join(ROOT, "open3d_slam_b200", "csrc", "state.cu")).read()
    body = re.search(r"inline long long submap_sections\(.*?\{(.*?)\n\}", src, re.S).group(1)
    body = re.sub(r"\s+", " ", body)
    for expect in ("len[B2S_SS_POSE] = B2S_STATE_POSE_SLOTS * 16 * 8;", "len[B2S_SS_OPTIONS] = st_pad8((long long)sizeof(b2s_mapper_options));",
                   "len[B2S_SS_MSTATE] = B2S_STATE_MSTATE_WORDS * 4;", "len[B2S_SS_BBOX] = 48;",
                   "len[B2S_SS_MAP_XYZ] = len[B2S_SS_MAP_NORMALS] = 24 * c.dn;",
                   "len[B2S_SS_VNEXT] = len[B2S_SS_PSTAMP] = len[B2S_SS_WFLAG] = fused ? st_pad8(4 * c.dn) : 0;",
                   "len[B2S_SS_DUPS] = st_pad8(4 * c.ndup);", "len[B2S_SS_WLIST] = st_pad8(4 * c.nw);",
                   "len[B2S_SS_VOXELS] = (long long)sizeof(b2s_state_voxel_record) * c.nv;", "len[B2S_SS_DENSE_USED] = dense ? 8 : 0;",
                   "len[B2S_SS_DENSE] = (long long)sizeof(b2s_state_dense_record) * c.nd;"):
        assert expect in body, f"submap_sections changed ({expect}): update tests/test_session_host.py and the format version"
    assert C.sizeof(L.MapperOptions) == 168


def test_parse_state_header_reads_a_blob_built_by_the_layout():
    """a synthetic blob laid out by the restated rules parses into the sections and parameters it was built from"""
    dn, nv, ndup, nw, nd = 5, 3, 1, 2, 4
    lens = submap_sections(dn, nv, ndup, nw, nd, True, True)
    w = np.zeros(32, dtype="<u8")
    w[L.STATE_W_MAGIC], w[L.STATE_W_VERSION], w[L.STATE_W_BYTE_ORDER] = L.STATE_MAGIC_SUBMAP, L.STATE_VERSION, L.STATE_BYTE_ORDER
    w[L.STATE_W_TOTAL_BYTES] = 256 + sum(lens)
    w[L.STATE_W_MAP_VOXEL] = np.array([0.1]).view("<u8")[0]
    w[L.STATE_W_N_SECTIONS] = len(lens)
    w[L.STATE_W_SECTIONS:L.STATE_W_SECTIONS + len(lens)] = lens
    params = dict(capacity=100, vcap=4096, stage_cap=64, dense_cap=4096, flags=5, dn=dn, n_voxels=nv, n_dups=ndup, n_wlist=nw, n_dense=nd)
    for k, name in enumerate(L.STATE_SUBMAP_PARAMS):
        w[L.STATE_W_PARAMS + k] = np.array([0.05]).view("<u8")[0] if name == "dense_voxel" else params[name]
    body = bytearray(sum(lens))
    blob = w.tobytes() + bytes(body)
    h = E.parseStateHeader(blob)
    assert h.kind == "submap" and h.total_bytes == len(blob) and h.map_voxel_size == 0.1 and h.params["dense_voxel"] == 0.05
    assert all(h.params[k] == v for k, v in params.items())
    off = 256
    for name, n in zip(L.STATE_SUBMAP_SECTIONS, lens):
        assert h.sections[name] == (off, n)
        off += n
    assert len(h.section(blob, "voxels", "voxels")) == nv and len(h.section(blob, "dense", "dense")) == nd
    assert len(h.section(blob, "map_xyz", "<f8")) == 3 * dn
    with pytest.raises(ValueError):
        E.parseStateHeader(bytes(256))


# ---- SegmentMapper.saveSession / loadSession over the oracle backend ----------------------------------------------------------------------
def same_tree(a, b):
    """equality of nested events / poses, numpy arrays bit for bit"""
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))
    if isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)):
        return len(a) == len(b) and all(same_tree(x, y) for x, y in zip(a, b))
    return a == b


def test_session_continues_exactly_over_the_oracle(tmp_path):
    """The closed lap with loop closures on, 10 m submaps (no dense map: the oracle's cannot be copied, and nothing the schedule decides
    reads it): saved after scan K (finished submaps with features, odometry constraints and pending ids), loaded into a new backend and
    finished.  Saving only reads, so the saved mapper finishing the lap is the uninterrupted run: every event and pose of the loaded one
    equals it, loop closure included."""
    import copy

    from oracle_backend_session import SessionOracleBackend
    from open3d_slam_b200 import slam as S
    from open3d_slam_b200 import workloads as W

    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()

    def mapper():
        lc = S.LoopClosingParameters.fromMapperParameters(p)
        lc.candidates.loopClosureSearchRadius = 10.0   # the search test_loop_closing_schedule_host.py closes the lap with
        return S.SegmentMapper(SessionOracleBackend(copy.deepcopy(p), carving=True, dense=False), S.SubmapParameters(radius=10.0),
                               isAttemptLoopClosures=True, loopClosing=lc)

    def run(m, ks):
        for k in ks:
            m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))

    N, K = 145, 100
    full = mapper()
    run(full, range(K))
    assert full.submaps.finishedSubmapsIdxs and any(r.feature is not None for r in full.submaps.submaps)
    n_events = len(full.submaps.events)
    path = str(tmp_path / "session.npz")
    full.saveSession(path)
    cont = S.SegmentMapper.loadSession(path, SessionOracleBackend(copy.deepcopy(p), carving=True, dense=False))
    assert cont.results == [] and cont.submaps.events == [] and cont._k == K
    run(full, range(K, N))
    run(cont, range(K, N))
    assert any(e[0] == "loop_closure_correction" for e in cont.submaps.events)
    assert same_tree(full.submaps.events[n_events:], cont.submaps.events)
    assert same_tree(full.poses, cont.poses) and len(cont.poses) == N
    for a, b in zip(full.submaps.submaps, cont.submaps.submaps):
        assert same_tree(a.handle.xyz, b.handle.xyz) and same_tree(a.handle.nrm, b.handle.nrm)
