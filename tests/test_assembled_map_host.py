"""CPU: the rules of the assembled map (DESIGN.md row A1, include/b2s.h) restated in numpy (tests/oracle_backend_assembly.py) and checked
against the oracle -- the palette with its float32 promotion and its wrap, the normals rule, the voxel path and the colour means -- and
SegmentMapper.getAssembledMapPointCloud over the oracle backend on a stretch of the closed lap."""
import copy

import numpy as np
import pytest

from oracle import oracle as O
from oracle_backend_assembly import PALETTE, AssemblyOracleBackend, assemble, assembled, colored, voxel_keys
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W


def patch(seed, n, offset=(0.0, 0.0, 0.0)):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-2.0, 2.0, (n, 3)) + np.asarray(offset)
    nrm = rng.normal(size=(n, 3))
    return xyz, nrm / np.linalg.norm(nrm, axis=1, keepdims=True)


def by_key(xyz, keys, *cols):
    o = np.lexsort(keys.T[::-1])
    return (xyz[o],) + tuple(c[o] for c in cols)


def test_palette_is_the_float32_colours_in_getColor_order():
    assert PALETTE.dtype == np.float64 and PALETTE.shape == (11, 3)
    assert tuple(PALETTE[0]) == (0.5, 0.5, 0.5) and tuple(PALETTE[1]) == (1.0, 0.0, 0.0) and tuple(PALETTE[5]) == (1.0, 0.5, 0.0)
    assert tuple(PALETTE[10]) == (0.7799999713897705, 0.0, 0.8999999761581421)   # Magenta (.78, 0, .9) through float32
    assert PALETTE[10, 0] != 0.78 and PALETTE[10, 2] != 0.9


@pytest.mark.parametrize("j, entry", [(0, 0), (10, 10), (11, 0), (12, 1), (22, 0), (23, 1)])
def test_palette_wraps_every_11_submaps(j, entry):
    maps = [(np.full((1, 3), float(k)), None) for k in range(j + 1)]
    _x, rgb = colored(maps, 0.0)
    assert np.array_equal(rgb[j], PALETTE[entry])


def test_assembly_is_the_concatenation_in_submap_order():
    a, b = patch(1, 50), patch(2, 30, (5, 0, 0))
    xyz, nrm, sub = assemble([a, (np.zeros((0, 3)), np.zeros((0, 3))), b])
    assert np.array_equal(xyz, np.concatenate([a[0], b[0]])) and np.array_equal(nrm, np.concatenate([a[1], b[1]]))
    assert np.array_equal(sub, np.r_[np.zeros(50), np.full(30, 2)])
    x0, n0 = assembled([a, b], 0.0)
    x1, n1 = assembled([a, b], -1.0)
    assert np.array_equal(x0, xyz) and np.array_equal(x1, xyz) and np.array_equal(n0, nrm) and np.array_equal(n1, nrm)


def test_normals_rule():
    a, b = patch(1, 40), patch(2, 40, (3, 0, 0))
    nan = np.full((40, 3), np.nan)
    empty_p2p = (np.zeros((0, 3)), np.zeros((0, 3)) * np.nan)
    assert assemble([a, b])[1] is not None                         # all with normals
    assert assemble([a, empty_p2p, b])[1] is not None              # an empty point-to-point map contributes nothing
    assert assemble([a, (b[0], nan)])[1] is None                   # mixed: no normals (the reference's cloud would be malformed)
    assert assemble([a, (b[0], None)])[1] is None
    assert assemble([(a[0], nan), (b[0], nan)])[1] is None         # all without
    assert assemble([])[1] is None and len(assemble([])[0]) == 0   # empty: no normals
    assert assemble([empty_p2p])[1] is None


@pytest.mark.parametrize("voxel", [0.1, 0.25, 1.0])
def test_voxel_path_is_the_oracle_on_the_concatenation(voxel):
    maps = [patch(k, 400, (1.5 * k, 0, 0)) for k in range(4)]
    xyz, nrm = np.concatenate([m[0] for m in maps]), np.concatenate([m[1] for m in maps])
    gx, gn = assembled(maps, voxel)
    ox, on, ok = O.voxel_down_sample(xyz, voxel, nrm, return_keys=True)
    assert np.array_equal(gx, ox) and np.array_equal(gn, on)
    # the key restated in numpy is the oracle's
    assert np.array_equal(np.unique(voxel_keys(xyz, voxel), axis=0), np.unique(ok.astype(np.int64), axis=0))


@pytest.mark.parametrize("voxel", [0.25, 1.0])
def test_colour_means_in_input_order(voxel):
    maps = [patch(k, 200, (0.7 * k, 0, 0)) for k in range(13)]     # 13 submaps: the palette wraps, and voxels mix colours
    cx, rgb = colored(maps, voxel)
    xyz, _n, sub = assemble(maps)
    ox, _on, ok = O.voxel_down_sample(xyz, voxel, return_keys=True)
    assert len(cx) == len(ox)
    keys = voxel_keys(xyz, voxel)
    uk = np.unique(keys, axis=0)
    (a,) = by_key(ox, ok.astype(np.int64))
    assert np.array_equal(cx, a)                                   # the same voxel means, ascending key order on both sides
    mixed = 0
    for v, k in enumerate(uk):                                     # AccumulatedPoint, one member after the other
        members = np.flatnonzero((keys == k).all(axis=1))
        s = np.zeros(3)
        for i in members:
            s = s + PALETTE[sub[i] % 11]
        assert np.array_equal(rgb[v], s / float(len(members)))
        mixed += len(np.unique(sub[members] % 11)) > 1
    assert mixed > 0


def test_segment_mapper_assembles_the_closed_lap_over_the_oracle():
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    be = AssemblyOracleBackend(copy.deepcopy(p), carving=True, dense=False)
    m = S.SegmentMapper(be, S.SubmapParameters(radius=3.0))
    for k in range(24):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    subs = m.submaps.submaps
    assert len(subs) >= 2
    c = m.getAssembledMapPointCloud()
    assert np.array_equal(c.xyz, np.concatenate([s.handle.xyz for s in subs])) and np.array_equal(c.nrm, np.concatenate([s.handle.nrm for s in subs]))
    assert m.submaps.getTotalNumPoints() == len(c)
    v = m.getAssembledMapPointCloud(0.25)
    ox, on = O.voxel_down_sample(c.xyz, 0.25, c.nrm)
    assert np.array_equal(v.xyz, ox) and np.array_equal(v.nrm, on)
    cc, rgb = m.assembleColoredPointCloud(0.0)
    assert np.array_equal(cc.xyz, c.xyz) and cc.nrm is None and len(rgb) == len(c)
    assert np.array_equal(rgb[:len(subs[0].handle.xyz)], np.broadcast_to(PALETTE[0], (len(subs[0].handle.xyz), 3)))
    assert np.array_equal(rgb[-1], PALETTE[(len(subs) - 1) % 11])


def test_visualization_parameters_are_the_lua_defaults():
    v = E.VisualizationParameters()
    assert (v.assembledMapVoxelSize, v.submapVoxelSize, v.visualizeEveryNmsec) == (0.1, 0.1, 250.0)
