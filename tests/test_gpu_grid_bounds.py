"""-m gpu: the scan-to-map index built from the submap's box (grid_index.cu, grid_zero_header_kernel) against the build that measures
its grid box with a pass over the map (B2S_GRID_BBOX_PASS=1), and the submap's box itself (fuse.cu).

  - the submap's box holds every live map slot after insertions, and is the exact box of the map after a rehash: carving,
    Submap::transform, setMapPointCloud and the initial map of a localisation;
  - an index built from the box holds exactly the map points the cropper accepts, each in the cell its position keys to (clamped to
    the border cells), for every bounded cropper kind and sensor positions from the middle of the map to beyond its border;
  - with the switch on and off (one process each: the library reads it once) every registration indexes the same points and has the
    same ICP outcome: iterations, correspondences and fitness equal, transforms to 1e-12; over a lap of the benchmark's chain, eager
    and replayed from a graph, the maps agree too.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from open3d_slam_b200 import _lib as L
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import synth
from open3d_slam_b200 import workloads as W

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CHILD = os.path.join(HERE, "grid_bounds_child.py")
from grid_bounds_child import CROPPERS, OFFSETS  # noqa: E402


def submap_box(sm):
    b = (C.c_double * 6)()
    L.check(L.lib().b2s_debug_submap_bbox(sm.eng._h, sm._s, b))
    return np.array(b[:3]), np.array(b[3:])


def assert_holds(sm, exact):
    xyz, _ = sm.getMapPointCloud()
    lo, hi = submap_box(sm)
    assert len(xyz) > 0
    assert (lo <= xyz.min(axis=0)).all() and (hi >= xyz.max(axis=0)).all(), (lo, hi, xyz.min(axis=0), xyz.max(axis=0))
    if exact:
        assert np.array_equal(lo, xyz.min(axis=0)) and np.array_equal(hi, xyz.max(axis=0))


def test_the_submap_box_holds_every_live_slot():
    lp = W.ClosedLoop()
    p = E.MapperParameters(seed=3)
    p.scanProcessing.downSamplingRatio = 0.3
    eng = E.Engine(p)
    mp = E.Mapper(eng, 760_000)
    lo, hi = submap_box(mp.submap)
    assert (lo == np.inf).all() and (hi == -np.inf).all()                   # the empty map
    mp.addRangeMeasurement(eng.cloud(lp.scan(0, seed=0)), None)
    for k in range(1, 35):                                                  # insertions
        mp.addRangeMeasurement(eng.cloud(lp.scan(k, seed=k)), lp.delta(k))
        if k % 6 == 0:
            assert_holds(mp.submap, exact=False)
    raw = eng.cloud(lp.scan(3, seed=3))
    mp.submap.carve(raw, lp.map_frame_pose(3), E.SpaceCarvingParameters(), force=True)   # carving: a rehash
    assert_holds(mp.submap, exact=True)
    mp.submap.transform(synth.se3(0.02, -0.01, 0.3, (4.0, -2.5, 0.5)))   # Submap::transform: a rehash
    assert_holds(mp.submap, exact=True)
    xyz, nrm = mp.submap.getMapPointCloud()
    sm = E.Submap(eng, 400_000)
    sm.setMapPointCloud(eng.cloud(xyz[::3], nrm[::3]))                      # setMapPointCloud
    assert_holds(sm, exact=True)
    sm.insertScan(None, eng.cloud(xyz[1::7] + 0.01, nrm[1::7]), np.eye(4))   # fusion after a load
    assert_holds(sm, exact=False)
    loc = E.Submap(eng, 400_000)
    cloud = eng.cloud(xyz, nrm)
    loc.setInitialMap(cloud, 0.2)                                           # the initial map of a localisation
    assert_holds(loc, exact=True)
    eng.close()


def run_child(out, env_extra):
    env = dict(os.environ)
    env.pop("B2S_GRID_BBOX_PASS", None)
    env.update(env_extra)
    proc = subprocess.run([sys.executable, "-s", CHILD, str(out)], env=env, capture_output=True, text=True, timeout=1800,
                          cwd=os.path.dirname(HERE))
    assert proc.returncode == 0, f"child {env_extra} exited with {proc.returncode}:\n{proc.stdout}\n{proc.stderr}"
    return dict(np.load(out))


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    d = tmp_path_factory.mktemp("grid_bounds")
    return run_child(d / "box.npz", {}), run_child(d / "pass.npz", {"B2S_GRID_BBOX_PASS": "1"})


def crop_in(xyz, c, kind, rmax, rmin, zmin, zmax):
    """crop_within, in its operation order (IEEE double, no FMA)"""
    d = xyz - c
    if kind == "Cylinder":
        r = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1])
        return (xyz[:, 2] >= zmin) & (xyz[:, 2] <= zmax) & (r <= rmax)
    r = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    return (r <= rmax) & (r >= rmin) if kind == "MinMaxRadius" else r <= rmax


def cases():
    for ci, crop in enumerate(CROPPERS):
        for k in (1, 6, 11):
            for oi in range(len(OFFSETS)):
                yield crop, f"patch_{ci}_{k}_{oi}"


def test_the_index_from_the_box_holds_the_cropped_map_cell_by_cell(runs):
    box, _ = runs
    xyz = box["patch_map"]
    empty = 0
    for crop, tag in cases():
        if box[f"{tag}_res"][0] == -1.0:
            empty += 1
            continue
        hdr, starts, orig = box[f"{tag}_hdr"], box[f"{tag}_starts"], box[f"{tag}_orig"]
        origin, cell, dims, ncell, n = hdr[:3], hdr[3], hdr[4:7].astype(int), int(hdr[7]), int(hdr[8])
        want = np.flatnonzero(crop_in(xyz, box[f"{tag}_pose"][:3, 3], *crop))
        assert n == len(want) and np.array_equal(np.sort(orig), want)
        p = xyz[orig]
        f = np.floor((p - origin) * (1.0 / cell))
        c = np.minimum(np.maximum(f, 0.0), dims - 1).astype(np.int64)
        got = np.repeat(np.arange(ncell), np.diff(starts))
        assert np.array_equal((c[:, 2] * dims[1] + c[:, 1]) * dims[0] + c[:, 0], got)
    assert empty > 0                                                        # the sensor beyond the map: nothing to index


def same_result(a, b):
    assert a.shape == b.shape
    if len(a) == 1:
        return
    assert np.array_equal(a[-3:], b[-3:])                                   # fitness, correspondences, iterations
    assert np.abs(a[:16] - b[:16]).max() <= 1e-12 * max(1.0, np.abs(b[:16]).max())


def test_both_builds_index_the_same_points_and_register_alike(runs):
    box, ref = runs
    for _crop, tag in cases():
        same_result(box[f"{tag}_res"], ref[f"{tag}_res"])
        if box[f"{tag}_res"][0] == -1.0:
            continue
        assert box[f"{tag}_hdr"][8] == ref[f"{tag}_hdr"][8]
        assert np.array_equal(np.sort(box[f"{tag}_orig"]), np.sort(ref[f"{tag}_orig"]))


@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_mapper_chain_matches_the_bbox_pass(runs, mode):
    box, ref = runs
    a, b = box[f"{mode}_res"], ref[f"{mode}_res"]
    assert a.shape == b.shape and len(a) > 100
    assert np.array_equal(a[:, -1], b[:, -1]), "iterations"
    assert np.array_equal(a[:, -2], b[:, -2]), "correspondences"
    assert np.abs(a[:, :16] - b[:, :16]).max() <= 1e-12
    ax, an = box[f"{mode}_xyz"], box[f"{mode}_nrm"]; bx, bn = ref[f"{mode}_xyz"], ref[f"{mode}_nrm"]
    assert len(ax) == len(bx) > 100_000
    oa = np.lexsort((ax[:, 2], ax[:, 1], ax[:, 0])); ob = np.lexsort((bx[:, 2], bx[:, 1], bx[:, 0]))
    assert np.abs(ax[oa] - bx[ob]).max() < 1e-9 and np.abs(an[oa] - bn[ob]).max() < 1e-9
    # the benchmark's map keeps its 0.25 m cells: the box from the submap needs no coarsening either
    print(f"{mode}: cell / ncell from the box {box[f'{mode}_hdr'][3]} / {int(box[f'{mode}_hdr'][7])}, "
          f"measured {ref[f'{mode}_hdr'][3]} / {int(ref[f'{mode}_hdr'][7])}")
    assert box[f"{mode}_hdr"][3] == ref[f"{mode}_hdr"][3] == 0.25
