"""-m "not gpu": the tile cover of the static map patch (tile_box in grid_index.cu) restated in numpy and checked against the CUDA
constants, in the way test_voxel_hash_rules.py checks the hash rules: every point crop_within accepts lies in a tile the box selects.
Sensors on tile faces and corners, beyond the map border, and 5 km from the origin; points on the cropper's boundary, an ulp in and out."""
import re
from pathlib import Path

import numpy as np
import pytest

CSRC = Path(__file__).resolve().parents[1] / "open3d_slam_b200" / "csrc"


def _constants():
    src = (CSRC / "common.cuh").read_text()
    edge = float(re.search(r"constexpr double TILE_EDGE = ([0-9.]+);", src).group(1))
    margin = int(re.search(r"constexpr int TILE_MARGIN = (\d+);", src).group(1))
    g = (CSRC / "grid_index.cu").read_text()
    # the gather takes the box the restatement below takes: c -/+ rmax per axis, the cylinder's absolute z range, floor -/+ the margin
    assert "lo[d] = c[d] - crop.rmax; hi[d] = c[d] + crop.rmax;" in g
    assert "if (crop.kind == B2S_CROP_CYLINDER) { lo[2] = crop.zmin; hi[2] = crop.zmax; }" in g
    assert "floor((lo[d] - g.origin[d]) * g.inv_cell) - TILE_MARGIN" in g and "floor((hi[d] - g.origin[d]) * g.inv_cell) + TILE_MARGIN" in g
    assert "grid_build(h, &sm->tile, map, TILE_EDGE, nullptr)" in g
    return edge, margin


EDGE, MARGIN = _constants()


def crop_within(kind, c, rmin, rmax, zmin, zmax, p):
    """common.cuh crop_within: (dx*dx + dy*dy) + dz*dz in round-to-nearest ops, then sqrt"""
    d = p - c
    if kind == "Cylinder":
        return (p[:, 2] >= zmin) & (p[:, 2] <= zmax) & (np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) <= rmax)
    r = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    return (r <= rmax) & (r >= rmin) if kind == "MinMaxRadius" else r <= rmax


def table(points):
    """grid_header_body over the map (no coarsening at these sizes) and grid_cell_of's clamped tile per point"""
    mn, mx = points.min(axis=0), points.max(axis=0)
    dims = (np.floor((mx - mn) / EDGE) + 1.0).astype(np.int64)
    inv = 1.0 / EDGE
    cell = np.clip(np.floor((points - mn) * inv), 0, dims - 1).astype(np.int64)
    return mn, inv, dims, cell


def tile_box(mn, inv, dims, kind, c, rmax, zmin, zmax):
    lo, hi = c - rmax, c + rmax
    if kind == "Cylinder":
        lo[2], hi[2] = zmin, zmax
    a = np.maximum(np.floor((lo - mn) * inv) - MARGIN, 0.0)
    b = np.minimum(np.floor((hi - mn) * inv) + MARGIN, (dims - 1).astype(np.float64))
    return a, b


def boundary_points(rng, c, rmin, rmax, zmin, zmax, n=4000):
    """points on the sphere / cylinder of radius rmax (and rmin), one ulp in and out, plus the cylinder's z faces"""
    u = rng.normal(size=(n, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    pts = []
    for r in (rmax, rmin):
        for s in (np.nextafter(r, 0.0), r, np.nextafter(r, np.inf)):
            pts.append(c + s * u)
    v = rng.normal(size=(n, 2)); v /= np.linalg.norm(v, axis=1, keepdims=True)
    for z in (zmin, zmax):
        for s in (np.nextafter(rmax, 0.0), rmax):
            pts.append(np.c_[c[0] + s * v[:, 0], c[1] + s * v[:, 1], np.full(n, z)])
    pts.append(c + rng.uniform(-rmax, rmax, (n, 3)))
    return np.concatenate(pts)


@pytest.mark.parametrize("kind", ["MaxRadius", "MinMaxRadius", "Cylinder"])
@pytest.mark.parametrize("origin", [(0.0, 0.0, 0.0), (5000.0, -5000.0, 30.0), (-5000.0, 0.0, -10.0)])
def test_every_accepted_point_lies_in_a_selected_tile(kind, origin):
    rng = np.random.default_rng(3)
    origin = np.asarray(origin)
    rmin, rmax = 2.0, 20.0
    world = origin + rng.uniform(-60.0, 60.0, (20000, 3)) * np.array([1.0, 1.0, 0.1])   # the map's extent
    mn0 = world.min(axis=0)
    sensors = [origin.copy(), world.max(axis=0) + 5.0, mn0 - 30.0]                       # centre, beyond both borders
    sensors += [mn0 + EDGE * np.array(k, dtype=np.float64) for k in ([10, 10, 1], [11, 10, 1], [10, 11, 2], [12, 12, 0])]   # faces, corners
    sensors += [s + np.array([0.0, 0.0, 1e-9]) for s in sensors[3:]]
    n_checked = 0
    for c in sensors:
        zmin, zmax = c[2] - 3.0, c[2] + 4.0
        pts = boundary_points(rng, c, rmin, rmax, zmin, zmax)
        pts = pts[(pts >= world.min(axis=0)).all(axis=1) & (pts <= world.max(axis=0)).all(axis=1)]   # map points lie in the map's box
        allp = np.concatenate([world, pts])
        mn, inv, dims, cell = table(allp)
        acc = crop_within(kind, c, rmin, rmax, zmin, zmax, allp)
        a, b = tile_box(mn, inv, dims, kind, c.copy(), rmax, zmin, zmax)
        inside = ((cell >= a) & (cell <= b)).all(axis=1)
        assert inside[acc].all(), (kind, c, np.flatnonzero(acc & ~inside)[:5])
        n_checked += int(acc.sum())
    assert n_checked > 1000


def test_box_beyond_the_table_is_clamped_or_empty():
    mn, inv, dims = np.zeros(3), 1.0 / EDGE, np.array([10, 10, 3])
    a, b = tile_box(mn, inv, dims, "MaxRadius", np.array([-500.0, 5.0, 1.0]), 20.0, 0, 0)
    assert a[0] > b[0]                                                       # wholly outside along x: no tile
    a, b = tile_box(mn, inv, dims, "MaxRadius", np.array([5.0, 5.0, 1.0]), 1e30, 0, 0)
    assert (a == 0).all() and (b == dims - 1).all()                          # an enormous radius selects the whole table
