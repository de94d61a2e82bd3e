"""The searches over the K-index grid (grid_index.cu) must follow the build's rules for their neighbours to match the oracle's bit
for bit: a coordinate's cell is floor((v - o) * inv_cell) clamped into the grid, a neighbour qualifies only if d2 < r2, neighbours
are ordered by (d2, original index), and a ring walk stops once the nearest block face with cells behind it lies beyond the k-th
best.  These rules are defined once, in common.cuh, and every search calls them; these tests read the CUDA sources and fail when a
source keeps its own copy again.  The ICP search in icp.cu is the one exception: it scans a register copy of the header (GridView)
with its own tuned cell_of / nn_scan_box / nn_scan_row / nn_phase2_warp / ring_bound, and shares only slab_gap.  No GPU needed."""
import glob
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open3d_slam_b200", "csrc")
HELPERS = ("grid_axis_cell", "nn_key_less", "slab_gap", "ring_bound", "grid_knn_walk", "grid_nearest")
# the ICP search's own GridView functions (see the module docstring)
ICP_OWN = ("cell_of", "nn_scan_box", "nn_scan_row", "nn_phase2_warp", "ring_bound")
SOURCES = sorted(os.path.basename(p) for p in glob.glob(os.path.join(CSRC, "*.cu")))


def source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def definitions(src, fn):
    """the signatures of every definition of fn (a declaration followed by a body)"""
    return re.findall(r"__device__ __forceinline__ [\w:<>]+ " + fn + r"\(([^;{]*)\)\s*\{", src)


def body(src, fn):
    """the body of the first definition of fn, braces matched"""
    m = re.search(r"\b" + fn + r"\([^;{]*\)\s*\{", src)
    assert m, f"{fn} not found"
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(src[i], 0)
        i += 1
    return src[m.end():i - 1]


def without(src, fns):
    for fn in fns:
        src = src.replace(body(src, fn), "")
    return src


def test_helpers_defined_once_in_common():
    common = source("common.cuh")
    for fn in HELPERS:
        assert len(definitions(common, fn)) == 1, f"common.cuh must define {fn} exactly once"
    for name in SOURCES:
        src = source(name)
        for fn in HELPERS:
            defs = definitions(src, fn)
            if name == "icp.cu" and fn == "ring_bound":
                assert len(defs) == 1 and defs[0].startswith("const GridView& g"), f"icp.cu: ring_bound other than its GridView one: {defs}"
                continue
            assert not defs, f"{name}: own definition of {fn}"


def test_shared_rules():
    common = source("common.cuh")
    assert "fmin(fmax(floor((v - o) * inv_cell), 0.0), (double)(n - 1))" in body(common, "grid_axis_cell")
    assert "return da < db || (da == db && ia < ib);" in common
    walk = body(common, "grid_knn_walk")
    for call in ("grid_axis_cell(", "slab_gap(", "nn_key_less(", "ring_bound(", "d < r2 &&"):
        assert call in walk, f"grid_knn_walk does not use {call}"
    assert "if (bound == INFINITY || bound * bound > fmin(kd, r2)) break;" in walk
    nearest = body(common, "grid_nearest")
    assert "d < r2 && nn_key_less(d, idx, bd, bi)" in nearest
    # the build files points with the shared cell rule
    assert body(source("grid_index.cu"), "grid_cell_of").count("grid_axis_cell(") == 3


@pytest.mark.parametrize("name", SOURCES)
def test_no_private_search_rule(name):
    """No source keeps its own slab gap, (d2, index) order or clamped cell: each calls the shared ones."""
    src = source(name)
    rest = without(src, ICP_OWN) if name == "icp.cu" else src
    assert not re.search(r"\bbool \w+\(double \w+, int \w+, double \w+, int \w+\)\s*\{", src), f"{name}: own (d2, index) order"
    assert "== db &&" not in src, f"{name}: own (d2, index) order"
    assert not re.search(r"double \w+\(double q, double o, double cell, int i, int n, double eps\)", src), f"{name}: own slab gap"
    assert "double lo = o + (double)i * cell" not in src, f"{name}: own slab gap"
    assert not re.search(r"inv(_cell)?\), 0\.0\)", rest), f"{name}: own clamped cell of a coordinate"


def test_searches_call_the_shared_walks():
    normals, features = source("normals.cu"), source("features.cu")
    for src, kernel, walk in ((normals, "normals_phase2_kernel", "grid_knn_walk<1, true>("),
                              (features, "fpfh_knn_kernel", "grid_knn_walk<FK_PER_LANE, false>(")):
        b = body(src, kernel)
        assert walk in b, f"{kernel} does not call {walk}"
        assert "__shfl_up_sync" not in b and "ring_bound(" not in b, f"{kernel}: own ring walk"
    select2 = body(normals, "normals_select2_kernel")
    assert select2.count("grid_axis_cell(") == 3 and "ring_bound(g, q, c, R, eps)" in select2
    for name, kernel in (("constraints.cu", "info_wide_kernel"), ("ransac.cu", "rs_validate_kernel")):
        assert "grid_nearest(" in body(source(name), kernel), f"{kernel} does not call grid_nearest"
