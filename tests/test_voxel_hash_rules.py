"""tests/voxel_hash.py restates the voxel-hash rules of the map-side kernels; these tests read the CUDA sources and fail, naming
the constant, when a rule there no longer matches.  Without them a changed hash or table size would quietly turn the probe-cluster
and capacity tests of test_gpu_map_boundaries.py into ordinary tests.  No GPU needed."""
import os
import re

import numpy as np
import pytest

import voxel_hash as VH

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open3d_slam_b200", "csrc")
TABLES = {"fuse.cu": ("fv", "dense"), "carve.cu": ("cv",), "overlap.cu": ("ov",), "voxelmap.cu": ("vm",)}
HINT = "update tests/voxel_hash.py (and the tests built on it) to the new rule"


def source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def body(src, fn):
    m = re.search(r"\b" + fn + r"\([^)]*\)\s*\{(.*?)\n\}", src, re.S)
    assert m, f"{fn} not found: {HINT}"
    return re.sub(r"\s+", " ", m.group(1))


@pytest.mark.parametrize("name", sorted(TABLES))
def test_pack_hash_and_key_limit(name):
    src = source(name)
    for prefix in TABLES[name]:
        h = body(src, prefix + "_hash")
        expect = f"k ^= k >> 33; k *= {VH.M1:#x}ull; k ^= k >> 33; k *= {VH.M2:#x}ull; k ^= k >> 33;"
        assert expect in h, f"{name}: {prefix}_hash is no longer the murmur3 finalizer ({h}): {HINT}"
        p = body(src, prefix + "_pack")
        for axis, shift in (("x", " << 42"), ("y", " << 21"), ("z", "")):
            assert f"(unsigned)({axis} + {VH.OFFSET}){shift}" in p, f"{name}: {prefix}_pack field {axis} moved ({p}): {HINT}"
    limits = set(re.findall(r"fabs\(f[xyz]\) < ([0-9.]+)", src))
    assert limits == {f"{VH.KEY_LIMIT}.0"}, f"{name}: key limit(s) {limits}, expected |k| < {VH.KEY_LIMIT}: {HINT}"


def test_table_sizes_and_fill_limits():
    fuse, carve, overlap, vmap = source("fuse.cu"), source("carve.cu"), source("overlap.cu"), source("voxelmap.cu")
    common, capi = source("common.cuh"), source("c_api.cu")
    assert f"constexpr int FUSE_DUP_CAP = 1 << {VH.FUSE_DUP_CAP.bit_length() - 1};" in common, f"FUSE_DUP_CAP: {HINT}"
    assert re.search(rf"size_t vcap = {VH.FUSE_TABLE_MIN};\s*while \(vcap < 2 \* sm->capacity\) vcap <<= 1;", fuse), f"fusion table size: {HINT}"
    assert "> mask - mask / 4) atomicOr(status, ST_HASH_FULL)" in fuse, f"fusion fill limit: {HINT}"
    assert "> cap - cap / 8) atomicOr(status, ST_HASH_FULL)" in fuse, f"dense fill limit: {HINT}"
    assert "> cap - cap / 8) atomicOr(status, ST_HASH_FULL)" in vmap, f"voxel-map fill limit: {HINT}"
    dense_sizes = re.findall(r"dense_init\(h, sm, \(size_t\)1 << (\d+),", capi)
    assert dense_sizes and set(dense_sizes) == {str(VH.DENSE_SLOTS.bit_length() - 1)}, f"dense slots {dense_sizes}: {HINT}"
    assert "dense_hash(key) % cap" in fuse, f"dense home slot: {HINT}"
    grow = rf"size_t cap = {VH.SCRATCH_TABLE_MIN};\s*while \(cap < 2 \* "
    assert re.search(grow + r"n_max\) cap <<= 1;", carve), f"sparse-carve table size: {HINT}"
    assert re.search(grow + r"\(ns \+ nt\)\) cap <<= 1;", overlap), f"overlap table size: {HINT}"
    assert re.search(grow + r"capacity_voxels\) cap <<= 1;", vmap), f"voxel-map table size: {HINT}"
    assert re.search(grow + r"n_max\) cap <<= 1;", fuse.split("op_dense_carve")[-1]), f"dense-carve ray table size: {HINT}"
    ray = body(fuse, "ray_home")
    assert "dense_hash(" in ray and "& m) << 42" in ray and f"+ {VH.OFFSET}u" in ray, f"dense-carve home slot ({ray}): {HINT}"


def test_inverse_finalizer():
    assert (VH.M1 * VH.M1_INV) & VH.U64 == 1 and (VH.M2 * VH.M2_INV) & VH.U64 == 1
    rng = np.random.default_rng(0)
    for k in rng.integers(0, 1 << 63, 200, dtype=np.int64):
        assert VH.fmix64_inv(VH.fmix64(int(k))) == int(k) and VH.fmix64(VH.fmix64_inv(int(k))) == int(k)
    for slots in (1024, VH.FUSE_TABLE_MIN, VH.DENSE_SLOTS):
        for slot in (0, slots - 1):
            keys = VH.keys_homed_at(slot, slots, 4, seed=slot)
            assert len(set(keys)) == 4 and all(VH.home(k, slots) == slot for k in keys)
    assert VH.grown(1024, 512) == 1024 and VH.grown(1024, 513) == 2048 and VH.fusion_slots(2048) == 4096 and VH.fusion_slots(2049) == 8192
    assert VH.dense_fill_limit() == 3_670_016
