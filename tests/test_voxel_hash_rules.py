"""tests/voxel_hash.py restates the voxel-hash rules of the map-side kernels; these tests read the CUDA sources and fail, naming
the constant, when a rule there no longer matches.  Without them a changed hash or table size would quietly turn the probe-cluster
and capacity tests of test_gpu_map_boundaries.py into ordinary tests.  The key, the hash and the probes are defined once, in
common.cuh; the table sizes and fill limits stay with each table's own source, and the fusion table keeps its own find-or-insert
loop over the shared hash.  No GPU needed."""
import os
import re

import numpy as np
import pytest

import voxel_hash as VH

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open3d_slam_b200", "csrc")
# the shared probes each table's source calls
TABLES = {"fuse.cu": ("voxel_key_claim", "voxel_key_find"), "carve.cu": ("voxel_key_claim", "voxel_key_find"),
          "overlap.cu": ("voxel_key_claim",), "voxelmap.cu": ("voxel_key_claim", "voxel_key_find")}
HINT = "update tests/voxel_hash.py (and the tests built on it) to the new rule"


def source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def body(src, fn):
    m = re.search(r"\b" + fn + r"\([^)]*\)\s*\{(.*?)\n\}", src, re.S)
    assert m, f"{fn} not found: {HINT}"
    return re.sub(r"\s+", " ", m.group(1))


def test_shared_key_rules():
    common = source("common.cuh")
    h = body(common, "voxel_key_hash")
    expect = f"k ^= k >> 33; k *= {VH.M1:#x}ull; k ^= k >> 33; k *= {VH.M2:#x}ull; k ^= k >> 33;"
    assert expect in h, f"voxel_key_hash is no longer the murmur3 finalizer ({h}): {HINT}"
    p = body(common, "voxel_key_pack")
    for axis, shift in (("x", " << 42"), ("y", " << 21"), ("z", "")):
        assert f"(unsigned)({axis} + {VH.OFFSET}){shift}" in p, f"voxel_key_pack field {axis} moved ({p}): {HINT}"
    u = body(common, "voxel_key_unpack")
    field = f"{(1 << VH.FIELD_BITS) - 1:#X}".replace("0X", "0x")
    for axis, shift in (("x", "(k >> 42)"), ("y", "(k >> 21)"), ("z", "k")):
        assert f"*{axis} = (int)({shift} & {field}) - {VH.OFFSET};" in u, f"voxel_key_unpack field {axis} moved ({u}): {HINT}"
    k = body(common, "voxel_key_of")
    limits = set(re.findall(r"fabs\(f[xyz]\) < ([0-9.]+)", k))
    assert limits == {f"{VH.KEY_LIMIT}.0"}, f"key limit(s) {limits}, expected |k| < {VH.KEY_LIMIT}: {HINT}"
    assert "floor(__dmul_rn(x, ix))" in k and "voxel_key_pack(" in k, f"voxel_key_of is no longer floor(p * inv) ({k}): {HINT}"
    for fn in ("voxel_key_find", "voxel_key_claim"):
        b = body(common, fn)
        assert "(size_t)voxel_key_hash(key) & mask" in b and "s = (s + 1) & mask" in b, f"{fn}: home slot / linear probe ({b}): {HINT}"
    # the dense-carve lookup by integer key applies the same limit
    int_limits = re.findall(r"abs\(k[xyz]\) < (\d+)", body(source("fuse.cu"), "dense_find_key"))
    assert int_limits == [str(VH.KEY_LIMIT)] * 3, f"dense_find_key key limit {int_limits}: {HINT}"


@pytest.mark.parametrize("name", sorted(TABLES) + ["voxel.cu"])
def test_no_private_key_copy(name):
    """The file keeps no copy of the key, the hash, the key limit or the point transforms: it calls the shared ones."""
    src = source(name)
    rest = re.sub(r"\bray_home\([^)]*\)\s*\{.*?\n\}", "", src, flags=re.S)   # the ray set's masked full-int32 key packing
    assert f"{VH.M1:#x}" not in src.lower() and f"{VH.M2:#x}" not in src.lower(), f"{name}: own copy of the hash finalizer"
    assert "<< 42" not in rest, f"{name}: own copy of the key packing"
    assert f"{VH.KEY_LIMIT}.0" not in src, f"{name}: own copy of the key limit"
    assert "__dmul_rn(T[12]" not in src, f"{name}: own copy of the homogeneous point transform"
    assert "fabs(T[i] - ((i % 5 == 0)" not in src, f"{name}: own copy of the near-identity test"
    assert re.findall(r"constexpr unsigned long long (\w+) = ~0ull", src) == (["RAY_EMPTY"] if name == "fuse.cu" else []), \
        f"{name}: own empty-slot constant"
    for fn in TABLES.get(name, ()):
        assert fn + "(" in src and "voxel_key_of(" in src, f"{name}: does not call the shared {fn} / voxel_key_of"


def test_table_sizes_fill_limits_and_dense_probe():
    fuse, carve, overlap, vmap = source("fuse.cu"), source("carve.cu"), source("overlap.cu"), source("voxelmap.cu")
    common, capi = source("common.cuh"), source("c_api.cu")
    assert f"constexpr int FUSE_DUP_CAP = 1 << {VH.FUSE_DUP_CAP.bit_length() - 1};" in common, f"FUSE_DUP_CAP: {HINT}"
    assert re.search(rf"size_t vcap = {VH.FUSE_TABLE_MIN};\s*while \(vcap < 2 \* sm->capacity\) vcap <<= 1;", fuse), f"fusion table size: {HINT}"
    assert "> mask - mask / 4) atomicOr(status, ST_HASH_FULL)" in fuse, f"fusion fill limit: {HINT}"
    fv = body(fuse, "fv_find_or_insert")
    assert "(size_t)voxel_key_hash(key) & mask" in fv and "s = (s + 1) & mask" in fv, f"fusion home slot / linear probe ({fv}): {HINT}"
    assert "> cap - cap / 8) atomicOr(status, ST_HASH_FULL)" in fuse, f"dense fill limit: {HINT}"
    assert "> cap - cap / 8) atomicOr(status, ST_HASH_FULL)" in vmap, f"voxel-map fill limit: {HINT}"
    dense_sizes = re.findall(r"dense_init\(h, sm, \(size_t\)1 << (\d+),", capi)
    assert dense_sizes and set(dense_sizes) == {str(VH.DENSE_SLOTS.bit_length() - 1)}, f"dense slots {dense_sizes}: {HINT}"
    # the dense map probes with the shared mask probe (its slot count is a power of two), home slot hash & (slots - 1)
    assert "voxel_key_claim(keys, cap - 1, key, &fresh)" in body(fuse, "dense_add_point"), f"dense insert probe: {HINT}"
    assert "voxel_key_find(keys, cap - 1, voxel_key_pack(kx, ky, kz))" in body(fuse, "dense_find_key"), f"dense carve probe: {HINT}"
    assert fuse.count("voxel_key_find(keys, cap - 1, key)") == 2, f"dense query / remove probe: {HINT}"
    assert "% cap" not in fuse, f"dense home slot: {HINT}"
    grow = rf"size_t cap = {VH.SCRATCH_TABLE_MIN};\s*while \(cap < 2 \* "
    assert re.search(grow + r"n_max\) cap <<= 1;", carve), f"sparse-carve table size: {HINT}"
    assert re.search(grow + r"\(ns \+ nt\)\) cap <<= 1;", overlap), f"overlap table size: {HINT}"
    assert re.search(grow + r"capacity_voxels\) cap <<= 1;", vmap), f"voxel-map table size: {HINT}"
    assert re.search(grow + r"n_max\) cap <<= 1;", fuse.split("op_dense_carve")[-1]), f"dense-carve ray table size: {HINT}"
    ray = body(fuse, "ray_home")
    assert "voxel_key_hash(" in ray and "& m) << 42" in ray and f"+ {VH.OFFSET}u" in ray, f"dense-carve home slot ({ray}): {HINT}"


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
