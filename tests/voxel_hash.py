"""The rules of the map-side voxel hashes, restated for the tests that aim at their edges.

Six open-addressing tables share one key scheme: the voxel index floor(p * (1/v)) on the global-origin grid, three 21-bit fields
offset by 2^20 in one 64-bit word, hashed by the murmur3 finalizer, linear probing.  They differ in their size:

    fusion hash     (fuse.cu, K-fuse)         4096 slots, doubled while < 2 x submap capacity; full past mask - mask / 4
    dense map       (fuse.cu, F3 / F2)        2^22 slots; full past 7/8 of them
    dense-carve rays(fuse.cu, C2)             1024 slots, doubled while < 2 x scan points; a key is three full int32 there
    sparse carve    (carve.cu, C1)            1024 slots, doubled while < 2 x map points
    overlap         (overlap.cu)              1024 slots, doubled while < 2 x (source + target points)
    voxel map       (voxelmap.cu)             1024 slots, doubled while < 2 x capacity_voxels; full past 7/8 of them

A key index is accepted while |floor(p * (1/v))| < KEY_LIMIT on every axis.  The finalizer is a bijection, so fmix64_inv gives the
keys whose home slot is any chosen slot.  The key, the hash and the probes are defined once, in open3d_slam_b200/csrc/common.cuh
(voxel_key_*); the sizes and fill limits live with each table.  test_voxel_hash_rules.py checks these constants against the CUDA
sources, so a change there fails loudly instead of turning the collision tests into ordinary ones.
"""
from __future__ import annotations

import numpy as np

FIELD_BITS = 21
OFFSET = 1 << 20
KEY_LIMIT = (1 << 20) - 1
M1, M2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
M1_INV, M2_INV = 0x4F74430C22A54005, 0x9CB4B2F8129337DB
U64 = (1 << 64) - 1

FUSE_DUP_CAP = 1 << 16
FUSE_TABLE_MIN = 4096
DENSE_SLOTS = 1 << 22
SCRATCH_TABLE_MIN = 1024


def pack(x: int, y: int, z: int) -> int:
    return ((x + OFFSET) << 42) | ((y + OFFSET) << 21) | (z + OFFSET)


def unpack(k: int) -> tuple[int, int, int]:
    f = (1 << FIELD_BITS) - 1
    return ((k >> 42) & f) - OFFSET, ((k >> 21) & f) - OFFSET, (k & f) - OFFSET


def fmix64(k: int) -> int:
    k ^= k >> 33; k = (k * M1) & U64; k ^= k >> 33; k = (k * M2) & U64; k ^= k >> 33
    return k


def fmix64_inv(h: int) -> int:
    h ^= h >> 33; h = (h * M2_INV) & U64; h ^= h >> 33; h = (h * M1_INV) & U64; h ^= h >> 33
    return h


def valid_key(k: int) -> bool:
    """k is the packed form of an accepted voxel index (bit 63 clear, every field within the key limit)."""
    return k >> 63 == 0 and all(abs(c) < KEY_LIMIT for c in unpack(k)) and pack(*unpack(k)) == k


def home(key_index, slots: int) -> int:
    return fmix64(pack(*key_index)) & (slots - 1)


def grown(minimum: int, n: int) -> int:
    """Slots of a table that starts at `minimum` and doubles while it is smaller than 2 n."""
    cap = minimum
    while cap < 2 * n:
        cap <<= 1
    return cap


def fusion_slots(capacity: int) -> int:
    return grown(FUSE_TABLE_MIN, capacity)


def dense_fill_limit(slots: int = DENSE_SLOTS) -> int:
    """Most distinct voxels a 7/8-full table takes (voxel map, dense map)."""
    return slots - slots // 8


def keys_homed_at(slot: int, slots: int, count: int, seed: int = 0, bound: int = KEY_LIMIT) -> list[tuple[int, int, int]]:
    """`count` distinct accepted voxel indices whose home slot is `slot`, every field within +-bound."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        h = (int(rng.integers(0, 1 << 62)) * slots + slot) & U64
        k = fmix64_inv(h)
        if valid_key(k) and all(abs(c) < bound for c in unpack(k)) and unpack(k) not in out:
            out.append(unpack(k))
    return out


def point_in(key_index, voxel: float) -> np.ndarray:
    """A point whose floor(p * (1/voxel)) is key_index, near the voxel's centre."""
    inv = 1.0 / voxel
    p = (np.asarray(key_index, dtype=np.float64) + 0.5) * voxel
    assert np.array_equal(np.floor(p * inv).astype(np.int64), np.asarray(key_index)), (key_index, p)
    return p


def key_of(p, voxel: float) -> tuple:
    return tuple(int(c) for c in np.floor(np.asarray(p, dtype=np.float64) * (1.0 / voxel)))
