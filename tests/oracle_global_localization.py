"""CPU restatement of b2s_submap_global_localization (include/b2s.h, steps 1-6; DESIGN.md row M3) for the tests (test infrastructure,
never imported by the package):

- rotations(), grid(): the hypothesis grid and the R_j table, built with Python's math as the library builds it with the C library.
- scores(): hits(h) of every hypothesis by the C restatement in tests/oracle_global_localization.c (OpenMP over hypotheses): the ground
  truth of the device's score kernel.  scores_np(): an independent numpy twin (a set of packed voxel keys) for small boxes.
- candidates(): the (hits desc, h asc) order, the pool of 64 n_candidates and the greedy suppression.
- decide(): winner, found and runner-up over the refined candidates.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import tempfile
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oracle_global_localization.c")
_lib = None
KEY_LIMIT = 1048575.0
TWO_PI = 2.0 * math.pi
POOL_PER_CANDIDATE = 64


def lib():
    """Compiles oracle_global_localization.c in a temporary directory and loads it (the tree stays untouched)."""
    global _lib
    if _lib is None:
        with tempfile.TemporaryDirectory(prefix="b2s_oracle_gl_") as tmp:
            out = os.path.join(tmp, "liboracle_gl.so")
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fopenmp", "-Wall", _SRC, "-o", out, "-lm"])
            _lib = C.CDLL(out)
            _lib.gl_scores.restype = C.c_int
            _lib.gl_scores.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p] + [C.c_double] * 5 + [C.c_int] * 4 + \
                [C.c_double, C.c_void_p]
    return _lib


@dataclass
class Params:
    """b2s_global_localization_params with its defaults (x_min > x_max: the live extent of the map)"""
    x_min: float = 1.0
    x_max: float = -1.0
    y_min: float = 1.0
    y_max: float = -1.0
    step: float = 0.25
    z0: float = 0.0
    z_step: float = 0.25
    n_z: int = 1
    n_yaw: int = 144
    yaw0: float = -math.pi
    yaw_step: float = TWO_PI / 144.0
    roll: float = 0.0
    pitch: float = 0.0
    score_voxel: float = 1.0
    n_candidates: int = 16
    nms_distance: float = 1.0
    nms_yaw: float = math.radians(10.0)

    @classmethod
    def of(cls, g):   # from engine.GlobalLocalizationParameters
        return cls(g.xMin, g.xMax, g.yMin, g.yMax, g.step, g.z0, g.zStep, g.nZ, g.nYaw, g.yaw0, g.yawStep, g.roll, g.pitch, g.scoreVoxel,
                   g.nCandidates, g.nmsDistance, g.nmsYaw)


@dataclass
class Grid:
    x_min: float
    y_min: float
    nx: int
    ny: int
    n_yaw: int
    n_z: int

    @property
    def n(self) -> int:
        return self.nx * self.ny * self.n_yaw * self.n_z


def _mul3(A, B):
    return [[(A[r][0] * B[0][c] + A[r][1] * B[1][c]) + A[r][2] * B[2][c] for c in range(3)] for r in range(3)]


def yaw_of(p: Params, j: int) -> float:
    return p.yaw0 + j * p.yaw_step


def rotations(p: Params) -> np.ndarray:
    """R_j = (Rz(yaw_j) Ry(pitch)) Rx(roll), n_yaw x 9 row-major"""
    cp, sp, cr, sr = math.cos(p.pitch), math.sin(p.pitch), math.cos(p.roll), math.sin(p.roll)
    Ry = [[cp, 0.0, sp], [0.0, 1.0, 0.0], [-sp, 0.0, cp]]
    Rx = [[1.0, 0.0, 0.0], [0.0, cr, -sr], [0.0, sr, cr]]
    out = np.zeros((p.n_yaw, 9))
    for j in range(p.n_yaw):
        y = yaw_of(p, j)
        cy, sy = math.cos(y), math.sin(y)
        Rz = [[cy, -sy, 0.0], [sy, cy, 0.0], [0.0, 0.0, 1.0]]
        out[j] = np.array(_mul3(_mul3(Rz, Ry), Rx)).reshape(9)
    return out


def live(map_xyz: np.ndarray) -> np.ndarray:
    return map_xyz[np.isfinite(map_xyz).all(axis=1)]


def grid(p: Params, map_xyz: np.ndarray) -> Grid:
    x_min, x_max, y_min, y_max = p.x_min, p.x_max, p.y_min, p.y_max
    if x_min > x_max:
        lv = live(map_xyz)
        x_min, x_max, y_min, y_max = lv[:, 0].min(), lv[:, 0].max(), lv[:, 1].min(), lv[:, 1].max()
    return Grid(float(x_min), float(y_min), int(math.floor((x_max - x_min) / p.step)) + 1, int(math.floor((y_max - y_min) / p.step)) + 1,
                p.n_yaw, p.n_z)


def decode(p: Params, g: Grid, h: int):
    """(t, yaw, j) of hypothesis h"""
    ix, r = h % g.nx, h // g.nx
    iy, r = r % g.ny, r // g.ny
    j, iz = r % g.n_yaw, r // g.n_yaw
    t = np.array([g.x_min + ix * p.step, g.y_min + iy * p.step, p.z0 + iz * p.z_step])
    return t, yaw_of(p, j), j


def pose(p: Params, g: Grid, rot: np.ndarray, h: int) -> np.ndarray:
    t, _y, j = decode(p, g, h)
    T = np.eye(4)
    T[:3, :3] = rot[j].reshape(3, 3)
    T[:3, 3] = t
    return T


def scores(q: np.ndarray, map_xyz: np.ndarray, p: Params, g: Grid | None = None) -> np.ndarray:
    g = g or grid(p, map_xyz)
    q = np.ascontiguousarray(q, dtype=np.float64)
    m = np.ascontiguousarray(live(map_xyz), dtype=np.float64)
    rot = np.ascontiguousarray(rotations(p))
    hits = np.zeros(g.n, dtype=np.int32)
    rc = lib().gl_scores(q.ctypes.data, len(q), m.ctypes.data, len(m), rot.ctypes.data, g.x_min, g.y_min, p.step, p.z0, p.z_step,
                         g.nx, g.ny, g.n_yaw, g.n_z, p.score_voxel, hits.ctypes.data)
    assert rc == 0
    return hits


def _keys(xyz: np.ndarray, inv: float):
    f = np.floor(xyz * inv)
    ok = (np.abs(f) < KEY_LIMIT).all(axis=1)
    k = (f.astype(np.int64) + (1 << 20))
    return ok, (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]


def scores_np(q: np.ndarray, map_xyz: np.ndarray, p: Params, g: Grid | None = None) -> np.ndarray:
    """the numpy twin: packed keys of the live map voxels, np.isin per hypothesis"""
    g = g or grid(p, map_xyz)
    inv = 1.0 / p.score_voxel
    ok, mk = _keys(live(map_xyz), inv)
    occ = np.unique(mk[ok])
    rot = rotations(p)
    hits = np.zeros(g.n, dtype=np.int32)
    for h in range(g.n):
        t, _y, j = decode(p, g, h)
        R = rot[j]
        rq = np.stack([(R[0] * q[:, 0] + R[1] * q[:, 1]) + R[2] * q[:, 2], (R[3] * q[:, 0] + R[4] * q[:, 1]) + R[5] * q[:, 2],
                       (R[6] * q[:, 0] + R[7] * q[:, 1]) + R[8] * q[:, 2]], axis=1)
        ok_q, qk = _keys(rq + t, inv)
        hits[h] = int(np.count_nonzero(ok_q & np.isin(qk, occ)))
    return hits


def close(p: Params, ta, ya, tb, yb) -> bool:
    """within nms_distance in translation and nms_yaw in wrapped yaw"""
    d = ta - tb
    dist = math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    return dist <= p.nms_distance and abs(math.remainder(ya - yb, TWO_PI)) <= p.nms_yaw


def order(hits: np.ndarray) -> np.ndarray:
    """hypothesis indices by (hits descending, h ascending)"""
    return np.lexsort((np.arange(len(hits)), -hits.astype(np.int64)))


def candidates(hits: np.ndarray, p: Params, g: Grid) -> list[int]:
    """greedy suppression over the first 64 n_candidates hypotheses of order(hits)"""
    pool = order(hits)[:POOL_PER_CANDIDATE * p.n_candidates]
    kept: list[tuple[int, np.ndarray, float]] = []
    for h in pool:
        if len(kept) >= p.n_candidates:
            break
        t, y, _j = decode(p, g, int(h))
        if not any(close(p, t, y, kt, ky) for _h, kt, ky in kept):
            kept.append((int(h), t, y))
    return [h for h, _t, _y in kept]


def decide(Ts, fitness, p: Params, min_fitness: float):
    """(winner rank, found, runner-up fitness) over the refined candidates (T_k, fitness_k) in rank order"""
    if not len(fitness):
        return -1, False, -1.0
    w = 0
    for k in range(1, len(fitness)):
        if fitness[k] > fitness[w]:
            w = k
    yw = math.atan2(Ts[w][1][0], Ts[w][0][0])
    ru = -1.0
    for k in range(len(fitness)):
        d = np.asarray(Ts[k])[:3, 3] - np.asarray(Ts[w])[:3, 3]
        dist = math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
        dyaw = abs(math.remainder(math.atan2(Ts[k][1][0], Ts[k][0][0]) - yw, TWO_PI))
        if (dist > p.nms_distance or dyaw > p.nms_yaw) and fitness[k] > ru:
            ru = float(fitness[k])
    return w, bool(fitness[w] >= min_fitness), ru
