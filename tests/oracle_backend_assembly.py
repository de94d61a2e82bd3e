"""The oracle backend with the assembled map (TEST INFRASTRUCTURE), and the numpy restatement of its rules (DESIGN.md row A1):
Mapper::getAssembledMapPointCloud (core/src/Mapper.cpp:183-208) is the concatenation of the submaps' maps in list order; the normals rule
keeps the normals only when every submap that contributes a point has them; voxelize is oracle.voxel_down_sample; the coloured map
(ros/open3d_slam_ros/src/helpers_ros.cpp:51-70) gives submap j the float32 colour getColor(j % 11 + 2), averaged per voxel in input
order -- the counterpart of slam.DeviceBackend.assembled_map / assembled_colored_map."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O
from oracle_backend import OracleBackend, OracleCloud

# Color.hpp:22-32 as std_msgs/ColorRGBA stores them (float32), promoted to double
PALETTE = np.array([[0.5, 0.5, 0.5], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, 0.5, 0], [0.5, 0, 1], [0.5, 1, 0], [0, 1, 1],
                    [1, 0, 0.5], [0.78, 0, 0.9]], dtype=np.float32).astype(np.float64)


def assemble(maps):
    """maps: [(xyz, normals or None)] in submap order -> (xyz, normals or None, submap index per point)"""
    xs = [np.asarray(x, dtype=np.float64).reshape(-1, 3) for x, _ in maps]
    xyz = np.concatenate(xs) if xs else np.zeros((0, 3))
    sub = np.concatenate([np.full(len(x), j, dtype=np.int64) for j, x in enumerate(xs)]) if xs else np.zeros(0, dtype=np.int64)
    contributing = [n for x, n in zip(xs, (n for _, n in maps)) if len(x)]
    # a map without normals: none given, or stored as NaN (a point-to-point map on the device)
    has = len(xyz) > 0 and all(n is not None and not np.isnan(n).all() for n in contributing)
    nrm = np.concatenate([np.asarray(n, dtype=np.float64).reshape(-1, 3) for x, n in zip(xs, (n for _, n in maps)) if len(x)]) if has else None
    return xyz, nrm, sub


def voxel_keys(xyz, voxel):
    """[O3D] VoxelDownSample's key of every point: floor((p - (min - v/2)) / v)"""
    vmin = xyz.min(axis=0) - voxel * 0.5
    return np.floor((xyz - vmin) / voxel).astype(np.int64)


def colored(maps, voxel):
    """(xyz, rgb) of assembleColoredPointCloud + voxelize(voxel); voxels in ascending key order"""
    xyz, _n, sub = assemble(maps)
    rgb = PALETTE[sub % 11]
    if voxel <= 0.0 or len(xyz) == 0:
        return xyz, rgb
    uk, inv = np.unique(voxel_keys(xyz, voxel), axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    cnt = np.bincount(inv, minlength=len(uk)).astype(np.float64)[:, None]
    sx = np.zeros((len(uk), 3)); sc = np.zeros((len(uk), 3))
    np.add.at(sx, inv, xyz)   # unbuffered, in index order: AccumulatedPoint's running sums
    np.add.at(sc, inv, rgb)
    return sx / cnt, sc / cnt


def assembled(maps, voxel):
    """(xyz, normals or None) of getAssembledMapPointCloud + voxelize(voxel), the voxel path through the oracle"""
    xyz, nrm, _ = assemble(maps)
    if voxel <= 0.0 or len(xyz) == 0:
        return xyz, nrm
    return O.voxel_down_sample(xyz, voxel, nrm)


class AssemblyOracleBackend(OracleBackend):
    def map_size(self, sm):
        return len(sm.xyz)

    def assembled_map(self, sms, voxelSize):
        return OracleCloud(*assembled([(s.xyz, s.nrm) for s in sms], voxelSize))

    def assembled_colored_map(self, sms, voxelSize):
        x, rgb = colored([(s.xyz, s.nrm) for s in sms], voxelSize)
        return OracleCloud(x), rgb
