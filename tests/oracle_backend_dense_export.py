"""The oracle backend with the dense-map export (TEST INFRASTRUCTURE), the counterpart of slam.DeviceBackend.dense_map_clouds (DESIGN.md
row A2): VoxelizedPointCloud::toPointCloud (core/src/Voxel.cpp:90-115) of every submap's dense map, restated by the oracle's DenseMap,
one n x 3 array per submap in list order; a submap without a dense map gives an empty array."""
from __future__ import annotations

import numpy as np

from oracle_backend import OracleBackend


def dense_cloud(sm):
    """toPointCloud of one oracle submap's dense map: the voxel means in the table's slot order"""
    return sm.dense.to_cloud()[0] if sm.dense is not None else np.zeros((0, 3))


class DenseExportOracleBackend(OracleBackend):
    def dense_map_clouds(self, sms):
        return [dense_cloud(s) for s in sms]
