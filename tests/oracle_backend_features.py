"""The oracle backend of tests/oracle_backend.py with the feature half of Submap::computeFeatures (TEST INFRASTRUCTURE):
compute_features = the C restatement of tests/oracle_submap_features.c, the counterpart of slam.DeviceBackend.compute_features
under slam.SubmapCollection.computeFeatures."""
from __future__ import annotations

import oracle_submap_features as OSF
from oracle_backend import OracleBackend, OracleCloud


class FeatureOracleBackend(OracleBackend):
    def compute_features(self, sm, params):
        """Submap::computeFeatures (Submap.cpp:239-244) over the C restatement: (sparse cloud, FPFH rows (n, 33))"""
        r = OSF.submap_features(sm.xyz, sm.nrm, params)
        return OracleCloud(r["xyz"], r["nrm"]), r["feature"]
