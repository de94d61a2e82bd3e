"""The session-capable oracle backend with localisation mode (rules 2-3 of M2) and global localisation over a set of submaps
(b2s_submaps_global_localization, DESIGN.md row M4) restated (TEST INFRASTRUCTURE), so SegmentMapper.relocalize runs on the CPU.

    rules 1-4   tests/oracle_global_localization.{c,py} on the concatenation of the submaps' live points
    assignment  closest(): SubmapCollection::findClosestSubmap (src/SubmapCollection.cpp:147-158) for each candidate's translation
    rule 5      ScanToMapRegistration on the candidate's submap: the scan-matcher crop around T_c, then point-to-plane ICP from T_c
    rule 6      oracle_global_localization.decide
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

import oracle_global_localization as G
from oracle import oracle as O
from oracle_backend import OracleCloud
from oracle_backend_localization import OracleLocalizationBackend
from oracle_backend_session import SessionOracleBackend
from open3d_slam_b200 import engine as E


def closest(t, centers) -> int:
    """the first submap whose centre is nearest to t, the distance summed as sqrt((dx^2 + dy^2) + dz^2)"""
    best, best_d = 0, 0.0
    for s, c in enumerate(np.asarray(centers, dtype=np.float64).reshape(-1, 3)):
        d = [float(t[0] - c[0]), float(t[1] - c[1]), float(t[2] - c[2])]
        dist = math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
        if s == 0 or dist < best_d:
            best, best_d = s, dist
    return best


def union_points(sms) -> np.ndarray:
    """the live points of every submap, concatenated in submap order"""
    parts = [G.live(sm.xyz) for sm in sms]
    return np.concatenate(parts) if parts else np.zeros((0, 3))


@dataclass
class Candidate:
    T_hypothesis: np.ndarray
    hypothesis: int
    hits: int
    icp: object


@dataclass
class Result:
    """the fields of engine.SubmapsGlobalLocalizationResult"""
    found: bool
    T: np.ndarray
    fitness: float
    inlier_rmse: float
    runner_up_fitness: float
    winner_rank: int
    n_hypotheses: int
    n_query: int
    candidates: list = field(default_factory=list)
    candidate_submaps: list = field(default_factory=list)
    winner_submap: int = -1


class RelocalizationOracleBackend(OracleLocalizationBackend, SessionOracleBackend):
    def query(self, raw, score_voxel: float) -> np.ndarray:
        """rule 1: the scan-matcher crop at identity, then VoxelDownSample(score_voxel)"""
        cropped, _ = O.crop(self.narrow, np.asarray(raw, dtype=np.float32).astype(np.float64))
        return O.voxel_down_sample(cropped, score_voxel)[0]

    def union_scores(self, sms, raw, params=None):
        """rules 1-3 over the union: (hits, query, grid)"""
        p = G.Params.of(params or E.GlobalLocalizationParameters())
        pts = union_points(sms)
        if len(pts) == 0:
            raise ValueError("every submap is empty")
        q = self.query(raw, p.score_voxel)
        g = G.grid(p, pts)
        return G.scores(q, pts, p, g), q, g

    def global_localization_submaps(self, sms, centers, raw, params=None) -> Result:
        gp = params or E.GlobalLocalizationParameters()
        p = G.Params.of(gp)
        hits, q, g = self.union_scores(sms, raw, gp)
        rot = G.rotations(p)
        _merge, (ax, _an) = self._process(raw)
        cands, owners, Ts, fits = [], [], [], []
        for h in G.candidates(hits, p, g):
            Tc = G.pose(p, g, rot, h)
            s = closest(Tc[:3, 3], centers)
            patch = self._cropper(self.p.scanProcessing.cropper, center=Tc[:3, 3])
            px, pn = O.crop(patch, sms[s].xyz, sms[s].nrm)
            if len(px) == 0:
                r = O.IcpResult(Tc.copy(), 0.0, 0.0, 0, 0, None)
            else:
                r = O.registration_icp_p2plane(ax, px, pn, self.p.icp.maxCorrespondenceDistance, Tc, max_iter=self.p.icp.maxNumIter)
            r.transformation_ = r.T; r.fitness_ = r.fitness; r.inlier_rmse_ = r.inlier_rmse
            cands.append(Candidate(Tc, int(h), int(hits[h]), r))
            owners.append(s); Ts.append(r.T); fits.append(r.fitness)
        w, found, ru = G.decide(Ts, fits, p, self.p.minRefinementFitness)
        if w < 0:
            return Result(False, np.zeros((4, 4)), 0.0, 0.0, -1.0, -1, g.n, len(q), [], [], -1)
        return Result(found, np.array(Ts[w]), float(fits[w]), float(cands[w].icp.inlier_rmse), ru, w, g.n, len(q), cands, owners, owners[w])

    def first_scan_at(self, sm, raw, T):
        (mx, mn), _ = self._process(raw)
        self._insert(sm, mx, mn, np.asarray(T))
        self.pose = np.array(T, dtype=np.float64)
        return OracleCloud(mx, mn)

    def restart_odometry(self, T):
        """the oracle runs addRangeMeasurement only: its odometry state is Mapper::mapToRangeSensorPrev_, which
        set_initial_transform sets"""
        self.pose = np.array(T, dtype=np.float64)
