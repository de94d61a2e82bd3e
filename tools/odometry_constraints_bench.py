"""Odometry constraints between consecutive 20 m submaps of the closed lap: the composition of the existing entry points against the
batched in-place call, and the information-matrix kernels on their own.

Submaps: Config4's 20 m-radius targets (6 scans 2 m apart fused at their true poses with S1 at ratio 1 + F1), built for consecutive
centres t = 0 .. P, kept resident; pair k = (submap k = parent, submap k + 1 = child).  For P in {1, 4, 16} and refinement off / on:
    (a) per pair: b2s_submap_to_cloud x 2, b2s_overlap (identity, 20 x map voxel), [b2s_register point-to-plane from I, r = 1.5 x map
        voxel, 100 iterations], b2s_information_matrix -- one pair after the other
    (b) one b2s_submap_odometry_constraints call for all P pairs
Each time is the median of --reps host-clock readings around calls that end in a device synchronisation, after --warmup calls.
Kernel times of the information matrix alone (refinement off): the ICP kernel group of the handle's CUDA-event profile
(b2s_profile_read), i.e. K-icp-iter's one-cluster evaluation in (a) and K-info-wide + its per-pair reduction in (b).  For context, one
pair through the C oracle on one host core (OMP_NUM_THREADS=1).  The card's name and power limit are read in the same run.

    python tools/odometry_constraints_bench.py [--pairs 1 4 16] [--reps 7] [--warmup 2] [--out /tmp/odometry_constraints.json]
"""
from __future__ import annotations

import os

os.environ.setdefault("OMP_NUM_THREADS", "1")   # the oracle's context number is one host core

import argparse
import json
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "not available"


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def build_submaps(eng, n):
    lp = W.ClosedLoop()
    c4 = W.Config4(lp)
    params = eng.params
    p_full = E.MapperParameters(seed=3)
    p_full.scanProcessing.downSamplingRatio = 1.0   # submaps keep every voxel of the scans they fuse (as Config4.build_target)
    eng.set_parameters(p_full)
    icp = E.ScanToMapIcp(eng)
    sms = []
    for t in range(n):
        sm = E.Submap(eng, 900_000)
        for k in c4.target_positions(t):
            raw = eng.cloud(lp.scan(k, seed=5000 + (k % lp.L)))
            ps = icp.processForScanMatchingAndMerging(raw)
            sm.insertScan(None, ps.merge_, lp.pose(k))
            raw.free(); ps.merge_.free(); ps.match_.free()
        sms.append(sm)
    eng.set_parameters(params)
    return sms


def composition(eng, parents, children, prm, reg):
    r = prm.voxelExpansionFactorIcpCorrespondenceDistance * prm.mapVoxelSize
    out = []
    for p, c in zip(parents, children):
        sc, tc = p.toCloud(), c.toCloud()
        so, to = E.computeOverlappingClouds(eng, sc, tc, np.eye(4), prm.voxelExpansionFactorOverlapComputation * prm.mapVoxelSize, 1)
        T = reg.registerClouds(so, to, np.eye(4)).transformation_ if reg is not None else np.eye(4)
        out.append(E.getInformationMatrixFromPointClouds(eng, so, to, r, T))
        for x in (sc, tc, so, to):
            x.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    eng = E.Engine(E.MapperParameters(seed=3))
    dev_name = card()
    P = max(a.pairs)
    sms = build_submaps(eng, P + 1)
    sizes = [s.size() for s in sms]
    rows = []
    for refine in (False, True):
        prm = E.OdometryConstraintParameters(isRefineOdometryConstraintsBetweenSubmaps=refine)
        reg = None
        if refine:
            pc = E.CloudRegistrationParameters(icp=E.IcpParameters(maxNumIter=prm.maxNumIter, maxCorrespondenceDistance=1.5 * prm.mapVoxelSize))
            reg = E.RegistrationIcpPointToPlane(eng, pc)
        for n in a.pairs:
            par, chi = sms[:n], sms[1:n + 1]
            res = E.buildOdometryConstraintsBatch(eng, par, chi, prm)
            ref = composition(eng, par, chi, prm, reg)
            worst = max(float(np.abs(x.informationMatrix_ - y).max() / np.abs(y).max()) for x, y in zip(res, ref))
            ta = median_ms(lambda: composition(eng, par, chi, prm, reg), a.reps, a.warmup)
            tb = median_ms(lambda: E.buildOdometryConstraintsBatch(eng, par, chi, prm), a.reps, a.warmup)
            row = {"pairs": n, "refine": refine, "a_composition_ms": round(ta, 3), "b_batched_ms": round(tb, 3), "speedup": round(ta / tb, 2),
                   "overlap_source": [r.nSourceOverlap for r in res], "overlap_target": [r.nTargetOverlap for r in res],
                   "info_max_rel_diff_a_vs_b": worst}
            if not refine:   # the information-matrix kernels alone, CUDA events of the handle's profile (ICP group)
                so = [E.Cloud(eng) for _ in par]; to = [E.Cloud(eng) for _ in par]
                E.buildOdometryConstraintsBatch(eng, par, chi, prm, so, to)
                eng.synchronize()
                eng.profile_enable(True)
                eng.profile_read()
                for _ in range(a.reps):
                    E.buildOdometryConstraintsBatch(eng, par, chi, prm)
                kb = eng.profile_read()["icp"]
                for _ in range(a.reps):
                    for x, y in zip(so, to):
                        E.getInformationMatrixFromPointClouds(eng, x, y, 1.5 * prm.mapVoxelSize, np.eye(4))
                ka = eng.profile_read()["icp"]
                eng.profile_enable(False)
                row["info_kernel_ms_cluster_a"] = round(ka[0] / a.reps, 3)
                row["info_kernel_ms_wide_b"] = round(kb[0] / a.reps, 3)
            rows.append(row)
            print(json.dumps(row), flush=True)
    # context: one pair through the C oracle on one host core
    from oracle import oracle as O  # noqa: E402 (test infrastructure, built by __graft_entry__.build)
    (px, pn), (cx, cn) = sms[0].getMapPointCloud(), sms[1].getMapPointCloud()
    t0 = time.perf_counter()
    fs, ft = O.overlap_flags(px, cx, np.eye(4), 2.0, 1)
    O.information_matrix(px[fs], cx[ft], 0.15, np.eye(4))
    t_oracle = (time.perf_counter() - t0) * 1e3
    summary = {"card": dev_name, "submap_points": sizes, "oracle_one_pair_one_core_ms": round(t_oracle, 1), "reps": a.reps, "warmup": a.warmup,
               "rows": rows}
    print(json.dumps({k: v for k, v in summary.items() if k != "rows"}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
