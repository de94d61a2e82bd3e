"""Loop-closure refinement of one 20 m submap against K candidates: today's composition against the one batched call, and the whole
buildLoopClosureConstraints with each.

Submaps: Config4's 20 m-radius targets (6 scans 2 m apart fused at their true poses with S1 at ratio 1 + F1) at the centres t0 - 8 ..
t0 + 8 of the closed lap, kept resident.  The source is the place t0 revisited: the same six positions scanned again with other noise
seeds, fused the same way.  Every map lives in the lap's frame, so the identity is each candidate's true sourceToTarget and the
initial guess of both arms; the K candidates are the K centres nearest t0 (t0 itself, the true closure, first), so their overlaps with
the source run from the whole map to a sliver.  For K in {1, 4, 16}:
    (a) slam.DeviceBackend: submap_as_cloud of the source and of every candidate, then slam.refineLoopClosures (b2s_overlap per pair,
        one b2s_register_batch, b2s_information_matrix per accepted pair)
    (b) slam.DeviceBackend.refine_loop_closures: one b2s_submap_loop_closure_refinement call
and slam.buildLoopClosureConstraints (RANSAC proposal, gates, refinement) with the refinement of (a) and of (b).  The arms alternate in
one process; each time is the median of --reps host-clock readings around calls that end in a device synchronisation, after --warmup
calls of each arm.  Before any time is printed, the outputs of (a) and (b) are checked to agree: overlap sizes and the accepted flags
equal, ICP T / fitness / rmse within 1e-12, information within 1e-12 relative (accepted pairs), the same decision log and constraints.
The card's name and power limit are read in the same run.

    python tools/loop_closure_refinement_bench.py [--k 1 4 16] [--reps 7] [--warmup 2] [--out /tmp/loop_closure_refinement.json]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import slam as S  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "not available"


class ComposedBackend(S.DeviceBackend):
    """arm (a): the refinement as buildLoopClosureConstraints composed it before the batched call"""

    def refine_loop_closures(self, source_sm, target_sms, inits, mapVoxelSize, lc=None):
        return S.refineLoopClosures(self, self.submap_as_cloud(source_sm), [self.submap_as_cloud(t) for t in target_sms], inits, mapVoxelSize, lc)


def build_submap(dev, lp, positions, seed0):
    eng = dev.eng
    icp = E.ScanToMapIcp(eng)
    sm = E.Submap(eng, 900_000)
    for k in positions:
        raw = eng.cloud(lp.scan(k, seed=seed0 + (k % lp.L)))
        ps = icp.processForScanMatchingAndMerging(raw)
        sm.insertScan(None, ps.merge_, lp.pose(k))
        raw.free(); ps.merge_.free(); ps.match_.free()
    return sm


def agree(a, b):
    """the tolerances of tests/test_gpu_loop_closure_refinement.py; the composition computes no information for a rejected pair"""
    for x, y in zip(a, b):
        assert (x["n_source_overlap"], x["n_target_overlap"], x["accepted"]) == (y["n_source_overlap"], y["n_target_overlap"], y["accepted"]), (x, y)
        assert np.abs(x["result"].transformation_ - y["result"].transformation_).max() <= 1e-12
        assert abs(x["result"].fitness_ - y["result"].fitness_) <= 1e-12 and abs(x["result"].inlier_rmse_ - y["result"].inlier_rmse_) <= 1e-12
        if x["accepted"]:
            d = np.abs(np.asarray(x["information"]) - np.asarray(y["information"])).max() / np.abs(np.asarray(x["information"])).max()
            assert d <= 1e-12, d


def median_pair(fa, fb, eng, reps, warmup):
    """alternating (a), (b): medians of host-clock readings around synchronised calls"""
    for _ in range(warmup):
        fa(); fb()
    ta, tb = [], []
    for _ in range(reps):
        for f, ts in ((fa, ta), (fb, tb)):
            eng.synchronize()
            t0 = time.perf_counter()
            f()
            eng.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ta)), float(np.median(tb))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    p = E.MapperParameters(seed=3)
    p_full = copy.deepcopy(p)
    p_full.scanProcessing.downSamplingRatio = 1.0   # submaps keep every voxel of the scans they fuse (as Config4.build_target)
    dev = ComposedBackend(p_full, carving=False, dense=False, graph=False)
    eng = dev.eng
    dev_name = card()
    lp = W.ClosedLoop()
    c4 = W.Config4(lp)
    K = max(a.k)
    t0 = 16
    offsets = sorted(range(-(K // 2), K - K // 2), key=lambda d: (abs(d), d))[:K]   # 0, -1, 1, -2, 2, ...
    cands = [build_submap(dev, lp, c4.target_positions(t0 + d), 5000) for d in offsets]
    src = build_submap(dev, lp, c4.target_positions(t0), 9000)
    sizes = [src.size()] + [c.size() for c in cands]
    pr = E.PlaceRecognitionParameters()
    # the records buildLoopClosureConstraints reads: the sparse cloud and the FPFH of every map
    coll = S.SubmapCollection(dev, S.SubmapParameters())
    for i, sm in enumerate([src] + cands):
        r = S.SubmapRecord(sm, i, 0, np.zeros(3))
        r.sparse, r.feature = dev.compute_features(sm, pr)
        coll.submaps.append(r)
    v = p.mapBuilder.mapVoxelSize
    rows = []
    for k in a.k:
        tg, inits = cands[:k], [np.eye(4)] * k
        arm_a = lambda: ComposedBackend.refine_loop_closures(dev, src, tg, inits, v)
        arm_b = lambda: S.DeviceBackend.refine_loop_closures(dev, src, tg, inits, v)
        ra, rb = arm_a(), arm_b()
        agree(ra, rb)
        ta, tb = median_pair(arm_a, arm_b, eng, a.reps, a.warmup)
        idx = list(range(1, 1 + k))
        build_a = lambda: S.buildLoopClosureConstraints(dev, coll, 0, idx, pr, v)
        build_b = lambda: S.buildLoopClosureConstraints(_AsDevice(dev), coll, 0, idx, pr, v)
        (ca, la), (cb, lb) = build_a(), build_b()
        assert la == lb and len(ca) == len(cb)
        for x, y in zip(ca, cb):
            assert np.abs(x.sourceToTarget - y.sourceToTarget).max() <= 1e-12
            assert np.abs(x.informationMatrix - y.informationMatrix).max() / np.abs(x.informationMatrix).max() <= 1e-12
        ba, bb = median_pair(build_a, build_b, eng, a.reps, a.warmup)
        row = {"K": k, "a_composition_ms": round(ta, 3), "b_batched_ms": round(tb, 3), "speedup": round(ta / tb, 2),
               "build_a_ms": round(ba, 3), "build_b_ms": round(bb, 3), "build_speedup": round(ba / bb, 2),
               "overlap_source": [r["n_source_overlap"] for r in rb], "overlap_target": [r["n_target_overlap"] for r in rb],
               "accepted": [bool(r["accepted"]) for r in rb], "log": [d for _, d, _ in lb]}
        rows.append(row)
        print(json.dumps(row), flush=True)
    summary = {"card": dev_name, "submap_points": sizes, "reps": a.reps, "warmup": a.warmup, "rows": rows}
    print(json.dumps({k: x for k, x in summary.items() if k != "rows"}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)
    dev.close()


class _AsDevice:
    """arm (b) of buildLoopClosureConstraints: the same backend object with DeviceBackend's own refine_loop_closures"""

    def __init__(self, dev):
        self._dev = dev

    def refine_loop_closures(self, *args, **kw):
        return S.DeviceBackend.refine_loop_closures(self._dev, *args, **kw)

    def __getattr__(self, name):
        return getattr(self._dev, name)


if __name__ == "__main__":
    main()
