"""Loop-closure refinement with each estimator: point-to-plane, point-to-point and generalized ICP, the one batched call against the
per-cloud composition with the same estimator.

Submaps and candidates are those of tools/loop_closure_refinement_bench.py: Config4's 20 m-radius targets (6 scans 2 m apart fused at
their true poses with S1 at ratio 1 + F1) at the centres t0 - 8 .. t0 + 8 of the closed lap, and the place t0 revisited with other
noise seeds as the source; the identity is every candidate's true sourceToTarget and the guess of both arms; the K candidates are the
K centres nearest t0.  For every estimator and K in {1, 4, 16}:
    (a) slam.DeviceBackend: submap_as_cloud of the source and of every candidate, then slam.refineLoopClosures with the estimator
        (b2s_overlap per pair, one b2s_register_batch of that type, b2s_information_matrix per accepted pair)
    (b) slam.DeviceBackend.refine_loop_closures: one b2s_submap_loop_closure_refinement call with reg_type = the estimator
The arms alternate in one process; each time is the median of --reps host-clock readings around calls that end in a device
synchronisation, after --warmup calls of each arm.  Before any time is printed, (a) and (b) are checked to agree (overlap sizes and
accepted flags equal, ICP T / fitness / rmse within 1e-12, information within 1e-12 relative for accepted pairs).  Each row also gives
the ICP iterations of every pair.  The card's name and power limit are read in the same run.

    python tools/loop_closure_refinement_estimators_bench.py [--k 1 4 16] [--reps 7] [--warmup 2] [--out /tmp/lc_estimators.json]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import loop_closure_refinement_bench as B  # noqa: E402  (the submaps, the agreement check and the alternating timer)
from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import slam as S  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402

ESTIMATORS = ["PointToPlaneIcp", "PointToPointIcp", "GeneralizedIcp"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    p = E.MapperParameters(seed=3)
    p_full = copy.deepcopy(p)
    p_full.scanProcessing.downSamplingRatio = 1.0
    dev = B.ComposedBackend(p_full, carving=False, dense=False, graph=False)
    eng = dev.eng
    dev_name = B.card()
    lp = W.ClosedLoop()
    c4 = W.Config4(lp)
    K = max(a.k)
    t0 = 16
    offsets = sorted(range(-(K // 2), K - K // 2), key=lambda d: (abs(d), d))[:K]   # 0, -1, 1, -2, 2, ...
    cands = [B.build_submap(dev, lp, c4.target_positions(t0 + d), 5000) for d in offsets]
    src = B.build_submap(dev, lp, c4.target_positions(t0), 9000)
    sizes = [src.size()] + [c.size() for c in cands]
    v = p.mapBuilder.mapVoxelSize
    rows = []
    for reg in ESTIMATORS:
        lc = S.LoopClosureParameters(registrationType=reg)
        for k in a.k:
            tg, inits = cands[:k], [np.eye(4)] * k
            arm_a = lambda: B.ComposedBackend.refine_loop_closures(dev, src, tg, inits, v, lc)
            arm_b = lambda: S.DeviceBackend.refine_loop_closures(dev, src, tg, inits, v, lc)
            ra, rb = arm_a(), arm_b()
            B.agree(ra, rb)
            ta, tb = B.median_pair(arm_a, arm_b, eng, a.reps, a.warmup)
            row = {"estimator": reg, "K": k, "a_composition_ms": round(ta, 3), "b_batched_ms": round(tb, 3), "speedup": round(ta / tb, 2),
                   "iters": [int(r["result"].iters) for r in rb], "fitness": [round(float(r["result"].fitness_), 4) for r in rb],
                   "overlap_source": [r["n_source_overlap"] for r in rb], "accepted": [bool(r["accepted"]) for r in rb]}
            rows.append(row)
            print(json.dumps(row), flush=True)
    summary = {"card": dev_name, "submap_points": sizes, "reps": a.reps, "warmup": a.warmup, "rows": rows}
    print(json.dumps({k: x for k, x in summary.items() if k != "rows"}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)
    dev.close()


if __name__ == "__main__":
    main()
