"""Wall clock of SegmentMapper on the closed lap with SlamWrapper's loop-closure schedule off and on (isAttemptLoopClosures), and the
breakdown of every attempt that ran: features, RANSAC, refinement, odometry
constraints, pose-graph solve and correction (submap transforms + the mapper's pose).  Device backend, 10 m submaps, carving and dense
map on, CUDA graph replay; host clock around each backend call with a device synchronise after it.
usage: python tools/loop_closing_mapper_bench.py [--scans 208] [--repeats 2]
prints one JSON line
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W

PHASES = {"compute_features": "features", "ransac": "ransac", "refine_loop_closures": "refinement",
          "odometry_constraints": "odometry_constraints", "global_optimization": "solve", "transform_submap": "correction",
          "loop_closure_update": "correction"}


def timed_backend(be, sink):
    """wrap the backend's loop-closure calls: each one's wall clock (ending in a device synchronise) goes to sink[phase]"""
    for name, phase in PHASES.items():
        fn = getattr(be, name)

        def wrapper(*a, _fn=fn, _phase=phase, **kw):
            t0 = time.perf_counter()
            out = _fn(*a, **kw)
            be.eng.synchronize()
            sink[_phase] = sink.get(_phase, 0.0) + (time.perf_counter() - t0) * 1e3
            return out
        setattr(be, name, wrapper)


def run(lp, n_scans, on: bool, search_radius: float):
    p = E.MapperParameters(seed=3)
    be = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=True)
    lcp = S.LoopClosingParameters.fromMapperParameters(p)
    lcp.candidates.loopClosureSearchRadius = search_radius
    m = S.SegmentMapper(be, S.SubmapParameters(radius=10.0), isAttemptLoopClosures=on, loopClosing=lcp)
    sink, attempts, per_scan = {}, [], []
    timed_backend(be, sink)
    scans = [(lp.scan(k, seed=k), lp.delta(k)) for k in range(n_scans)]
    for k, (raw, d) in enumerate(scans):
        sink.clear()
        t0 = time.perf_counter()
        m.addRangeMeasurement(raw, d)
        be.eng.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        per_scan.append(ms)
        if sink:
            attempts.append({"scan": k, "ms_scan_total": ms, **{ph: round(v, 3) for ph, v in sink.items()}})
    truth = [lp.map_frame_pose(k) for k in range(n_scans)]
    err = float(np.mean([np.linalg.norm(P[:3, 3] - G[:3, 3]) for P, G in zip(m.poses, truth)]))
    ev = m.submaps.events
    a = np.array(per_scan[5:])
    out = {"loop_closing": on, "ms_per_scan_mean": float(a.mean()), "ms_per_scan_median": float(np.median(a)),
           "ms_per_scan_p95": float(np.percentile(a, 95)), "ms_per_scan_max": float(a.max()), "ms_total": float(sum(per_scan)),
           "submaps": len(m.submaps.submaps), "mean_translation_error_m": err,
           "candidates": [e[3] for e in ev if e[0] == "loop_closure_candidates" and e[3]],
           "decisions": [[(i, d) for i, d, _n in e[3]] for e in ev if e[0] == "loop_closure_decisions" and e[3]],
           "corrections": [(e[1], e[2]) for e in ev if e[0] == "loop_closure_correction"],
           "attempts": [a_ for a_ in attempts if on]}
    be.close()
    return out


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=208)
    ap.add_argument("--repeats", type=int, default=2)
    # 10 m: on this 16 m courtyard loop the default 20 m reaches submaps across the courtyard, whose maps can alias
    ap.add_argument("--search-radius", type=float, default=10.0)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("loop_closing_mapper_bench: no CUDA device")
    lp = W.ClosedLoop()
    run(lp, 20, False, args.search_radius)   # warm-up: module load, graph capture paths
    runs = []
    for r in range(args.repeats):   # alternate off / on
        runs.append(run(lp, args.scans, False, args.search_radius))
        runs.append(run(lp, args.scans, True, args.search_radius))
    print(json.dumps({"gpu": gpu_info(), "scans": args.scans, "submap_radius_m": 10.0, "search_radius_m": args.search_radius, "runs": runs}))


if __name__ == "__main__":
    main()
