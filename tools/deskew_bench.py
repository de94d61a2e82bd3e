#!/usr/bin/env python
"""What motion compensation (de-skew of both inputs, b2s_odometry_set_motion_compensation) adds per scan: the combined odometry +
mapper graph (b2s_slam_step_async, graph mode) with de-skew on against the same graph with it off.

Workload: odometry_bench.py's -- workloads.ClosedLoop steady state, Lua defaults, downsampling ratio 0.3 (--ratio), every chain
pre-grown over one lap (untimed), scans resident in HBM and copied into the graph's staging cloud; device time from CUDA events on the
main stream around every step (one scan per chain per step), after a warm-up of the same shape.  The step times of the two arms differ by
the de-skew launches AND by the ICP's work on the de-skewed scans (other iteration counts), so the de-skew kernels' own device time is
also read, with torch.profiler over replayed steps of one chain.  Prints one JSON line (and writes it to --out): ms per step and
scans/s at each chain count, kernel launches and graph captures per scan, the de-skew kernels' device time per scan, and the card
name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402
from odometry_bench import TICKS_PER_SCAN, Arm, card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", default="1,16")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--ratio", type=float, default=0.3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("deskew_bench.py: no CUDA device -- the b2s engine has no CPU fallback")
    chains = sorted(int(x) for x in args.chains.split(",") if x)
    n_max = max(chains)
    lp = W.ClosedLoop()
    sets = min(n_max, 4)
    clouds = [[lp.scan_moving(k, seed=1000 * s + k) for k in range(lp.L)] for s in range(sets)]
    params = E.MapperParameters(seed=3)
    params.scanProcessing.downSamplingRatio = args.ratio
    odo_params = E.OdometryParameters(seed=5)
    odo_params.scanProcessing.downSamplingRatio = args.ratio
    main_s = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in range(n_max)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    arms = {"deskew_off": Arm(True, n_max, lp, clouds, params, odo_params, streams, 900_000),
            "deskew_on": Arm(True, n_max, lp, clouds, params, odo_params, streams, 900_000)}
    mc = E.ConstantVelocityMotionCompensationParameters(isUndistortInputCloud=True)
    for arm in arms.values():
        for o in arm.odos:
            o.pushMapToRangeSensor(TICKS_PER_SCAN, np.eye(4))   # Mapper.cpp:112: the first scan's pose (Arm inserted it at this time)
    for o in arms["deskew_on"].odos:   # before any graph is captured: the first capture includes both de-skews
        o.setMotionCompensation(mc)
    for arm in arms.values():          # the rest of lap 0: the maps reach steady state
        timed(arm, n_max, lp.L - 1, main_s, streams, flush)
    result = {"tool": "deskew_bench", "workload": "workloads.ClosedLoop.scan_moving steady state (one lap pre-grown), Lua defaults, ratio %g"
              % args.ratio, "steps": args.steps, "warmup": args.warmup, "card": card()}
    for name, arm in arms.items():
        r = {}
        for n in chains:
            timed(arm, n, args.warmup, main_s, streams, flush)
            l0, c0 = arm.launches(n), arm.captures(n)
            ms = timed(arm, n, args.steps, main_s, streams, flush)
            r[str(n)] = {"scans_per_s": n * args.steps / (sum(ms) * 1e-3), "ms_per_step_median": float(np.median(ms)),
                         "launches_per_scan": (arm.launches(n) - l0) / (n * args.steps),
                         "captures_per_scan": (arm.captures(n) - c0) / (n * args.steps)}
        result[name] = r
    for n in chains:
        on, off = result["deskew_on"][str(n)], result["deskew_off"][str(n)]
        result.setdefault("added", {})[str(n)] = {"ms_per_step": on["ms_per_step_median"] - off["ms_per_step_median"],
                                                   "launches_per_scan": on["launches_per_scan"] - off["launches_per_scan"]}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        timed(arms["deskew_on"], 1, args.steps, main_s, streams, flush)
    ev = [e for e in prof.key_averages() if "deskew_kernel" in e.key]
    result["deskew_kernels_us_per_scan"] = sum(e.device_time_total for e in ev) / args.steps if ev else None
    result["deskew_kernel_launches_per_scan"] = sum(e.count for e in ev) / args.steps if ev else None
    m = arms["deskew_on"].odos[0].fetchMotionCompensation(0)
    result["deskew_on_sanity"] = {"odometry_applied": m.odometryApplied, "map_applied": m.mapApplied,
                                  "map_linear_velocity": m.mapLinearVelocity.tolist()}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
