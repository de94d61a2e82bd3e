#!/usr/bin/env python
"""Does de-skew help?  CPU only: the oracle composition of SlamWrapper's two workers (tests/motion_compensation.py, DeskewBackend: the
odometry and the mapper on one submap, no carving) over a lap of rolling-shutter scans (ClosedLoop.scan_moving, one scan period = one
scan_duration = 0.1 s), with motion compensation off and on.  Prints one JSON line: the final, mean and largest translation error and
the final and mean rotation error of mapToRangeSensor against ClosedLoop.map_frame_pose."""
from __future__ import annotations

import argparse
import copy
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402
from motion_compensation import DeskewBackend  # noqa: E402
from test_gpu_odometry import odo_params  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=0, help="default: one lap")
    args = ap.parse_args()
    lp = W.ClosedLoop()
    n = args.scans or lp.L
    scans = [lp.scan_moving(k, seed=k) for k in range(n)]
    times = [12345 + k * 1_000_000 for k in range(n)]
    out = {"tool": "deskew_accuracy", "scans": n}
    for on in (False, True):
        mc = E.ConstantVelocityMotionCompensationParameters(isUndistortInputCloud=on)
        be = DeskewBackend(copy.deepcopy(E.MapperParameters(seed=3)), odo_params(), mc, carving=False, dense=False)
        sm = be.new_submap()
        be.first_scan_with_odometry(sm, scans[0], times[0])
        te, re = [], []
        for k in range(1, n):
            be.step_with_odometry(sm, scans[k], times[k])
            gt = lp.map_frame_pose(k)
            te.append(float(np.linalg.norm(be.pose[:3, 3] - gt[:3, 3])))
            R = be.pose[:3, :3].T @ gt[:3, :3]
            re.append(float(np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1)))))
        out["deskew_on" if on else "deskew_off"] = {"final_m": te[-1], "mean_m": float(np.mean(te)), "max_m": float(np.max(te)),
                                                     "final_deg": re[-1], "mean_deg": float(np.mean(re))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
