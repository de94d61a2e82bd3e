#!/usr/bin/env python
"""What the device-resident odometry adds per scan: the combined odometry + mapper graph (b2s_slam_step_async, graph mode)
against the mapper-only graph fed the odometry motion from the host (b2s_mapper_step_async, graph mode, bench.py's path).

Workload: bench.py's steady state -- workloads.ClosedLoop, Lua defaults (odometry and mapper both voxel 0.1 m, MinMaxRadius 2-30 m,
knn 20 / 3 m, max corr. 1 m, PointToPlaneIcp), downsampling ratio 0.3 for both (--ratio sets both), every chain pre-grown over one lap
(untimed), scans resident
in HBM and copied into the graph's staging cloud.  Device time from CUDA events on the main stream around every step (one scan per
chain per step), after a warm-up of the same shape.  Prints one JSON line (and writes it to --out): single-chain ms per scan of both
arms, scans/s at 1, 4, 8, 16 chains, kernel launches and graph captures per scan (0 in steady state: every step is a replay), and the
card name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open3d_slam_b200 import _lib as L  # noqa: E402
from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402

TICKS_PER_SCAN = 1_000_000   # 0.1 s in UniversalTimeScaleClock ticks


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = (v.strip() for v in q.split(","))
    except Exception as e:   # the number still stands, but without its context: say so
        out["power_limit"] = f"unread ({e})"
    return out


class Arm:
    """n chains (engine + stream + submap each) of one arm, pre-grown over one lap"""

    def __init__(self, combined, n, lp, clouds, params, odo_params, streams, capacity):
        self.combined, self.lp = combined, lp
        n_lap = lp.L
        self.engs = [E.Engine(params, cuda_stream=streams[c].cuda_stream) for c in range(n)]
        self.maps = [E.Mapper(e, capacity) for e in self.engs]
        self.clouds = [[e.cloud(clouds[c % len(clouds)][k]) for k in range(n_lap)] for c, e in enumerate(self.engs)]
        self.odos = [E.DeviceLidarOdometry(e, odo_params, 65536) for e in self.engs] if combined else None
        for c in range(n):
            self.maps[c].addRangeMeasurement(self.clouds[c][0], None)
            self.maps[c].submap.setPose(np.eye(4))
            if combined:
                self.odos[c].addRangeScan(self.clouds[c][0], TICKS_PER_SCAN)
        self.staging = [(self.odos[c].enableGraph(65536) if combined else self.maps[c].enableGraph(65536)) for c in range(n)]
        self.k = [1] * n
        self.deltas = [np.ascontiguousarray(lp.delta(k)) for k in range(1, n_lap + 1)]

    def one(self, c):
        k = self.k[c]
        n_lap = self.lp.L
        L.check(L.lib().b2s_cloud_copy(self.engs[c]._h, self.clouds[c][k % n_lap]._c, self.staging[c]._c))
        if self.combined:
            self.maps[c].addRangeMeasurementWithOdometry(self.odos[c], self.staging[c], (k + 1) * TICKS_PER_SCAN)
        else:
            self.maps[c].addRangeMeasurementAsync(self.staging[c], self.deltas[(k - 1) % n_lap])
        self.k[c] = k + 1

    def launches(self, n):
        return sum(e.launches for e in self.engs[:n])

    def captures(self, n):
        return sum(e.graphCaptures for e in self.engs[:n])


def timed(arm, n, steps, main, streams, flush):
    import torch
    evs = []
    for _ in range(steps):
        flush.zero_()
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(main)
        for s in streams[:n]:
            s.wait_event(a)
        for c in range(n):
            arm.one(c)
        for s in streams[:n]:
            d = torch.cuda.Event(); d.record(s); main.wait_event(d)
        b.record(main)
        evs.append((a, b))
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in evs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", default="1,4,8,16")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--ratio", type=float, default=0.3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("odometry_bench.py: no CUDA device -- the b2s engine has no CPU fallback")
    chains = sorted(int(x) for x in args.chains.split(",") if x)
    n_max = max(chains)
    lp = W.ClosedLoop()
    sets = min(n_max, 4)
    clouds = [[lp.scan(k, seed=1000 * s + k) for k in range(lp.L)] for s in range(sets)]
    params = E.MapperParameters(seed=3)
    params.scanProcessing.downSamplingRatio = args.ratio
    odo_params = E.OdometryParameters(seed=5)
    odo_params.scanProcessing.downSamplingRatio = args.ratio
    main_s = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in range(n_max)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    arms = {"combined": Arm(True, n_max, lp, clouds, params, odo_params, streams, 900_000),
            "mapper_only": Arm(False, n_max, lp, clouds, params, odo_params, streams, 900_000)}
    for arm in arms.values():   # the rest of lap 0: the maps reach steady state
        timed(arm, n_max, lp.L - 1, main_s, streams, flush)
    result = {"tool": "odometry_bench", "workload": "workloads.ClosedLoop steady state (one lap pre-grown), Lua defaults, ratio %g" % args.ratio,
              "steps": args.steps, "warmup": args.warmup, "card": card()}
    for name, arm in arms.items():
        r = {}
        for n in chains:
            timed(arm, n, args.warmup, main_s, streams, flush)
            l0, c0 = arm.launches(n), arm.captures(n)
            ms = timed(arm, n, args.steps, main_s, streams, flush)
            launches = (arm.launches(n) - l0) / (n * args.steps)
            r[str(n)] = {"scans_per_s": n * args.steps / (sum(ms) * 1e-3), "ms_per_step_median": float(np.median(ms)),
                         "launches_per_scan": launches, "captures_per_scan": (arm.captures(n) - c0) / (n * args.steps)}
        r["single_chain_ms_per_scan"] = r[str(chains[0])]["ms_per_step_median"] if chains[0] == 1 else None
        result[name] = r
    for c in range(min(n_max, 4)):   # sanity: the combined chains track the trajectory and the odometry succeeds
        s = arms["combined"].odos[c].fetchSlamResult(0)
        result.setdefault("combined_sanity", []).append({"odometry_outcome": s.odometry.outcome, "odom_used": s.odomUsed,
                                                         "mapper_fitness": s.mapper.fitness_})
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
