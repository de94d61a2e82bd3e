"""Pose-graph optimisation (b2s_global_optimization) on synthetic graphs: N = 16, 64, 128, 256, 500 nodes, a random-walk trajectory
with noisy odometry edges and one true loop closure per 8 nodes, the Lua GlobalOptimizationOption (parameter_structure_definitions.lua:
45-50) and [O3D]'s default criteria.

Per size: the whole call (host clock around the synchronising call, median after warm-up), the factorisation's kernel time per LM try
(torch.profiler over one call: the device time of K-pg-diag + K-pg-panel + K-pg-trailing, divided by the tries of both passes -- the
factorisation runs inside the try's CUDA graph, so events around it alone are not available from here), the achieved fp64 rate of the
factorisation from (6N)^3 / 3 flops over that time, the LM tries per call, and the launches per call and per try.  The numpy restatement
(tests/oracle_pose_graph.py, one host thread) is timed at the sizes where it finishes in reasonable time.  Prints the card and its power
limit first.  Usage: python tools/pose_graph_bench.py [--reps 7] [--numpy-max 256] [--out DIR]"""
import os

os.environ.setdefault("OMP_NUM_THREADS", "1")          # the restatement on one host core
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
os.environ.setdefault("MKL_NUM_THREADS", "1")

import argparse
import json
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import oracle_pose_graph as PG  # noqa: E402
from open3d_slam_b200 import engine as E  # noqa: E402

FACTOR_KERNELS = ("pg_diag_kernel", "pg_panel_kernel", "pg_trailing_kernel")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as ex:   # the numbers below still need the card beside them: say that it could not be read
        return f"unknown ({ex})"


def pose_graph(init, edges):
    return E.PoseGraph([E.PoseGraphNode(np.array(T)) for T in init],
                       [E.PoseGraphEdge(e.source, e.target, np.array(e.T), np.array(e.information), bool(e.uncertain)) for e in edges])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,64,128,256,500")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--numpy-max", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    print("card:", card())
    eng = E.Engine()
    rows = []
    for n in [int(s) for s in a.sizes.split(",")]:
        _truth, init, edges = PG.random_graph(n, seed=n, loop_every=8)
        st = E.globalOptimization(eng, pose_graph(init, edges))   # warm-up: buffers, graph capture
        E.globalOptimization(eng, pose_graph(init, edges))
        times = []
        for _ in range(a.reps):
            g = pose_graph(init, edges)
            t0 = time.perf_counter()
            st = E.globalOptimization(eng, g)   # synchronises (the poses come back)
            times.append(time.perf_counter() - t0)
        tries = sum(s.lm_tries for s in st)
        l0 = eng.launches
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            E.globalOptimization(eng, pose_graph(init, edges))
            torch.cuda.synchronize()
        launches = eng.launches - l0
        fac_us = sum(ev.device_time_total for ev in prof.key_averages() if any(k in ev.key for k in FACTOR_KERNELS))
        per_fac = fac_us * 1e-6 / max(tries, 1)
        flops = (6.0 * n) ** 3 / 3.0
        row = {"N": n, "edges": len(edges), "call_ms_median": 1e3 * statistics.median(times), "lm_tries": tries,
               "accepted": sum(s.accepted_steps for s in st), "factor_ms_per_try": 1e3 * per_fac,
               "factor_gflops": flops / per_fac / 1e9 if per_fac > 0 else None, "launches_per_call": launches,
               "launches_per_try": 5 * ((6 * n + 63) // 64) + 2}
        if n <= a.numpy_max:
            t0 = time.perf_counter()
            _o, _k, _c, rst = PG.global_optimization(init, edges)
            row["numpy_ms"] = 1e3 * (time.perf_counter() - t0)
            row["numpy_tries"] = sum(s.lm_tries for s in rst)
        else:
            row["numpy_ms"] = None
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "pose_graph_bench.json"), "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
