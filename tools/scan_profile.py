"""Kernel table of the steady-state odometry scan (GPU box): where one eager scan's device time goes.

One chain is driven over a full lap of the closed loop (the bench.py workload: Lua defaults, PointToPlaneIcp, ratio 0.3), so
that its map is in steady state; then `--scans` further scans run eagerly under torch.profiler, each followed by a device
synchronise.  The table lists, per kernel, launches, device microseconds and an SM-microsecond estimate per scan:
duration x min(#SMs, #CTAs) -- what a launch takes away from concurrent chains when the GPU is shared.  The launches of the
ICP target index build over the map (from compose_kernel to grid_scatter_kernel) are reported as their own group.

usage: python tools/scan_profile.py [--scans 10] [--out DIR]   (DIR: the table and the chrome trace; default a temporary directory)"""
import argparse
import json
import os
import re
import sys
import tempfile
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def short_name(name):
    base = re.sub(r"^void\s+", "", name)
    base = base.split("(")[0]
    m = re.match(r"((?:[\w:]+::)?)(\w+)(<.*>)?", base)
    if not m:
        return name[:60]
    return m.group(2) + (m.group(3) or "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "b2s_scan_profile"))
    ap.add_argument("--map-capacity", type=int, default=760_000)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from open3d_slam_b200 import engine as E
    from open3d_slam_b200 import workloads as W

    if not torch.cuda.is_available():
        raise SystemExit("scan_profile.py: no CUDA device")
    dev = torch.device("cuda", 0)
    props = torch.cuda.get_device_properties(dev)
    n_sm = props.multi_processor_count
    lp = W.ClosedLoop()
    params = E.MapperParameters(seed=3)
    stream = torch.cuda.Stream(device=dev)
    eng = E.Engine(params, device=0, cuda_stream=stream.cuda_stream)
    mp = E.Mapper(eng, args.map_capacity)
    n_total = lp.L + 3 + args.scans
    clouds = [eng.cloud(lp.scan(k, seed=k % lp.L)) for k in range(lp.L)]
    mp.addRangeMeasurement(clouds[0], None)
    mp.submap.setPose(np.eye(4))
    eng.synchronize()
    for k in range(1, lp.L + 3):
        mp.addRangeMeasurementAsync(clouds[k % lp.L], lp.delta(k), slot=k % 256)
    eng.synchronize()
    map_pts = mp.submap.size()

    ev = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(lp.L + 3, n_total):
            a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
            a.record(stream)
            mp.addRangeMeasurementAsync(clouds[k % lp.L], lp.delta(k), slot=k % 256)
            b.record(stream)
            torch.cuda.synchronize(dev)
            ev.append((a, b))
    scan_ms = [a.elapsed_time(b) for a, b in ev]
    res = [mp.fetchResult(k % 256) for k in range(n_total - args.scans, n_total)]
    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "scan_profile.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    gpu = [e for e in events if e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy") and e.get("ph") == "X"]
    gpu.sort(key=lambda e: e["ts"])

    rows = defaultdict(lambda: [0, 0.0, 0.0])     # name -> launches, us, SM-us
    group = defaultdict(lambda: [0, 0.0, 0.0])
    in_map_index = False
    for e in gpu:
        cat = e["cat"]
        name = short_name(e["name"]) if cat == "kernel" else cat
        dur = float(e["dur"])
        if cat == "kernel":
            g = e.get("args", {}).get("grid", [1, 1, 1])
            blocks = int(np.prod(g))
            sm_us = dur * min(n_sm, blocks)
        else:
            sm_us = 0.0
        if name == "compose_kernel":
            in_map_index = True
        r = rows[name]; r[0] += 1; r[1] += dur; r[2] += sm_us
        gname = "map_index_build" if (in_map_index and name != "compose_kernel") else "other"
        gr = group[gname]; gr[0] += 1; gr[1] += dur; gr[2] += sm_us
        if in_map_index and name == "grid_scatter_kernel":
            in_map_index = False

    K = args.scans
    tot_us = sum(r[1] for r in rows.values()); tot_sm = sum(r[2] for r in rows.values())
    lines = [f"device: {props.name}, {n_sm} SMs; map points {map_pts}; {K} eager steady-state scans, "
             f"scan time (events) median {np.median(scan_ms):.3f} ms; ICP iterations {[r.iters for r in res]}",
             f"{'kernel':44s} {'launch/scan':>11s} {'us/scan':>9s} {'share':>7s} {'SM-us/scan':>11s} {'share':>7s}"]
    for name, (n, us, sm) in sorted(rows.items(), key=lambda kv: -kv[1][2]):
        lines.append(f"{name[:44]:44s} {n / K:11.2f} {us / K:9.1f} {100 * us / tot_us:6.1f}% {sm / K:11.0f} {100 * sm / tot_sm:6.1f}%")
    lines.append("")
    for gname, (n, us, sm) in sorted(group.items()):
        lines.append(f"group {gname:38s} {n / K:11.2f} {us / K:9.1f} {100 * us / tot_us:6.1f}% {sm / K:11.0f} {100 * sm / tot_sm:6.1f}%")
    text = "\n".join(lines)
    print(text)
    with open(os.path.join(args.out, "scan_profile.txt"), "w") as f:
        f.write(text + "\n")
    summary = {"device": props.name, "map_points": int(map_pts), "scan_ms_median": float(np.median(scan_ms)),
               "groups": {g: {"launches_per_scan": v[0] / K, "us_per_scan": v[1] / K, "sm_us_per_scan": v[2] / K,
                              "us_share": v[1] / tot_us, "sm_us_share": v[2] / tot_sm} for g, v in group.items()}}
    print(json.dumps(summary))
    mp.submap.free()
    for c in clouds:
        c.free()
    eng.close()


if __name__ == "__main__":
    main()
