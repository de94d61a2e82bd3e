"""Session state (DESIGN.md row A3): export and import of the 64 Config4 submaps, with the assembled map (A1) and the dense-map export (A2)
of the same submaps beside them for reference (those are outputs only, not state).

Submaps: Config4's 20 m-radius targets, each with its 6 lap scans (2 m apart) fused by S1 (ratio 1) + F1 into the sparse map and fed by
b2s_submap_insert_dense into the dense map at their true poses (default 0.1 m map voxel, 0.05 m dense voxel), resident.  Timed, each the
median of --reps host-clock readings around calls that end in a device synchronisation, after --warmup calls:
    export   E.exportSubmapStates of every submap: the size call and the fill call, blobs in host memory
    import   E.importSubmapState of every blob into a new submap (allocation and table initialisation included), then a synchronize
    A1 + A2  getAssembledMapPointCloud and assembleDenseMaps of the same list, each downloaded to the host
The re-export of the imports is compared byte for byte with the export.  The card's name and power limit are read in the same run.

    python tools/session_state_bench.py [--targets 64] [--reps 5] [--warmup 1] [--out /tmp/session_state.json]
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
    return float(np.median(ts)), [round(t, 2) for t in ts]


def build_submaps(eng, params, n, capacity):
    lp = W.ClosedLoop()
    c4 = W.Config4(lp, n_targets=n)
    p_full = copy.deepcopy(params); p_full.scanProcessing.downSamplingRatio = 1.0   # Config4's targets keep every voxel of their scans
    eng.set_parameters(p_full)
    icp = E.ScanToMapIcp(eng)
    sms = []
    for t in range(n):
        sm = E.Submap(eng, capacity)
        for k in c4.target_positions(t):
            raw = eng.cloud(lp.scan(k, seed=5000 + (k % lp.L)))
            ps = icp.processForScanMatchingAndMerging(raw)
            sm.insertScan(None, ps.merge_, lp.pose(k))
            sm.insertScanDenseMap(raw, lp.pose(k))
            raw.free(); ps.merge_.free(); ps.match_.free()
        sms.append(sm)
    eng.set_parameters(params)
    eng.synchronize()
    return sms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--targets", type=int, default=64)
    ap.add_argument("--capacity", type=int, default=400_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev_name = card()
    params = E.MapperParameters(seed=3)
    eng = E.Engine(params)
    t0 = time.perf_counter()
    sms = build_submaps(eng, params, a.targets, a.capacity)
    build_s = time.perf_counter() - t0
    points = sum(s.size() for s in sms)
    voxels = sum(s.denseSize() for s in sms)

    blobs = E.exportSubmapStates(eng, sms)
    hdrs = [E.parseStateHeader(b) for b in blobs]
    dense_bytes = sum(h.sections["dense"][1] for h in hdrs)
    total_bytes = sum(len(b) for b in blobs)

    t_export, export_all = median_ms(lambda: E.exportSubmapStates(eng, sms), a.reps, a.warmup)

    other = E.Engine(params)
    held = []

    def do_import():
        for s in held:
            s.free()
        held.clear()
        held.extend(E.importSubmapState(other, b) for b in blobs)
        other.synchronize()

    t_import, import_all = median_ms(do_import, a.reps, a.warmup)
    identical = E.exportSubmapStates(other, held) == blobs
    for s in held:
        s.free()

    def outputs():
        E.getAssembledMapPointCloud(eng, sms).download()
        E.assembleDenseMaps(eng, sms)[0].download()

    t_out, out_all = median_ms(outputs, a.reps, a.warmup)
    res = {"card": dev_name, "submaps": a.targets, "capacity": a.capacity, "build_s": round(build_s, 1), "map_points": int(points),
           "dense_voxels": int(voxels), "blob_bytes": int(total_bytes), "sparse_state_bytes": int(total_bytes - dense_bytes),
           "dense_record_bytes": int(dense_bytes), "reexport_identical": bool(identical),
           "export_ms": round(t_export, 2), "export_GB_per_s": round(total_bytes / (t_export * 1e-3) / 1e9, 2), "export_ms_all": export_all,
           "import_ms": round(t_import, 2), "import_GB_per_s": round(total_bytes / (t_import * 1e-3) / 1e9, 2), "import_ms_all": import_all,
           "a1_plus_a2_download_ms": round(t_out, 2), "a1_plus_a2_ms_all": out_all}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
