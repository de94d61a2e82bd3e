"""The dense-map export (saveDenseSubmaps / publishDenseMap; DESIGN.md row A2) over 16 and 64 submaps of the closed lap.

Submaps: Config4's 20 m-radius targets, each with the dense map of its 6 lap scans (2 m apart) inserted by b2s_submap_insert_dense at their
true poses with the default 0.05 m dense voxel, resident (2^22-slot tables: about 15 GB of HBM for 64).  Timed, each the median of --reps
host-clock readings around calls that end in a device synchronisation, after --warmup calls:
    (a) one b2s_assemble_dense_maps call, alone (ended by b2s_synchronize) and with the download of its cloud to the host
    (b) what a caller does today: b2s_submap_dense_download for every submap (Submap.getDenseMap)
The outputs of (a) and (b) are compared bit for bit.  The bytes the call must move are computed from the table sizes and the live counts:
the count array read twice (count and gather passes), plus 24 B read (the position sums) and 24 B written per live voxel; the achieved
rate of (a) alone is reported against the H100 SXM's 3.35 TB/s.  The card's name and power limit are read in the same run.

    python tools/dense_map_export_bench.py [--targets 16,64] [--reps 5] [--warmup 2] [--out /tmp/dense_map_export.json]
"""
from __future__ import annotations

import argparse
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

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


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
    scans = {}
    sms = []
    for t in range(n):
        sm = E.Submap(eng, 1000)
        for k in c4.target_positions(t):
            if k not in scans:
                scans[k] = eng.cloud(lp.scan(k, seed=5000 + (k % lp.L)))
            sm.insertScanDenseMap(scans[k], lp.pose(k))
        sms.append(sm)
    for c in scans.values():
        c.free()
    eng.synchronize()
    return sms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--targets", default="16,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    counts = [int(v) for v in a.targets.split(",")]
    dev_name = card()
    eng = E.Engine(E.MapperParameters(seed=3))
    t0 = time.perf_counter()
    all_sms = build_submaps(eng, max(counts))
    build_s = time.perf_counter() - t0
    out = E.Cloud(eng)
    rows = []
    for n in counts:
        sms = all_sms[:n]
        live = [s.denseSize() for s in sms]
        slots = n * (1 << 22)
        moved = 2 * 4 * slots + 48 * sum(live)

        def call():
            E.assembleDenseMaps(eng, sms, out)
            eng.synchronize()

        def call_download():
            E.assembleDenseMaps(eng, sms, out)
            return out.download()[0]

        def loop():
            return [s.getDenseMap()[0] for s in sms]

        got = call_download()
        ref = np.concatenate(loop())
        identical = bool(got.shape == ref.shape and np.array_equal(got.view(np.uint64), ref.view(np.uint64)))
        del got, ref
        t_call = median_ms(call, a.reps, a.warmup)
        t_call_dl = median_ms(call_download, a.reps, a.warmup)
        t_loop = median_ms(loop, max(1, a.reps // 2), 1)
        rows.append({"submaps": n, "live_voxels_total": int(sum(live)), "live_voxels_min": int(min(live)), "live_voxels_max": int(max(live)),
                     "table_slots_total": slots, "export_equals_downloads_bitwise": identical,
                     "export_ms": round(t_call, 3), "export_and_download_ms": round(t_call_dl, 2), "per_submap_downloads_ms": round(t_loop, 1),
                     "bytes_moved": int(moved), "export_GB_per_s": round(moved / (t_call * 1e-3) / 1e9, 1),
                     "export_share_of_3.35_TB_per_s": round(moved / (t_call * 1e-3) / HBM_BYTES_PER_S, 3)})
    res = {"card": dev_name, "build_s": round(build_s, 1), "rows": rows}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
