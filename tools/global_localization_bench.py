"""Global localisation in a prior map (b2s_submap_global_localization, DESIGN.md row M3): the time of one call on maps of growing size.

The map is the closed lap's prior map (every scan of one lap moved by map_frame_pose(k), voxelized at mapVoxelSize) replicated R x R
times on a 60 m pitch, R = 1, 2, 4; the search box is the default (the map's live extent), so it grows with the map.  The query is a
lap-2 scan.  Per size, two alternated runs of:
  - the whole call, host clock around the synchronising call, median of --reps calls after --warmup;
  - one traced call (torch.profiler, CUDA activities): the score kernel's device time, and the share of the call's device span that
    follows the candidate selection (the refinement: patch builds and the batched ICP);
  - hypotheses x query points per second of the score kernel.
The card's name and power limit are read in the same run.  Prints one JSON line per (run, size) and writes them to --out.

    python tools/global_localization_bench.py --out /tmp/global_localization_bench.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import slam as S  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402

PITCH = 60.0


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return name, limit
    except Exception as e:   # the numbers are then reported without the card, which makes them worthless: say so
        return f"unknown ({e})", "unknown"


def lap_map(lp, voxel):
    parts = []
    for k in range(lp.L):
        T = lp.map_frame_pose(k)
        parts.append(lp.scan(k, seed=k).astype(np.float64) @ T[:3, :3].T + T[:3, 3])
    xyz = np.concatenate(parts)
    key = np.floor(xyz / voxel).astype(np.int64)
    _u, inv, cnt = np.unique(key, axis=0, return_inverse=True, return_counts=True)
    out = np.zeros((len(cnt), 3))
    np.add.at(out, inv.reshape(-1), xyz)
    return out / cnt[:, None]


def setup(base, p, R):
    xyz = np.concatenate([base + [PITCH * i, PITCH * j, 0.0] for i in range(R) for j in range(R)])
    dev = S.DeviceBackend(p, carving=False, dense=False, graph=False, submap_capacity=len(xyz) + 1024)
    m = S.SegmentMapper(dev, S.SubmapParameters(radius=1e6))
    m.setInitialMap(xyz)
    return dev, m.submaps.getActiveSubmap().handle


def trace(dev, sm, c, gp):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sm.globalLocalization(c, gp, 0.7)
        dev.eng.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ks = sorted(((e.time_range.start, e.time_range.end, e.name) for e in ev), key=lambda t: t[0])
    score = sum(b - a for a, b, n in ks if "gl_score_kernel" in n)
    nms_end = max((b for a, b, n in ks if "gl_nms_kernel" in n), default=None)
    span = ks[-1][1] - ks[0][0] if ks else 0
    refine = (ks[-1][1] - nms_end) / span if nms_end is not None and span else None
    return score / 1e3, refine   # us -> ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,2,4")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    lp = W.ClosedLoop()
    p = E.MapperParameters(seed=3, isUseInitialMap=True, isMergeScansIntoMap=False)
    base = lap_map(lp, p.mapBuilder.mapVoxelSize)
    raw = lp.scan(25 + lp.L, seed=4025)
    gp = E.GlobalLocalizationParameters()
    rows = []
    sizes = [int(s) for s in a.sizes.split(",")]
    envs = {R: setup(base, p, R) for R in sizes}
    for run in range(a.runs):
        for R in (sizes if run % 2 == 0 else sizes[::-1]):    # alternated order between the runs
            dev, sm = envs[R]
            c = dev.eng.cloud(raw)
            for _ in range(a.warmup):
                r = sm.globalLocalization(c, gp, 0.7)
            ts = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                r = sm.globalLocalization(c, gp, 0.7)   # synchronises before it returns
                ts.append(time.perf_counter() - t0)
            score_ms, refine_share = trace(dev, sm, c, gp)
            row = dict(run=run, replicas=f"{R}x{R}", map_points=int(len(base) * R * R), hypotheses=r.n_hypotheses, query_points=r.n_query,
                       call_ms_median=1e3 * float(np.median(ts)), call_ms_min=1e3 * float(min(ts)), score_kernel_ms=score_ms,
                       probes_per_s=(r.n_hypotheses * r.n_query / (score_ms * 1e-3)) if score_ms else None,
                       refinement_share_of_device_span=refine_share, found=r.found, fitness=r.fitness,
                       runner_up_fitness=r.runner_up_fitness, gpu=name, power_limit=limit)
            print(json.dumps(row), flush=True)
            rows.append(row)
            c.free()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    for dev, _sm in envs.values():
        dev.close()


if __name__ == "__main__":
    main()
