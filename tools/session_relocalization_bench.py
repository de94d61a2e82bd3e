"""Relocalisation in a session (b2s_submaps_global_localization, DESIGN.md row M4): one search over the union of every submap against the
one-submap search (b2s_submap_global_localization, row M3) run on every submap in turn, keeping the best.

Submaps: the 64 Config4 submaps of the closed lap, built as tools/session_state_bench.py builds them (6 lap scans each, fused at their true
poses), resident on one handle; centres = the mean of each map (Submap::getMapToSubmapCenter once finished).  The query is a lap-2 scan;
default search parameters (the box is the live extent of the union, or of each submap).  Timed, each the median of --reps host-clock
readings around calls that end in a device synchronisation, after --warmup calls, the two alternated:
    union      one E.globalLocalizationInSubmaps call over the 64 submaps
    per_submap E.globalLocalization on each submap in turn, the best fitness kept
Then one traced call of each (torch.profiler, CUDA activities), its kernel time split into occupancy (the box and occupancy kernels),
score (gl_score_kernel), selection (histogram, threshold, compaction, suppression) and refinement (everything after gl_nms_kernel: patch
builds and the batched ICP).  The card's name, power limit and clocks are read in the same run.

    python tools/session_relocalization_bench.py [--targets 64] [--reps 5] [--warmup 1] [--out /tmp/session_relocalization.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from open3d_slam_b200 import engine as E  # noqa: E402
from open3d_slam_b200 import workloads as W  # noqa: E402
from session_state_bench import build_submaps, card  # noqa: E402

OCCUPANCY = ("gl_union_box_kernel", "gl_union_occ_kernel", "gl_occ_kernel", "bbox")


def split_trace(fn):
    """kernel milliseconds of one traced call by stage: the kernels before gl_score_kernel (occupancy, or the scan processing and the
    query), the score kernel, the ones after it up to gl_nms_kernel (selection), the ones after that (refinement)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ks = sorted(((e.time_range.start, e.time_range.end, e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                key=lambda t: t[0])
    out = dict(occupancy=0.0, score=0.0, selection=0.0, refinement=0.0, query_and_scan=0.0)
    phase = "query_and_scan"
    for a, b, n in ks:
        if "gl_score_kernel" in n:
            k, phase = "score", "selection"
        elif "gl_nms_kernel" in n:
            k, phase = "selection", "refinement"
        elif phase == "query_and_scan" and any(s in n for s in OCCUPANCY):
            k = "occupancy"
        else:
            k = phase
        out[k] += (b - a) / 1e3
    return out


def summed(parts):
    return {k: round(sum(p[k] for p in parts), 3) for k in parts[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--targets", type=int, default=64)
    ap.add_argument("--capacity", type=int, default=400_000)
    ap.add_argument("--position", type=int, default=47, help="lap position of the query scan")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev_name = card()
    params = E.MapperParameters(seed=3)
    eng = E.Engine(params)
    sms = build_submaps(eng, params, a.targets, a.capacity)
    centers = np.array([sm.getMapPointCloud()[0].mean(axis=0) for sm in sms])
    lp = W.ClosedLoop()
    truth = lp.pose(a.position)
    raw = eng.cloud(lp.scan(a.position + lp.L, seed=8000 + a.position))
    gp = E.GlobalLocalizationParameters()
    fit = params.minRefinementFitness

    def union():
        return E.globalLocalizationInSubmaps(eng, sms, centers, raw, gp, fit)

    def per_submap():
        rs = [E.globalLocalization(eng, sm, raw, gp, fit) for sm in sms]
        best = max(range(len(rs)), key=lambda s: (rs[s].fitness, -s))
        return rs, best

    for _ in range(a.warmup):
        union(); per_submap()
    tu, tp = [], []
    for _ in range(a.reps):   # alternated
        t0 = time.perf_counter(); ru = union(); tu.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter(); rp, best = per_submap(); tp.append((time.perf_counter() - t0) * 1e3)
    err = lambda T: round(float(np.linalg.norm(np.asarray(T)[:3, 3] - truth[:3, 3])), 4)   # noqa: E731
    res = {"card": dev_name, "submaps": a.targets, "map_points": int(sum(s.size() for s in sms)), "query_points": ru.n_query,
           "union_ms": round(float(np.median(tu)), 2), "union_ms_all": [round(t, 2) for t in tu],
           "per_submap_ms": round(float(np.median(tp)), 2), "per_submap_ms_all": [round(t, 2) for t in tp],
           "union_hypotheses": ru.n_hypotheses, "per_submap_hypotheses": int(sum(r.n_hypotheses for r in rp)),
           "union_found": ru.found, "union_fitness": round(ru.fitness, 4), "union_winner_submap": ru.winner_submap,
           "union_error_m": err(ru.T), "per_submap_fitness": round(rp[best].fitness, 4), "per_submap_best": best,
           "per_submap_error_m": err(rp[best].T),
           "union_kernel_ms": summed([split_trace(union)]),
           "per_submap_kernel_ms": summed([split_trace(lambda sm=sm: E.globalLocalization(eng, sm, raw, gp, fit)) for sm in sms]),
           "timing": "host clock around synchronising calls, median of %d after %d warm-up; kernel split from one traced call" % (a.reps, a.warmup)}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
