"""The assembled map (getAssembledMapPointCloud, saveMap / publishMaps; DESIGN.md row A1) on the 64 Config4 submaps of the closed lap.

Submaps: Config4's 64 20 m-radius targets (6 scans 2 m apart fused at their true poses with S1 at ratio 1 + F1), resident.  Timed, each the
median of --reps host-clock readings around calls that end in a device synchronisation, after --warmup calls:
    (a) b2s_assemble_map unvoxelized, voxelized at 0.1; b2s_assemble_colored_map at 0.1 (colours copied to the host)
    (b) the per-submap composition: b2s_submap_to_cloud for every submap, the clouds concatenated on the device (export into one torch
        buffer, import as one cloud), b2s_voxel_down_sample at 0.1
    (c) the download path: b2s_submap_download for every submap + numpy concatenation; the host VoxelDownSample is the C oracle on one
        core (OMP_NUM_THREADS=1) over the first --host-points points of that concatenation
The outputs of (a) and (b) are compared bit for bit.  The card's name and power limit are read in the same run.

    python tools/assembled_map_bench.py [--targets 64] [--reps 5] [--warmup 1] [--host-points 2000000] [--out /tmp/assembled_map.json]
"""
from __future__ import annotations

import os

os.environ.setdefault("OMP_NUM_THREADS", "1")   # the host voxelize is one core

import argparse
import json
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
    return float(np.median(ts))


def build_submaps(eng, n):
    lp = W.ClosedLoop()
    c4 = W.Config4(lp)
    params = eng.params
    p_full = E.MapperParameters(seed=3)
    p_full.scanProcessing.downSamplingRatio = 1.0   # submaps keep every voxel of the scans they fuse (as Config4.build_target)
    eng.set_parameters(p_full)
    icp = E.ScanToMapIcp(eng)
    sms = []
    for t in range(n):
        sm = E.Submap(eng, 900_000)
        for k in c4.target_positions(t):
            raw = eng.cloud(lp.scan(k, seed=5000 + (k % lp.L)))
            ps = icp.processForScanMatchingAndMerging(raw)
            sm.insertScan(None, ps.merge_, lp.pose(k))
            raw.free(); ps.merge_.free(); ps.match_.free()
        sms.append(sm)
    eng.set_parameters(params)
    return sms


def composition(eng, sms, voxel, buf):
    """b2s_submap_to_cloud per submap, concatenated on the device, then b2s_voxel_down_sample"""
    import torch
    o = 0
    for s in sms:
        c = s.toCloud()
        n = c.export_device(buf[0][o:].data_ptr(), buf[1][o:].data_ptr(), buf[0].shape[0] - o)
        c.free()
        o += n
    cat = eng.cloud().import_device(buf[0].data_ptr(), buf[1].data_ptr(), o)
    torch.cuda.synchronize()
    if voxel <= 0.0:
        return cat
    v = E.voxelize(eng, cat, voxel)
    v.size()
    return v


def download_path(sms):
    parts = [s.getMapPointCloud() for s in sms]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def main():
    import torch
    from oracle import oracle as O
    ap = argparse.ArgumentParser()
    ap.add_argument("--targets", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--host-points", type=int, default=2_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev_name = card()
    eng = E.Engine(E.MapperParameters(seed=3))
    sms = build_submaps(eng, a.targets)
    sizes = [s.size() for s in sms]
    total = int(sum(sizes))
    buf = (torch.empty((total + 16, 3), dtype=torch.float64, device="cuda"), torch.empty((total + 16, 3), dtype=torch.float64, device="cuda"))

    # outputs of (a) and (b), bit for bit
    ga = E.getAssembledMapPointCloud(eng, sms).download()
    gb = composition(eng, sms, 0.0, buf).download()
    va = E.getAssembledMapPointCloud(eng, sms, 0.1).download()
    vb = composition(eng, sms, 0.1, buf).download()
    same = lambda x, y: x[0].shape == y[0].shape and np.array_equal(x[0].view(np.uint64), y[0].view(np.uint64)) and \
        np.array_equal(x[1].view(np.uint64), y[1].view(np.uint64))
    identical = bool(same(ga, gb) and same(va, vb))
    n_vox = int(len(va[0]))
    del ga, gb, va, vb

    t_asm = median_ms(lambda: E.getAssembledMapPointCloud(eng, sms), a.reps, a.warmup)
    t_asm_v = median_ms(lambda: E.getAssembledMapPointCloud(eng, sms, 0.1), a.reps, a.warmup)
    t_asm_c = median_ms(lambda: E.assembleColoredPointCloud(eng, sms, 0.1), a.reps, a.warmup)
    t_comp = median_ms(lambda: composition(eng, sms, 0.0, buf), a.reps, a.warmup)
    t_comp_v = median_ms(lambda: composition(eng, sms, 0.1, buf), a.reps, a.warmup)
    t_dl = median_ms(lambda: download_path(sms), max(1, a.reps // 2), 1)
    hx, hn = download_path(sms)
    m = min(a.host_points, len(hx))
    t0 = time.perf_counter()
    O.voxel_down_sample(hx[:m], 0.1, hn[:m])
    t_host_vox = (time.perf_counter() - t0) * 1e3

    res = {"card": dev_name, "submaps": len(sms), "points_total": total, "points_min": int(min(sizes)), "points_max": int(max(sizes)),
           "voxels_at_0.1": n_vox, "assembly_equals_composition_bitwise": identical,
           "assemble_ms": round(t_asm, 2), "assemble_voxel_0.1_ms": round(t_asm_v, 2), "assemble_colored_0.1_ms": round(t_asm_c, 2),
           "composition_ms": round(t_comp, 2), "composition_voxel_0.1_ms": round(t_comp_v, 2),
           "download_concat_ms": round(t_dl, 2), "host_voxel_0.1_points": int(m), "host_voxel_0.1_ms_one_core": round(t_host_vox, 1)}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
