"""Localisation against a growing prior map: per-scan time of the tile path (static map patch) and of the full path (B2S_PATCH_FULL=1).

Prior maps: the device map of the first half lap of ClosedLoop, replicated at 100 m offsets (1x1, 2x2, 4x4 copies), so the patch around
the sensor stays the same while the map grows.  Every chain localises lap-2 scans from the true pose with merging off, as one CUDA graph
per scan (b2s_mapper_step_host_async, all chains enqueued, then one synchronisation per step).  The library reads B2S_PATCH_FULL once
per process, so each setting runs in child processes of its own, alternated.  Also reported: the one-off tile-table build (the first
registration minus a steady one, one chain) and the initial-map load (normals + voxel down-sample) of the largest map.

    python tools/localization_bench.py [--steps 30] [--warmup 5] [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def child(steps, warmup):
    import numpy as np
    import torch
    from open3d_slam_b200 import engine as E
    from open3d_slam_b200 import slam as S
    from open3d_slam_b200 import workloads as W

    lp = W.ClosedLoop()
    p = E.MapperParameters(seed=3)
    dev = S.DeviceBackend(p, carving=False, dense=False, graph=False, submap_capacity=2_000_000)
    m = S.SegmentMapper(dev, S.SubmapParameters(radius=1e4))
    for k in range(lp.L // 2):
        m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
    base, nrm = dev.map_cloud(m.submaps.submaps[0].handle)
    dev.close()
    k0 = 2
    scans = [np.ascontiguousarray(lp.scan(k0 + 1 + i + lp.L, seed=900 + i)) for i in range(warmup + steps)]
    out = {"base_points": int(len(base)), "maps": {}}
    for R in (1, 2, 4):
        off = np.array([(100.0 * i, 100.0 * j, 0.0) for i in range(R) for j in range(R)])
        xyz = np.concatenate([base + o for o in off]); nn = np.concatenate([nrm] * len(off))
        res = {"map_points": int(len(xyz))}
        for chains in (1, 16):
            mps = []
            for _ in range(chains):
                eng = E.Engine(p)
                mp = E.Mapper(eng, len(xyz) + 16)
                c = eng.cloud(xyz, nn)
                mp.submap.setMapPointCloud(c)
                mp.submap.setMergeScans(False)
                mp.enableGraph(70_000)
                mp.setMapToRangeSensorInitial(lp.map_frame_pose(k0))
                pin = torch.empty((70_000, 3), dtype=torch.float32).pin_memory()
                outp = torch.empty(256, dtype=torch.uint8).pin_memory()
                mps.append((eng, mp, pin, outp))
            if chains == 1 and R == 1:   # the table build: the first registration after merge went off, minus a steady one
                eng, mp, _, _ = mps[0]
                sc = eng.cloud(scans[0]); ps = mp.scan2MapReg_.processForScanMatchingAndMerging(sc)
                T = lp.map_frame_pose(k0)
                eng.synchronize(); t0 = time.perf_counter(); mp.scan2MapReg_.scanToMapRegistration(ps.match_, mp.submap, T, T)
                t1 = time.perf_counter(); mp.scan2MapReg_.scanToMapRegistration(ps.match_, mp.submap, T, T); t2 = time.perf_counter()
                out["first_registration_ms"] = 1e3 * (t1 - t0); out["steady_registration_ms"] = 1e3 * (t2 - t1)
            times = []
            for i, s in enumerate(scans):
                k = k0 + 1 + i
                t0 = time.perf_counter()
                for eng, mp, pin, outp in mps:
                    pin[:len(s)].copy_(torch.from_numpy(s))
                    mp.addRangeMeasurementHostAsync(pin.data_ptr(), len(s), lp.delta(k), outp.data_ptr())
                for eng, *_ in mps:
                    eng.synchronize()
                if i >= warmup:
                    times.append(time.perf_counter() - t0)
            res[f"chains{chains}_ms_per_step"] = 1e3 * float(np.median(times))
            res[f"chains{chains}_captures"] = int(sum(e.graphCaptures for e, *_ in mps))
            for eng, mp, *_ in mps:
                mp.submap.free()
        out["maps"][f"{R}x{R}"] = res
    # the initial-map load of the largest map: normals on the full cloud, then the voxelized load
    eng = E.Engine(p); mp = E.Mapper(eng, len(xyz) + 16)
    p.isUseInitialMap = True
    c = eng.cloud(np.ascontiguousarray(xyz))
    eng.synchronize(); t0 = time.perf_counter()
    mp.scan2MapReg_.prepareInitialMap(c); eng.synchronize(); t1 = time.perf_counter()
    mp.submap.setInitialMap(c, p.mapBuilder.mapVoxelSize); eng.synchronize(); t2 = time.perf_counter()
    out["initial_map_load"] = {"points": int(len(xyz)), "normals_ms": 1e3 * (t1 - t0), "voxel_load_ms": 1e3 * (t2 - t1)}
    print("RESULT " + json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    if a.child:
        return child(a.steps, a.warmup)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    runs = {"tile": [], "full": []}
    for rep in range(a.reps):
        for mode in (("tile", "full") if rep % 2 == 0 else ("full", "tile")):
            env = dict(os.environ)
            env.pop("B2S_PATCH_FULL", None)
            if mode == "full":
                env["B2S_PATCH_FULL"] = "1"
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--steps", str(a.steps), "--warmup", str(a.warmup)],
                               env=env, capture_output=True, text=True)
            line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
            if r.returncode or not line:
                sys.exit(f"child ({mode}) failed:\n{r.stderr[-3000:]}")
            runs[mode].append(json.loads(line[0][7:]))
    print(json.dumps({"card": card, "runs": runs}))


if __name__ == "__main__":
    main()
