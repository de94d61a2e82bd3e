"""Loop-closure features of real submaps (b2s_submap_compute_features, DESIGN.md row K-features): the feature-cloud front end of
Submap::computeFeatures -- voxel down-sample of the map at 0.5 m, normals (k 20, r 2.0) with the voxel-mean normals as priors,
FPFH (k 100, r 2.5) -- timed per submap with CUDA events after warm-up, next to the C restatement of the same step
(tests/oracle_submap_features.c, one host core) on the same map.  The submaps are built by the engine's own mapper (SegmentMapper over
the device backend, 20 m submap radius) on the closed lap.  Prints one line per submap and a JSON summary with the card name and
its power limit; a number from this script is only meaningful together with those two.
usage: python tools/features_bench.py [--scans N] [--radius 20] [--warmup 2] [--reps 10] [--out FILE]
"""
import argparse, copy, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the C restatement is test infrastructure
import numpy as np
import torch
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W
import oracle_submap_features as OSF

ap = argparse.ArgumentParser()
ap.add_argument("--scans", type=int, default=0, help="scans of the closed lap to map (0 = two laps)")
ap.add_argument("--radius", type=float, default=20.0)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--out", default="")
args = ap.parse_args()


def power_limit_w():
    """read-only query of the enforced power limit (W); None when nvidia-smi is not available"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                             text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


stream = torch.cuda.Stream()
p = E.MapperParameters(seed=3)
lp = W.ClosedLoop()
n_scans = args.scans or 2 * lp.L
dev = S.DeviceBackend(copy.deepcopy(p), cuda_stream=stream.cuda_stream, carving=True, dense=False, graph=True)
m = S.SegmentMapper(dev, S.SubmapParameters(radius=args.radius))
for k in range(n_scans):
    m.addRangeMeasurement(lp.scan(k, seed=k), lp.delta(k))
prm = E.PlaceRecognitionParameters()
rows = []
for rec in m.submaps.submaps:
    sm = rec.handle
    for _ in range(args.warmup):
        sm.computeFeatures(prm)
    ms = []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        sm.computeFeatures(prm)
        b.record(stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    x, n = sm.getMapPointCloud()
    t0 = time.perf_counter()
    ref = OSF.submap_features(x, n, prm)
    host_ms = 1e3 * (time.perf_counter() - t0)
    row = {"submap": rec.id, "finished": rec.id in m.submaps.finishedSubmapsIdxs, "map_points": int(len(x)),
           "sparse_points": int(len(sm.getSparseMapPointCloud())), "device_ms_median": float(np.median(ms)), "device_ms_min": float(np.min(ms)),
           "host_c_ms": host_ms, "host_sparse_points": int(len(ref["xyz"]))}
    rows.append(row)
    print(f"submap {row['submap']}: map {row['map_points']} pts -> sparse {row['sparse_points']} pts; device {row['device_ms_median']:.3f} ms "
          f"(min {row['device_ms_min']:.3f}); C restatement, one host core {host_ms:.1f} ms")
res = {"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "scans": n_scans, "submap_radius": args.radius,
       "params": vars(prm), "submaps": rows}
line = json.dumps(res)
print(line)
if args.out:
    with open(args.out, "w") as f:
        f.write(line + "\n")
dev.close()
