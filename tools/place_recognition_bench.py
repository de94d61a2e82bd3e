"""Loop-closure proposal on the device (DESIGN.md row K-ransac) at the Lua parameters: one 20 m source submap against K = 1, 4 and 16
candidate submaps built by the Config4 target builder on the closed lap (candidate 0 is the source's place, fused from other scans).
CUDA-event times of the feature correspondences (b2s_feature_correspondences, per pair), of the batched RANSAC and of the whole
slam.buildLoopClosureConstraints (proposal, gate, consistency, refinement), the hypotheses and validations per pair, and the C
restatement's time for the matching pair on one host core.  Prints a JSON line with the card name and its power limit; a number
from this script is only meaningful together with those two.
usage: python tools/place_recognition_bench.py [--warmup 1] [--reps 3] [--out FILE]
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
import oracle_ransac as OR

ap = argparse.ArgumentParser()
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--reps", type=int, default=3)
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


def timed(fn):
    for _ in range(args.warmup):
        out = fn()
    ms = []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        out = fn()
        b.record(stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), out


p = E.MapperParameters(seed=3)
dev = S.DeviceBackend(copy.deepcopy(p), cuda_stream=stream.cuda_stream, carving=False, dense=False, graph=False)
eng = dev.eng
lp = W.ClosedLoop()
c4 = W.Config4(lp, n_pairs=16, n_targets=16)
icp = E.ScanToMapIcp(eng)
prm = E.PlaceRecognitionParameters()


def as_submap(cloud):
    sm = E.Submap(eng, 900_000)
    sm.setMapPointCloud(cloud)
    cloud.free()
    sm.computeFeatures(prm)
    return sm


# the source: the place of candidate 0 from the scans between its scans (positions shifted by 2 = 1 m)
shifted = copy.copy(c4)
shifted.target_positions = lambda t: [k + 2 for k in W.Config4.target_positions(c4, t)]
source = as_submap(shifted.build_target(E, eng, icp, p, 0))
cands = [as_submap(c4.build_target(E, eng, icp, p, t)) for t in range(16)]
sc = S.SubmapCollection(dev, S.SubmapParameters())
for k, sm in enumerate([source] + cands):
    r = S.SubmapRecord(sm, k, 0, np.zeros(3))
    r.sparse, r.feature = sm.getSparseMapPointCloud(), sm.getFeatures()
    sc.submaps.append(r)
src = sc.submaps[0]
corr_ms, _ = timed(lambda: E.featureCorrespondences(eng, src.feature, sc.submaps[1].feature))
rows = []
for K in (1, 4, 16):
    tg = sc.submaps[1:1 + K]
    ransac_ms, res = timed(lambda: dev.ransac(src.sparse, src.feature, [t.sparse for t in tg], [t.feature for t in tg], prm))
    build_ms, (cons, log) = timed(lambda: S.buildLoopClosureConstraints(dev, sc, 0, list(range(1, 1 + K)), prm, p.mapBuilder.mapVoxelSize))
    rows.append({"K": K, "ransac_ms": ransac_ms, "build_loop_closure_constraints_ms": build_ms,
                 "hypotheses": [r.hypotheses for r in res], "validations": [r.validations for r in res], "inliers": [r.n_corr for r in res],
                 "decisions": [d for _, d, _ in log]})
    print(f"K={K}: RANSAC {ransac_ms:.2f} ms, buildLoopClosureConstraints {build_ms:.2f} ms; hypotheses {rows[-1]['hypotheses']} "
          f"validations {rows[-1]['validations']} decisions {rows[-1]['decisions']}")
sx, _ = src.sparse.download(); sf = src.feature.data_.T
tx, _ = sc.submaps[1].sparse.download(); tf = sc.submaps[1].feature.data_.T
t0 = time.perf_counter()
ref = OR.ransac(sx, sf, tx, tf, OR.Params.of(prm))
host_ms = 1e3 * (time.perf_counter() - t0)
res = {"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "params": vars(prm),
       "source_sparse_points": len(sx), "candidate_sparse_points": [len(t.sparse) for t in sc.submaps[1:]],
       "correspondences_ms_per_pair": corr_ms, "runs": rows,
       "host_c_restatement_ms_matching_pair": host_ms, "host_hypotheses": ref.hypotheses, "host_validations": ref.validations,
       "timing": f"CUDA events on the engine's stream, median of {args.reps} after {args.warmup} warm-up; correspondences include the D2H copy"}
line = json.dumps(res)
print(line)
if args.out:
    with open(args.out, "w") as f:
        f.write(line + "\n")
dev.close()
