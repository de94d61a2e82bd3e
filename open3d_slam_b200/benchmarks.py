"""Device-timed runs of BASELINE.json's configs 3, 4 and 5 (SURVEY.md section 8d), shared by bench.py (extra keys of its JSON
line) and tools/.  CUDA events on the launching stream, L2 flushed (256 MiB write) between repetitions, max over ranks.
torch is plumbing here: streams, events, the flush buffer and torch.distributed (NCCL)."""
from __future__ import annotations

import ctypes as C
import time

import numpy as np

from . import _lib as L
from . import dist as D
from . import engine as E
from . import slam as S
from . import workloads as W


def hbm_peak():
    return 3350.0, "H100 SXM data sheet (HBM3, 700 W card); not a measured figure"


class Timer:
    """CUDA-event timing of fn() on `stream` with an L2 flush before every repetition."""

    def __init__(self, dev, stream):
        import torch
        self.torch, self.dev, self.stream = torch, dev, stream
        self.flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def __call__(self, fn, reps=5, warm=2, before=None):
        torch = self.torch
        ts = []
        for r in range(reps + warm):
            with torch.cuda.stream(self.stream):
                self.flush.fill_(r & 0xFF)
                if before is not None:
                    before()
                a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
                a.record(self.stream); fn(); b.record(self.stream)
            self.stream.synchronize()
            if r >= warm:
                ts.append(a.elapsed_time(b))
        return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


# ----------------------------------------------------------------------------------------------------------------------
# config 3: voxel down-sample + normals on 2^20 points
# ----------------------------------------------------------------------------------------------------------------------
def run_config3(dev, stream, reps=8):
    VOXEL, KNN, RADIUS = 0.1, 20, 3.0
    xyz = W.config3_cloud()
    N = xyz.shape[0]
    p = E.MapperParameters()
    p.icp.knn = KNN; p.icp.maxDistanceKnn = RADIUS
    eng = E.Engine(p, device=dev.index or 0, cuda_stream=stream.cuda_stream)
    raw = eng.cloud(xyz); vox = E.Cloud(eng)
    lib = L.lib()
    t = Timer(dev, stream)
    l0 = eng.launches
    ms_vox = t(lambda: L.check(lib.b2s_voxel_down_sample(eng._h, raw._c, C.c_double(VOXEL), vox._c)), reps, 3)
    launches_vox = (eng.launches - l0) // (reps + 3)
    M = len(vox)
    l0 = eng.launches
    ms_nrm = t(lambda: L.check(lib.b2s_estimate_normals(eng._h, vox._c, C.c_int32(KNN), C.c_double(RADIUS))), reps, 3)
    launches_nrm = (eng.launches - l0) // (reps + 3)
    peak, peak_src = hbm_peak()
    bv, bn = 24.0 * N + 24.0 * M, 24.0 * M * (KNN + 2)       # algorithmic bytes in the engine's fp64 layout (DESIGN.md section 5)
    out = {"workload": "config3: voxel down-sample + normals, 2^20 returns of 21 scans of 64x1024 in the map frame", "N": N, "M": M,
           "voxel_size": VOXEL, "knn": KNN, "radius": RADIUS,
           "voxel": {"ms_median": ms_vox[0], "ms_min": ms_vox[1], "launches": int(launches_vox), "algorithmic_bytes": bv,
                     "achieved_gbs": bv / ms_vox[0] / 1e6, "frac_of_hbm_peak": bv / ms_vox[0] / 1e6 / peak, "mpoints_per_s": N / ms_vox[0] / 1e3},
           "normals": {"ms_median": ms_nrm[0], "ms_min": ms_nrm[1], "launches": int(launches_nrm), "algorithmic_bytes": bn,
                       "achieved_gbs": bn / ms_nrm[0] / 1e6, "frac_of_hbm_peak": bn / ms_nrm[0] / 1e6 / peak, "mpoints_per_s": M / ms_nrm[0] / 1e3},
           "peak_gbs": peak, "peak_source": peak_src, "timing": "CUDA events on the launching stream, median of %d, 256 MiB L2 flush before each" % reps}
    raw.free(); vox.free(); eng.close()
    return out


# ----------------------------------------------------------------------------------------------------------------------
# config 4: 512 scan-submap pairs over 64 shared targets, strong scaling over the ranks
# ----------------------------------------------------------------------------------------------------------------------
def run_config4(dev, stream, world, rank, loop=None, n_pairs=512, n_targets=64, reps=5):
    import torch
    loop = loop or W.ClosedLoop()
    p = E.MapperParameters(seed=3)
    eng = E.Engine(p, device=dev.index or 0, cuda_stream=stream.cuda_stream)
    icp = E.ScanToMapIcp(eng)
    c4 = W.Config4(loop, n_pairs, n_targets)
    mine = list(D.shard_range(n_pairs, world, rank))
    needed = sorted({c4.target_of(i) for i in mine})
    # every target is built ONCE, by its owner (round robin), and broadcast to the ranks that register against it
    t0 = time.perf_counter()
    owned = {}
    for t in range(n_targets):
        if D.owner_of(t, world) == rank:
            owned[t] = c4.build_target(E, eng, icp, p, t)
    local = {}
    for t, c in owned.items():
        n = len(c)
        x = torch.empty((n, 3), dtype=torch.float64, device=dev); nr = torch.empty((n, 3), dtype=torch.float64, device=dev)
        c.export_device(x.data_ptr(), nr.data_ptr(), n)
        local[t] = (x, nr)
    with torch.cuda.stream(stream):
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(stream)
        shared, recv_bytes = D.broadcast_point_sets(local, n_targets, world, rank, dev, needed)
        b.record(stream)
    stream.synchronize()
    bcast_ms = a.elapsed_time(b)
    targets = {}
    for t in needed:
        if t in owned:
            targets[t] = owned[t]
        else:
            x, nr = shared[t]
            targets[t] = E.Cloud(eng).import_device(x.data_ptr(), nr.data_ptr(), x.shape[0])
    eng.synchronize()
    sources = [c4.build_source(E, eng, icp, i) for i in mine]
    inits = [c4.init(i) for i in mine]
    tgt_list = [targets[c4.target_of(i)] for i in mine]
    build_s = time.perf_counter() - t0
    reg = c4.registration(E, eng, p)
    tm = Timer(dev, stream)
    res_box = {}

    def batch():
        res_box["r"] = reg.registerCloudsBatch(sources, tgt_list, inits)

    def sync_ranks():
        if world > 1:
            import torch.distributed as dist
            dist.barrier()

    ms = tm(batch, reps, 2, before=sync_ranks)
    eng.profile_enable(True); eng.profile_read()
    batch()
    prof = {k: round(v[0], 3) for k, v in eng.profile_read().items() if v[1] > 0}
    eng.profile_enable(False)
    res = res_box["r"]
    ms_max = D.max_over_ranks(ms[0], world, dev)
    tab = np.array([[*r.transformation_.ravel(), r.fitness_, r.inlier_rmse_, r.iters, r.n_corr] for r in res]).reshape(len(res), 20)
    err = np.array([np.linalg.norm(r.transformation_[:3, 3] - c4.truth(i)[:3, 3]) for r, i in zip(res, mine)]).reshape(len(res), 1)
    nsrc = np.array([r.n_corr / max(r.fitness_, 1e-12) for r in res]).reshape(len(res), 1)
    full = D.gather_results(np.c_[tab, err, nsrc], n_pairs, world, rank, dev)
    recv_total = D.max_over_ranks(float(recv_bytes), world, dev)
    peak, peak_src = hbm_peak()
    out = None
    if rank == 0:
        iters, n_src = full[:, 18], full[:, 21]
        bytes_icp = float(np.sum(72.0 * n_src * (iters + 1)))          # algorithmic bytes of all ICP evaluations (fp64 layout)
        icp_ms = prof.get("icp", float("nan"))
        out = {"workload": "config4: %d scan-submap pairs over %d shared 20 m-radius targets, r=0.3, max_iter=100" % (n_pairs, n_targets),
               "pairs": n_pairs, "targets": n_targets, "n_gpus": world, "scaling": "strong", "ms_per_batch": ms_max,
               "registrations_per_s": n_pairs / ms_max * 1e3, "mean_source_points": float(n_src.mean()),
               "mean_target_points": float(np.mean([len(t) for t in targets.values()])), "mean_iters": float(iters.mean()),
               "min_fitness": float(full[:, 16].min()), "median_translation_error_m": float(np.median(full[:, 20])),
               "frac_within_10cm": float((full[:, 20] < 0.1).mean()),
               "kernel_group_ms_rank0": prof,
               "roofline": {"bound": "hbm", "kernel": "icp (batched)", "bytes": bytes_icp / world, "ms": icp_ms,
                            "achieved": bytes_icp / world / icp_ms / 1e6 if icp_ms == icp_ms else None, "peak": peak, "unit": "GB/s",
                            "frac": bytes_icp / world / icp_ms / 1e6 / peak if icp_ms == icp_ms else None, "peak_source": peak_src},
               "shared_targets": {"collective": "broadcast of each target's {point, normal} per voxel from its owner (round robin)" if world > 1 else None,
                                  "nccl_bytes_received_per_rank_max": recv_total, "broadcast_ms_rank0": bcast_ms},
               "setup_s_rank0": build_s,
               "timing": "CUDA events around b2s_register_batch (index build per distinct target + one batched ICP launch + D2H of results), "
                         "median of %d, barrier + 256 MiB L2 flush before each, max over ranks" % reps}
    for c in list(targets.values()) + sources:
        c.free()
    eng.close()
    return out


# ----------------------------------------------------------------------------------------------------------------------
# config 5: the full mapper (one robot per GPU)
# ----------------------------------------------------------------------------------------------------------------------
def lua_mapper_parameters(seed=3):
    """The Lua defaults of the mapper around the hot path: carving voxel 0.2 / truncation 0.3 / every 10 scans, submap size 20 m,
    10 scans minimum, 10 overlap scans, revisit fitness 0.5 (param/default/parameter_structure_definitions.lua:87-100), dense map off."""
    p = E.MapperParameters(seed=seed)
    p.mapBuilder.carving.voxelSize = 0.2
    p.mapBuilder.carving.truncationDistance = 0.3
    sp = S.SubmapParameters(radius=20.0, minNumRangeData=10, adjacencyBasedRevisitingMinFitness=0.5, numScansOverlap=10)
    return p, sp


def run_config5(dev, stream, world, rank, loop=None, n_scans=354, submap_radius=10.0):
    """One robot per GPU: n_scans (3 laps) through SegmentMapper on the device backend -- per scan ONE C call with host buffers
    (float32 scan in, RegistrationResult out) replaying the captured chain S1 -> S2 -> gates -> carving -> F1, host decisions
    (hand-over, revisit) in between; after every hand-over the loop-closure refinement between the finished submap and the others.
    Wall-clock per scan is the number: this is the latency path of one robot.  submap_radius 10 m (default 20) so that the
    16 m x 16 m loop produces hand-overs."""
    import torch
    loop = loop or W.ClosedLoop()
    p, sp = lua_mapper_parameters()
    sp.radius = submap_radius
    be = S.DeviceBackend(p, device=dev.index or 0, cuda_stream=stream.cuda_stream, carving=True, dense=False, graph=True)
    m = S.SegmentMapper(be, sp)
    scans = [loop.scan(k, seed=k) for k in range(min(n_scans, loop.L))]
    deltas = [loop.delta(k) for k in range(n_scans)]
    lc_ms, lc_n, lc_acc = 0.0, 0, 0
    seen_finished = 0
    l0 = be.eng.launches
    torch.cuda.synchronize(dev)
    t_all = time.perf_counter()
    t_steps = 0.0
    lat = []
    for k in range(n_scans):
        t0 = time.perf_counter()
        m.addRangeMeasurement(scans[k % loop.L], deltas[k])
        dt = time.perf_counter() - t0
        t_steps += dt
        lat.append(dt)
        fin = m.submaps.finishedSubmapsIdxs
        if len(fin) > seen_finished:    # a submap was finished: refine loop closures against every other submap, one batch
            seen_finished = len(fin)
            src = fin[-1]
            others = [i for i in range(len(m.submaps.submaps)) if i != src]
            t1 = time.perf_counter()
            sc = be.submap_as_cloud(m.submaps.submaps[src].handle)
            tcs = [be.submap_as_cloud(m.submaps.submaps[i].handle) for i in others]
            out = S.refineLoopClosures(be, sc, tcs, [np.eye(4) for _ in others], p.mapBuilder.mapVoxelSize)
            be.eng.synchronize()
            lc_ms += (time.perf_counter() - t1) * 1e3
            lc_n += len(others); lc_acc += sum(1 for o in out if o["accepted"])
            for c in [sc] + tcs:
                c.free()
    be.eng.synchronize()
    wall = time.perf_counter() - t_all
    gt = loop.map_frame_pose(n_scans - 1)
    err = float(np.linalg.norm(m.mapToRangeSensor[:3, 3] - gt[:3, 3]))
    cnt = [be.counters(s.handle) for s in m.submaps.submaps]
    lat_ms = np.array(lat[5:]) * 1e3
    out = {"workload": "config5: full mapper, %d scans (%.1f laps of the closed loop), carving every 10 insertions (Lua defaults), submap radius %.0f m, "
                       "hand-overs + overlap buffer + revisit check, loop-closure refinement (overlap -> batched ICP -> information matrix) per finished submap"
                       % (n_scans, n_scans / loop.L, submap_radius),
           "scans": n_scans, "scans_per_s_per_robot": n_scans / wall, "robots": world, "scans_per_s": world * n_scans / wall,
           "ms_per_scan_median": float(np.median(lat_ms)), "ms_per_scan_p95": float(np.percentile(lat_ms, 95)), "mapping_steps_s": t_steps,
           "loop_closure": {"batches": seen_finished, "registrations": lc_n, "accepted": lc_acc, "ms_total": lc_ms},
           "submaps": len(m.submaps.submaps), "hand_overs": sum(1 for e in m.submaps.events if e[0] == "active_submap_changed"),
           "revisit_checks": sum(1 for e in m.submaps.events if e[0] == "revisit_check"),
           "carve_runs": int(sum(c["carve_runs"] for c in cnt)), "carved_points": int(sum(c["carved_points_total"] for c in cnt)),
           "map_points": [int(len(be.map_cloud(s.handle)[0])) for s in m.submaps.submaps],
           "final_pose_err_m": err, "gpu_launches": int(be.eng.launches - l0),
           "timing": "host wall clock around the whole run (one synchronous C call per scan: H2D of the float32 scan, graph replay, D2H of the result)"}
    be.close()
    return out
