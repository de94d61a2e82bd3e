"""GPU test of slam.loopClosureCycle end to end on the closed lap: SegmentMapper over the device backend and over the oracle backend
(tests/oracle_backend_pose_graph.py), one loop closure refined on the device, then the cycle on both: odometry constraints (one batched
device call), the solve (b2s_global_optimization against the numpy restatement), the correction of every submap and of the mapper."""
import copy

import numpy as np
import pytest

from oracle_backend_pose_graph import PoseGraphOracleBackend
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import slam as S
from open3d_slam_b200 import workloads as W

pytestmark = pytest.mark.gpu

N_SCANS = 208


def test_loop_closure_cycle_on_the_closed_lap():
    p = E.MapperParameters(seed=3)
    lp = W.ClosedLoop()
    sp = S.SubmapParameters(radius=10.0)
    dev = S.DeviceBackend(copy.deepcopy(p), carving=True, dense=True, graph=True)
    ora = PoseGraphOracleBackend(copy.deepcopy(p), carving=True, dense=True)
    md, mo = S.SegmentMapper(dev, sp), S.SegmentMapper(ora, sp)
    for k in range(N_SCANS):
        raw, d = lp.scan(k, seed=k), lp.delta(k)
        md.addRangeMeasurement(raw, d)
        mo.addRangeMeasurement(raw, d)
    sc, so = md.submaps, mo.submaps
    assert len(sc.submaps) == len(so.submaps) >= 3
    # one loop closure: the last finished submap against submap 0, refined on the device from the identity (the lap closes on itself)
    src = max(sc.finishedSubmapsIdxs)
    assert src >= 2
    ref = S.refineLoopClosures(dev, dev.submap_as_cloud(sc.submaps[src].handle), [dev.submap_as_cloud(sc.submaps[0].handle)], [np.eye(4)],
                               p.mapBuilder.mapVoxelSize)[0]
    T = np.array(ref["result"].transformation_)
    info = dev.information_matrix(dev.submap_as_cloud(sc.submaps[src].handle), dev.submap_as_cloud(sc.submaps[0].handle), 0.3, T)
    lc = S.Constraint(T, src, 0, np.array(info))

    # the device maps as they are, copied into fresh submaps: the increment the cycle applies must move them bit for bit alike
    copies = []
    for rec in sc.submaps:
        cp = E.Submap(dev.eng, dev.submap_capacity)
        c = rec.handle.toCloud()
        cp.setMapPointCloud(c)
        c.free()
        copies.append(cp)
    applied = {}
    orig = dev.transform_submap

    def recording(sm, sparse, T):
        applied[id(sm)] = np.array(T)
        orig(sm, sparse, T)

    dev.transform_submap = recording
    truth = [np.linalg.inv(lp.pose(0)) @ lp.pose(k) for k in range(N_SCANS)]   # in the mapper's frame (scan 0 at the identity)

    def translation_error(mapper):
        return float(np.mean([np.linalg.norm(P[:3, 3] - G[:3, 3]) for P, G in zip(mapper.poses, truth)]))

    pd_, po_ = S.OptimizationProblem(dev), S.OptimizationProblem(ora)
    err_before = translation_error(md)
    dTd = S.loopClosureCycle(dev, md, pd_, [lc])
    dTo = S.loopClosureCycle(ora, mo, po_, [copy.deepcopy(lc)])
    sd, so_ = pd_.lastStats, po_.lastStats
    for a, b in zip(sd, so_):
        assert (a.valid, a.n_edges, a.lm_tries, a.accepted_steps, a.stop_reason) == (b.valid, b.n_edges, b.lm_tries, b.accepted_steps, b.stop_reason)
    nd, no = pd_.poseGraphOptimized_.nodes_, po_.poseGraphOptimized_.nodes_
    assert len(nd) == len(no)
    for a, b in zip(nd, no):
        assert np.abs(a.pose_ - b.pose_).max() < 1e-6
    assert np.abs(dTd - dTo).max() < 1e-6
    # the mapper's trajectory corrected from here on: the reference moves the pose, not the history; the latest pose's error
    last_gt = truth[-1][:3, 3]
    err_last_before = float(np.linalg.norm(md.poses[-1][:3, 3] - last_gt))
    err_last_after = float(np.linalg.norm(md.mapToRangeSensor[:3, 3] - last_gt))
    print(f"submaps {len(sc.submaps)}, loop closure {src} -> 0 fitness {ref['result'].fitness_:.3f}; stats {sd}; mean trajectory error "
          f"{err_before:.4f} m; latest pose error {err_last_before:.4f} m before the cycle, {err_last_after:.4f} m after")
    assert err_last_after < err_last_before   # observed on an H100: 0.0121 m -> 0.0063 m (9 submaps, loop closure 7 -> 0)
    # every device map equals b2s_submap_transform of its copy with the increment the cycle applied to it
    for rec, cp in zip(sc.submaps, copies):
        Tinc = applied[id(rec.handle)]
        cp.transform(Tinc)
        a, _ = rec.handle.getMapPointCloud()
        b, _ = cp.getMapPointCloud()
        assert a.shape == b.shape and np.array_equal(a, b)
        cp.free()
    # the active submap's slot holds dT * (the mapper pose before): the next step replays its graph and agrees with the oracle
    assert np.allclose(sc.getActiveSubmap().handle.getPose(), md.mapToRangeSensor, rtol=0, atol=1e-12)
    caps = dev.eng.graphCaptures
    raw, d = lp.scan(N_SCANS, seed=N_SCANS), lp.delta(N_SCANS)
    rd = md.addRangeMeasurement(raw, d)
    ro = mo.addRangeMeasurement(raw, d)
    assert dev.eng.graphCaptures == caps
    assert np.abs(np.asarray(rd.transformation_) - np.asarray(ro.transformation_)).max() < 1e-6
    dev.close()
