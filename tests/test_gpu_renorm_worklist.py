"""-m gpu: K3's renormalisation worklist leaves the map bit-identical to the pass over every map slot (B2S_RENORM_FULL=1).

K3 applies the reference's normalized(n / 1) to the untouched in-cropper points of the map.  Only the slots whose normal is not yet
a fixed point of that operation are visited; the rest are skipped, which is exact only if no slot leaves the worklist too early and
every slot whose normal is rewritten (by K2, a rehash, Submap::transform or setMapPointCloud) joins it again.  The same runs go
through a child process per setting, since the library reads the knob once per process:
  - scans of the closed loop with host-made normals fused at fixed poses over more than a lap, with a carve (a rehash) every 10
    insertions and a cropper that holds every point: no merge depends on the order of the map's slots, so the final map is
    bit-identical keyed by voxel, positions and normals;
  - a loaded map with normals of arbitrary length and NaN normals, crossed by a sensor whose cropper covers a strip of it at a
    time, fed small scans at fixed poses: entries outside the cropper that are not fixed points must stay on the worklist until
    they enter it.  The map is bit-identical to the full pass, and the normals of the map points no scan came near equal a numpy
    replay of normalized() bit for bit, applied once per insertion that had the point inside the cropper;
  - the benchmark's chain over the same lap, eager and under graph replay, with carving every 10 insertions: per-scan iterations
    and correspondences identical, transforms to 1e-12 (the documented phase-2 summation noise, which also reaches the fused
    positions of the two runs), the final maps equal point for point to 1e-9;
  - a point-to-point submap loaded without normals (NaN), fed scans without normals and some with normals of arbitrary
    length, moved by Submap::transform, with part of the map outside the cropper: the same NaN normals, the rest to 1e-12
    (after the move, several map points of one voxel merge in the order of their slots, which comes from atomics).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CHILD = os.path.join(HERE, "renorm_child.py")
V = 0.1   # MapperParameters' map voxel


def run_child(out, env_extra):
    env = dict(os.environ)
    env.pop("B2S_RENORM_FULL", None)
    env.update(env_extra)
    proc = subprocess.run([sys.executable, "-s", CHILD, str(out)], env=env, capture_output=True, text=True, timeout=1800,
                          cwd=os.path.dirname(HERE))
    assert proc.returncode == 0, f"child {env_extra} exited with {proc.returncode}:\n{proc.stdout}\n{proc.stderr}"
    return dict(np.load(out))


def keyed_bits(xyz, nrm):
    """The map as a set keyed by voxel: rows ordered by key, then position; positions and normals as raw bits."""
    k = np.floor(xyz * (1.0 / V)).astype(np.int64)
    order = np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0], k[:, 2], k[:, 1], k[:, 0]))
    return xyz[order].view(np.int64), nrm[order].view(np.int64)


def assert_map_identical(a_xyz, a_nrm, b_xyz, b_nrm, what):
    assert len(a_xyz) == len(b_xyz), (what, len(a_xyz), len(b_xyz))
    ax, an = keyed_bits(a_xyz, a_nrm); bx, bn = keyed_bits(b_xyz, b_nrm)
    assert np.array_equal(ax, bx), what
    bad = np.any(an != bn, axis=1)
    assert not bad.any(), (what, int(bad.sum()), an[bad][:3].view(np.float64), bn[bad][:3].view(np.float64))


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    d = tmp_path_factory.mktemp("renorm")
    return run_child(d / "worklist.npz", {}), run_child(d / "full.npz", {"B2S_RENORM_FULL": "1"})


@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_mapper_chain_matches_the_full_pass(runs, mode):
    wl, full = runs
    a, b = wl[f"{mode}_res"], full[f"{mode}_res"]
    assert a.shape == b.shape and len(a) > 100
    assert np.array_equal(a[:, -1], b[:, -1]), "iterations"
    assert np.array_equal(a[:, -2], b[:, -2]), "correspondences"
    assert np.abs(a[:, :16] - b[:, :16]).max() <= 1e-12
    assert np.array_equal(wl[f"{mode}_counters"], full[f"{mode}_counters"])
    assert wl[f"{mode}_counters"].max() > 0
    ax, an = wl[f"{mode}_xyz"], wl[f"{mode}_nrm"]; bx, bn = full[f"{mode}_xyz"], full[f"{mode}_nrm"]
    assert len(ax) == len(bx) > 100_000
    oa = np.lexsort((ax[:, 2], ax[:, 1], ax[:, 0])); ob = np.lexsort((bx[:, 2], bx[:, 1], bx[:, 0]))
    assert np.abs(ax[oa] - bx[ob]).max() < 1e-9 and np.abs(an[oa] - bn[ob]).max() < 1e-9


def test_fixed_pose_fusion_matches_the_full_pass_bit_for_bit(runs):
    wl, full = runs
    assert len(full["fixed_xyz"]) > 100_000
    assert_map_identical(wl["fixed_xyz"], wl["fixed_nrm"], full["fixed_xyz"], full["fixed_nrm"], "fixed poses")


def renormalized(n):
    """K3's normalized(n / 1), row-wise, in the kernel's operation order (IEEE double, no FMA): bit-exact with the device."""
    n = np.where(np.isnan(n).any(axis=1, keepdims=True), 0.0, n)
    zz = (n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2]
    sn = np.sqrt(np.where(zz > 0.0, zz, 1.0))
    return np.where((zz > 0.0)[:, None], n / sn[:, None], n)


def test_points_entering_the_cropper_are_renormalised_bit_for_bit(runs):
    wl, full = runs
    assert_map_identical(wl["crop_xyz"], wl["crop_nrm"], full["crop_xyz"], full["crop_nrm"], "cropped")
    from scipy.spatial import cKDTree
    x0, n0, poses, R = wl["crop_map0_xyz"], wl["crop_map0_nrm"], wl["crop_poses"], float(wl["crop_r"])
    far = cKDTree(wl["crop_scan_world"]).query(x0)[0] > 0.3            # no scan point in or next to the point's voxel
    n = n0.copy()
    inside_at = np.zeros(len(x0), dtype=int); outside_first = np.zeros(len(x0), dtype=bool)
    for k, T in enumerate(poses):
        d = x0 - T[:3, 3]
        r = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        assert np.abs(r[far] - R).min() > 1e-9
        inside = r <= R
        n[inside] = renormalized(n[inside])
        outside_first |= (inside_at == 0) & ~inside
        inside_at += inside
    # the case under test: points outside at first, with a normal that is not a fixed point, that entered the cropper later
    late = far & outside_first & (inside_at > 0) & np.any(renormalized(n0).view(np.int64) != n0.view(np.int64), axis=1)
    assert late.sum() > 1000 and (late & np.isnan(n0).any(axis=1)).sum() > 100
    got = {x.tobytes(): m for x, m in zip(wl["crop_xyz"], wl["crop_nrm"])}
    idx = np.flatnonzero(far)
    assert len(idx) > 2000
    g = np.array([got[x0[i].tobytes()] for i in idx])
    bad = np.any(g.view(np.int64) != n[idx].view(np.int64), axis=1)
    assert not bad.any(), (int(bad.sum()), g[bad][:3], n[idx][bad][:3])


def test_nan_normal_point_to_point_map_matches_the_full_pass(runs):
    wl, full = runs
    n = full["p2p_nrm"]
    assert np.isnan(n).any() and (np.abs(np.linalg.norm(n, axis=1) - 1.0) > 0.0).any()   # NaN and not-yet-unit normals were kept
    ax, an = wl["p2p_xyz"], wl["p2p_nrm"]; bx, bn = full["p2p_xyz"], full["p2p_nrm"]
    assert len(ax) == len(bx)
    oa = np.lexsort((ax[:, 2], ax[:, 1], ax[:, 0])); ob = np.lexsort((bx[:, 2], bx[:, 1], bx[:, 0]))
    assert np.abs(ax[oa] - bx[ob]).max() < 1e-12
    an, bn = an[oa], bn[ob]
    assert np.array_equal(np.isnan(an), np.isnan(bn))
    assert np.nanmax(np.abs(an - bn)) < 1e-12
