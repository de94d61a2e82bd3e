"""-m gpu: the registration's single-thread pose solves against high-precision references (test_pose_solver_references.py), far from
the origin and at degenerate inputs.

One-iteration point-to-point ICP (max_iter = 1) on targets spaced more than twice the correspondence distance apart: the nearest
neighbour of every source point is its own target, so the device's first update is the Umeyama / Kabsch solution of known
correspondences, and T = update * init.  It is compared with the 50-digit Kabsch answer at
    |dR| <= 1e-13 and |dt| <= 1e-14 max(1, |offset|)
(a two-pass fp64 Umeyama meets this at every offset; the raw-moment one-pass form misses it from about 1e2-1e3 m on).
Where the init is not the identity, the device moves the source by it with the rounding of its own product, which
`moved_like_the_device` repeats bit for bit, and the reference solves from those points.
"""
import numpy as np
import pytest

from oracle import oracle as O
from open3d_slam_b200 import engine as E
from open3d_slam_b200 import synth
from test_pose_solver_references import (SKEW, kabsch_mp, kabsch_pose_mp, lattice_pairs, mp_to_np, nearest_pairs_are_exact,
                                         rotation, solve_exact, vec6_to_mat4)

pytestmark = pytest.mark.gpu


def moved_like_the_device(G, P):
    """icp_kernel's application of a non-identity init: ((G0 x + G1 y) + G2 z) + G3 per row, every operation rounded"""
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    return np.stack([((G[r, 0] * x + G[r, 1] * y) + G[r, 2] * z) + G[r, 3] for r in range(3)], 1)


def rigid(R, t):
    G = np.eye(4)
    G[:3, :3] = R; G[:3, 3] = t
    return G


def one_p2p_update(eng, src, tgt, max_corr, init=np.eye(4)):
    p = E.CloudRegistrationParameters(regType="PointToPointIcp", icp=E.IcpParameters(maxNumIter=1, maxCorrespondenceDistance=max_corr))
    return E.cloudRegistrationFactory(eng, p).registerClouds(eng.cloud(src), eng.cloud(tgt), init)


def assert_within_bound(T, Tref, offset):
    dR = np.abs(T[:3, :3] - Tref[:3, :3]).max()
    dt = np.abs(T[:3, 3] - Tref[:3, 3]).max()
    assert dR <= 1e-13 and dt <= 1e-14 * max(1.0, abs(offset)), (dR, dt)


def check_one_update(eng, src, tgt, max_corr, init, offset):
    assert nearest_pairs_are_exact(moved_like_the_device(init, src) if not np.array_equal(init, np.eye(4)) else src, tgt, max_corr)
    res = one_p2p_update(eng, src, tgt, max_corr, init)
    assert res.iters == 1 and res.n_corr == len(src)
    moved = src if np.array_equal(init, np.eye(4)) else moved_like_the_device(init, src)
    assert_within_bound(res.transformation_, kabsch_pose_mp(moved, tgt, init), offset)
    return res


# ---- 2. point-to-point far from the origin ------------------------------------------------------------------------------------
@pytest.mark.parametrize("rot", ["small", "large"])
@pytest.mark.parametrize("spread", [0.5, 5.0, 30.0])
@pytest.mark.parametrize("offset", [0.0, 1e2, 1e3, 1e4, 1e5])
def test_point_to_point_update_far_from_the_origin(engine_factory, offset, spread, rot):
    """small: an update of 1e-3 rad from the identity.  large: an update of 0.04 rad (the most a nearest-neighbour step can see on
    this lattice) composed with an init of 2.5 rad about a skew axis through the clouds' centre."""
    eng = engine_factory()
    src, tgt, mc = lattice_pairs(offset, spread, 1e-3 if rot == "small" else 0.04, seed=7 + int(spread))
    init = np.eye(4)
    if rot == "large":
        c = tgt.mean(0)
        RG = rotation([-0.6, 0.2, 0.9], 2.5)
        init = rigid(RG, c - RG @ c)
        src = (src - c) @ RG + c                        # RG^T (src - c) + c: the init carries it back next to the targets
    check_one_update(eng, src, tgt, mc, init, offset)


@pytest.mark.parametrize("offset", [0.0, 1e2, 1e3, 1e4, 1e5])
def test_point_to_point_icp_far_from_the_origin_matches_oracle(engine_factory, offset):
    """Full runs on the config-1 clouds moved off the origin along a skew direction: same iterations and correspondences as the
    oracle (two-pass Umeyama), T to 1e-9."""
    src, tgt, _, _ = synth.planar_cloud_config1(noise=0.01)
    base = offset * SKEW
    src, tgt = src + base, tgt + base
    p = E.MapperParameters()
    p.icp.maxCorrespondenceDistance = 1.0
    p.icp.maxNumIter = 50
    eng = engine_factory(p)
    reg = E.cloudRegistrationFactory(eng, E.CloudRegistrationParameters(regType="PointToPointIcp", icp=p.icp))
    for init in (np.eye(4), synth.se3(0.01, -0.02, 0.03, (0.05, 0.02, -0.01))):
        G = rigid(np.eye(3), base) @ init @ rigid(np.eye(3), -base)         # the same perturbation about the moved clouds
        res = reg.registerClouds(eng.cloud(src), eng.cloud(tgt), G)
        ref = O.registration_icp_p2point(src, tgt, 1.0, G, max_iter=50)
        assert res.iters == ref.iters and res.n_corr == ref.n_corr
        assert np.abs(res.transformation_[:3, :3] - ref.T[:3, :3]).max() < 1e-9
        assert np.abs(res.transformation_[:3, 3] - ref.T[:3, 3]).max() < 1e-9 * max(1.0, offset)


# ---- 4. degenerate Umeyama / SVD inputs ------------------------------------------------------------------------------------
def _planar(offset):
    """a level 8 x 8 plane: with a power-of-two count and correspondence distance (the grid cell is a quarter of it) the target row
    of the device's cross-covariance, (t - c)_z - (mt - c)_z, is exactly zero at every offset"""
    rng = np.random.default_rng(21)
    g = np.arange(-4, 4) * 0.5
    tgt0 = np.c_[np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2), np.zeros(64)]
    src0 = tgt0 @ rotation([0.4, -0.3, 0.2], 0.01).T + rng.uniform(-0.01, 0.01, tgt0.shape) * np.array([1, 1, 0])
    return src0, tgt0, 0.125


def _reflection(offset):
    """two thin layers, the lower one shifted by half a cell; the source is the targets mirrored through the mid-plane"""
    g = np.arange(-3.0, 4.0)
    xy = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
    tgt0 = np.r_[np.c_[xy, np.full(len(xy), 0.0625)], np.c_[xy + 0.5, np.full(len(xy), -0.0625)]]
    return tgt0 * np.array([1.0, 1.0, -1.0]), tgt0, 0.2


def _octahedron(offset):
    tgt0 = np.r_[np.eye(3), -np.eye(3)] * 2.0
    src0 = tgt0 @ rotation([0.5, 0.5, -0.7], 0.05).T
    return src0, tgt0, 0.6


DEGENERATE = {"planar": _planar, "reflection": _reflection, "octahedron": _octahedron}


@pytest.mark.parametrize("offset", [0.0, 1e3, 1e5])
@pytest.mark.parametrize("case", sorted(DEGENERATE))
def test_point_to_point_update_at_degenerate_inputs(engine_factory, case, offset):
    """planar (rank-2 cross-covariance, R still unique), an exact reflection (det U det V < 0: the rule flips the smallest singular
    direction) and the regular octahedron (three equal singular values): the same bound as far from the origin."""
    src0, tgt0, mc = DEGENERATE[case](offset)
    base = np.round(offset * SKEW)                    # integer metres: the moved coordinates keep the sets' exact structure
    src, tgt = src0 + base, tgt0 + base
    _, _, sgn = kabsch_mp(src, tgt)
    assert (sgn < 0) == (case == "reflection")
    check_one_update(engine_factory(), src, tgt, mc, np.eye(4), offset)


@pytest.mark.parametrize("axis", ["x", "y", "z", "skew"])
def test_point_to_point_update_composed_with_an_init_near_pi(engine_factory, axis):
    """An init within 1e-6 rad of pi (about each axis and a skew one) far from the origin: the update is still the Kabsch solution
    of the moved source, and T = update * init to the same bound."""
    ax = {"x": [1, 0, 0], "y": [0, 1, 0], "z": [0, 0, 1], "skew": [0.3, -0.8, 0.5]}[axis]
    src, tgt, mc = lattice_pairs(1e4, 5.0, 0.01, seed=31)
    c = tgt.mean(0)
    RG = rotation(ax, np.pi - 1e-6)
    init = rigid(RG, c - RG @ c)
    check_one_update(engine_factory(), (src - c) @ RG + c, tgt, mc, init, 1e4)


@pytest.mark.parametrize("offset", [0.0, 1e4])
def test_point_to_point_update_on_collinear_sets(engine_factory, offset):
    """Collinear sets (rank-1 cross-covariance): the rotation is not unique.  It must be proper and orthonormal to 1e-14, carry the
    source line's direction onto the target line's, and T must carry the source centroid onto the target centroid."""
    k = np.arange(-6, 7)[:, None]
    base = np.round(offset * SKEW)
    tgt = base + k * np.array([3.0, 0.0, 4.0]) / 10.0
    src = base + (k * np.array([3.0, 0.0, 4.0]) / 10.0) @ rotation([0.0, 1.0, 0.0], 0.02).T + np.array([0.01, -0.02, 0.005])

    def direction(P):                                  # principal direction of the points as stored (fp64 rounding included)
        d = np.linalg.svd(P - P.mean(0))[2][0]
        return d if d[2] > 0 else -d

    assert nearest_pairs_are_exact(src, tgt, 0.2)
    res = one_p2p_update(engine_factory(), src, tgt, 0.2)
    assert res.iters == 1 and res.n_corr == len(src)
    T = res.transformation_
    R = T[:3, :3]
    assert abs(np.linalg.det(R) - 1.0) < 1e-14 and np.abs(R.T @ R - np.eye(3)).max() < 1e-14
    assert np.abs(R @ direction(src) - direction(tgt)).max() < 1e-13 * max(1.0, offset / 1e3)
    assert np.abs(R @ src.mean(0) + T[:3, 3] - tgt.mean(0)).max() < 1e-14 * max(1.0, offset)


# ---- 5. the point-to-plane 6x6 solve with exact inputs --------------------------------------------------------------------
def _plane_system(src, tgt, nrm):
    """J = [p x n ; n], r = (p - q) . n per correspondence i -> i: JTJ and -JTr, exact for these dyadic inputs"""
    J = np.c_[np.cross(src, nrm), nrm]
    r = np.einsum("ij,ij->i", src - tgt, nrm)
    return J.T @ J, -(J.T @ r)


def _dyadic_walls(kind, seed):
    """Correspondences spaced 1 m apart with coordinates in 1/8 m and normals in {-1, -1/2, 0, 1/2, 1}: every product and partial sum
    of JTJ / JTr is exact in fp64, so any summation order gives the same system"""
    rng = np.random.default_rng(seed)
    pts, nrm = [], []
    g = np.arange(-3, 4, 1.0)
    walls = {"box": [(0, 1.0), (1, 1.0), (2, 1.0), (0, 0.5)], "plane": [(2, 1.0)], "corridor": [(0, 1.0), (2, 1.0)]}[kind]
    for axis, s in walls:
        for a in g:
            for b in g:
                p = np.zeros(3); p[axis] = 4.0 if axis != 2 else -2.0
                p[[i for i in range(3) if i != axis]] = [a, b]
                n = np.zeros(3); n[axis] = s
                if kind == "box" and axis == 0 and s == 0.5:   # a tilted wall makes the system fully ranked but not diagonal
                    p[0] = -4.0; n = np.array([0.5, 0.5, 0.0])
                pts.append(p); nrm.append(n)
    tgt = np.array(pts); nrm = np.array(nrm)
    src = tgt + rng.integers(-1, 2, tgt.shape) / 8.0
    return src, tgt, nrm


@pytest.mark.parametrize("kind", ["box", "plane", "corridor"])
def test_point_to_plane_update_with_exact_inputs(engine_factory, kind):
    """The device's first point-to-plane update is vec6_to_mat4 of the exact solution of the exact JTJ x = -JTr (to a bound from the
    condition number), and equals the oracle's one-iteration run to 1e-15: the inputs make the oracle's JTJ / JTr the same exact
    system, so that run is orc_ldlt6_solve on it followed by its vec6_to_mat4.  For the singular systems (one plane; a corridor of
    walls and floor) the unobservable components are exactly zero, as D^+ gives."""
    src, tgt, nrm = _dyadic_walls(kind, seed=5)
    A, b = _plane_system(src, tgt, nrm)
    x_exact = np.array([float(v) for v in solve_exact(A, b)])
    p = E.MapperParameters()
    p.icp.maxCorrespondenceDistance = 0.45
    p.icp.maxNumIter = 1
    eng = engine_factory(p)
    res = E.RegistrationIcpPointToPlane(eng).registerClouds(eng.cloud(src), eng.cloud(tgt, nrm), np.eye(4))
    assert res.iters == 1 and res.n_corr == len(src)
    T = res.transformation_
    obs = np.abs(A).sum(1) > 0
    ev = np.linalg.eigvalsh(A[np.ix_(obs, obs)])
    cond = ev.max() / ev.min()
    assert np.abs(T - vec6_to_mat4(x_exact)).max() <= 64 * np.finfo(float).eps * cond * max(1.0, np.abs(x_exact).max())
    ref = O.registration_icp_p2plane(src, tgt, nrm, 0.45, np.eye(4), max_iter=1)
    assert np.abs(T - ref.T).max() <= 1e-15
    if kind != "box":
        zero_t = [i - 3 for i in range(3, 6) if not obs[i]]
        assert all(T[i, 3] == 0.0 for i in zero_t)
        if not obs[2]:                                   # rotation about z unobservable: sin(x2) = 0 exactly
            assert T[1, 0] == 0.0


# ---- point-to-point scan-to-map far from the origin -----------------------------------------------------------------------
@pytest.mark.parametrize("offset", [0.0, 1e4])
def test_point_to_point_scan_to_map_far_from_the_origin(engine_factory, offset):
    """ScanToMapIcp with PointToPointIcp, the map and the trajectory moved `offset` metres off the origin: every scan-to-map
    registration against the cropped submap (the ICP reference point is the centre of the cropped map's grid) matches the oracle's
    restatement of the same steps -- same iterations and correspondences, rotation to 1e-13, translation to 1e-14 max(1, offset) m
    (on an H100 the device stays within 3e-15 and 5e-11 m at 1e4 m; raw moments were 5e-11 off in rotation there).  (A comparison with
    the same run at the origin, moved back, cannot be this tight: these runs stop on the 1e-6 relative fitness / RMSE criterion, and
    moving the map by even 1 m changes the voxel means in their last bits and the converged pose by up to 1e-5.)"""
    p = E.MapperParameters(seed=3)
    p.scanToMapRegType = "PointToPointIcp"
    p.scanProcessing.downSamplingRatio = 0.5
    eng = engine_factory(p)
    icp = E.ScanToMapIcp(eng)
    sm = E.Submap(eng, 600_000)
    sc = synth.Scene(); poses = synth.loop_trajectory(8)
    M = rigid(np.eye(3), np.round(offset * SKEW)) @ np.linalg.inv(poses[0])
    wide = O.cropper("MinMaxRadius", 2.0, 30.0)
    map_x = np.zeros((0, 3)); map_n = np.zeros((0, 3))
    for k in range(4):
        raw = synth.lidar_scan(sc, poses[k], seed=300 + k)
        ps = icp.processForScanMatchingAndMerging(eng.cloud(raw))
        (mx, mn), (ax, an) = O.process_scan(raw.astype(np.float64), wide, wide, 0.1, 20, 3.0, 0.5, 3)
        pose = M @ poses[k]
        if k > 0:
            prev = M @ poses[k - 1]
            guess = pose @ synth.se3(0.004, -0.003, 0.01, (0.05, -0.03, 0.01))
            got = icp.scanToMapRegistration(ps.match_, sm, prev, guess)
            px, _ = O.crop(O.cropper("MinMaxRadius", 2.0, 30.0, center=prev[:3, 3]), map_x, map_n)
            ref = O.registration_icp_p2point(ax, px, 1.0, guess, max_iter=50)
            assert ref.fitness > 0.7
            assert got.iters == ref.iters and got.n_corr == ref.n_corr
            assert np.abs(got.transformation_[:3, :3] - ref.T[:3, :3]).max() < 1e-13
            assert np.abs(got.transformation_[:3, 3] - ref.T[:3, 3]).max() < 1e-14 * max(1.0, offset)
        sm.insertScan(None, ps.merge_, pose)
        map_x, map_n = O.submap_insert_scan(map_x, map_n, mx, mn, pose, 0.1, O.cropper("MinMaxRadius", 2.0, 30.0, center=pose[:3, 3]))


# ---- 6. the pose buffer's interpolation on general rotations ----------------------------------------------------------------
@pytest.mark.parametrize("size", [2000, 5, 1])
def test_map_pose_buffer_interpolation_on_general_rotations(engine_factory, size):
    """b2s_slam_map_pose_push / b2s_slam_map_lookup (the same buffer view and interpolation as the odometry's buffer) on the pushes of
    buffer_pushes(): the device to tests/odometry_buffer.py at 1e-14 and to the 50-digit geodesic at 1e-12 on every query, clamped
    at both ends, with eviction (size 5) and a single entry (size 1).  1e-14, not 1e-15: the device's acos / sin are not the host
    libm's, and slerp's weights sin(t theta) / sin(theta) carry their last-ulp differences into the rotation (up to 1.3e-15 seen
    on an H100)."""
    from odometry_buffer import TransformInterpolationBuffer
    from test_pose_solver_references import buffer_pushes, buffer_queries, lookup_mp
    eng = engine_factory()
    odo = E.DeviceLidarOdometry(eng, E.OdometryParameters(bufferSize=size), 1024)
    buf = TransformInterpolationBuffer(size)
    pushes = buffer_pushes()
    for t, T in pushes:
        odo.pushMapToRangeSensor(t, T)
        buf.push(t, T)
    kept = pushes[-size:]
    for q in buffer_queries(pushes):
        T, has = odo._map_lookup(q)
        assert has == buf.has(q)
        assert np.abs(T - buf.get_transform(q)).max() <= 1e-14, q
        assert np.abs(T - lookup_mp(kept, q)).max() < 1e-12, q
    odo.free()
