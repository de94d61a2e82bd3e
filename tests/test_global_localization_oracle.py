"""CPU: the restatement of b2s_submap_global_localization (tests/oracle_global_localization.{c,py}) checked on hand-built inputs --
the C scores against the numpy twin, the hypothesis enumeration and tie rule, the suppression (also across +-pi), points on voxel
faces, the key limit, the default box and the runner-up rule."""
import math

import numpy as np

import oracle_global_localization as G


def _box(**kw):
    p = G.Params(x_min=-2.0, x_max=2.0, y_min=-1.5, y_max=1.5, step=0.5, n_yaw=8, yaw_step=2 * math.pi / 8, score_voxel=0.5)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _scene(seed):
    rng = np.random.default_rng(seed)
    m = rng.uniform(-4, 4, (400, 3)) * [1, 1, 0.2]
    m[::37] = np.nan                                                        # tombstones
    q = rng.uniform(-3, 3, (60, 3)) * [1, 1, 0.2]
    q[:10] = np.round(q[:10] * 2) / 2                                       # on voxel faces of the 0.5 m grid
    return m, q


def test_c_scores_equal_the_numpy_twin():
    for seed, kw in ((1, {}), (2, dict(n_z=3, z0=-0.5, z_step=0.5)), (3, dict(roll=0.1, pitch=-0.05, score_voxel=1.0)), (4, dict(step=0.3))):
        m, q = _scene(seed)
        p = _box(**kw)
        g = G.grid(p, m)
        a, b = G.scores(q, m, p, g), G.scores_np(q, m, p, g)
        assert a.shape == (g.n,) and np.array_equal(a, b), seed
        assert a.max() > 0


def test_enumeration_order_and_counts():
    p = _box(n_z=2, z0=1.0, z_step=0.25)
    g = G.grid(p, np.zeros((1, 3)))
    assert (g.nx, g.ny, g.n_yaw, g.n_z) == (9, 7, 8, 2)
    h = ((1 * 8 + 3) * 7 + 2) * 9 + 5                                        # h = ((iz n_yaw + j) n_y + iy) n_x + ix
    t, y, j = G.decode(p, g, h)
    assert j == 3 and y == -math.pi + 3 * (2 * math.pi / 8)
    assert np.array_equal(t, [-2.0 + 5 * 0.5, -1.5 + 2 * 0.5, 1.0 + 0.25])
    assert G.grid(_box(x_max=2.2), np.zeros((1, 3))).nx == 9                 # floor((x_max - x_min) / step) + 1


def test_order_and_tie_rule():
    hits = np.array([3, 5, 5, 1, 5, 0, 3], dtype=np.int32)
    assert list(G.order(hits)) == [1, 2, 4, 0, 6, 3, 5]


def test_suppression_keeps_distinct_and_wraps_at_pi():
    p = _box(n_candidates=3, nms_distance=0.6, nms_yaw=math.radians(50))
    g = G.grid(p, np.zeros((1, 3)))
    hits = np.zeros(g.n, dtype=np.int32)

    def hid(ix, iy, j):
        return (j * g.ny + iy) * g.nx + ix
    hits[hid(0, 0, 0)] = 9         # yaw -pi
    hits[hid(0, 0, 7)] = 8         # yaw +3pi/4: 45 degrees from -pi across the wrap -> suppressed
    hits[hid(1, 0, 0)] = 7         # 0.5 m away, same yaw -> suppressed
    hits[hid(2, 0, 0)] = 6         # 1.0 m away -> kept
    hits[hid(0, 0, 2)] = 6         # same place, 90 degrees -> kept, after hid(2, 0, 0) (equal hits, higher h)
    kept = G.candidates(hits, p, g)
    assert kept == [hid(0, 0, 0), hid(2, 0, 0), hid(0, 0, 2)]
    assert G.close(p, *G.decode(p, g, hid(0, 0, 0))[:2], *G.decode(p, g, hid(0, 0, 7))[:2])


def test_fewer_candidates_than_asked_and_pool_limit():
    p = _box(n_candidates=2, nms_distance=100.0, nms_yaw=4.0)                # everything is close to the first
    g = G.grid(p, np.zeros((1, 3)))
    hits = np.arange(g.n, dtype=np.int32)[::-1].copy()
    assert G.candidates(hits, p, g) == [0]


def test_points_on_voxel_faces():
    m = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]])                         # voxels (0,0,0) and (1,0,0) of a 1 m grid
    q = np.array([[-0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [2.0, 0.0, 0.0], [-1e-300, 0.0, 0.0]])
    p = G.Params(x_min=0.0, x_max=1.0, y_min=0.0, y_max=0.0, step=1.0, n_yaw=1, yaw0=0.0, yaw_step=0.0, score_voxel=1.0)
    g = G.grid(p, m)
    want = np.array([2, 2], dtype=np.int32)   # t = 0: keys 0, 1 hit, 2, -1 miss; t = 1: x = 1 and -1e-300 + 1 = 1 hit, 2 and 3 miss
    assert np.array_equal(G.scores(q, m, p, g), want)
    assert np.array_equal(G.scores_np(q, m, p, g), want)


def test_key_limit_is_a_miss():
    big = 1048574.0                                                          # |k| = 2^20 - 2: the largest valid key
    m = np.array([[big, 0.0, 0.0], [big + 1.0, 0.0, 0.0], [0.0, 0.0, 0.0]])  # the second is beyond the limit: never occupied
    q = np.array([[0.0, 0.0, 0.0]])
    p = G.Params(x_min=big - 1.0, x_max=big + 1.0, y_min=0.0, y_max=0.0, step=1.0, n_yaw=1, yaw0=0.0, yaw_step=0.0, score_voxel=1.0)
    g = G.grid(p, m)
    assert np.array_equal(G.scores(q, m, p, g), [0, 1, 0])
    assert np.array_equal(G.scores_np(q, m, p, g), [0, 1, 0])


def test_default_box_is_the_live_extent():
    m = np.array([[-3.0, 2.0, 0.0], [4.1, -1.0, 5.0], [np.nan, np.nan, np.nan], [0.0, 7.3, 0.0]])
    g = G.grid(G.Params(), m)
    assert (g.x_min, g.y_min) == (-3.0, -1.0)
    assert g.nx == math.floor(7.1 / 0.25) + 1 and g.ny == math.floor(8.3 / 0.25) + 1
    assert g.n_yaw == 144 and g.n_z == 1


def test_rotations_are_exact_for_zero_attitude():
    p = G.Params()
    rot = G.rotations(p)
    for j in (0, 17, 143):
        y = p.yaw0 + j * p.yaw_step
        assert np.array_equal(rot[j], [math.cos(y), -math.sin(y), 0, math.sin(y), math.cos(y), 0, 0, 0, 1])


def _T(x, y, yaw):
    T = np.eye(4)
    T[:2, :2] = [[math.cos(yaw), -math.sin(yaw)], [math.sin(yaw), math.cos(yaw)]]
    T[:2, 3] = [x, y]
    return T


def test_runner_up_rule():
    p = G.Params()
    Ts = [_T(0, 0, 0), _T(0.5, 0, 0.05), _T(5, 0, 0), _T(0, 0, math.pi)]
    w, found, ru = G.decide(Ts, [0.8, 0.9, 0.6, 0.7], p, 0.7)
    assert (w, found) == (1, True)
    assert ru == 0.7                                                         # index 0 is within 1 m / 10 degrees of the winner
    w, found, ru = G.decide(Ts[:2], [0.5, 0.5], p, 0.7)
    assert (w, found, ru) == (0, False, -1.0)                                # ties -> lower rank; nothing beyond the winner
    assert G.decide([], [], p, 0.7) == (-1, False, -1.0)
