"""CPU checks of the numpy TransformInterpolationBuffer / interpolate restatement (tests/odometry_buffer.py) against answers
computed another way: the GPU odometry tests use that restatement as their reference."""
import numpy as np
from scipy.spatial.transform import Rotation

from odometry_buffer import TransformInterpolationBuffer, interpolate, quat_from_rot, rot_from_quat, slerp


def rz(angle, t=(0.0, 0.0, 0.0)):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_euler("z", angle).as_matrix()
    T[:3, 3] = t
    return T


def test_quaternion_conversions_match_scipy():
    rng = np.random.default_rng(0)
    for R in Rotation.random(200, random_state=1).as_matrix():
        q = quat_from_rot(R)
        ref = Rotation.from_matrix(R).as_quat()            # (x, y, z, w), sign free
        assert min(np.abs(q - ref).max(), np.abs(q + ref).max()) < 1e-12
        assert np.abs(rot_from_quat(q) - R).max() < 1e-12
    for angle in (np.pi, -np.pi + 1e-9, 0.0):              # the trace <= 0 branches
        R = Rotation.from_rotvec(angle * rng.normal(size=3) / np.linalg.norm(rng.normal(size=3))).as_matrix()
        assert np.abs(rot_from_quat(quat_from_rot(R)) - R).max() < 1e-9


def test_slerp_about_one_axis_is_angle_interpolation():
    a, b = 0.3, 1.4
    for f in (0.0, 0.25, 0.5, 0.9, 1.0):
        q = slerp(quat_from_rot(rz(a)[:3, :3]), quat_from_rot(rz(b)[:3, :3]), f)
        assert np.abs(rot_from_quat(q) - rz(a + f * (b - a))[:3, :3]).max() < 1e-12


def test_slerp_takes_the_shortest_path_when_the_dot_product_is_negative():
    """Eigen's matrix -> quaternion conversion fixes the sign by its branch, so two nearby rotations can come out with a negative
    dot product; slerp must still take the short way round, which is what scipy's Slerp (relative rotation vector) does."""
    from scipy.spatial.transform import Slerp
    rng = np.random.default_rng(2)
    seen = 0
    for _ in range(4000):
        Ra = Rotation.random(random_state=rng)
        Rb = Rotation.from_rotvec(rng.normal(scale=0.6, size=3)) * Ra
        qa, qb = quat_from_rot(Ra.as_matrix()), quat_from_rot(Rb.as_matrix())
        if np.dot(qa, qb) >= 0.0:
            continue
        seen += 1
        ref = Slerp([0.0, 1.0], Rotation.from_matrix([Ra.as_matrix(), Rb.as_matrix()]))
        for f in (0.25, 0.5, 0.75):
            assert np.abs(rot_from_quat(slerp(qa, qb, f)) - ref([f]).as_matrix()[0]).max() < 1e-12
    assert seen >= 20


def test_slerp_of_nearly_identical_rotations_uses_linear_weights():
    qa = quat_from_rot(rz(0.7)[:3, :3])
    for f in (0.0, 0.3, 1.0):
        q = slerp(qa, qa, f)                                # |d| >= 1 - eps: (1 - f) qa + f qa, no 0 / 0
        assert np.all(np.isfinite(q)) and np.abs(q - qa).max() < 1e-15


def test_interpolation_factor_has_the_microsecond_denominator():
    A, B = rz(0.0, (0.0, 0.0, 0.0)), rz(0.0, (1.0, 0.0, 0.0))
    # 10 ticks = 1e-6 s between the entries: halfway in time is a factor of 5e-7 / (1e-6 + 1e-6) = 0.25
    assert abs(interpolate(A, 0, B, 10, 5)[0, 3] - 0.25) < 1e-15
    # a second apart the denominator hardly matters: 0.5 / (1 + 1e-6)
    assert abs(interpolate(A, 0, B, 10_000_000, 5_000_000)[0, 3] - 0.5 / (1.0 + 1e-6)) < 1e-15


def test_buffer_clamps_hits_exactly_and_interpolates_between():
    buf = TransformInterpolationBuffer()
    assert not buf.has(0)
    T = [rz(0.1 * k, (k, 2.0 * k, 0.0)) for k in range(3)]
    for k in range(3):
        buf.push(1_000_000 * (k + 1), T[k])
    assert buf.has(1_000_000) and buf.has(3_000_000) and buf.has(2_500_000)
    assert not buf.has(999_999) and not buf.has(3_000_001)
    assert np.array_equal(buf.get_transform(0), T[0])              # before the earliest: the earliest
    assert np.array_equal(buf.get_transform(10_000_000), T[2])     # after the latest: the latest
    for k in range(3):
        assert np.array_equal(buf.get_transform(1_000_000 * (k + 1)), T[k])
    f = 0.5e6 / 1e7 / (0.1 + 1e-6)
    mid = buf.get_transform(1_500_000)
    assert np.abs(mid[:3, 3] - (T[0][:3, 3] + (T[1][:3, 3] - T[0][:3, 3]) * f)).max() < 1e-15
    assert np.abs(mid[:3, :3] - rz(0.1 * f)[:3, :3]).max() < 1e-12


def test_buffer_evicts_the_oldest_at_its_size_limit():
    buf = TransformInterpolationBuffer(3)
    for k in range(5):
        buf.push(10 * (k + 1), rz(0.0, (k, 0.0, 0.0)))
    assert [t for t, _ in buf.entries] == [30, 40, 50]
    assert not buf.has(20) and buf.has(30)
    assert buf.get_transform(10)[0, 3] == 2.0                      # clamps to what is left
