"""numpy restatement of the reference's TransformInterpolationBuffer (src/TransformInterpolationBuffer.cpp) and interpolate
(src/Transform.cpp:16-41) with Eigen's quaternion conversions and slerp -- the reference the device odometry buffer is checked
against (TEST INFRASTRUCTURE).  Times are UniversalTimeScaleClock ticks (100 ns); transforms are 4x4 numpy arrays."""
from __future__ import annotations

import numpy as np

EPS = np.finfo(np.float64).eps   # NumTraits<double>::epsilon()


def quat_from_rot(R) -> np.ndarray:
    """Eigen's Quaterniond(const Matrix3d&): (x, y, z, w)"""
    R = np.asarray(R, dtype=np.float64)
    t = R[0, 0] + R[1, 1] + R[2, 2]
    q = np.zeros(4)
    if t > 0.0:
        t = np.sqrt(t + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0] = (R[2, 1] - R[1, 2]) * t
        q[1] = (R[0, 2] - R[2, 0]) * t
        q[2] = (R[1, 0] - R[0, 1]) * t
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (R[k, j] - R[j, k]) * t
        q[j] = (R[j, i] + R[i, j]) * t
        q[k] = (R[k, i] + R[i, k]) * t
    return q


def rot_from_quat(q) -> np.ndarray:
    """Eigen's QuaternionBase::toRotationMatrix (no normalisation)"""
    x, y, z, w = (float(v) for v in q)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1.0 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1.0 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1.0 - (txx + tyy)]])


def slerp(qa, qb, t: float) -> np.ndarray:
    """Eigen's QuaternionBase::slerp: shortest path (the second quaternion's sign follows the dot product), linear weights when
    the two are within an epsilon of each other"""
    one = 1.0 - EPS
    d = float(np.dot(qa, qb))
    absD = abs(d)
    if absD >= one:
        s0, s1 = 1.0 - t, t
    else:
        theta = np.arccos(absD)
        sinTheta = np.sin(theta)
        s0 = np.sin((1.0 - t) * theta) / sinTheta
        s1 = np.sin(t * theta) / sinTheta
    if d < 0.0:
        s1 = -s1
    return s0 * np.asarray(qa) + s1 * np.asarray(qb)


def interpolate(Ta, ta: int, Tb, tb: int, t: int) -> np.ndarray:
    """Transform.cpp:16-41: factor = toSeconds(t - ta) / (toSeconds(tb - ta) + 1e-6)"""
    duration = (tb - ta) / 1e7
    factor = ((t - ta) / 1e7) / (duration + 1e-6)
    out = np.eye(4)
    out[:3, :3] = rot_from_quat(slerp(quat_from_rot(Ta[:3, :3]), quat_from_rot(Tb[:3, :3]), factor))
    out[:3, 3] = Ta[:3, 3] + (Tb[:3, 3] - Ta[:3, 3]) * factor
    return out


class TransformInterpolationBuffer:
    def __init__(self, size_limit: int = 2000):
        self.size_limit = size_limit
        self.entries: list[tuple[int, np.ndarray]] = []

    def push(self, t: int, T) -> None:   # the callers push in increasing time order
        self.entries.append((int(t), np.array(T, dtype=np.float64)))
        while len(self.entries) > self.size_limit:
            self.entries.pop(0)

    def has(self, t: int) -> bool:
        return bool(self.entries) and self.entries[0][0] <= t <= self.entries[-1][0]

    def lookup(self, t: int) -> np.ndarray:
        assert self.has(t)
        if len(self.entries) == 1:
            return self.entries[0][1].copy()
        i = next(k for k, (ti, _) in enumerate(self.entries) if t <= ti)
        if self.entries[i][0] == t:
            return self.entries[i][1].copy()
        (ta, Ta), (tb, Tb) = self.entries[i - 1], self.entries[i]
        return interpolate(Ta, ta, Tb, tb, t)

    def get_transform(self, t: int) -> np.ndarray:
        """getTransform(t, buffer): clamped to the earliest / latest entry"""
        if t < self.entries[0][0]:
            return self.lookup(self.entries[0][0])
        if t > self.entries[-1][0]:
            return self.lookup(self.entries[-1][0])
        return self.lookup(t)
