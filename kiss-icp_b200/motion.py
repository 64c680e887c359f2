"""Sampled motion: deskew and predict scans from IMU or wheel-odometry samples (DESIGN.md section 4.17).

A ``Motion`` is the LiDAR's trajectory sampled at ``times``: its pose T_k at times[k] in any fixed frame. Between two
samples the pose is T(t) = T_k Exp(alpha Log(T_k^-1 T_k+1)), alpha = (t - t_k) / (t_k+1 - t_k); before the first and
after the last sample the first and last intervals are extrapolated. Passed with a scan to ``KissICP.register_frame``
or ``register_frames``, it replaces the constant-velocity model for that scan:
  * deskew: a point with stamp s becomes T(end_time)^-1 T(s + stamp_offset) p (with deskewing on and stamps given);
  * prediction: when the previous scan had a Motion whose end_time lies within this one's samples, the initial guess
    is last_pose T(prev_end)^-1 T(end_time).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as N

MAX_SAMPLES = 65536  # KB_MOTION_MAX_SAMPLES


class Motion:
    """Sampled LiDAR poses for one scan.

    ``times`` (m,) strictly increasing on the sample clock, ``poses`` (m, 4, 4) SE(3), the LiDAR's pose at each time in
    any fixed frame, 2 <= m <= MAX_SAMPLES. ``stamp_offset`` is added to every point stamp to put it on the sample
    clock (per-scan relative stamps: the scan's start time). ``end_time`` is the sample-clock time the scan's pose
    refers to; None: max(stamps) + stamp_offset for a scan with stamps, stamp_offset for one without (KISS-ICP's
    deskew target is the end of the sweep). Checked by kb_motion_check: ValueError for a malformed motion."""

    def __init__(self, times, poses, stamp_offset: float = 0.0, end_time: float | None = None):
        self.times = np.ascontiguousarray(np.asarray(times, dtype=np.float64).reshape(-1))
        self.poses = np.ascontiguousarray(np.asarray(poses, dtype=np.float64))
        if self.poses.shape != (len(self.times), 4, 4):
            raise ValueError(f"poses must be ({len(self.times)}, 4, 4), not {self.poses.shape}")
        self.stamp_offset = float(stamp_offset)
        self.end_time = None if end_time is None else float(end_time)
        s = self._struct(0.0 if end_time is None else self.end_time)
        st = N.lib().kb_motion_check(C.byref(s))
        if st != N.KB_OK:
            raise ValueError(N.lib().kb_last_error().decode())

    def resolved_end_time(self, stamps) -> float:
        """end_time for a scan with these stamps"""
        if self.end_time is not None:
            return self.end_time
        ts = np.asarray(stamps, dtype=np.float64).reshape(-1)
        if ts.size and np.isfinite(ts).any():
            return float(np.nanmax(ts)) + self.stamp_offset
        return self.stamp_offset

    def _struct(self, end_time: float) -> N.Motion:
        s = N.Motion()
        s.times = self.times.ctypes.data
        s.poses = self.poses.ctypes.data
        s.m = len(self.times)
        s.stamp_offset = self.stamp_offset
        s.end_time = float(end_time)
        return s


def deskew(points, stamps, motion: Motion) -> np.ndarray:
    """The deskew of one scan alone (kb_deskew_motion): T(end_time)^-1 T(s + stamp_offset) p per point, no range crop;
    without stamps the points as they are."""
    if not isinstance(motion, Motion):
        raise TypeError(f"motion must be a Motion, not {type(motion).__name__}")
    pts = N.points_arg(points)
    ts = np.ascontiguousarray(np.asarray(stamps, dtype=np.float64).reshape(-1))
    s = motion._struct(motion.resolved_end_time(ts))
    out = np.empty_like(pts)
    N.check(N.lib().kb_deskew_motion(N.ptr(pts), len(pts), N.ptr(ts), len(ts), C.byref(s), N.ptr(out)))
    return out


def _so3_exp(w):
    th = float(np.linalg.norm(w))
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1.0 - np.cos(th)) / th ** 2 * (K @ K)


def motion_from_gyro(times, rates, lidar_velocity, imu_to_lidar_rotation=None, stamp_offset: float = 0.0,
                     end_time: float | None = None) -> Motion:
    """A Motion from gyroscope samples (host only, numpy).

    ``times`` (m,) on the IMU clock, ``rates`` (m, 3) body angular rates [rad/s] in the IMU frame at those times,
    ``lidar_velocity`` (3,) the velocity of the LiDAR origin [m/s], constant over the samples, expressed in the LiDAR
    frame at times[0]. ``imu_to_lidar_rotation`` (3, 3) maps IMU-frame vectors to the LiDAR frame (identity if None).
    Poses are relative to the LiDAR frame at times[0]:
      * rotation, zero-order hold: R_0 = I, R_k+1 = R_k Exp(w_k (t_k+1 - t_k)) with w_k the rate in the LiDAR frame
        (C rates[k], C = imu_to_lidar_rotation), i.e. C R_imu C^T;
      * translation: lidar_velocity (t_k - t_0).
    Without a better source of velocity (wheel odometry, a GNSS/INS), take it from the pipeline's own motion model:
    ``kiss.last_delta[:3, 3] / scan_period`` is the last scan's mean velocity in the LiDAR frame at its start, which for
    a scan that turns little is the frame at this scan's start up to the turn."""
    t = np.asarray(times, dtype=np.float64).reshape(-1)
    w = np.asarray(rates, dtype=np.float64).reshape(-1, 3)
    if w.shape[0] != t.shape[0]:
        raise ValueError("times and rates differ in length")
    Cm = np.eye(3) if imu_to_lidar_rotation is None else np.asarray(imu_to_lidar_rotation, dtype=np.float64)
    v = np.asarray(lidar_velocity, dtype=np.float64).reshape(3)
    poses = np.tile(np.eye(4), (len(t), 1, 1))
    R = np.eye(3)
    for k in range(len(t)):
        poses[k, :3, :3] = R
        poses[k, :3, 3] = v * (t[k] - t[0])
        if k + 1 < len(t):
            R = R @ _so3_exp((Cm @ w[k]) * (t[k + 1] - t[k]))
    return Motion(t, poses, stamp_offset=stamp_offset, end_time=end_time)
