"""Multi-LiDAR rigs: scans of several sensors merged into one base-frame scan on the device (DESIGN.md section 4.18).

A ``Rig`` is 1 to MAX_SENSORS ``Sensor``s mounted on a base (the vehicle). Sensor i has an extrinsic E_i (4x4 SE(3),
base <- sensor) and a range crop (min_range_i, max_range_i) measured in its own frame. A rig frame is one (N_i, 3) scan
per sensor, optionally with per-point stamps (for every sensor with points or for none) and a per-sensor stamp offset
that puts its stamps on the common clock. Its merged frame concatenates the sensors' points in sensor order, turns a
point outside its sensor's crop into NaN (the pipeline's own crop drops it), maps each point to the base, q = E_i p, and
stamps it s + stamp_offset_i. ``KissICP.register_rig_frame`` / ``register_rig_frames`` register merged frames: poses,
the map and every report then refer to the base, and a ``Motion`` passed with a rig frame holds the base's poses.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from . import _native as N
from .motion import Motion

MAX_SENSORS = 16  # KB_RIG_MAX_SENSORS


class Sensor:
    """One LiDAR of a rig: ``extrinsic`` (4, 4) SE(3), base <- sensor; its points are kept iff
    min_range < |p| < max_range in its own frame (0 and inf: no crop)."""

    def __init__(self, extrinsic, min_range: float = 0.0, max_range: float = math.inf):
        self.extrinsic = np.array(extrinsic, dtype=np.float64)
        if self.extrinsic.shape != (4, 4):
            raise ValueError(f"an extrinsic is a 4x4 matrix, not {self.extrinsic.shape}")
        self.min_range, self.max_range = float(min_range), float(max_range)

    def __repr__(self):
        return f"Sensor(extrinsic={self.extrinsic.tolist()}, min_range={self.min_range}, max_range={self.max_range})"


class Rig:
    """The sensors of a rig, in the order their scans are merged. Checked by kb_rig_check: ValueError for a rig without
    sensors or with more than MAX_SENSORS, an extrinsic outside SE(3), or a NaN, negative or inverted range."""

    def __init__(self, sensors):
        self.sensors = [s if isinstance(s, Sensor) else Sensor(*s) for s in sensors]
        n = len(self.sensors)
        self._structs = (N.Sensor * max(n, 1))()
        for st, s in zip(self._structs, self.sensors):
            st.extrinsic[:] = [float(x) for x in s.extrinsic.reshape(-1)]
            st.min_range, st.max_range = s.min_range, s.max_range
        status = N.lib().kb_rig_check(self._structs if n else None, n)
        if status != N.KB_OK:
            raise ValueError(N.lib().kb_last_error().decode())

    def __len__(self):
        return len(self.sensors)

    @property
    def n_sensors(self) -> int:
        return len(self.sensors)


def _check_rig(rig):
    if not isinstance(rig, Rig):
        raise TypeError(f"rig must be a Rig, not {type(rig).__name__}")


def _frame(scans, rig: Rig, timestamps, stamp_offsets, f32: bool):
    """one rig frame's arrays: (points, stamps, offsets), each a list of S arrays / floats"""
    S = rig.n_sensors
    if len(scans) != S:
        raise ValueError(f"a frame of this rig has {S} scans, not {len(scans)}")
    if f32:
        pts = [np.ascontiguousarray(np.asarray(a, dtype=np.float32)) for a in scans]
    else:
        pts = [N.points_arg(a) for a in scans]
    if timestamps is None:
        ts = [np.empty(0)] * S
    else:
        if len(timestamps) != S:
            raise ValueError(f"a frame of this rig has {S} stamp arrays, not {len(timestamps)}")
        ts = [np.ascontiguousarray(np.asarray(t, dtype=np.float64).ravel()) for t in timestamps]
    offs = [0.0] * S if stamp_offsets is None else [float(o) for o in stamp_offsets]
    if len(offs) != S:
        raise ValueError(f"a frame of this rig has {S} stamp offsets, not {len(offs)}")
    return pts, ts, offs


def _end_time(motion: Motion, ts, offs) -> float:
    """the motion's end_time for a rig frame: by default the latest merged stamp + the motion's stamp_offset"""
    if motion.end_time is not None:
        return motion.end_time
    ends = [float(np.nanmax(t)) + o for t, o in zip(ts, offs) if t.size and np.isfinite(t).any()]
    return (max(ends) if ends else 0.0) + motion.stamp_offset


def merge_rig(scans, rig: Rig, timestamps=None, stamp_offsets=None, motion: Motion | None = None):
    """The merge of one rig frame alone (kb_merge_rig) -> (points (N, 3), stamps (N,) or (0,)): the merged base-frame
    points, deskewed along ``motion`` (the base's poses) when it is given and the frame has stamps, without the
    pipeline's crop; the merged stamps s + stamp_offset_i when the frame has stamps."""
    _check_rig(rig)
    if motion is not None and not isinstance(motion, Motion):
        raise TypeError(f"motion must be a Motion, not {type(motion).__name__}")
    pts, ts, offs = _frame(scans, rig, timestamps, stamp_offsets, False)
    S = rig.n_sensors
    X = (C.c_void_p * S)(*[a.ctypes.data for a in pts])
    T = (C.c_void_p * S)(*[t.ctypes.data if t.size else None for t in ts])
    n = (N.sz * S)(*[len(a) for a in pts])
    nt = (N.sz * S)(*[len(t) for t in ts])
    O = (N.dbl * S)(*offs)
    total = sum(len(a) for a in pts)
    out = np.empty((total, 3))
    out_ts = np.empty(total)
    m = C.byref(motion._struct(_end_time(motion, ts, offs))) if motion is not None else None
    N.check(N.lib().kb_merge_rig(rig._structs, S, X, n, T, nt, O, m, N.ptr(out), N.ptr(out_ts)))
    stamped = any(len(t) for t, a in zip(ts, pts) if len(a))
    return out, (out_ts if stamped else np.empty(0))
