"""voxel_down_sample — python/kiss_icp/voxelization.py:28-30 surface over kb_voxel_down_sample."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as N
from .mapping import check_value


def voxel_down_sample(points: np.ndarray, voxel_size: float):
    pts = N.points_arg(points)
    out = np.empty_like(pts)
    n = N.sz(0)
    check_value(N.lib().kb_voxel_down_sample(N.ptr(pts), len(pts), float(voxel_size), N.ptr(out), len(pts), C.byref(n)))
    return out[: n.value]
