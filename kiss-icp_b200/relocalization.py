"""Relocalization: a global pose search in a bounded region of a prior map (kb_reloc_hypotheses, kb_relocalize).

No reference counterpart. A scan is placed in a map without an initial pose: every hypothesis of a grid in x, y and
yaw around a centre pose is scored on the device (the source points whose voxel the map holds), the best peaks of the
scores are refined by one batched ICP launch, and the refined candidate with the most inliers wins. Whether to accept
the winner is the caller's decision: compare its inliers with n_source and with the runner-up's.
"""
from __future__ import annotations

import ctypes as C
import operator
from dataclasses import dataclass

import numpy as np

from . import _native as N
from .mapping import VoxelHashMap, check_value


@dataclass
class RelocalizationSearch:
    """The hypotheses of a relocalization (kb_reloc_search). Hypothesis h = (k Ny + (j + half_cells_y)) Nx +
    (i + half_cells_x), with Nx = 2 half_cells_x + 1, Ny = 2 half_cells_y + 1, i and j in [-half_cells, half_cells]
    and k in [0, n_yaw): rotation Rz((k - n_yaw // 2) yaw_step) @ R_center, translation center + (i step, j step, 0).
    z, roll and pitch come from the centre. The yaw axis wraps when n_yaw * yaw_step is 2 pi. At most 2^24 hypotheses;
    top_k (1..256) peaks are refined with max_correspondence_distance and kernel_scale."""
    center: np.ndarray
    half_cells_x: int
    half_cells_y: int
    step: float
    n_yaw: int
    yaw_step: float
    top_k: int = 16
    max_correspondence_distance: float = 3.0
    kernel_scale: float = 1.0

    @property
    def shape(self):
        """(n_yaw, Ny, Nx): the layout of the scores"""
        return (int(self.n_yaw), 2 * int(self.half_cells_y) + 1, 2 * int(self.half_cells_x) + 1)

    def _struct(self):
        """-> (kb_reloc_search, number of hypotheses); ValueError for a field the library rejects"""
        c = np.asarray(self.center, dtype=np.float64)
        if c.shape != (4, 4):
            raise ValueError(f"center must be a 4x4 pose, not shape {c.shape}")
        s = N.RelocSearch()
        s.center[:] = [float(x) for x in c.ravel()]
        for name in ("half_cells_x", "half_cells_y", "n_yaw", "top_k"):
            v = operator.index(getattr(self, name))  # TypeError for a non-integer
            if not -2 ** 31 <= v < 2 ** 31:
                raise ValueError(f"{name} = {v} is out of range")
            setattr(s, name, v)
        for name in ("step", "yaw_step", "max_correspondence_distance", "kernel_scale"):
            setattr(s, name, float(getattr(self, name)))
        n = N.sz(0)
        check_value(N.lib().kb_reloc_hypotheses(C.byref(s), None, 0, C.byref(n)))
        return s, n.value

    def hypotheses(self) -> np.ndarray:
        """the (H, 4, 4) poses that are scored, in order h (host only)"""
        s, H = self._struct()
        out = np.empty((H, 4, 4))
        n = N.sz(0)
        check_value(N.lib().kb_reloc_hypotheses(C.byref(s), N.ptr(out), H, C.byref(n)))
        return out


@dataclass
class RelocalizationResult:
    """pose, inliers, iterations: the winner after refinement; rank: its index among the candidates. runner_up_pose /
    runner_up_inliers: the best refined candidate farther than 2 step in xy or 2 yaw_step in angle from the winner
    (None / -1 when there is none). candidates (K, 4, 4): the coarse poses of the peaks that were refined, with their
    candidate_scores (K,). scores: (n_yaw, Ny, Nx) coarse scores when asked for, else None."""
    pose: np.ndarray
    inliers: int
    iterations: int
    rank: int
    n_source: int
    n_hypotheses: int
    n_peaks: int
    runner_up_pose: np.ndarray | None
    runner_up_inliers: int
    candidates: np.ndarray
    candidate_scores: np.ndarray
    scores: np.ndarray | None = None


def relocalize(reg_handle, points, voxel_map, search: RelocalizationSearch, return_scores: bool = False):
    """kb_relocalize on a registration handle (Registration.relocalize)"""
    if not isinstance(search, RelocalizationSearch):
        raise TypeError(f"search must be a RelocalizationSearch, not {type(search).__name__}")
    if not isinstance(voxel_map, VoxelHashMap):
        raise TypeError(f"voxel_map must be a VoxelHashMap, not {type(voxel_map).__name__}")
    pts = N.points_arg(points)
    s, _ = search._struct()
    K = int(search.top_k)
    cand = np.empty((K, 4, 4))
    cand_scores = np.empty(K, dtype=np.int32)
    scores = np.empty(search.shape, dtype=np.int32) if return_scores else None
    r = N.RelocResult()
    check_value(N.lib().kb_relocalize(reg_handle, N.ptr(pts), len(pts), voxel_map._h, C.byref(s), C.byref(r),
                                      N.ptr(cand), N.ptr(cand_scores), N.ptr(scores) if scores is not None else None))
    k = r.n_candidates
    return RelocalizationResult(
        pose=np.array(r.pose[:]).reshape(4, 4), inliers=r.inliers, iterations=r.iterations, rank=r.rank,
        n_source=r.n_source, n_hypotheses=r.n_hypotheses, n_peaks=r.n_peaks,
        runner_up_pose=np.array(r.runner_up_pose[:]).reshape(4, 4) if r.runner_up_inliers >= 0 else None,
        runner_up_inliers=r.runner_up_inliers, candidates=cand[:k].copy(), candidate_scores=cand_scores[:k].copy(),
        scores=scores)
