"""Free-space evidence of a voxel map: remove moving objects with the rays of a run's scans (C-ABI kb_map_free_space).

A ray from the sensor to its endpoint passes the map points it goes through on its way; a car that was there when the
map was built and has left since is passed by later rays, while the ground, the walls and thin static objects are not
(include/kiss_icp_b200.h, "free space", states the rule in full)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _native as N


@dataclass
class FreeSpaceParams:
    """kb_free_space_params. A field left as None takes its default for the map's voxel size v: pass_radius 0.1 v,
    end_margin 2.0 v, min_incidence asin(2 pass_radius / end_margin) [rad], min_planarity 0.3, min_passes 20, ratio 0.1
    (DESIGN.md §4.13 has the measurements behind them)."""
    pass_radius: float | None = None
    end_margin: float | None = None
    min_incidence: float | None = None
    min_planarity: float | None = None
    min_passes: int | None = None
    ratio: float | None = None

    def resolve(self, voxel_size: float) -> "FreeSpaceParams":
        """every field set: the given ones as they are, the others from the voxel size (min_incidence from the
        resolved pass_radius and end_margin)"""
        d = N.FreeSpaceParams()
        N.lib().kb_free_space_params_default(C.byref(d), float(voxel_size))
        eps = d.pass_radius if self.pass_radius is None else float(self.pass_radius)
        delta = d.end_margin if self.end_margin is None else float(self.end_margin)
        if self.min_incidence is not None:
            inc = float(self.min_incidence)
        else:
            inc = float(np.arcsin(min(1.0, 2.0 * eps / delta))) if delta > 0 else float(np.pi / 2)
        return FreeSpaceParams(eps, delta, inc, d.min_planarity if self.min_planarity is None else float(self.min_planarity),
                               d.min_passes if self.min_passes is None else int(self.min_passes),
                               d.ratio if self.ratio is None else float(self.ratio))

    def _c(self) -> N.FreeSpaceParams:
        if self.min_passes < 0 or self.min_passes >= 2**32:
            raise ValueError("min_passes must be in [1, 2^32)")
        return N.FreeSpaceParams(self.pass_radius, self.end_margin, self.min_incidence, self.min_planarity,
                                 int(self.min_passes), self.ratio)


@dataclass
class FreeSpaceReport:
    """kb_free_space_report"""
    rays: int
    scans: int
    points: int
    voxels: int
    points_removed: int
    voxels_removed: int
    ray_point_tests: int


@dataclass
class FreeSpace:
    """The evidence of one call, aligned with VoxelHashMap.dump(): passes (P,) per point, hits (V,) per voxel, and
    removed (P,) = passes >= min_passes and passes >= ratio * hits of the point's voxel."""
    passes: np.ndarray
    hits: np.ndarray
    removed: np.ndarray
    report: FreeSpaceReport
    params: FreeSpaceParams


def _scan_args(scans, poses):
    scans = [N.points_arg(s) for s in scans]
    P = np.ascontiguousarray(poses, dtype=np.float64)
    if P.shape != (len(scans), 4, 4):
        raise ValueError(f"poses must be ({len(scans)}, 4, 4), one per scan")
    offset = np.zeros(len(scans) + 1, dtype=np.uintp)
    offset[1:] = np.cumsum([len(s) for s in scans], dtype=np.uint64)
    xyz = np.ascontiguousarray(np.concatenate(scans) if scans else np.empty((0, 3)))
    return xyz, offset, P


def count(vmap, scans, poses, params: FreeSpaceParams | None, out=None) -> FreeSpace:
    """kb_map_free_space of vmap (a VoxelHashMap) with the scans (list of (N_s, 3)) at poses (S, 4, 4); out (a
    VoxelHashMap or None) receives the kept points. ValueError for a rejected argument."""
    vs = N.dbl(0)
    N.check(N.lib().kb_map_params(vmap._h, C.byref(vs), None, None))
    prm = (params or FreeSpaceParams()).resolve(vs.value)
    cp = prm._c()
    xyz, offset, P = _scan_args(scans, poses)
    passes = np.zeros(vmap.num_points(), dtype=np.uint32)
    hits = np.zeros(vmap.num_voxels(), dtype=np.uint32)
    rep = N.FreeSpaceReport()
    st = N.lib().kb_map_free_space(vmap._h, N.ptr(xyz), len(xyz), offset.ctypes.data_as(C.c_void_p), len(P), N.ptr(P),
                                   C.byref(cp), N.ptr(passes), N.ptr(hits), out._h if out is not None else None,
                                   C.byref(rep))
    if st in (N.KB_ERR_INVALID_ARG, N.KB_ERR_NOT_SE3):
        raise ValueError(N.lib().kb_last_error().decode())
    N.check(st)
    _, counts, _ = vmap.dump() if len(hits) else (None, np.zeros(0, np.int32), None)
    vox_of_point = np.repeat(np.arange(len(counts)), counts)
    removed = (passes >= prm.min_passes) & (passes.astype(np.float64) >= prm.ratio * hits[vox_of_point].astype(np.float64))
    report = FreeSpaceReport(*(int(getattr(rep, f)) for f, _ in N.FreeSpaceReport._fields_))
    return FreeSpace(passes, hits, removed, report, prm)
