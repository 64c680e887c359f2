"""VoxelHashMap — same Python surface as python/kiss_icp/mapping.py:37-68, backed by the HBM
voxel table (C-ABI kb_map_*)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as N
from .config import KISSConfig


class MapInUseError(N.KissB200Error):
    """A call that would change or free a VoxelHashMap while localizers read it (KissICP(config, prior_map=...)).
    A RuntimeError; the map is unchanged. It works again once the last localizer using it is gone."""


def check_value(status: int):
    """N.check, except that a rejected argument (KB_ERR_INVALID_ARG) raises ValueError: the checkpoint loads report
    bad input the way numpy and the reference's Python do"""
    if status == N.KB_ERR_INVALID_ARG:
        raise ValueError(N.lib().kb_last_error().decode())
    N.check(status)


def _int32_arg(a, name):
    a = np.asarray(a)
    if a.size and a.dtype.kind not in "iu":
        raise ValueError(f"{name} must be integers")
    b = np.ascontiguousarray(a, dtype=np.int32)
    if not np.array_equal(a, b):
        raise ValueError(f"{name} out of int32 range")
    return b


def get_voxel_hash_map(config: KISSConfig):
    return VoxelHashMap(
        voxel_size=config.mapping.voxel_size,
        max_distance=config.data.max_range,
        max_points_per_voxel=config.mapping.max_points_per_voxel,
    )


class VoxelHashMap:
    """The mutators (clear, update, add_points, remove_far_away_points, compact, load) raise MapInUseError while a
    localizer uses the map as its prior map."""

    def __init__(self, voxel_size: float, max_distance: float, max_points_per_voxel: int, _borrowed=None, _owner=None):
        self._owner = _owner
        self._borrowed = _borrowed is not None
        if self._borrowed:
            self._h = N.vp(_borrowed)
        else:
            self._h = N.vp()
            N.check(N.lib().kb_map_create(float(voxel_size), float(max_distance), int(max_points_per_voxel), C.byref(self._h)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and not self._borrowed and N._lib is not None:
            N._lib.kb_map_destroy(h)
            self._h = None

    def readers(self) -> int:
        """localizers using this map as their prior map (while > 0 the map cannot be changed)"""
        r = N.i32(0)
        N.check(N.lib().kb_map_readers(self._h, C.byref(r)))
        return r.value

    def _mutated(self, status: int, check=N.check):
        if status == N.KB_ERR_INVALID_ARG and self.readers() > 0:
            raise MapInUseError(N.lib().kb_last_error().decode())
        check(status)

    # -- reference surface ---------------------------------------------------------------------
    def clear(self):
        self._mutated(N.lib().kb_map_clear(self._h))

    def empty(self):
        e = N.i32(0)
        N.check(N.lib().kb_map_empty(self._h, C.byref(e)))
        return bool(e.value)

    def update(self, points: np.ndarray, pose: np.ndarray = np.eye(4)):
        """points + (4,4) pose  -> VoxelHashMap::Update(points, pose)   (VoxelHashMap.cpp:89-95)
        points + (3,) origin    -> VoxelHashMap::Update(points, origin) (VoxelHashMap.cpp:83-87)
        ValueError for a non-finite point or origin, or a point whose voxel coordinates do not fit in an int."""
        pts = N.points_arg(points)
        x = np.ascontiguousarray(pose, dtype=np.float64)
        if x.shape == (4, 4):
            self._mutated(N.lib().kb_map_update_pose(self._h, N.ptr(pts), len(pts), N.ptr(x)), check_value)
        elif x.shape == (3,):
            self._mutated(N.lib().kb_map_update_origin(self._h, N.ptr(pts), len(pts), N.ptr(x)), check_value)
        else:
            raise TypeError("_update(): incompatible function arguments (pose (4,4) or origin (3,))")

    def add_points(self, points):
        pts = N.points_arg(points)
        self._mutated(N.lib().kb_map_add_points(self._h, N.ptr(pts), len(pts)), check_value)

    def remove_far_away_points(self, origin):
        o = np.ascontiguousarray(origin, dtype=np.float64).reshape(3)
        self._mutated(N.lib().kb_map_remove_far(self._h, N.ptr(o)))

    def point_cloud(self) -> np.ndarray:
        n = N.sz(0)
        N.check(N.lib().kb_map_pointcloud(self._h, None, 0, C.byref(n)))
        out = np.empty((n.value, 3))
        if n.value:
            N.check(N.lib().kb_map_pointcloud(self._h, N.ptr(out), n.value, C.byref(n)))
        return out

    # -- extras (no reference counterpart in Python; C++ has GetClosestNeighbor) ----------------
    def compact(self):
        """rebuild the table at the smallest capacity (load <= 0.5, no tombstones)"""
        self._mutated(N.lib().kb_map_compact(self._h))

    def num_points(self) -> int:
        n = N.sz(0)
        N.check(N.lib().kb_map_num_points(self._h, C.byref(n)))
        return n.value

    def num_voxels(self) -> int:
        n = N.sz(0)
        N.check(N.lib().kb_map_num_voxels(self._h, C.byref(n)))
        return n.value

    def dump(self):
        """(voxels (V,3) int32 ascending, counts (V,), points (P,3) per-voxel insertion order)."""
        nv, npnt = self.num_voxels(), self.num_points()
        vox = np.empty((nv, 3), dtype=np.int32)
        cnt = np.empty(nv, dtype=np.int32)
        pts = np.empty((npnt, 3))
        a, b = N.sz(0), N.sz(0)
        N.check(N.lib().kb_map_dump(self._h, N.ptr(vox), N.ptr(cnt), N.ptr(pts), nv, npnt, C.byref(a), C.byref(b)))
        return vox, cnt, pts

    def load(self, voxels, counts, points):
        """The inverse of dump(): replace the map's contents with (voxels (V,3), counts (V,), points (P,3)); the
        voxels may come in any order. Validated on the device and all or nothing: a duplicate voxel, a count outside
        [1, max_points_per_voxel], P != counts.sum(), a non-finite coordinate or a point outside the voxel it is
        listed under raises ValueError and leaves the map as it was."""
        vox, cnt = _int32_arg(voxels, "voxels"), _int32_arg(counts, "counts")
        pts = np.ascontiguousarray(points, dtype=np.float64)
        if vox.ndim != 2 or vox.shape[1] != 3 or cnt.shape != (len(vox),) or pts.ndim != 2 or pts.shape[1] != 3:
            raise ValueError("expected voxels (V, 3), counts (V,) and points (P, 3)")
        self._mutated(N.lib().kb_map_load(self._h, N.ptr(vox), N.ptr(cnt), N.ptr(pts), len(vox), len(pts)), check_value)

    def free_space(self, scans, poses, params=None):
        """Count the free-space evidence of the scans (a list of (N_s, 3) arrays in their sensor frames) at poses
        (S, 4, 4, world <- sensor) for this map -> FreeSpace (passes, hits, removed, report), aligned with dump().
        Only reads the map: it works while localizers use it. params: a FreeSpaceParams (None: the defaults)."""
        from . import free_space
        return free_space.count(self, scans, poses, params)

    def cleaned(self, scans, poses, params=None):
        """-> (VoxelHashMap, FreeSpace): a new map with this one's voxel size, maximum distance and points per voxel that
        holds the points free_space() does not remove, in per-voxel insertion order. This map is unchanged."""
        from . import free_space
        vs, md, mp = N.dbl(0), N.dbl(0), N.u32(0)
        N.check(N.lib().kb_map_params(self._h, C.byref(vs), C.byref(md), C.byref(mp)))
        out = VoxelHashMap(vs.value, md.value, mp.value)
        fs = free_space.count(self, scans, poses, params, out=out)
        return out, fs

    def closest_neighbors(self, queries):
        """batched VoxelHashMap::GetClosestNeighbor (VoxelHashMap.cpp:46-70). ValueError for a non-finite query or
        one whose voxel coordinates do not fit in an int."""
        q = N.points_arg(queries)
        outp = np.empty_like(q)
        outd = np.empty(len(q))
        check_value(N.lib().kb_map_closest_neighbors(self._h, N.ptr(q), len(q), N.ptr(outp), N.ptr(outd)))
        return outp, outd
