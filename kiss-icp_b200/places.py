"""Place recognition: a database of Scan Context descriptors, searched on the device over every entry and heading
(kb_place_* in include/kiss_icp_b200.h, which states every rule).

No reference counterpart. A mapping run stores the descriptor of the scan at each keyframe pose; a query scan is
compared with every entry at every cyclic shift, and the best entries, rotated by their shift, are initial guesses for
a batched ICP refinement against a prior map (Registration.relocalize_in_places, KissICP.relocalize_by_place). With
max_entry, the same query over the entries older than the recent ones gives loop-closure candidates.

The query and the entries must describe the same kind of cloud: the preprocessed frame in its sensor frame, for
example ``pre, _ = odometry.register_frame(scan, timestamps); db.add(pre, odometry.last_pose)`` every ~2 m.
"""
from __future__ import annotations

import ctypes as C
import operator
from dataclasses import dataclass

import numpy as np

from . import _native as N
from .mapping import check_value

STATE_FORMAT_VERSION = 1  # of PlaceDatabase.state_dict()


@dataclass
class PlaceDescriptorParams:
    """The Scan Context grid (kb_place_params): n_rings in [1, 64], n_sectors in [3, 720], n_rings * n_sectors <= 4096,
    max_radius finite and > 0 [m], z_offset finite [m] (added to z: the sensor's height above the ground)."""
    n_rings: int = 20
    n_sectors: int = 60
    max_radius: float = 80.0
    z_offset: float = 2.0

    def _struct(self):
        p = N.PlaceParams()
        for name in ("n_rings", "n_sectors"):
            v = operator.index(getattr(self, name))
            if not -2 ** 31 <= v < 2 ** 31:
                raise ValueError(f"{name} = {v} is out of range")
            setattr(p, name, v)
        p.max_radius, p.z_offset = float(self.max_radius), float(self.z_offset)
        return p


@dataclass
class PlaceMatch:
    """one candidate: the entry, the shift s (the query's column k matches the entry's column k + s), yaw = s 2 pi /
    n_sectors, the distance and the query's pose guess T_entry Rz(yaw)"""
    entry: int
    shift: int
    yaw: float
    distance: float
    guess: np.ndarray


@dataclass
class PlaceRelocalizationResult:
    """pose, inliers, iterations: the winner after refinement; rank: its index among the candidates. runner_up_pose /
    runner_up_inliers: the best refined candidate farther than `separation` in xy or 2 sector widths in angle from the
    winner (None / -1 when there is none). candidates: the PlaceMatch list that was refined."""
    pose: np.ndarray
    inliers: int
    iterations: int
    rank: int
    n_source: int
    n_entries: int
    runner_up_pose: np.ndarray | None
    runner_up_inliers: int
    candidates: list


def _matches(buf, n):
    return [PlaceMatch(entry=m.entry, shift=m.shift, yaw=m.yaw, distance=m.distance,
                       guess=np.array(m.guess[:]).reshape(4, 4)) for m in buf[:n]]


def _int32(v, name):
    v = operator.index(v)
    if not -2 ** 31 <= v < 2 ** 31:
        raise ValueError(f"{name} = {v} is out of range")
    return v


class PlaceDatabase:
    """Scan Context descriptors with their keyframe poses, on the calling thread's device."""

    def __init__(self, params: PlaceDescriptorParams | None = None):
        self.params = PlaceDescriptorParams() if params is None else params
        if not isinstance(self.params, PlaceDescriptorParams):
            raise TypeError(f"params must be a PlaceDescriptorParams, not {type(self.params).__name__}")
        self._h = N.vp()
        check_value(N.lib().kb_place_db_create(C.byref(self.params._struct()), C.byref(self._h)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and N._lib is not None:
            N._lib.kb_place_db_destroy(h)
            self._h = None

    @property
    def shape(self):
        return (int(self.params.n_rings), int(self.params.n_sectors))

    def __len__(self):
        n = N.sz(0)
        N.check(N.lib().kb_place_db_size(self._h, C.byref(n)))
        return n.value

    def descriptor(self, points) -> np.ndarray:
        """the (n_rings, n_sectors) descriptor of ``points`` (N, 3) in their sensor frame; nothing is added"""
        pts = N.points_arg(points)
        out = np.empty(self.shape)
        check_value(N.lib().kb_place_descriptor(self._h, N.ptr(pts), len(pts), N.ptr(out)))
        return out

    def add(self, points, pose) -> int:
        """append the descriptor of ``points`` (the cloud in its sensor frame) taken at keyframe ``pose`` (4x4)"""
        pts = N.points_arg(points)
        T = N.mat4_arg(pose)
        idx = N.sz(0)
        check_value(N.lib().kb_place_db_add(self._h, N.ptr(pts), len(pts), N.ptr(T), C.byref(idx)))
        return idx.value

    def _dump(self):
        n = N.sz(0)
        N.check(N.lib().kb_place_db_dump(self._h, None, None, 0, C.byref(n)))
        d = np.empty((n.value, *self.shape))
        p = np.empty((n.value, 4, 4))
        if n.value:
            N.check(N.lib().kb_place_db_dump(self._h, N.ptr(d), N.ptr(p), n.value, C.byref(n)))
        return d, p

    @property
    def poses(self) -> np.ndarray:
        """the (N, 4, 4) keyframe poses"""
        return self._dump()[1]

    def query(self, points, top_k: int = 8, max_entry: int = -1, separation: float = 3.0,
              return_distances: bool = False):
        """the candidates (a list of PlaceMatch, best first) of ``points`` among the entries [0, max_entry) (all of
        them when max_entry < 0), no two closer than ``separation`` metres in xy. With return_distances also every
        searched entry's distance and shift: (matches, distances (M,), shifts (M,))."""
        pts = N.points_arg(points)
        top_k, max_entry = _int32(top_k, "top_k"), _int32(max_entry, "max_entry")
        M = len(self) if max_entry < 0 else min(max_entry, len(self))
        buf = (N.PlaceMatch * max(top_k, 1))()
        n = N.sz(0)
        dist = np.empty(M) if return_distances else None
        shift = np.empty(M, dtype=np.int32) if return_distances else None
        check_value(N.lib().kb_place_query(self._h, N.ptr(pts), len(pts), max_entry, float(separation), top_k, buf,
                                           C.byref(n), N.ptr(dist) if dist is not None else None,
                                           N.ptr(shift) if shift is not None else None))
        m = _matches(buf, n.value)
        return (m, dist, shift) if return_distances else m

    def match(self, queries: "PlaceDatabase | None" = None, top_k: int = 8, max_entry=None, separation: float = 3.0,
              return_report: bool = False):
        """every entry of ``queries`` (None: this database) as a query of this one, in one device search
        (kb_place_db_match): one PlaceMatch list per query, each equal to what query() gives for the cloud that entry
        was added from. max_entry: None (every entry), an int for all queries or a (Q,) array; < 0 searches every
        entry, and an empty range gives an empty list. With return_report also the counts (N.PlaceMatchReport)."""
        q = self if queries is None else queries
        if not isinstance(q, PlaceDatabase):
            raise TypeError(f"queries must be a PlaceDatabase, not {type(q).__name__}")
        top_k = _int32(top_k, "top_k")
        Q = len(q)
        if max_entry is None:
            me = None
        else:
            me = np.asarray(max_entry)
            if me.ndim == 0:
                me = np.full(Q, _int32(int(me), "max_entry"), dtype=np.int64)
            if me.shape != (Q,) or not np.issubdtype(me.dtype, np.integer):
                raise ValueError(f"max_entry must be None, an int or ({Q},) integers, not {me.dtype} {me.shape}")
            if Q and (me.min() < -2 ** 31 or me.max() >= 2 ** 31):
                raise ValueError("max_entry is out of range")
            me = np.ascontiguousarray(me, dtype=np.int32)
        buf = (N.PlaceMatch * max(Q * max(top_k, 1), 1))()
        n = np.zeros(max(Q, 1), dtype=np.int32)
        rep = N.PlaceMatchReport()
        check_value(N.lib().kb_place_db_match(self._h, q._h, N.ptr(me) if me is not None else None, float(separation),
                                              top_k, buf, N.ptr(n), C.byref(rep)))
        K = max(top_k, 1)
        out = [_matches(buf[i * K:(i + 1) * K], int(n[i])) for i in range(Q)]
        return (out, rep) if return_report else out

    def pair_distances(self, queries: "PlaceDatabase | None" = None):
        """(distances (Q, N), shifts (Q, N)): every query's distance and shift to every entry, from match()'s kernel
        (kb_debug_place_match_pairs)"""
        q = self if queries is None else queries
        Q, M = len(q), len(self)
        d = np.empty((Q, M))
        s = np.empty((Q, M), dtype=np.int32)
        check_value(N.lib().kb_debug_place_match_pairs(self._h, q._h, N.ptr(d), N.ptr(s)))
        return d, s

    def state_dict(self):
        """the database as numpy arrays (np.savez-safe): format_version, the parameters, descriptors (N, n_rings,
        n_sectors) and poses (N, 4, 4)"""
        d, p = self._dump()
        return {"format_version": np.array(STATE_FORMAT_VERSION), "n_rings": np.array(int(self.params.n_rings)),
                "n_sectors": np.array(int(self.params.n_sectors)), "max_radius": np.array(float(self.params.max_radius)),
                "z_offset": np.array(float(self.params.z_offset)), "descriptors": d, "poses": p}

    def load_state_dict(self, state):
        """replace the entries by those of a state_dict(), all or nothing: on ValueError nothing has changed. The
        parameters must equal this database's."""
        d = {k: np.asarray(v) for k, v in state.items()}
        if int(d["format_version"]) != STATE_FORMAT_VERSION:
            raise ValueError(f"state format {int(d['format_version'])}, expected {STATE_FORMAT_VERSION}")
        got = (int(d["n_rings"]), int(d["n_sectors"]), float(d["max_radius"]), float(d["z_offset"]))
        have = (int(self.params.n_rings), int(self.params.n_sectors), float(self.params.max_radius),
                float(self.params.z_offset))
        if got != have:
            raise ValueError(f"state of a database with parameters {got}; this one has {have}")
        desc = np.ascontiguousarray(d["descriptors"], dtype=np.float64)
        poses = np.ascontiguousarray(d["poses"], dtype=np.float64)
        if desc.ndim != 3 or desc.shape[1:] != self.shape or poses.shape != (len(desc), 4, 4):
            raise ValueError(f"descriptors {desc.shape} and poses {poses.shape} do not match (N, {self.shape[0]}, "
                             f"{self.shape[1]}) and (N, 4, 4)")
        check_value(N.lib().kb_place_db_load(self._h, N.ptr(desc), N.ptr(poses), len(desc)))


def relocalize_in_places(reg_handle, descriptor_points, source, voxel_map, places: PlaceDatabase, top_k=8,
                         separation=3.0, max_correspondence_distance=3.0, kernel_scale=1.0, max_entry=-1):
    """kb_place_relocalize on a registration handle (Registration.relocalize_in_places)"""
    from .mapping import VoxelHashMap
    if not isinstance(places, PlaceDatabase):
        raise TypeError(f"places must be a PlaceDatabase, not {type(places).__name__}")
    if not isinstance(voxel_map, VoxelHashMap):
        raise TypeError(f"voxel_map must be a VoxelHashMap, not {type(voxel_map).__name__}")
    dp, src = N.points_arg(descriptor_points), N.points_arg(source)
    s = N.PlaceSearch()
    s.top_k, s.max_entry = _int32(top_k, "top_k"), _int32(max_entry, "max_entry")
    s.separation = float(separation)
    s.max_correspondence_distance, s.kernel_scale = float(max_correspondence_distance), float(kernel_scale)
    buf = (N.PlaceMatch * max(s.top_k, 1))()
    r = N.PlaceResult()
    check_value(N.lib().kb_place_relocalize(reg_handle, places._h, N.ptr(dp), len(dp), N.ptr(src), len(src),
                                            voxel_map._h, C.byref(s), C.byref(r), buf))
    return PlaceRelocalizationResult(
        pose=np.array(r.pose[:]).reshape(4, 4), inliers=r.inliers, iterations=r.iterations, rank=r.rank,
        n_source=r.n_source, n_entries=r.n_entries,
        runner_up_pose=np.array(r.runner_up_pose[:]).reshape(4, 4) if r.runner_up_inliers >= 0 else None,
        runner_up_inliers=r.runner_up_inliers, candidates=_matches(buf, r.n_candidates))
