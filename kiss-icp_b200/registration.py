"""Registration — python/kiss_icp/registration.py:36-65 surface over kb_registration_*."""
from __future__ import annotations

import ctypes as C
import sys

import numpy as np

from . import _native as N
from .config import KISSConfig
from .constraints import Constraints, _from_struct
from .mapping import VoxelHashMap, check_value
from .places import PlaceDatabase, PlaceRelocalizationResult, relocalize_in_places
from .relocalization import RelocalizationResult, RelocalizationSearch, relocalize


def _torch_if_cuda(x):
    """the torch module when x is a torch CUDA tensor (torch is imported only if the caller already did)"""
    torch = sys.modules.get("torch")
    return torch if torch is not None and isinstance(x, torch.Tensor) and x.is_cuda else None


def _guesses_arg(G) -> np.ndarray:
    a = np.ascontiguousarray(G, dtype=np.float64)
    if a.ndim != 3 or a.shape[1:] != (4, 4):
        raise RuntimeError("Unable to cast Python instance to C++ type (expected (B, 4, 4) initial guesses)")
    return a


def _ranges_arg(ranges, n_points: int, B: int):
    """(offsets, counts) as uint64 (size_t); no ranges: each of the B hypotheses uses all points"""
    if ranges is None:
        return np.zeros(B, dtype=np.uint64), np.full(B, n_points, dtype=np.uint64)
    r = np.asarray(ranges)
    if r.ndim != 2 or r.shape[1] != 2 or (r.size and r.dtype.kind not in "iu"):
        raise RuntimeError("ranges must be a (B, 2) integer array of (offset, count)")
    r = r.astype(np.int64)
    bad = (r[:, 0] < 0) | (r[:, 1] < 0) | (r[:, 0] + r[:, 1] > n_points)
    if bad.any():
        k = int(np.argmax(bad))
        raise IndexError(f"ranges[{k}] = ({r[k, 0]}, {r[k, 1]}) is outside the {n_points} points")
    return np.ascontiguousarray(r[:, 0], dtype=np.uint64), np.ascontiguousarray(r[:, 1], dtype=np.uint64)


def _per_hypothesis(x, B: int) -> np.ndarray:
    a = np.asarray(x, dtype=np.float64)
    if a.ndim > 1 or (a.ndim == 1 and a.shape[0] != B):
        raise RuntimeError(f"expected a scalar or {B} values, got shape {a.shape}")
    return np.ascontiguousarray(np.broadcast_to(a, (B,)))


def get_registration(config: KISSConfig):
    return Registration(
        max_num_iterations=config.registration.max_num_iterations,
        convergence_criterion=config.registration.convergence_criterion,
        max_num_threads=config.registration.max_num_threads,
    )


class Registration:
    def __init__(self, max_num_iterations: int, convergence_criterion: float, max_num_threads: int = 0):
        self._h = N.vp()
        N.check(N.lib().kb_registration_create(int(max_num_iterations), float(convergence_criterion),
                                               int(max_num_threads), C.byref(self._h)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and N._lib is not None:
            N._lib.kb_registration_destroy(h)
            self._h = None

    def align_points_to_map(self, points: np.ndarray, voxel_map: VoxelHashMap, initial_guess: np.ndarray,
                            max_correspondance_distance: float, kernel: float) -> np.ndarray:
        pts = N.points_arg(points)
        g = N.mat4_arg(initial_guess)
        out = np.empty((4, 4))
        check_value(N.lib().kb_registration_align_points_to_map(self._h, N.ptr(pts), len(pts), voxel_map._h, N.ptr(g),
                                                                float(max_correspondance_distance), float(kernel), N.ptr(out)))
        return out

    def constraints(self, points, voxel_map: VoxelHashMap, pose, max_correspondance_distance: float) -> Constraints:
        """The plane constraints (constraints.Constraints) of ``points`` mapped by ``pose`` against ``voxel_map``, for
        the correspondences closer than ``max_correspondance_distance``: those of the fit. Read-only, so it works on a
        localizer's prior map. ValueError for a pose outside SE(3)."""
        pts = N.points_arg(points)
        T = N.mat4_arg(pose)
        c = N.Constraints()
        N.check(N.lib().kb_registration_constraints(self._h, N.ptr(pts), len(pts), voxel_map._h, N.ptr(T),
                                                    float(max_correspondance_distance), C.byref(c)))
        return _from_struct(c)

    def align_points_to_map_batch(self, points, voxel_map: VoxelHashMap, initial_guesses, max_correspondance_distance,
                                  kernel, ranges=None, return_inliers: bool = False):
        """B independent align_points_to_map problems against one map, run side by side in one launch
        (relocalization, loop-closure checks, multi-hypothesis starts). Each result equals, bit for bit, what
        align_points_to_map returns for that hypothesis alone.

        points: one (N, 3) cloud with ``ranges`` (B, 2) rows of (offset, count) — ranges may overlap or repeat; no
        ranges: every hypothesis uses the whole cloud — or a list of B (n_b, 3) clouds. initial_guesses: (B, 4, 4).
        max_correspondance_distance, kernel: scalars or (B,) arrays.
        Returns (poses (B, 4, 4), iterations (B,)) and, with return_inliers, inliers (B,): the correspondence count
        build_system gives for the source mapped by its pose. Torch CUDA tensors in give torch CUDA tensors out
        (the device entry point); anything else goes through host arrays."""
        torch = _torch_if_cuda(points[0] if isinstance(points, (list, tuple)) and len(points) else points)
        if torch is not None:
            return self._align_batch_dev(torch, points, voxel_map, initial_guesses, max_correspondance_distance, kernel,
                                         ranges, return_inliers)
        g = _guesses_arg(initial_guesses)
        B = len(g)
        if isinstance(points, (list, tuple)):
            if ranges is not None:
                raise RuntimeError("ranges go with a single (N, 3) cloud, not with a list of clouds")
            clouds = [N.points_arg(p) for p in points]
            counts = np.array([len(c) for c in clouds], dtype=np.uint64)
            pts = np.concatenate(clouds) if clouds else np.empty((0, 3))
            offsets = (np.cumsum(counts) - counts).astype(np.uint64)
        else:
            pts = N.points_arg(points)
            offsets, counts = _ranges_arg(ranges, len(pts), B)
        if len(counts) != B:
            raise RuntimeError(f"{len(counts)} point ranges for {B} initial guesses")
        md = _per_hypothesis(max_correspondance_distance, B)
        ks = _per_hypothesis(kernel, B)
        poses = np.empty((B, 4, 4))
        iters = np.empty(B, dtype=np.int32)
        inl = np.empty(B, dtype=np.int32) if return_inliers else None
        N.check(N.lib().kb_registration_align_batch(
            self._h, N.ptr(pts), len(pts), N.ptr(offsets), N.ptr(counts), B, voxel_map._h, N.ptr(g), N.ptr(md), N.ptr(ks),
            N.ptr(poses), N.ptr(iters), N.ptr(inl) if inl is not None else None))
        return (poses, iters, inl) if return_inliers else (poses, iters)

    def _align_batch_dev(self, torch, points, voxel_map, initial_guesses, max_dist, kernel, ranges, return_inliers):
        if isinstance(points, (list, tuple)):
            if ranges is not None:
                raise RuntimeError("ranges go with a single (N, 3) cloud, not with a list of clouds")
            counts = np.array([p.shape[0] for p in points], dtype=np.uint64)
            offsets = (np.cumsum(counts) - counts).astype(np.uint64)
            points = torch.cat(list(points))
        else:
            offsets = counts = None
        dev = points.device
        if points.ndim != 2 or points.shape[1] != 3:
            raise RuntimeError("Unable to cast Python instance to C++ type (expected an (N, 3) array)")
        pts = points.to(torch.float64).contiguous()
        g = torch.as_tensor(initial_guesses, dtype=torch.float64, device=dev).contiguous()
        if g.ndim != 3 or g.shape[1:] != (4, 4):
            raise RuntimeError("Unable to cast Python instance to C++ type (expected (B, 4, 4) initial guesses)")
        B = g.shape[0]
        if counts is None:
            offsets, counts = _ranges_arg(None if ranges is None else np.asarray(torch.as_tensor(ranges).cpu()), len(pts), B)
        if len(counts) != B:
            raise RuntimeError(f"{len(counts)} point ranges for {B} initial guesses")
        as_dev = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), device=dev).to(dt).contiguous()
        off_d = as_dev(offsets.astype(np.int64), torch.int64)  # (size_t on the device: non-negative int64, same bits)
        cnt_d = as_dev(counts.astype(np.int64), torch.int64)
        md = as_dev(_per_hypothesis(np.asarray(torch.as_tensor(max_dist).cpu()), B), torch.float64)
        ks = as_dev(_per_hypothesis(np.asarray(torch.as_tensor(kernel).cpu()), B), torch.float64)
        poses = torch.empty((B, 4, 4), dtype=torch.float64, device=dev)
        iters = torch.empty(B, dtype=torch.int32, device=dev)
        inl = torch.empty(B, dtype=torch.int32, device=dev) if return_inliers else None
        p = lambda t: C.c_void_p(t.data_ptr())
        torch.cuda.current_stream(dev).synchronize()  # the inputs were made on torch's stream, the map has its own
        N.check(N.lib().kb_registration_align_batch_dev(
            self._h, p(pts), len(pts), p(off_d), p(cnt_d), B, voxel_map._h, p(g), p(md), p(ks), p(poses), p(iters),
            p(inl) if inl is not None else None))
        N.check(N.lib().kb_map_sync(voxel_map._h))
        return (poses, iters, inl) if return_inliers else (poses, iters)

    def relocalize(self, source, voxel_map: VoxelHashMap, search: RelocalizationSearch,
                   return_scores: bool = False) -> RelocalizationResult:
        """Find the pose of ``source`` (N, 3) in ``voxel_map`` without an initial pose: score every hypothesis of
        ``search`` on the device, refine its top_k peaks with align_points_to_map_batch (bit for bit that call's
        poses, iterations and inliers) and return the candidate with the most inliers, with the runner-up and, with
        return_scores, the (n_yaw, Ny, Nx) coarse scores. Only reads the map. Accepting the result is the caller's
        decision. kb_relocalize in include/kiss_icp_b200.h states every rule."""
        return relocalize(self._h, source, voxel_map, search, return_scores)

    def relocalize_in_places(self, descriptor_points, source, voxel_map: VoxelHashMap, places: PlaceDatabase, top_k=8,
                             separation=3.0, max_correspondence_distance=3.0, kernel_scale=1.0,
                             max_entry=-1) -> PlaceRelocalizationResult:
        """Find the pose of ``source`` (N, 3) in ``voxel_map`` without any pose: the top_k candidates of
        ``descriptor_points`` (the preprocessed frame the entries of ``places`` describe) among the database's entries,
        no two closer than ``separation`` metres, refined from their guesses with align_points_to_map_batch (bit for
        bit that call's poses, iterations and inliers); the candidate with the most inliers wins. Only reads the map.
        Accepting the result is the caller's decision. kb_place_relocalize in include/kiss_icp_b200.h states every
        rule."""
        return relocalize_in_places(self._h, descriptor_points, source, voxel_map, places, top_k, separation,
                                    max_correspondence_distance, kernel_scale, max_entry)

    @property
    def last_iterations(self) -> int:
        it = N.i32(0)
        N.check(N.lib().kb_registration_last_iterations(self._h, C.byref(it)))
        return it.value

    def build_system(self, points_in_map_frame, voxel_map: VoxelHashMap, max_correspondance_distance: float, kernel: float):
        """one DataAssociation + BuildLinearSystem pass (Registration.cpp:60-121): (JTJ, JTr, n)."""
        pts = N.points_arg(points_in_map_frame)
        JTJ = np.empty((6, 6))
        JTr = np.empty(6)
        nc = N.i32(0)
        check_value(N.lib().kb_registration_build_system(self._h, N.ptr(pts), len(pts), voxel_map._h,
                                                         float(max_correspondance_distance), float(kernel), N.ptr(JTJ),
                                                         N.ptr(JTr), C.byref(nc)))
        return JTJ, JTr, nc.value
