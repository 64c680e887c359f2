"""KissICP — same surface as python/kiss_icp/kiss_icp.py:33-80.

Two execution modes:
  * fused (default): ``register_frame`` is ONE call into kb_pipeline_register_frame, i.e. one
    persistent CUDA kernel doing kiss_icp::pipeline::KissICP::RegisterFrame
    (cpp/kiss_icp/pipeline/KissICP.cpp:35-68) with all state resident in HBM.
  * modular (``fused=False`` or a fixed threshold, which only the Python reference has): the
    reference's own module-by-module sequence (kiss_icp.py:43-75) through the per-module C-ABI.

``KissICP(config, prior_map=vmap)`` is a localizer: the same statement against the prior map ``vmap`` without
``local_map.update``. The map is never written, ``last_fit`` reports how well each scan fits it, and while the
localizer exists the map's mutators raise MapInUseError. Build a prior map with existing calls, for example a
VoxelHashMap with a large max_distance and ``vmap.update(frame_downsample, pose)`` per scan of an odometry run, or
``vmap.load(...)`` from a state_dict (INTEGRATION.md section 4).

``KissICP(config, report_fit=True)`` is an odometry pipeline that also reports, in ``last_fit`` and
``register_frames(..., return_fits=True)``, how well each scan fit the map it was registered in: the pipeline's own map
before the scan's ``local_map.update``. Poses, thresholds and the map are the same as without it.

``report_constraints=True`` (a localizer, or odometry, where it turns fit reporting on too) also reports, in
``last_constraints`` and ``register_frames(..., return_constraints=True)``, the plane constraints of each scan's fit
(constraints.Constraints): which directions the scan pins down. Poses, fits and the map are the same as without it.

``degeneracy_ratio=rho`` (0 < rho < 1; a localizer, or odometry, where it turns fit reporting on too) holds the
prediction along directions a scan does not constrain: before ICP, the plane information at the initial guess
(centred at its position) is eigen-decomposed blockwise, axes with an eigenvalue below rho times their block's largest
are held, and every ICP step is projected off them (DESIGN.md section 4.16). ``last_degeneracy`` and
``register_frames(..., return_degeneracy=True)`` report it per scan (constraints.ScanDegeneracy). A scan that holds
nothing registers bit for bit as without it. ``constraints.RECOMMENDED_DEGENERACY_RATIO`` is the ratio to start from.

``register_frame(frame, timestamps, motion=Motion(...))`` and ``register_frames(..., motions=[...])`` take the LiDAR's
trajectory sampled by an IMU or wheel odometry (motion.Motion, DESIGN.md section 4.17) in place of the constant-velocity
model: the scan is deskewed along it, and predicted from it when the previous scan's Motion ends within its samples.

``register_rig_frame(scans, rig, ...)`` and ``register_rig_frames(frames, rig, ...)`` register frames of a multi-LiDAR rig
(rig.Rig, DESIGN.md section 4.18): each frame's per-sensor scans are cropped per sensor, mapped to the base and merged on
the device; the pipeline then tracks the base.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math
from collections import namedtuple

import numpy as np

from . import _native as N
from .config import KISSConfig, load_config
from .constraints import Constraints, ScanDegeneracy, _constraints_of, _from_struct, _from_structs, _scan_degeneracy
from .mapping import VoxelHashMap, check_value, get_voxel_hash_map
from .motion import Motion
from .places import PlaceDatabase, PlaceRelocalizationResult
from .preprocess import Preprocessor, get_preprocessor
from .registration import get_registration
from .relocalization import RelocalizationResult, RelocalizationSearch
from .rig import Rig, _check_rig, _end_time, _frame
from .threshold import AdaptiveThreshold, get_threshold_estimator
from .voxelization import voxel_down_sample

STATE_FORMAT_VERSION = 1  # of KissICP.state_dict()
MAP_KEYS = ("voxels", "counts", "points")  # the map's part of an odometry state_dict()

# the fit of a scan at its final pose (kb_fit): correspondences closer than 3 sigma, source points,
# sqrt(sum |r|^2 / n_correspondences) (NaN without correspondences), and the 6x6 information matrix J^T W J
Fit = namedtuple("Fit", ["n_correspondences", "n_source", "rmse", "information"])


def _fit_of(n_corr, n_src, sse, JTJ):
    """a Fit from the raw values; array arguments give a Fit of arrays"""
    n = np.asarray(n_corr)
    with np.errstate(invalid="ignore", divide="ignore"):
        rmse = np.where(n > 0, np.sqrt(np.asarray(sse, dtype=np.float64) / np.maximum(n, 1)), np.nan)
    if n.ndim == 0:
        return Fit(int(n), int(n_src), float(rmse), np.asarray(JTJ, dtype=np.float64).reshape(6, 6))
    return Fit(n.astype(np.int64), np.asarray(n_src, dtype=np.int64), rmse, np.asarray(JTJ, dtype=np.float64).reshape(-1, 6, 6))


def _fits_from_structs(fs) -> Fit:
    """a Fit of arrays from an array of kb_fit"""
    return _fit_of([f.n_correspondences for f in fs], [f.n_source for f in fs], [f.sum_sq_residual for f in fs],
                   np.array([f.JTJ[:] for f in fs]).reshape(-1, 36))


def se3_params_from_matrix(T) -> np.ndarray:
    """4x4 SE(3) -> {qx,qy,qz,qw,tx,ty,tz}, the quaternion exactly as the library computes it from a matrix
    (Eigen's Quaterniond(Matrix3d); se3.cuh q_from_matrix, same operations in the same order)"""
    m = [[float(T[i][j]) for j in range(3)] for i in range(3)]
    c = [0.0] * 4
    t = m[0][0] + m[1][1] + m[2][2]
    if t > 0.0:
        t = math.sqrt(t + 1.0)
        c[3] = 0.5 * t
        t = 0.5 / t
        c[0] = (m[2][1] - m[1][2]) * t
        c[1] = (m[0][2] - m[2][0]) * t
        c[2] = (m[1][0] - m[0][1]) * t
    else:
        i = 0
        if m[1][1] > m[0][0]:
            i = 1
        if m[2][2] > m[i][i]:
            i = 2
        j = (i + 1) % 3
        k = (j + 1) % 3
        t = math.sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0)
        c[i] = 0.5 * t
        t = 0.5 / t
        c[3] = (m[k][j] - m[j][k]) * t
        c[j] = (m[j][i] + m[i][j]) * t
        c[k] = (m[k][i] + m[i][k]) * t
    return np.array(c + [float(T[0][3]), float(T[1][3]), float(T[2][3])])


def _params_arg(a):
    a = np.asarray(a, dtype=np.float64).reshape(-1)
    if a.shape != (7,):
        raise ValueError("an SE(3) parameter vector has 7 values {qx,qy,qz,qw,tx,ty,tz}")
    return a


def _pose_arg(T):
    a = np.array(T, dtype=np.float64)
    if a.shape != (4, 4) or not np.isfinite(a).all():
        raise ValueError("a pose is a finite 4x4 matrix")
    return a


class _PipelineThreshold:
    """read-only view of the device-resident adaptive threshold of a fused pipeline"""

    def __init__(self, owner):
        self._owner = owner

    def get_threshold(self):
        return self._owner._sigma_next()


class KissICP:
    def __init__(self, config: KISSConfig | None = None, fused: bool = True, prior_map: VoxelHashMap | None = None,
                 report_fit: bool = False, report_constraints: bool = False, degeneracy_ratio: float = 0.0):
        if prior_map is not None and not isinstance(prior_map, VoxelHashMap):
            raise TypeError(f"prior_map must be a VoxelHashMap, not {type(prior_map).__name__}")
        self.config = config if config is not None else load_config()
        if self.config.mapping.voxel_size is None:
            self.config.mapping.voxel_size = float(self.config.data.max_range / 100.0)
        self.fused = bool(fused) and self.config.adaptive_threshold.fixed_threshold is None
        self.localizer = prior_map is not None
        self._report_constraints = bool(report_constraints)
        rho = float(degeneracy_ratio)
        if not 0.0 <= rho < 1.0:  # (NaN fails too)
            raise ValueError(f"degeneracy_ratio {degeneracy_ratio} is not in [0, 1)")
        if rho > 0.0 and not (bool(fused) and self.config.adaptive_threshold.fixed_threshold is None):
            raise ValueError("degeneracy_ratio needs the fused pipeline (fused=True, an adaptive threshold)")
        self._degeneracy_ratio = rho
        # (a localizer always reports fits; plane constraints and the degeneracy pass run next to the fit)
        self._report_fit = self.localizer or bool(report_fit) or self._report_constraints or rho > 0.0
        self._h = None
        self._seen_motion = False  # (state_dict() carries motion_end_time once a Motion was registered)
        if self.localizer:
            self._check_prior(prior_map)
        if self.fused:
            c = N.Config()
            c.voxel_size = self.config.mapping.voxel_size
            c.max_range = self.config.data.max_range
            c.min_range = self.config.data.min_range
            c.max_points_per_voxel = self.config.mapping.max_points_per_voxel
            c.min_motion_th = self.config.adaptive_threshold.min_motion_th
            c.initial_threshold = self.config.adaptive_threshold.initial_threshold
            c.max_num_iterations = self.config.registration.max_num_iterations
            c.convergence_criterion = self.config.registration.convergence_criterion
            c.max_num_threads = self.config.registration.max_num_threads
            c.deskew = int(self.config.data.deskew)
            self._h = N.vp()
            if self.localizer:
                # (self.local_map holds the prior: it cannot be collected while the localizer reads it)
                check_value(N.lib().kb_pipeline_create_localizer(C.byref(c), prior_map._h, C.byref(self._h)))
                self.local_map = prior_map
            else:
                N.check(N.lib().kb_pipeline_create(C.byref(c), C.byref(self._h)))
                self.local_map = VoxelHashMap(c.voxel_size, c.max_range, c.max_points_per_voxel,
                                              _borrowed=N.lib().kb_pipeline_voxel_map(self._h), _owner=self)
                if self._report_fit:
                    N.check(N.lib().kb_pipeline_set_fit_reporting(self._h, 1))
            if self._report_constraints:
                N.check(N.lib().kb_pipeline_set_constraint_reporting(self._h, 1))
            if rho > 0.0:
                N.check(N.lib().kb_pipeline_set_degeneracy_ratio(self._h, rho))
            self.adaptive_threshold = _PipelineThreshold(self)
        else:
            self._last_pose = np.eye(4)
            self._last_delta = np.eye(4)
            self.adaptive_threshold = get_threshold_estimator(self.config)
            self.preprocessor = get_preprocessor(self.config)
            self.registration = get_registration(self.config)
            self.local_map = prior_map if self.localizer else get_voxel_hash_map(self.config)
            self._last_fit = _fit_of(0, 0, 0.0, np.zeros(36))
            self._last_constraints = _constraints_of(0, 0.0, 0.0, np.zeros(36))

    def _check_prior(self, prior_map):
        vs, mp = N.dbl(0), N.u32(0)
        N.check(N.lib().kb_map_params(prior_map._h, C.byref(vs), None, C.byref(mp)))
        c = self.config.mapping
        if vs.value != float(c.voxel_size) or mp.value != int(c.max_points_per_voxel):
            raise ValueError(f"prior map with voxel_size {vs.value}, max_points_per_voxel {mp.value}; the config has "
                             f"{c.voxel_size}, {c.max_points_per_voxel}")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and N._lib is not None:
            N._lib.kb_pipeline_destroy(h)
            self._h = None

    # -- pose()/delta() (KissICP.hpp:81-85) -----------------------------------------------------
    @property
    def last_pose(self):
        if not self.fused:
            return self._last_pose
        M = np.empty((4, 4))
        N.check(N.lib().kb_pipeline_pose(self._h, N.ptr(M)))
        return M

    @last_pose.setter
    def last_pose(self, T):
        if not self.fused:
            self._last_pose = np.array(T, dtype=np.float64)
        else:
            N.check(N.lib().kb_pipeline_set_pose(self._h, N.ptr(N.mat4_arg(T))))

    @property
    def last_delta(self):
        if not self.fused:
            return self._last_delta
        M = np.empty((4, 4))
        N.check(N.lib().kb_pipeline_delta(self._h, N.ptr(M)))
        return M

    @last_delta.setter
    def last_delta(self, T):
        if not self.fused:
            self._last_delta = np.array(T, dtype=np.float64)
        else:
            N.check(N.lib().kb_pipeline_set_delta(self._h, N.ptr(N.mat4_arg(T))))

    @property
    def report_fit(self) -> bool:
        """whether every scan gets a fit (a localizer, or KissICP(config, report_fit=True))"""
        return self._report_fit

    def _check_reports_fits(self):
        if not self._report_fit:
            raise ValueError("fits are computed by localizers and by odometry pipelines that report them: "
                             "KissICP(config, prior_map=...) or KissICP(config, report_fit=True)")

    @property
    def last_fit(self) -> Fit:
        """the fit of the last scan at its final pose (zeros before the first scan): against the prior map of a
        localizer, or against the map of an odometry pipeline with report_fit=True before the scan's update"""
        self._check_reports_fits()
        if not self.fused:
            return self._last_fit
        f = N.Fit()
        N.check(N.lib().kb_pipeline_last_fit(self._h, C.byref(f)))
        return _fit_of(f.n_correspondences, f.n_source, f.sum_sq_residual, np.array(f.JTJ[:]))

    @property
    def report_constraints(self) -> bool:
        """whether every scan gets plane constraints (KissICP(config, report_constraints=True))"""
        return self._report_constraints

    def _check_reports_constraints(self):
        if not self._report_constraints:
            raise ValueError("plane constraints are reported by pipelines created with report_constraints=True")

    @property
    def last_constraints(self) -> Constraints:
        """the plane constraints of the last scan's fit (zeros before the first scan), against the map the fit is
        against"""
        self._check_reports_constraints()
        if not self.fused:
            return self._last_constraints
        c = N.Constraints()
        N.check(N.lib().kb_pipeline_last_constraints(self._h, C.byref(c)))
        return _from_struct(c)

    @property
    def degeneracy_ratio(self) -> float:
        """the degeneracy ratio (0: off), KissICP(config, degeneracy_ratio=...)"""
        return self._degeneracy_ratio

    def _check_degeneracy(self):
        if self._degeneracy_ratio <= 0.0:
            raise ValueError("degeneracy results are reported by pipelines created with degeneracy_ratio > 0")

    @property
    def last_degeneracy(self) -> ScanDegeneracy:
        """the degeneracy-aware ICP's result of the last scan (zeros before the first)"""
        self._check_degeneracy()
        d = N.Degeneracy()
        N.check(N.lib().kb_pipeline_last_degeneracy(self._h, C.byref(d)))
        return _scan_degeneracy(d)

    @property
    def motion_end_time(self) -> float:
        """the end_time of the last scan if it was registered with a Motion, else NaN: a scan whose Motion covers it
        is predicted from it"""
        v = N.dbl(0)
        N.check(N.lib().kb_pipeline_motion_time(self._h, C.byref(v)))
        return v.value

    def _sigma_next(self):
        s = N.dbl(0)
        N.check(N.lib().kb_pipeline_threshold(self._h, C.byref(s)))
        return s.value

    @property
    def last_sigma(self):
        s = N.dbl(0)
        N.check(N.lib().kb_pipeline_last_sigma(self._h, C.byref(s)))
        return s.value

    @property
    def last_iterations(self):
        if not self.fused:
            return self.registration.last_iterations
        it = N.i32(0)
        N.check(N.lib().kb_pipeline_last_iterations(self._h, C.byref(it)))
        return it.value

    @property
    def last_profile_us(self):
        """device-side phase durations of the last fused RegisterFrame [us]:
        preprocess, downsample 0.5v, downsample 1.5v, ICP, map update, epilogue"""
        us = np.zeros(6)
        N.check(N.lib().kb_pipeline_last_profile(self._h, N.ptr(us), 6))
        return us

    def set_profiling(self, enabled: bool):
        """in-kernel phase timestamps (last_profile_us, history phase_us): off by default, ~10 us/scan when on"""
        N.check(N.lib().kb_pipeline_set_profiling(self._h, int(bool(enabled))))

    def grow_retries(self) -> int:
        """frames the kernel vetoed because the voxel table was sized too optimistically (grown + replayed)"""
        v = C.c_ulonglong(0)
        N.check(N.lib().kb_pipeline_grow_retries(self._h, C.byref(v)))
        return int(v.value)

    def start_history(self, capacity: int):
        """log per-frame statistics of the next ``capacity`` fused RegisterFrame calls (host side)"""
        N.check(N.lib().kb_pipeline_set_history(self._h, int(capacity)))

    def history(self):
        n = N.sz(0)
        N.check(N.lib().kb_pipeline_get_history(self._h, None, 0, C.byref(n)))
        arr = (N.FrameStats * n.value)()
        if n.value:
            N.check(N.lib().kb_pipeline_get_history(self._h, arr, n.value, C.byref(n)))
        return list(arr)

    # -- RegisterFrame ---------------------------------------------------------------------------
    def register_frame(self, frame, timestamps, return_clouds: bool = True, motion: Motion | None = None):
        """-> (preprocessed frame, source) like the reference; ``return_clouds=False`` skips the
        two device-to-host cloud copies (the pose is available as ``last_pose`` either way).
        ``motion``: the scan's sampled trajectory (motion.Motion) in place of the constant-velocity model."""
        if motion is not None:  # (a blocking frame is a queue of one)
            self.register_frames([frame], [timestamps], motions=[motion])
            return self._last_clouds() if return_clouds else (None, None)
        if not self.fused:
            return self._register_frame_modular(frame, timestamps)
        ts = np.ascontiguousarray(np.asarray(timestamps).ravel(), dtype=np.float64)
        f = np.asarray(frame)
        if f.dtype == np.float32 and f.ndim == 2 and f.shape[1] == 3:
            # float32 clouds (KITTI .bin, PointCloud2) go to the device as they are: half the H2D bytes,
            # widened exactly on the device (the reference does .astype(np.float64) on the host)
            pts = np.ascontiguousarray(f)
            N.check(N.lib().kb_pipeline_register_frame_f32(self._h, N.ptr(pts), len(pts), N.ptr(ts), len(ts)))
        else:
            pts = N.points_arg(frame)
            N.check(N.lib().kb_pipeline_register_frame(self._h, N.ptr(pts), len(pts), N.ptr(ts), len(ts)))
        if not return_clouds:
            return None, None
        return self._last_clouds()

    def _last_clouds(self):
        a, b = N.sz(0), N.sz(0)
        N.check(N.lib().kb_pipeline_last_cloud_sizes(self._h, C.byref(a), C.byref(b)))
        pre = np.empty((a.value, 3))
        src = np.empty((b.value, 3))
        N.check(N.lib().kb_pipeline_last_clouds(self._h, N.ptr(pre), a.value, N.ptr(src), b.value))
        return pre, src

    def register_frames(self, frames, timestamps=None, return_fits: bool = False, return_constraints: bool = False,
                        return_degeneracy: bool = False, motions=None):
        """Register a whole sequence (the dataset loop of python/kiss_icp/pipeline.py:106-112) -> poses (K,4,4).

        Same results as K ``register_frame`` calls; the frames are queued on the device (copy of frame k+1
        overlaps the registration of frame k, results are read behind the queue). ``frames`` is a sequence of
        (N_k,3) arrays, all float64 or all float32; ``timestamps`` a matching sequence (or None).
        ``return_fits`` (localizers and report_fit=True only) -> (poses, fits): a Fit of arrays, one entry per frame.
        ``return_constraints`` (report_constraints=True only) appends a Constraints of arrays: (poses, [fits,] constraints).
        ``return_degeneracy`` (degeneracy_ratio > 0 only) appends a ScanDegeneracy of arrays, one entry per frame.
        ``motions``: a matching sequence of motion.Motion or None (None: the constant-velocity model for that frame)."""
        K = len(frames)
        self._check_motions(motions, K)
        if return_fits:
            self._check_reports_fits()
        if return_constraints:
            self._check_reports_constraints()
        if return_degeneracy:
            self._check_degeneracy()
        if timestamps is None:
            timestamps = [np.empty(0)] * K
        if len(timestamps) != K:
            raise ValueError("frames and timestamps differ in length")
        if not self.fused:
            poses = np.empty((K, 4, 4))
            fits, cons = [], []
            for k in range(K):
                self._register_frame_modular(frames[k], timestamps[k])
                poses[k] = self._last_pose
                if return_fits:
                    fits.append(self._last_fit)
                if return_constraints:
                    cons.append(self._last_constraints)
            out = [poses]
            if return_fits:
                out.append(_fit_of([f.n_correspondences for f in fits], [f.n_source for f in fits],
                                   [f.rmse ** 2 * f.n_correspondences if f.n_correspondences else 0.0 for f in fits],
                                   np.array([f.information for f in fits]).reshape(-1, 36)))
            if return_constraints:
                out.append(_constraints_of([c.n_planes for c in cons], [c.weight_sum for c in cons],
                                           [c.plane_rmse ** 2 * c.weight_sum if c.weight_sum > 0 else 0.0 for c in cons],
                                           np.array([c.information for c in cons]).reshape(-1, 36)))
            return out[0] if len(out) == 1 else tuple(out)
        arrs = [np.asarray(f) for f in frames]
        f32 = K > 0 and all(a.dtype == np.float32 and a.ndim == 2 and a.shape[1] == 3 for a in arrs)
        pts = [np.ascontiguousarray(a) for a in arrs] if f32 else [N.points_arg(a) for a in arrs]
        ts = [np.ascontiguousarray(np.asarray(t).ravel(), dtype=np.float64) for t in timestamps]
        mstructs = None
        if motions is not None and any(m is not None for m in motions):
            mstructs = [m._struct(m.resolved_end_time(t)) if m is not None else None for m, t in zip(motions, ts)]
        return self._register_frames_raw([N.ptr(a) for a in pts], [len(a) for a in pts], [N.ptr(t) for t in ts],
                                         [len(t) for t in ts], 1 if f32 else 0, return_fits=return_fits,
                                         return_constraints=return_constraints, return_degeneracy=return_degeneracy,
                                         motions=mstructs)

    def _check_motions(self, motions, K):
        if motions is None:
            return
        if len(motions) != K:
            raise ValueError("frames and motions differ in length")
        if any(m is not None and not isinstance(m, Motion) for m in motions):
            raise TypeError("motions holds Motion objects or None")
        if not self.fused and any(m is not None for m in motions):
            raise ValueError("a Motion needs the fused pipeline (fused=True, an adaptive threshold)")

    def register_rig_frame(self, scans, rig: Rig, timestamps=None, stamp_offsets=None, motion: Motion | None = None,
                           return_clouds: bool = True):
        """Register one frame of a multi-LiDAR rig: ``scans`` one (N_i, 3) array per sensor of ``rig``, ``timestamps``
        None or one stamp array per sensor, ``stamp_offsets`` None or one offset per sensor (added to its stamps),
        ``motion`` the base's sampled trajectory (motion.Motion) or None. -> (preprocessed frame, source) like
        register_frame: the merged base-frame cloud after the pipeline's crop, and its source."""
        self.register_rig_frames([scans], rig, None if timestamps is None else [timestamps],
                                 None if stamp_offsets is None else [stamp_offsets],
                                 motions=None if motion is None else [motion])
        return self._last_clouds() if return_clouds else (None, None)

    def register_rig_frames(self, frames, rig: Rig, timestamps=None, stamp_offsets=None, motions=None,
                            return_fits: bool = False, return_constraints: bool = False, return_degeneracy: bool = False):
        """Register a sequence of rig frames, queued like register_frames -> poses (K, 4, 4) of the base, with the
        same ``return_fits`` / ``return_constraints`` / ``return_degeneracy`` rules. ``frames`` is a sequence of frames,
        each one (N_i, 3) array per sensor (all float64 or all float32); ``timestamps`` and ``stamp_offsets`` None or one
        entry per frame as in register_rig_frame; ``motions`` None or one Motion (the base's poses) or None per frame.
        Everything is checked before anything is registered, except a frame's own arrays: an invalid frame stops the
        sequence after the frames before it."""
        _check_rig(rig)
        if not self.fused:
            raise ValueError("a rig needs the fused pipeline (fused=True, an adaptive threshold)")
        K = len(frames)
        self._check_motions(motions, K)
        if return_fits:
            self._check_reports_fits()
        if return_constraints:
            self._check_reports_constraints()
        if return_degeneracy:
            self._check_degeneracy()
        timestamps = [None] * K if timestamps is None else timestamps
        stamp_offsets = [None] * K if stamp_offsets is None else stamp_offsets
        if len(timestamps) != K or len(stamp_offsets) != K:
            raise ValueError("frames, timestamps and stamp_offsets differ in length")
        f32 = K > 0 and all(isinstance(a, np.ndarray) and a.dtype == np.float32 and a.ndim == 2 and a.shape[1] == 3
                            for f in frames for a in f)
        parts = [_frame(f, rig, t, o, f32) for f, t, o in zip(frames, timestamps, stamp_offsets)]
        pts = [a for p in parts for a in p[0]]
        ts = [t for p in parts for t in p[1]]
        offs = [o for p in parts for o in p[2]]
        mstructs = None
        if motions is not None and any(m is not None for m in motions):
            mstructs = [m._struct(_end_time(m, p[1], p[2])) if m is not None else None for m, p in zip(motions, parts)]
        return self._register_rig_frames_raw(rig, [N.ptr(a) for a in pts], [len(a) for a in pts],
                                             [N.ptr(t) if t.size else None for t in ts], [len(t) for t in ts], offs,
                                             1 if f32 else 0, return_fits=return_fits,
                                             return_constraints=return_constraints,
                                             return_degeneracy=return_degeneracy, motions=mstructs)

    def _register_rig_frames_raw(self, rig: Rig, xyz_ptrs, sizes, ts_ptrs, ts_sizes, stamp_offsets, layout,
                                 return_fits: bool = False, return_constraints: bool = False,
                                 return_degeneracy: bool = False, motions=None):
        """raw-pointer form of register_rig_frames (host or device addresses, S per frame, layout as
        _register_frames_raw); stamp_offsets: None or one float per array; motions: None or one _native.Motion (None:
        no motion) per frame, with its end_time resolved"""
        S = rig.n_sensors
        K = len(xyz_ptrs) // S
        if len(xyz_ptrs) != K * S:
            raise ValueError(f"{len(xyz_ptrs)} arrays are not frames of {S} sensors")
        as_vp = lambda v: v if isinstance(v, C.c_void_p) else C.c_void_p(int(v) if v else None)
        X = (C.c_void_p * (K * S))(*[as_vp(v) for v in xyz_ptrs])
        T = (C.c_void_p * (K * S))(*[as_vp(v) for v in ts_ptrs])
        n = (N.sz * (K * S))(*sizes)
        nt = (N.sz * (K * S))(*ts_sizes)
        O = None if stamp_offsets is None else (N.dbl * (K * S))(*stamp_offsets)
        M = None
        if motions is not None:
            M = (N.Motion * K)(*[m if m is not None else N.Motion() for m in motions])
            self._seen_motion = True
        poses = np.empty((K, 4, 4))
        fits = (N.Fit * K)() if return_fits else None
        cons = (N.Constraints * K)() if return_constraints else None
        degs = (N.Degeneracy * K)() if return_degeneracy else None
        N.check(N.lib().kb_pipeline_register_rig_frames(self._h, rig._structs, S, X, n, T, nt, O, M, K, int(layout),
                                                        N.ptr(poses), fits, cons, degs))
        return self._results(poses, fits, cons, degs)

    @staticmethod
    def _results(poses, fits, cons, degs):
        out = [poses]
        if fits is not None:
            out.append(_fits_from_structs(fits))
        if cons is not None:
            out.append(_from_structs(cons))
        if degs is not None:
            out.append(_scan_degeneracy(degs))
        return out[0] if len(out) == 1 else tuple(out)

    def _register_frames_raw(self, xyz_ptrs, sizes, ts_ptrs, ts_sizes, layout, return_fits: bool = False,
                             return_constraints: bool = False, return_degeneracy: bool = False, motions=None):
        """raw-pointer form (host or device addresses): layout 0 host f64, 1 host f32, 2 device f64; motions: None or
        one _native.Motion (None: no motion) per frame, with its end_time resolved"""
        K = len(xyz_ptrs)
        as_vp = lambda v: v if isinstance(v, C.c_void_p) else C.c_void_p(int(v) if v else None)
        X = (C.c_void_p * K)(*[as_vp(v) for v in xyz_ptrs])
        T = (C.c_void_p * K)(*[as_vp(v) for v in ts_ptrs])
        n = (N.sz * K)(*sizes)
        nt = (N.sz * K)(*ts_sizes)
        poses = np.empty((K, 4, 4))
        fits = (N.Fit * K)() if return_fits else None
        cons = (N.Constraints * K)() if return_constraints else None
        degs = (N.Degeneracy * K)() if return_degeneracy else None
        if motions is not None:
            M = (N.Motion * K)(*[m if m is not None else N.Motion() for m in motions])
            self._seen_motion = True
            N.check(N.lib().kb_pipeline_register_frames_motion(self._h, X, n, T, nt, M, K, int(layout), N.ptr(poses),
                                                               fits, cons, degs))
        elif return_degeneracy:
            N.check(N.lib().kb_pipeline_register_frames_degeneracy(self._h, X, n, T, nt, K, int(layout), N.ptr(poses),
                                                                   fits, cons, degs))
        else:
            N.check(N.lib().kb_pipeline_register_frames_constraints(self._h, X, n, T, nt, K, int(layout), N.ptr(poses),
                                                                    fits, cons))
        return self._results(poses, fits, cons, degs)

    def _register_frame_modular(self, frame, timestamps):
        # python/kiss_icp/kiss_icp.py:43-75, line for line, on the per-module device API
        frame = self.preprocessor.preprocess(frame, np.asarray(timestamps), self._last_delta)
        source, frame_downsample = self.voxelize(frame)
        sigma = self.adaptive_threshold.get_threshold()
        initial_guess = self._last_pose @ self._last_delta
        new_pose = self.registration.align_points_to_map(
            points=source,
            voxel_map=self.local_map,
            initial_guess=initial_guess,
            max_correspondance_distance=3 * sigma,
            kernel=sigma,
        )
        model_deviation = np.linalg.inv(initial_guess) @ new_pose
        self.adaptive_threshold.update_model_deviation(model_deviation)
        if self._report_fit:  # against the map the scan was registered in: before local_map.update adds it
            self._last_fit = self._fit_modular(source, new_pose, sigma)
        if self._report_constraints:
            self._last_constraints = self.registration.constraints(source, self.local_map, new_pose, 3 * sigma)
        if not self.localizer:  # (a localizer has no local_map.update)
            self.local_map.update(frame_downsample, new_pose)
        self._last_delta = np.linalg.inv(self._last_pose) @ new_pose
        self._last_pose = new_pose
        return frame, source

    def _fit_modular(self, source, pose, sigma):
        mapped = source @ pose[:3, :3].T + pose[:3, 3]
        JTJ, _, n = self.registration.build_system(mapped, self.local_map, 3 * sigma, sigma)
        _, d = self.local_map.closest_neighbors(mapped)
        near = d < 3 * sigma
        return _fit_of(n, len(source), float(np.sum(d[near] ** 2)), JTJ)

    # -- relocalization ------------------------------------------------------------------------------
    def relocalize(self, frame, search: RelocalizationSearch) -> RelocalizationResult:
        """Find the localizer's pose in its prior map from one scan, without a pose to start from (at power-up, or
        after the track was lost), and continue the track from there.

        The scan's source is built as register_frame builds it, but without deskewing (there is no motion to deskew
        with): preprocessing, then the 0.5 voxel_size and 1.5 voxel_size downsamples. Registration.relocalize searches
        ``search`` with the refinement thresholds of the pipeline's current sigma (3 sigma, sigma): they override the
        search's max_correspondence_distance and kernel_scale. Then last_pose is the winner and last_delta the
        identity; the adaptive threshold's state is unchanged. Returns the RelocalizationResult; accepting it (for
        example by its inliers against n_source and against the runner-up's) is the caller's decision."""
        if not self.localizer:
            raise ValueError("relocalization needs a prior map: KissICP(config, prior_map=...)")
        if not isinstance(search, RelocalizationSearch):
            raise TypeError(f"search must be a RelocalizationSearch, not {type(search).__name__}")
        pre, reg = self._relocalizer()
        frame = pre.preprocess(frame, np.empty(0), np.eye(4))
        source, _ = self.voxelize(frame)
        sigma = self._sigma_next() if self.fused else self.adaptive_threshold.get_threshold()
        result = reg.relocalize(source, self.local_map,
                                dataclasses.replace(search, max_correspondence_distance=3 * sigma, kernel_scale=sigma))
        self.last_pose = result.pose
        self.last_delta = np.eye(4)
        return result

    def relocalize_by_place(self, frame, places: PlaceDatabase, top_k: int = 8,
                            separation: float = 3.0) -> PlaceRelocalizationResult:
        """Find the localizer's pose in its prior map from one scan without any pose, through the place database
        ``places`` built from the same run as the map, and continue the track from there.

        The scan is preprocessed as relocalize() does (without deskewing). The preprocessed frame is the descriptor
        cloud, the source is built from it by voxelize(). Registration.relocalize_in_places refines the top_k
        candidates with the thresholds of the pipeline's current sigma (3 sigma, sigma). Then last_pose is the winner
        and last_delta the identity; the adaptive threshold's state is unchanged. Returns the
        PlaceRelocalizationResult; accepting it is the caller's decision."""
        if not self.localizer:
            raise ValueError("relocalization needs a prior map: KissICP(config, prior_map=...)")
        if not isinstance(places, PlaceDatabase):
            raise TypeError(f"places must be a PlaceDatabase, not {type(places).__name__}")
        pre, reg = self._relocalizer()
        frame = pre.preprocess(frame, np.empty(0), np.eye(4))
        source, _ = self.voxelize(frame)
        sigma = self._sigma_next() if self.fused else self.adaptive_threshold.get_threshold()
        result = reg.relocalize_in_places(frame, source, self.local_map, places, top_k=top_k, separation=separation,
                                          max_correspondence_distance=3 * sigma, kernel_scale=sigma)
        self.last_pose = result.pose
        self.last_delta = np.eye(4)
        return result

    def _relocalizer(self):
        """(the preprocessor without deskewing, a registration) of the relocalization calls"""
        if getattr(self, "_reloc", None) is None:
            c = self.config
            self._reloc = (Preprocessor(c.data.max_range, c.data.min_range, False, c.registration.max_num_threads),
                           self.registration if not self.fused else get_registration(c))
        return self._reloc

    # -- checkpoint / restore -----------------------------------------------------------------------
    def state_dict(self):
        """The sequence's whole state as a dict of numpy arrays (it survives np.savez / np.load):
        format_version; the config fields; pose_qt, delta_qt (Sophus::SE3d::params() order {qx,qy,qz,qw,tx,ty,tz})
        and pose, delta (4x4); the adaptive threshold's model_sse, num_samples (NaN and 0 under a fixed threshold);
        the map as voxels, counts, points (VoxelHashMap.dump()). A localizer's state has no map: its prior map is not
        part of it.

        The fused pipeline's pose and delta are the device's quaternions and translations, bit for bit. In modular
        mode the 4x4 matrices are the state and pose_qt / delta_qt are derived from them."""
        c = self.config
        fixed = c.adaptive_threshold.fixed_threshold
        d = {"format_version": np.array(STATE_FORMAT_VERSION),
             "voxel_size": np.array(float(c.mapping.voxel_size)), "max_range": np.array(float(c.data.max_range)),
             "min_range": np.array(float(c.data.min_range)), "deskew": np.array(bool(c.data.deskew)),
             "max_points_per_voxel": np.array(int(c.mapping.max_points_per_voxel)),
             "max_num_iterations": np.array(int(c.registration.max_num_iterations)),
             "convergence_criterion": np.array(float(c.registration.convergence_criterion)),
             "initial_threshold": np.array(float(c.adaptive_threshold.initial_threshold)),
             "min_motion_th": np.array(float(c.adaptive_threshold.min_motion_th)),
             "fixed_threshold": np.array(np.nan if fixed is None else float(fixed))}
        if self.fused:
            s = N.PipelineState()
            N.check(N.lib().kb_pipeline_get_state(self._h, C.byref(s)))
            pose_qt, delta_qt = np.array(s.pose[:]), np.array(s.delta[:])
            pose, delta, sse, ns = self.last_pose, self.last_delta, s.model_sse, s.num_samples
        else:
            pose, delta = np.array(self._last_pose, dtype=np.float64), np.array(self._last_delta, dtype=np.float64)
            pose_qt, delta_qt = se3_params_from_matrix(pose), se3_params_from_matrix(delta)
            sse, ns = (np.nan, 0)  # a fixed threshold has no state
            if isinstance(self.adaptive_threshold, AdaptiveThreshold):
                sse, ns = self.adaptive_threshold.get_state()
        d.update(pose_qt=pose_qt, delta_qt=delta_qt, pose=pose, delta=delta, model_sse=np.array(float(sse)),
                 num_samples=np.array(int(ns)))
        if self._seen_motion:  # the end_time of the last scan if it had a Motion (NaN: none), for its successor's prediction
            d["motion_end_time"] = np.array(self.motion_end_time)
        if not self.localizer:  # (a localizer's prior map is not part of its state)
            vox, cnt, pts = self.local_map.dump()
            d.update(voxels=vox, counts=cnt, points=pts)
        return d

    def load_state_dict(self, state):
        """Restore a state_dict() taken in either mode (or an equivalent dict of the oracle's state), all or nothing: on ValueError
        nothing has changed. A localizer rejects a dict that carries a map; an odometry pipeline one that does not.

        voxel_size and max_points_per_voxel must equal this pipeline's (ValueError otherwise): the map's voxels
        and its per-voxel cap depend on them. Every other config field of the dict is ignored; the receiving
        pipeline keeps its own (max_range, thresholds, iterations ...). A fused pipeline restores pose and delta
        from pose_qt / delta_qt, exactly; modular mode takes the 4x4 pose / delta. A fixed threshold has no state
        and ignores model_sse / num_samples; an adaptive one rejects NaN, negative model_sse and num_samples < 1."""
        d = {k: np.asarray(v) for k, v in state.items()}
        if int(d["format_version"]) != STATE_FORMAT_VERSION:
            raise ValueError(f"state format {int(d['format_version'])}, expected {STATE_FORMAT_VERSION}")
        has_map = [k in d for k in MAP_KEYS]
        if self.localizer and any(has_map):
            raise ValueError("the prior map is not part of a localizer's state: the state carries a map")
        if not self.localizer and not all(has_map):
            raise ValueError("the state carries no map (voxels, counts, points): a localizer's state cannot restore "
                             "an odometry pipeline")
        c = self.config
        if float(d["voxel_size"]) != float(c.mapping.voxel_size) or \
                int(d["max_points_per_voxel"]) != int(c.mapping.max_points_per_voxel):
            raise ValueError(f"state of a map with voxel_size {float(d['voxel_size'])}, max_points_per_voxel "
                             f"{int(d['max_points_per_voxel'])}; this pipeline has {c.mapping.voxel_size}, "
                             f"{c.mapping.max_points_per_voxel}")
        sse, ns = float(d["model_sse"]), int(d["num_samples"])
        load_map = (lambda: None) if self.localizer else (lambda: self.local_map.load(d["voxels"], d["counts"], d["points"]))
        if self.fused:
            new, old = N.PipelineState(), N.PipelineState()
            new.pose[:] = [float(x) for x in _params_arg(d["pose_qt"])]
            new.delta[:] = [float(x) for x in _params_arg(d["delta_qt"])]
            new.model_sse, new.num_samples = sse, ns
            mt = float(d["motion_end_time"]) if "motion_end_time" in d else math.nan
            if math.isinf(mt):
                raise ValueError("motion_end_time is not finite")
            N.check(N.lib().kb_pipeline_get_state(self._h, C.byref(old)))
            check_value(N.lib().kb_pipeline_set_state(self._h, C.byref(new)))
            try:
                load_map()
            except Exception:
                N.check(N.lib().kb_pipeline_set_state(self._h, C.byref(old)))
                raise
            N.check(N.lib().kb_pipeline_set_motion_time(self._h, mt))
            self._seen_motion = self._seen_motion or "motion_end_time" in d
            return
        pose, delta = _pose_arg(d["pose"]), _pose_arg(d["delta"])
        if isinstance(self.adaptive_threshold, AdaptiveThreshold):
            old = self.adaptive_threshold.get_state()
            self.adaptive_threshold.set_state(sse, ns)
            try:
                load_map()
            except Exception:
                self.adaptive_threshold.set_state(*old)
                raise
        else:
            load_map()
        self._last_pose, self._last_delta = pose, delta

    def voxelize(self, iframe):
        if self.fused:
            pts = N.points_arg(iframe)
            src = np.empty_like(pts)
            ds = np.empty_like(pts)
            a, b = N.sz(0), N.sz(0)
            N.check(N.lib().kb_pipeline_voxelize(self._h, N.ptr(pts), len(pts), N.ptr(src), len(pts), C.byref(a),
                                                 N.ptr(ds), len(pts), C.byref(b)))
            return src[: a.value], ds[: b.value]
        frame_downsample = voxel_down_sample(iframe, self.config.mapping.voxel_size * 0.5)
        source = voxel_down_sample(frame_downsample, self.config.mapping.voxel_size * 1.5)
        return source, frame_downsample
