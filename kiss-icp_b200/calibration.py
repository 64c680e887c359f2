"""Extrinsic calibration of a multi-LiDAR rig from a recorded run (kb_calibrate_rig, DESIGN.md section 4.19).

A rig's extrinsics usually come from a drawing or a tape measure, and a few centimetres or a degree off smear every
merged scan. ``calibrate_rig`` refines them without targets: a reference sensor's scans, placed at the base poses T_k,
make a map, and every other sensor's extrinsic E_j is moved until its scans, placed at T_k E_j, fit that map best
(KISS-ICP's Geman-McClure point-to-point cost summed over every frame). Each refined sensor gets a report at its
returned extrinsic: the fit (``Fit``, information matrix in the sensor's own tangent) and the plane constraints
(``Constraints``), so that ``degeneracy(cal.sensors[j].constraints)`` tells which of the sensor's own axes the run
pins down. A run along a tunnel, for instance, does not fix a sensor's offset along the tunnel.

``calibrate_rig_clocks`` (kb_calibrate_rig_clocks, DESIGN.md section 4.20) also refines each sensor's clock offset o_j
from a run with per-point stamps: every point is placed along the base trajectory at its own time, s + stamp offset +
o_j, so sweeps that span a moving 0.1 s are not read as extrinsic error. Register with the result by adding
``time_offsets[j]`` to sensor j's ``stamp_offsets``.
"""
from __future__ import annotations

import ctypes as C
from collections import namedtuple

import numpy as np

from . import _native as N
from .config import load_config
from .constraints import _from_struct
from .kiss_icp import KissICP, _fit_of
from .mapping import VoxelHashMap, check_value
from .motion import Motion, _so3_exp
from .rig import Rig, Sensor, _check_rig, _end_time, merge_rig

# The stages of calibrate_rig, (max_correspondence_distance, kernel_scale) in voxel sizes: a coarse gate that admits
# the ~1 m a degree of rotation error makes at 60 m, then a fine one (DESIGN.md section 4.19 has the basin measured).
DEFAULT_STAGES_VOXELS = ((3.0, 1.0), (1.0, 1.0 / 3.0))

# iterations: summed over the stages; converged: of the last stage; fit / constraints: at the returned extrinsic
SensorCalibration = namedtuple("SensorCalibration", ["iterations", "converged", "fit", "constraints"])
# rig: the calibrated Rig (every crop kept); extrinsics: (S, 4, 4); sensors: one SensorCalibration per sensor (zeros
# for a sensor that was not refined)
RigCalibration = namedtuple("RigCalibration", ["rig", "extrinsics", "sensors"])

# |do| [s] below which calibrate_rig_clocks' offset has converged: 10 us, 0.1 mm at 10 m/s (the extrinsic's
# convergence_criterion of 1e-4 is of the same size)
DEFAULT_TIME_CONVERGENCE = 1e-5
# iterations: summed over the stages; converged: of the last stage; fit / constraints: at the returned values;
# time_information: s = H_oo - H_oe H_ee^-1 H_eo, the offset's information with the extrinsic free [1/s^2 in the
# Geman-McClure-weighted metres of the fit]; time_coupling: s / H_oo, 1 when the offset is independent of the
# extrinsic and 0 when the run confounds them (0 also without any information, H_oo = 0)
SensorClockCalibration = namedtuple("SensorClockCalibration", ["iterations", "converged", "fit", "constraints",
                                                               "time_information", "time_coupling"])
# rig: the calibrated Rig; extrinsics: (S, 4, 4); time_offsets: (S,) [s], to be added to each sensor's stamp offsets;
# sensors: one SensorClockCalibration per sensor (zeros for a sensor neither refined nor timed)
RigClockCalibration = namedtuple("RigClockCalibration", ["rig", "extrinsics", "time_offsets", "sensors"])


def _calibrate(voxel_map: VoxelHashMap, poses, rig: Rig, ptrs, sizes, layout: int, refine, max_dist: float,
               kscale: float, max_iter: int, conv: float):
    """one kb_calibrate_rig call on raw frame pointers (ptrs[k S + j], sizes[k S + j], host or device addresses as
    ``layout`` says) -> (extrinsics (S, 4, 4), [kb_sensor_calibration] * S)"""
    S = rig.n_sensors
    P = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 16)
    K = len(P)
    if len(ptrs) != K * S or len(sizes) != K * S:
        raise ValueError(f"{len(ptrs)} arrays are not {K} frames of {S} sensors")
    X, n = _frame_arrays(ptrs, sizes)
    opt = N.RigCalibrationOptions(float(max_dist), float(kscale), int(max_iter), float(conv))
    E = np.empty((S, 4, 4))
    rep = (N.SensorCalibration * S)()
    check_value(N.lib().kb_calibrate_rig(voxel_map._h, N.ptr(P), K, rig._structs, S, _flag_array(refine, S), X, n,
                                         int(layout), C.byref(opt), N.ptr(E), rep))
    return E, list(rep)


def _frame_arrays(ptrs, sizes):
    X = (C.c_void_p * max(len(ptrs), 1))(*[C.c_void_p(int(p)) if p else None for p in ptrs])
    return X, (N.sz * max(len(sizes), 1))(*sizes)


def _flag_array(flags, S: int):
    return None if flags is None else (N.i32 * S)(*[int(bool(r)) for r in flags])


def _check_run(rig: Rig, frames: list, reference, *per_frame) -> tuple[int, int, int]:
    """K frames of S scans (and of S entries in each of per_frame's K lists) and a reference sensor -> (S, K, reference)"""
    S, K = rig.n_sensors, len(frames)
    if any(len(x) != K for x in per_frame):
        raise ValueError("frames, timestamps and stamp_offsets differ in length")
    for f in zip(frames, *per_frame):
        if any(len(x) != S for x in f):
            raise ValueError(f"a frame of this rig has {S} scans, stamp arrays and stamp offsets" if per_frame else
                             f"a frame of this rig has {S} scans, not {len(f[0])}")
    if not 0 <= int(reference) < S:
        raise ValueError(f"reference {reference} is not a sensor of this {S}-sensor rig")
    return S, K, int(reference)


def _config_stages(config, stages):
    """the KISSConfig (default: load_config(); voxel size defaulted to max_range / 100 as the pipeline does) and the
    stages in metres (default: DEFAULT_STAGES_VOXELS times the voxel size) -> (cfg, voxel size, stages)"""
    cfg = config if config is not None else load_config()
    if cfg.mapping.voxel_size is None:
        cfg.mapping.voxel_size = float(cfg.data.max_range / 100.0)
    v = float(cfg.mapping.voxel_size)
    stages = [(d * v, k * v) for d, k in DEFAULT_STAGES_VOXELS] if stages is None else [tuple(s) for s in stages]
    if not stages or any(len(s) != 2 for s in stages):
        raise ValueError("stages: one or more pairs (max_correspondence_distance, kernel_scale)")
    return cfg, v, stages


def _run_stages(rig: Rig, stages, call):
    """call(rig, max_dist, kscale) -> (extrinsics (S, 4, 4), reports) once per stage, each stage on the rig the last
    one returned -> (the calibrated Rig, the last extrinsics, the last reports, iterations summed over the stages)"""
    cur = rig
    iters = np.zeros(rig.n_sensors, dtype=np.int64)
    for max_dist, kscale in stages:
        E, rep = call(cur, max_dist, kscale)
        iters += [r.iterations for r in rep]
        cur = Rig([Sensor(E[j], s.min_range, s.max_range) for j, s in enumerate(rig.sensors)])
    return cur, E, rep, iters


def _fit_and_constraints(r):
    return (_fit_of(r.fit.n_correspondences, r.fit.n_source, r.fit.sum_sq_residual, np.array(r.fit.JTJ[:])),
            _from_struct(r.constraints))


def _crop(points, sensor: Sensor) -> np.ndarray:
    p = N.points_arg(points)
    with np.errstate(invalid="ignore"):
        r = np.linalg.norm(p, axis=1)
        return p[(r > sensor.min_range) & (r < sensor.max_range)]


def calibrate_rig(frames, rig: Rig, poses=None, reference: int = 0, refine=None, voxel_map: VoxelHashMap | None = None,
                  config=None, stages=None) -> RigCalibration:
    """Refine the extrinsics of ``rig`` from a recorded run.

    ``frames``: K rig frames, each one (N_j, 3) scan per sensor in its own frame, without stamps (as
    ``KissICP.register_rig_frames`` takes them). Each scan is cropped to its sensor's range and downsampled in its own
    frame with the pipeline's source rule (``KissICP.voxelize``).
    ``poses``: (K, 4, 4) base poses (world <- base). None: odometry on the ``reference`` sensor alone (a one-sensor
    rig with its extrinsic, ``KissICP.register_rig_frames``).
    ``voxel_map``: the map to align to, in the poses' frame (a survey map, ``LoopCloser.global_map()``); it is only read,
    so a localizer may hold it. None: the reference sensor's frame-downsampled scans at T_k E_ref, nothing evicted;
    a caller's map needs the poses.
    ``refine``: the sensors to refine (default: every sensor but ``reference``). The others come back unchanged.
    ``config``: the KISSConfig that sets the voxel size, the map's points per voxel, ``max_num_iterations`` and
    ``convergence_criterion`` (default: load_config()).
    ``stages``: (max_correspondence_distance, kernel_scale) pairs in metres, one kb_calibrate_rig call each, every
    one starting from the last one's result (default: DEFAULT_STAGES_VOXELS times the voxel size)."""
    _check_rig(rig)
    frames = list(frames)
    S, K, reference = _check_run(rig, frames, reference)
    sel = _flags(refine, S, [j != reference for j in range(S)], "refine")
    cfg, v, stages = _config_stages(config, stages)
    if voxel_map is not None and poses is None:
        raise ValueError("a caller's voxel_map needs the poses in its frame")
    if poses is None:
        odo = KissICP(cfg)
        poses = odo.register_rig_frames([[f[reference]] for f in frames], Rig([rig.sensors[reference]]))
    poses = np.ascontiguousarray(poses, dtype=np.float64)
    if poses.shape != (K, 4, 4):
        raise ValueError(f"poses must be ({K}, 4, 4), not {poses.shape}")
    # the pipeline's source rule, in each sensor's own frame
    vox = KissICP(cfg)
    sources = [[np.empty((0, 3))] * S for _ in range(K)]
    ref_ds = []  # the reference's frame-downsampled scans (for the map)
    for k, f in enumerate(frames):
        for j in range(S):
            if sel[j] or (voxel_map is None and j == reference):
                src, ds = vox.voxelize(_crop(f[j], rig.sensors[j]))
                if sel[j]:
                    sources[k][j] = src
                if j == reference:
                    ref_ds.append(ds)
    if voxel_map is None:
        voxel_map = VoxelHashMap(v, cfg.data.max_range, cfg.mapping.max_points_per_voxel)
        E_ref = rig.sensors[reference].extrinsic
        for k in range(K):
            M = poses[k] @ E_ref
            if len(ref_ds[k]):
                voxel_map.add_points(ref_ds[k] @ M[:3, :3].T + M[:3, 3])
    flat = [a for f in sources for a in f]
    ptrs = [a.ctypes.data if len(a) else None for a in flat]
    sizes = [len(a) for a in flat]
    cur, E, rep, iters = _run_stages(rig, stages, lambda cur, max_dist, kscale: _calibrate(
        voxel_map, poses, cur, ptrs, sizes, 0, sel, max_dist, kscale,  # (0: KB_FRAMES_HOST_F64)
        cfg.registration.max_num_iterations, cfg.registration.convergence_criterion))
    sensors = [SensorCalibration(int(iters[j]), bool(r.converged), *_fit_and_constraints(r)) for j, r in enumerate(rep)]
    return RigCalibration(cur, E, sensors)


def _calibrate_clocks(voxel_map: VoxelHashMap, trajectory: Motion, rig: Rig, ptrs, sizes, stamps, stamp_offsets,
                      layout: int, refine, refine_time, time_offsets, max_dist: float, kscale: float, max_iter: int,
                      conv: float, tconv: float):
    """one kb_calibrate_rig_clocks call on raw frame pointers (ptrs[k S + j], sizes[k S + j] host or device addresses
    as ``layout`` says; stamps[k S + j] host float64 arrays, stamp_offsets[k S + j] floats)
    -> (extrinsics (S, 4, 4), time offsets (S,), [kb_sensor_clock_calibration] * S)"""
    S = rig.n_sensors
    KS = len(ptrs)
    if KS % S or len(sizes) != KS or len(stamps) != KS or len(stamp_offsets) != KS:
        raise ValueError(f"{len(ptrs)} arrays are not frames of {S} sensors with stamps and stamp offsets")
    stamps = [np.ascontiguousarray(np.asarray(t, dtype=np.float64).ravel()) for t in stamps]
    X, n = _frame_arrays(ptrs, sizes)
    T, nt = _frame_arrays([t.ctypes.data if t.size else None for t in stamps], [t.size for t in stamps])
    so = (N.dbl * max(KS, 1))(*[float(o) for o in stamp_offsets])
    o0 = None if time_offsets is None else (N.dbl * S)(*[float(o) for o in time_offsets])
    opt = N.RigClockCalibrationOptions(float(max_dist), float(kscale), int(max_iter), float(conv), float(tconv))
    E = np.empty((S, 4, 4))
    o = np.empty(S)
    rep = (N.SensorClockCalibration * S)()
    m = trajectory._struct(0.0)  # (end_time is not used)
    check_value(N.lib().kb_calibrate_rig_clocks(voxel_map._h, C.byref(m), rig._structs, S, _flag_array(refine, S),
                                                _flag_array(refine_time, S), o0, X, n, T, nt, so, KS // S, int(layout),
                                                C.byref(opt), N.ptr(E), N.ptr(o), rep))
    return E, o, list(rep)


def _crop_stamped(points, stamps, sensor: Sensor):
    p = N.points_arg(points)
    t = np.asarray(stamps, dtype=np.float64).ravel()
    if len(t) != len(p):
        raise ValueError(f"{len(p)} points need as many stamps, not {len(t)}")
    with np.errstate(invalid="ignore"):
        r = np.linalg.norm(p, axis=1)
        keep = (r > sensor.min_range) & (r < sensor.max_range)
    return p[keep], t[keep]


def _first_rows(rows: np.ndarray, of: np.ndarray) -> np.ndarray:
    """the index in ``of`` of the first row equal, bit for bit, to each row of ``rows`` (each one is there)"""
    key = np.dtype([("x", "<u8"), ("y", "<u8"), ("z", "<u8")])
    a = np.ascontiguousarray(of, dtype=np.float64).view(np.uint64).view(key).ravel()
    b = np.ascontiguousarray(rows, dtype=np.float64).view(np.uint64).view(key).ravel()
    u, first = np.unique(a, return_index=True)
    pos = np.minimum(np.searchsorted(u, b), len(u) - 1)
    if not (u[pos] == b).all():
        raise AssertionError("a downsampled row is not an input row")
    return first[pos]


def _se3_log_exp_pose(T0, T1, alpha: float) -> np.ndarray:
    """T0 Exp(alpha Log(T0^-1 T1)) (host, numpy)"""
    D = np.linalg.inv(T0) @ T1
    R, t = D[:3, :3], D[:3, 3]
    c = min(1.0, max(-1.0, (np.trace(R) - 1.0) / 2.0))
    th = float(np.arccos(c))
    vee = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    w = vee * (0.5 if th < 1e-9 else th / (2.0 * np.sin(th)))
    W = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    V = np.eye(3) + 0.5 * W + (W @ W) / 12.0 if th < 1e-6 else \
        np.eye(3) + (1 - np.cos(th)) / th ** 2 * W + (th - np.sin(th)) / th ** 3 * (W @ W)
    u = np.linalg.solve(V, t)
    wa, ua = alpha * w, alpha * u
    tha = float(np.linalg.norm(wa))
    Wa = np.array([[0.0, -wa[2], wa[1]], [wa[2], 0.0, -wa[0]], [-wa[1], wa[0], 0.0]])
    Va = np.eye(3) + 0.5 * Wa + (Wa @ Wa) / 6.0 if tha < 1e-6 else \
        np.eye(3) + (1 - np.cos(tha)) / tha ** 2 * Wa + (tha - np.sin(tha)) / tha ** 3 * (Wa @ Wa)
    X = np.eye(4)
    X[:3, :3] = _so3_exp(wa)
    X[:3, 3] = Va @ ua
    return T0 @ X


def trajectory_pose(trajectory: Motion, t: float) -> np.ndarray:
    """T(t) of a Motion's samples, t on its sample clock (host, numpy): T_i Exp(alpha Log(T_i^-1 T_i+1)), the first
    and last intervals extrapolated; a sample's own time gives its pose exactly"""
    times, poses = trajectory.times, trajectory.poses
    i = int(np.clip(np.searchsorted(times, t, side="right") - 1, 0, len(times) - 2))
    alpha = (t - times[i]) / (times[i + 1] - times[i])
    return poses[i].copy() if alpha == 0.0 else _se3_log_exp_pose(poses[i], poses[i + 1], alpha)


def _flags(names, S: int, default, what: str):
    if names is None:
        return list(default)
    sel = [False] * S
    for j in names:
        if not 0 <= int(j) < S:
            raise ValueError(f"{what}: {j} is not a sensor of this {S}-sensor rig")
        sel[int(j)] = True
    return sel


def calibrate_rig_clocks(frames, timestamps, stamp_offsets, rig: Rig, trajectory: Motion | None = None,
                         reference: int = 0, refine=None, refine_time=None, time_offsets=None,
                         voxel_map: VoxelHashMap | None = None, config=None, stages=None) -> RigClockCalibration:
    """Refine the extrinsics and the clock offsets of ``rig`` from a recorded run with per-point stamps.

    ``frames``: K rig frames, each one (N_j, 3) scan per sensor in its own frame; ``timestamps``: K frames of S stamp
    arrays (one stamp per point); ``stamp_offsets``: K frames of S offsets that put each sensor's stamps on the run's
    clock, all on one clock (e.g. each sweep's start time), as ``KissICP.register_rig_frames`` takes them. Sensor j's
    unknown clock offset o_j is added to its stamps: a point is at time s + stamp_offset + o_j.
    ``trajectory``: the base's poses over the whole run (a Motion, world <- base; its stamp_offset is added to every
    point time, its end_time is not used). None: odometry on the ``reference`` sensor alone (a one-sensor rig with its
    stamps and stamp offsets through ``KissICP.register_rig_frames``), its poses at each frame's end time (the latest
    stamp plus offset), so that the offsets are relative to the reference sensor's clock.
    ``voxel_map``: the map to align to, in the trajectory's frame; only read (a localizer may hold it). None: the
    reference sensor's scans deskewed along the trajectory (``merge_rig``), frame-downsampled and placed at T(end_k);
    a caller's map needs the trajectory.
    ``refine`` / ``refine_time``: the sensors whose extrinsic / offset to refine (default: every sensor but
    ``reference``); the reference's offset is held at ``time_offsets[reference]`` unless ``refine_time`` names it.
    ``time_offsets``: (S,) initial offsets [s] (default 0).
    ``config`` and ``stages`` as in ``calibrate_rig``; the offset is refined in every stage. Each scan is cropped to its
    sensor's range and downsampled in its own frame with the pipeline's source rule; each kept point keeps its stamp.
    To register with the result, add ``time_offsets[j]`` to sensor j's ``stamp_offsets`` (and use ``rig``)."""
    _check_rig(rig)
    frames = list(frames)
    timestamps = list(timestamps)
    stamp_offsets = [[float(o) for o in f] for f in stamp_offsets]
    S, K, reference = _check_run(rig, frames, reference, timestamps, stamp_offsets)
    others = [j != reference for j in range(S)]
    sel = _flags(refine, S, others, "refine")
    sel_t = _flags(refine_time, S, others, "refine_time")
    o0 = np.zeros(S) if time_offsets is None else np.array(time_offsets, dtype=np.float64).reshape(-1)
    if o0.shape != (S,):
        raise ValueError(f"time_offsets must hold {S} offsets")
    cfg, v, stages = _config_stages(config, stages)
    if voxel_map is not None and trajectory is None:
        raise ValueError("a caller's voxel_map needs the trajectory in its frame")
    if trajectory is not None and not isinstance(trajectory, Motion):
        raise TypeError(f"trajectory must be a Motion, not {type(trajectory).__name__}")
    ref_rig = Rig([rig.sensors[reference]])
    ref_ts = [np.asarray(t[reference], dtype=np.float64).ravel() for t in timestamps]
    ref_off = [o[reference] + o0[reference] if o0[reference] else o[reference] for o in stamp_offsets]
    if trajectory is None:
        poses = KissICP(cfg).register_rig_frames([[f[reference]] for f in frames], ref_rig,
                                                 timestamps=[[t] for t in ref_ts],
                                                 stamp_offsets=[[o] for o in ref_off])
        ends = [float(np.nanmax(t)) + o if t.size and np.isfinite(t).any() else o for t, o in zip(ref_ts, ref_off)]
        trajectory = Motion(ends, poses)
    vox = KissICP(cfg)
    if voxel_map is None:
        voxel_map = VoxelHashMap(v, cfg.data.max_range, cfg.mapping.max_points_per_voxel)
        for k, f in enumerate(frames):
            merged, _ = merge_rig([f[reference]], ref_rig, [ref_ts[k]], [ref_off[k]], motion=trajectory)
            merged = merged[np.isfinite(merged).all(axis=1)]
            if not len(merged):
                continue
            _, ds = vox.voxelize(merged)
            M = trajectory_pose(trajectory, _end_time(trajectory, [ref_ts[k]], [ref_off[k]]))  # (merge_rig's target)
            voxel_map.add_points(ds @ M[:3, :3].T + M[:3, 3])
    # the pipeline's source rule in each sensor's own frame, each kept point with its stamp
    proc = [a or b for a, b in zip(sel, sel_t)]
    srcs, src_ts, offs = [], [], []
    for k, f in enumerate(frames):
        for j in range(S):
            offs.append(stamp_offsets[k][j])
            if not proc[j]:
                srcs.append(np.empty((0, 3)))
                src_ts.append(np.empty(0))
                continue
            p, t = _crop_stamped(f[j], timestamps[k][j], rig.sensors[j])
            src = vox.voxelize(p)[0] if len(p) else np.empty((0, 3))
            srcs.append(np.ascontiguousarray(src))
            src_ts.append(t[_first_rows(src, p)] if len(src) else np.empty(0))
    ptrs = [a.ctypes.data if len(a) else None for a in srcs]
    sizes = [len(a) for a in srcs]
    o = o0.copy()

    def stage(cur, max_dist, kscale):  # (each stage starts from the last one's offsets)
        nonlocal o
        E, o, rep = _calibrate_clocks(voxel_map, trajectory, cur, ptrs, sizes, src_ts, offs, 0, sel, sel_t, o,
                                      max_dist, kscale, cfg.registration.max_num_iterations,
                                      cfg.registration.convergence_criterion, DEFAULT_TIME_CONVERGENCE)
        return E, rep

    cur, E, rep, iters = _run_stages(rig, stages, stage)
    sensors = [SensorClockCalibration(int(iters[j]), bool(r.converged), *_fit_and_constraints(r), float(r.time_schur),
                                      float(r.time_schur / r.time_row[6]) if r.time_row[6] > 0 else 0.0)
               for j, r in enumerate(rep)]
    return RigClockCalibration(cur, E, o, sensors)
