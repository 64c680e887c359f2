"""Extrinsic calibration of a multi-LiDAR rig from a recorded run (kb_calibrate_rig, DESIGN.md section 4.19).

A rig's extrinsics usually come from a drawing or a tape measure, and a few centimetres or a degree off smear every
merged scan. ``calibrate_rig`` refines them without targets: a reference sensor's scans, placed at the base poses T_k,
make a map, and every other sensor's extrinsic E_j is moved until its scans, placed at T_k E_j, fit that map best
(KISS-ICP's Geman-McClure point-to-point cost summed over every frame). Each refined sensor gets a report at its
returned extrinsic: the fit (``Fit``, information matrix in the sensor's own tangent) and the plane constraints
(``Constraints``), so that ``degeneracy(cal.sensors[j].constraints)`` tells which of the sensor's own axes the run
pins down. A run along a tunnel, for instance, does not fix a sensor's offset along the tunnel.
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
from .rig import Rig, Sensor, _check_rig

# The stages of calibrate_rig, (max_correspondence_distance, kernel_scale) in voxel sizes: a coarse gate that admits
# the ~1 m a degree of rotation error makes at 60 m, then a fine one (DESIGN.md section 4.19 has the basin measured).
DEFAULT_STAGES_VOXELS = ((3.0, 1.0), (1.0, 1.0 / 3.0))

# iterations: summed over the stages; converged: of the last stage; fit / constraints: at the returned extrinsic
SensorCalibration = namedtuple("SensorCalibration", ["iterations", "converged", "fit", "constraints"])
# rig: the calibrated Rig (every crop kept); extrinsics: (S, 4, 4); sensors: one SensorCalibration per sensor (zeros
# for a sensor that was not refined)
RigCalibration = namedtuple("RigCalibration", ["rig", "extrinsics", "sensors"])


def _calibrate(voxel_map: VoxelHashMap, poses, rig: Rig, ptrs, sizes, layout: int, refine, max_dist: float,
               kscale: float, max_iter: int, conv: float):
    """one kb_calibrate_rig call on raw frame pointers (ptrs[k S + j], sizes[k S + j], host or device addresses as
    ``layout`` says) -> (extrinsics (S, 4, 4), [kb_sensor_calibration] * S)"""
    S = rig.n_sensors
    P = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 16)
    K = len(P)
    if len(ptrs) != K * S or len(sizes) != K * S:
        raise ValueError(f"{len(ptrs)} arrays are not {K} frames of {S} sensors")
    X = (C.c_void_p * max(K * S, 1))(*[C.c_void_p(int(p)) if p else None for p in ptrs])
    n = (N.sz * max(K * S, 1))(*sizes)
    ref = None if refine is None else (N.i32 * S)(*[int(bool(r)) for r in refine])
    opt = N.RigCalibrationOptions(float(max_dist), float(kscale), int(max_iter), float(conv))
    E = np.empty((S, 4, 4))
    rep = (N.SensorCalibration * S)()
    check_value(N.lib().kb_calibrate_rig(voxel_map._h, N.ptr(P), K, rig._structs, S, ref, X, n, int(layout),
                                         C.byref(opt), N.ptr(E), rep))
    return E, list(rep)


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
    S = rig.n_sensors
    frames = list(frames)
    K = len(frames)
    for f in frames:
        if len(f) != S:
            raise ValueError(f"a frame of this rig has {S} scans, not {len(f)}")
    if not 0 <= int(reference) < S:
        raise ValueError(f"reference {reference} is not a sensor of this {S}-sensor rig")
    reference = int(reference)
    sel = [j != reference for j in range(S)] if refine is None else [False] * S
    if refine is not None:
        for j in refine:
            if not 0 <= int(j) < S:
                raise ValueError(f"refine: {j} is not a sensor of this {S}-sensor rig")
            sel[int(j)] = True
    cfg = config if config is not None else load_config()
    if cfg.mapping.voxel_size is None:
        cfg.mapping.voxel_size = float(cfg.data.max_range / 100.0)
    v = float(cfg.mapping.voxel_size)
    stages = [(d * v, k * v) for d, k in DEFAULT_STAGES_VOXELS] if stages is None else [tuple(s) for s in stages]
    if not stages or any(len(s) != 2 for s in stages):
        raise ValueError("stages: one or more pairs (max_correspondence_distance, kernel_scale)")
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
    cur = rig
    iters = np.zeros(S, dtype=np.int64)
    for max_dist, kscale in stages:
        E, rep = _calibrate(voxel_map, poses, cur, ptrs, sizes, 0, sel, max_dist, kscale,  # (0: KB_FRAMES_HOST_F64)
                            cfg.registration.max_num_iterations, cfg.registration.convergence_criterion)
        iters += [r.iterations for r in rep]
        cur = Rig([Sensor(E[j], s.min_range, s.max_range) for j, s in enumerate(rig.sensors)])
    sensors = [SensorCalibration(int(iters[j]), bool(r.converged),
                                 _fit_of(r.fit.n_correspondences, r.fit.n_source, r.fit.sum_sq_residual,
                                         np.array(r.fit.JTJ[:])),
                                 _from_struct(r.constraints)) for j, r in enumerate(rep)]
    return RigCalibration(cur, E, sensors)
