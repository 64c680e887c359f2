"""Multi-LiDAR rigs on the device (kb_merge_rig, kb_pipeline_register_rig_frames, KissICP.register_rig_frames, DESIGN.md
section 4.18): the merge against the numpy restatement of tests/test_rig.py, rig frames against the same frames merged
and registered as single frames, queue replay, a localizer, degeneracy-aware ICP, checkpoints and errors."""
import math

import numpy as np
import pytest

from test_motion import _exp_np, _random_motion
from test_rig import _front_rear, merge_np, random_extrinsic

pytestmark = pytest.mark.gpu


def _rig(K, sensors):
    return K.Rig([K.Sensor(E, lo, hi) for E, lo, hi in sensors])


def test_merge_rig_matches_restatement(K):
    rng = np.random.default_rng(21)
    times, poses = _random_motion(rng, m=6)
    sensors = [(np.eye(4), 1.0, 45.0), (random_extrinsic(rng), 2.0, math.inf), (np.eye(4), 0.0, math.inf),
               (random_extrinsic(rng), 0.0, 30.0), (np.eye(4), 0.0, math.inf)]
    scans = [rng.uniform(-50, 50, (n, 3)) for n in (4000, 3000, 0, 2500, 1500)]
    scans[0][:3] = [[1.0, 0.0, 0.0], [45.0, 0.0, 0.0], [-0.0, 0.0, -0.0]]  # on the crop's bounds: cropped
    # an identity sensor without crop passes its points unchanged: signed zeros, its origin, non-finite points
    scans[4][:5] = [[-0.0, 0.0, -0.0], [0.0, -0.0, 0.0], [-0.0, -0.0, -0.0], [np.inf, 1.0, 2.0], [np.nan, 0.0, 1.0]]
    stamps = [rng.uniform(times[0], times[-1], len(s)) - 3.0 for s in scans]
    offsets = [3.0, 3.02, 2.9, 2.95, 3.01]
    rig = _rig(K, sensors)
    for motion in (None, K.Motion(times, poses, stamp_offset=0.001, end_time=times[-1] - 0.01)):
        got, got_ts = K.merge_rig(scans, rig, stamps, offsets, motion)
        ref, ref_ts = merge_np(scans, sensors, stamps, offsets,
                               None if motion is None else (times, poses, 0.001, motion.end_time))
        assert np.array_equal(got_ts, ref_ts)  # stamp offsets: bit for bit
        assert np.array_equal(np.isfinite(got).all(1), np.isfinite(ref).all(1))
        assert np.isnan(got[:3]).all()
        ok = np.isfinite(ref).all(1)
        if motion is None:
            ident = np.zeros(len(ref), bool)
            ident[:4000] = ident[-1500:] = True
            # identity sensors, with and without a crop: bit for bit (the sign of every zero included)
            assert got[ident & ok].tobytes() == ref[ident & ok].tobytes()
            assert got[-1500:].tobytes() == scans[4].tobytes()
            assert np.abs(got[ok] - ref[ok]).max() < 1e-12
        else:
            assert np.abs(got[ok] - ref[ok]).max() < 1e-11
    # without stamps: points only; one sensor, identity, motion: exactly kb_deskew_motion
    got, got_ts = K.merge_rig(scans, rig)
    assert got_ts.size == 0 and np.array_equal(np.isnan(got), np.isnan(merge_np(scans, sensors)[0]))
    M = K.Motion(times, poses)
    one = _rig(K, [(np.eye(4), 0.0, math.inf)])
    assert np.array_equal(K.merge_rig([scans[1]], one, [stamps[1]], motion=M)[0], K.deskew(scans[1], stamps[1], M))


def _stream(K, n_frames, stamps="column"):
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=3, beams=32, cols=512, stamps=stamps)
    return L, [L.scan(k) for k in range(n_frames)]


def _state(kiss):
    vox, cnt, pts = kiss.local_map.dump()
    return kiss.last_pose, kiss.last_delta, vox, cnt, pts


def _same_state(a, b):
    return all(np.array_equal(x, y) for x, y in zip(_state(a), _state(b)))


@pytest.mark.parametrize("layout", ["f64", "f32", "dev"])
@pytest.mark.parametrize("mode", ["none", "stamps", "motion"])
def test_one_sensor_rig_equals_register_frames(K, layout, mode):
    import torch
    L, frames = _stream(K, 7, stamps="none" if mode == "none" else ("sweep" if mode == "motion" else "column"))
    pts = [f[0].astype(np.float32) if layout == "f32" else f[0] for f in frames]
    ts = [f[1] for f in frames]
    motions = None
    if mode == "motion":
        motions = [K.Motion(*L.motion_samples(k, 100.0)[:2], stamp_offset=L.scan_start_time(k)) for k in range(len(pts))]
    rig = _rig(K, [(np.eye(4), 0.0, math.inf)])
    a, b = K.KissICP(K.load_config(), report_fit=True), K.KissICP(K.load_config(), report_fit=True)
    if layout == "dev":
        d = [torch.tensor(p, device="cuda") for p in pts]
        dt = [torch.tensor(t, device="cuda") for t in ts]
        ms = None if motions is None else [m._struct(m.resolved_end_time(t)) for m, t in zip(motions, ts)]
        args = ([x.data_ptr() for x in d], [len(p) for p in pts], [t.data_ptr() if t.numel() else None for t in dt],
                [t.numel() for t in dt])
        Pa, Fa = a._register_rig_frames_raw(rig, *args, None, 2, return_fits=True, motions=ms)
        Pb, Fb = b._register_frames_raw(*args, 2, return_fits=True, motions=ms)
    else:
        Pa, Fa = a.register_rig_frames([[p] for p in pts], rig, [[t] for t in ts], motions=motions, return_fits=True)
        Pb, Fb = b.register_frames(pts, ts, motions=motions, return_fits=True)
    assert np.array_equal(Pa, Pb)
    assert all(np.array_equal(x, y, equal_nan=True) for x, y in zip(Fa, Fb))  # (rmse: NaN without correspondences)
    assert _same_state(a, b)
    assert all(np.array_equal(x, y) for x, y in zip(a._last_clouds(), b._last_clouds()))


def _two_sensor_frames(K, n_frames, stamps):
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=4, beams=32, cols=512)
    F, R = _front_rear()
    body = ((-2.3, -1.0, -1.6), (2.3, 1.0, -0.1))
    rig = synthetic.RigLidar(L, [F, R], shapes=[None, (16, 256, (-20.0, 10.0))], phases=[0.0, 0.3], stamps=stamps,
                             body=body)
    sensors = [(F, 4.0, math.inf), (R, 4.0, 90.0)]
    return rig, sensors, [rig.scan(k) for k in range(n_frames)]


def test_multi_sensor_rig_equals_merged_frames(K):
    """constant velocity: the merged frame and merged stamps through register_frames; motion: the deskewed merge without
    stamps, with the same Motions (their prediction)"""
    rig_l, sensors, frames = _two_sensor_frames(K, 8, "sweep")
    rig = _rig(K, sensors)
    a, b = K.KissICP(K.load_config()), K.KissICP(K.load_config())
    Pa = a.register_rig_frames([f[0] for f in frames], rig, [f[1] for f in frames], [f[2] for f in frames])
    merged = [K.merge_rig(f[0], rig, f[1], f[2]) for f in frames]
    Pb = b.register_frames([m[0] for m in merged], [m[1] for m in merged])
    assert np.array_equal(Pa, Pb) and _same_state(a, b)
    motions = []
    for k, f in enumerate(frames):
        times, poses, _, _ = rig_l.lidar.motion_samples(k, 100.0)
        motions.append(K.Motion(times, poses, stamp_offset=rig_l.lidar.scan_start_time(k), end_time=k / rig_l.lidar.hz))
    a, b = K.KissICP(K.load_config()), K.KissICP(K.load_config())
    Pa = a.register_rig_frames([f[0] for f in frames], rig, [f[1] for f in frames], [f[2] for f in frames],
                               motions=motions)
    desk = [K.merge_rig(f[0], rig, f[1], f[2], motion=m)[0] for f, m in zip(frames, motions)]
    Pb = b.register_frames(desk, None, motions=motions)
    assert np.array_equal(Pa, Pb) and _same_state(a, b)


@pytest.mark.parametrize("with_motion", [False, True])
def test_queued_equals_blocking_with_replay(K, with_motion, monkeypatch):
    """sparse two-sensor frames from the minimal voxel table: frames 0 and 4 outgrow it and are vetoed and replayed"""
    monkeypatch.setenv("KB_MAP_RESERVE_SLOTS", "0")
    rng = np.random.default_rng(8)
    xi = np.array([1.0, 0.1, 0.0, 0.0, 0.0, 0.3])
    E = _exp_np(np.array([0.5, -0.2, 0.1, 0.0, 0.0, 3.0]))[0]
    rig = _rig(K, [(np.eye(4), 0.0, math.inf), (E, 1.0, 200.0)])
    frames, motions = [], []
    for k in range(9):
        n = 15000 if k in (0, 4, 5) else 1500
        scans = [rng.uniform(-150, 150, size=(n, 3)) * [1.0, 1.0, 0.2] for _ in range(2)]
        frames.append((scans, [rng.uniform(0.0, 0.1, n), rng.uniform(0.0, 0.1, n)], [0.1 * (k - 1), 0.1 * (k - 1) + 0.002]))
        times = 0.1 * (k - 1) + np.array([0.0, 0.05, 0.1])
        motions.append(K.Motion(times, _exp_np(times[:, None] * xi), end_time=0.1 * k) if with_motion else None)
    cfg = K.load_config(max_range=300.0, voxel_size=1.0)
    a = K.KissICP(cfg)
    P_q = a.register_rig_frames([f[0] for f in frames], rig, [f[1] for f in frames], [f[2] for f in frames],
                                motions=motions)
    b = K.KissICP(cfg)
    P_b = []
    for f, m in zip(frames, motions):
        b.register_rig_frame(f[0], rig, f[1], f[2], motion=m, return_clouds=False)
        P_b.append(b.last_pose)
    assert a.grow_retries() >= 2
    assert np.array_equal(P_q, np.array(P_b)) and _same_state(a, b)


def test_localizer_degeneracy_and_checkpoint(K):
    rig_l, sensors, frames = _two_sensor_frames(K, 12, "none")
    rig = _rig(K, sensors)
    cfg = K.load_config()
    odo = K.KissICP(cfg)
    P = odo.register_rig_frames([f[0] for f in frames], rig)
    # a localizer in the odometry's map tracks the same rig run
    prior = K.VoxelHashMap(cfg.mapping.voxel_size, 1e4, cfg.mapping.max_points_per_voxel)
    prior.load(*odo.local_map.dump())
    loc = K.KissICP(cfg, prior_map=prior)
    loc.last_pose = P[0]
    Pl, fits = loc.register_rig_frames([f[0] for f in frames[1:]], rig, return_fits=True)
    assert max(np.linalg.norm(Pl[:, :3, 3] - P[1:, :3, 3], axis=1)) < 0.05
    assert (fits.n_correspondences > 0.8 * fits.n_source).all()
    # degeneracy-aware ICP on this well-conditioned rig run (box city, walls on all sides) holds nothing: bit for bit
    # the plain run, and the pass saw plane information in every scan after the first
    deg = K.KissICP(cfg, degeneracy_ratio=0.02)
    Pd, dg = deg.register_rig_frames([f[0] for f in frames], rig, return_degeneracy=True)
    assert not dg.translation_held.any() and not dg.rotation_held.any()
    assert (dg.n_planes[1:] > 0).all()
    assert np.array_equal(Pd, P)
    # a checkpoint taken mid-run restores and continues bit for bit
    a = K.KissICP(cfg)
    a.register_rig_frames([f[0] for f in frames[:6]], rig)
    b = K.KissICP(cfg)
    b.load_state_dict(a.state_dict())
    rest = [f[0] for f in frames[6:]]
    assert np.array_equal(a.register_rig_frames(rest, rig), b.register_rig_frames(rest, rig))
    assert np.array_equal(b.last_pose, P[-1]) and _same_state(a, b)


def test_errors_register_nothing(K):
    rig_l, sensors, frames = _two_sensor_frames(K, 3, "sweep")
    rig = _rig(K, sensors)
    kiss = K.KissICP(K.load_config())
    kiss.register_rig_frames([f[0] for f in frames[:1]], rig, [f[1] for f in frames[:1]], [f[2] for f in frames[:1]])
    before = _state(kiss)
    fs = [f[0] for f in frames[1:]]
    with pytest.raises(ValueError):  # a frame with one scan for a rig of two
        kiss.register_rig_frames([fs[0], fs[1][:1]], rig)
    with pytest.raises(K._native.KissB200Error):  # mixed stamps in the first frame
        kiss.register_rig_frames(fs, rig, [[frames[1][1][0], np.empty(0)], frames[2][1]])
    with pytest.raises(ValueError):  # a bad extrinsic
        kiss.register_rig_frames(fs, _rig(K, [(np.diag([1.0, 1.0, -1.0, 1.0]), 0.0, math.inf)] * 2))
    with pytest.raises(ValueError):
        K.KissICP(K.load_config(), fused=False).register_rig_frames(fs, rig)
    with pytest.raises(ValueError):  # a bad motion: checked before anything is registered
        kiss.register_rig_frames(fs, rig, motions=[None, K.Motion([0.0, 1.0], [np.eye(4)] * 2, end_time=np.inf)])
    assert all(np.array_equal(x, y) for x, y in zip(before, _state(kiss)))


def test_front_rear_rig_accuracy(K):
    """tools/rig_accuracy.py's scene without a body (seed 0, 150 scans from rest): the front/rear rig tracks the base
    better than either sensor alone. Measured on an H100: ATE 1.22 m / RTE 0.0252 m for the rig, 1.72 / 0.0308 front,
    1.36 / 0.0288 rear (DESIGN.md section 4.18)."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import rig_accuracy
    r = rig_accuracy.run(150, 0, False)["ate_rte_m"]
    print("front/rear rig without body:", r)
    assert r["rig"][0] < 1.5 and r["rig"][1] < 0.028
    assert r["rig"][0] < 0.95 * min(r["front"][0], r["rear"][0])
    assert r["rig"][1] < 0.95 * min(r["front"][1], r["rear"][1])


def test_sensor_crop_removes_self_hits(K):
    """with the body, a per-sensor min_range just beyond the self-hits' reach leaves no point of the body in the merged
    base-frame cloud, and keeps every scene point farther from its sensor"""
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=0, beams=32, cols=512)
    F, R = _front_rear()
    lo, hi = np.array([-2.3, -1.0, -1.6]), np.array([2.3, 1.0, -0.1])
    rig_l = synthetic.RigLidar(L, [F, R], body=(lo, hi))
    frames = [rig_l.scan(k, body_mask=True) for k in range(3)]
    reach = max(float(np.linalg.norm(p[m], axis=1).max()) for f in frames for p, m in zip(f[0], f[3]))
    rig = _rig(K, [(F, reach + 0.05, math.inf), (R, reach + 0.05, math.inf)])
    for pts, _, _, masks in frames:
        merged, _ = K.merge_rig(pts, rig)
        kept = merged[np.isfinite(merged).all(1)]
        inside = ((kept > lo - 0.1) & (kept < hi + 0.1)).all(1)
        assert masks[0].any() and masks[1].any() and not inside.any()
        far = sum(int((np.linalg.norm(p[~m], axis=1) > reach + 0.05).sum()) for p, m in zip(pts, masks))
        assert len(kept) == far
