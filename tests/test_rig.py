"""Multi-LiDAR rigs (kb_sensor, rig.Rig, DESIGN.md section 4.18), without a device: the rig's checks, the synthetic rig
streams, and the merge restated twice, in plain numpy (4x4 matrices, the motion's numpy statement of test_motion) and over
the oracle's SE(3) functions. tests/test_rig_device.py checks the device against the numpy restatement."""
import ctypes as C
import hashlib
import math

import numpy as np
import pytest

from test_motion import _deskew_np, _exp_np, _oracle_deskew, _random_motion


# ---------------------------------------------------------------------------------------------- restatements
def random_extrinsic(rng, identity=False):
    if identity:
        return np.eye(4)
    return _exp_np(np.concatenate([rng.normal(0, 2.0, 3), rng.normal(0, 1.0, 3)]))[0]


def merge_np(scans, sensors, stamps=None, offsets=None, motion=None):
    """the merged frame in numpy: per sensor (E, min_range, max_range) the crop in its frame (no crop for [0, inf]), then
    E p; stamps s + offset_i; with motion = (times, poses, stamp_offset, end_time) and stamps, the deskew of
    test_motion._deskew_np at the merged stamp + stamp_offset. -> (points, stamps or None)"""
    S = len(scans)
    offsets = [0.0] * S if offsets is None else offsets
    pts, ts = [], []
    for i, (p, (E, lo, hi)) in enumerate(zip(scans, sensors)):
        p = np.asarray(p, dtype=np.float64).copy()
        if not (lo == 0.0 and hi == math.inf):
            r = np.sqrt((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2])
            p[~((r > lo) & (r < hi))] = np.nan
        if not np.array_equal(E, np.eye(4)):
            p = p @ E[:3, :3].T + E[:3, 3]
        pts.append(p)
        if stamps is not None:
            ts.append(np.asarray(stamps[i], dtype=np.float64)[: len(p)] + offsets[i])
    P = np.concatenate(pts) if pts else np.empty((0, 3))
    T = np.concatenate(ts) if stamps is not None else None
    if motion is not None and T is not None:
        times, poses, off, end = motion
        P = _deskew_np(P, T, times, poses, off, end)
    return P, T


def merge_oracle(O, scans, sensors, stamps=None, offsets=None, motion=None):
    """the same merge stated point by point over the oracle's SE(3) functions and the library's interval statement"""
    S = len(scans)
    offsets = [0.0] * S if offsets is None else offsets
    out, ts = [], []
    for i, (p, (E, lo, hi)) in enumerate(zip(scans, sensors)):
        for j, q in enumerate(np.asarray(p, dtype=np.float64)):
            r = float(np.linalg.norm(q))
            if (lo != 0.0 or hi != math.inf) and not (lo < r < hi):
                q = np.full(3, np.nan)
            out.append(O.se3_act(E, q[None])[0])
            if stamps is not None:
                ts.append(stamps[i][j] + offsets[i])
    P, T = np.array(out).reshape(-1, 3), (np.array(ts) if stamps is not None else None)
    if motion is not None and T is not None:
        times, poses, off, end = motion
        P = _oracle_deskew(O, P, T, times, poses, off, end)
    return P, T


def _sensor_struct(N, E, lo=0.0, hi=math.inf):
    s = N.Sensor()
    s.extrinsic[:] = [float(x) for x in np.asarray(E, dtype=np.float64).reshape(-1)]
    s.min_range, s.max_range = lo, hi
    return s


# ---------------------------------------------------------------------------------------------- without a device
def test_rig_check_rejects_malformed(K):
    from kiss_icp_b200 import _native as N
    lib = N.lib()
    ok = _sensor_struct(N, np.eye(4))
    arr = lambda *ss: (N.Sensor * len(ss))(*ss)
    assert lib.kb_rig_check(arr(ok), 1) == N.KB_OK
    assert lib.kb_rig_check(arr(*[ok] * 16), 16) == N.KB_OK
    assert lib.kb_rig_check(arr(_sensor_struct(N, np.eye(4), 0.5, 80.0)), 1) == N.KB_OK
    assert lib.kb_rig_check(None, 1) == N.KB_ERR_INVALID_ARG
    assert lib.kb_rig_check(arr(ok), 0) == N.KB_ERR_INVALID_ARG
    assert lib.kb_rig_check(arr(*[ok] * 17), 17) == N.KB_ERR_INVALID_ARG
    reflect = np.diag([1.0, 1.0, -1.0, 1.0])
    scaled = np.diag([1.1, 1.0, 1.0, 1.0])
    bottom = np.eye(4)
    bottom[3, 0] = 0.5
    nan = np.eye(4)
    nan[0, 3] = np.nan
    for E in (reflect, scaled, bottom, nan):
        assert lib.kb_rig_check(arr(ok, _sensor_struct(N, E)), 2) == N.KB_ERR_NOT_SE3
    for lo, hi in ((np.nan, 10.0), (-1.0, 10.0), (math.inf, math.inf), (0.0, np.nan), (5.0, 5.0), (6.0, 5.0)):
        assert lib.kb_rig_check(arr(ok, _sensor_struct(N, np.eye(4), lo, hi)), 2) == N.KB_ERR_INVALID_ARG, (lo, hi)
    for bad in ([], [K.Sensor(reflect)], [K.Sensor(np.eye(4), 3.0, 2.0)], [K.Sensor(np.eye(4))] * 17):
        with pytest.raises(ValueError):
            K.Rig(bad)
    with pytest.raises(ValueError):
        K.Sensor(np.eye(3))
    assert len(K.Rig([K.Sensor(np.eye(4)), K.Sensor(np.eye(4), 1.0)])) == 2


def _front_rear():
    F = np.eye(4)
    F[:3, 3] = [2.0, 0.0, 0.0]
    R = np.diag([-1.0, -1.0, 1.0, 1.0])
    R[:3, 3] = [-2.0, 0.0, 0.0]
    return F, R


def test_synthetic_rig_streams(K):
    """rig streams are deterministic, each sensor sees the scene from its mount, body hits are close to their sensor,
    and the default single-sensor streams give the arrays they always gave"""
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=2, beams=8, cols=128)
    F, R = _front_rear()
    body = ((-2.3, -1.0, -1.6), (2.3, 1.0, -0.1))
    rig = synthetic.RigLidar(L, [F, R], shapes=[None, (4, 64, (-15.0, 5.0))], phases=[0.0, 0.5], stamps="sweep", body=body)
    a, b = rig.scan(3, body_mask=True), rig.scan(3, body_mask=True)
    for x, y in zip(a[0] + a[1] + a[3], b[0] + b[1] + b[3]):
        assert np.array_equal(x, y)
    assert a[2] == [0.0, 0.5 / L.hz]
    assert len(a[0][1]) <= 4 * 64 and a[3][0].any() and a[3][1].any()
    for p, m in zip(a[0], a[3]):
        assert np.linalg.norm(p[m], axis=1).max() < 5.0
    # without the body, the front sensor's points are the single sensor's scan of a lidar mounted at F
    plain = synthetic.RigLidar(L, [np.eye(4)])
    p, ts, offs = plain.scan(2)
    assert len(p) == 1 and ts[0].size == 0 and offs == [0.0]
    assert np.abs(np.sort(np.linalg.norm(p[0], axis=1)) - np.sort(np.linalg.norm(L.scan(2)[0], axis=1))).max() < 0.2
    h = hashlib.sha256()
    for stamps in ("none", "column", "sweep"):
        S = synthetic.small_shape(seed=5, beams=8, cols=128, stamps=stamps)
        for k in (0, 3):
            q, t = S.scan(k)
            h.update(q.tobytes())
            h.update(t.tobytes())
    h.update(synthetic.Tunnel(beams=4, cols=32).scan(2)[0].tobytes())
    assert h.hexdigest() == DEFAULT_STREAMS_SHA256


# of the streams above at the commit before rigs were added (synthetic.SyntheticLidar and Tunnel are unchanged)
DEFAULT_STREAMS_SHA256 = "4b9a2c00378191401e97414a8573be2787f7b114488bca6c9974c035367a4a52"


def test_merge_restatements_agree(O):
    rng = np.random.default_rng(11)
    times, poses = _random_motion(rng, m=6)
    sensors = [(random_extrinsic(rng, identity=True), 0.0, math.inf), (random_extrinsic(rng), 2.0, 40.0),
               (random_extrinsic(rng), 0.0, 25.0)]
    scans = [rng.uniform(-50, 50, (n, 3)) for n in (300, 0, 250)]
    scans[1] = np.empty((0, 3))
    scans[0][5] = 0.0  # at the origin of a sensor without crop: passes
    scans[2][7] = [30.0, 0.0, 0.0]  # beyond its sensor's max_range: NaN
    stamps = [rng.uniform(times[0], times[-1], len(s)) - 5.0 for s in scans]
    offsets = [5.0, 5.1, 4.97]
    for motion in (None, (times, poses, 0.0, times[-1] - 0.01)):
        P, T = merge_np(scans, sensors, stamps, offsets, motion)
        Q, U = merge_oracle(O, scans, sensors, stamps, offsets, motion)
        assert np.array_equal(np.isnan(P), np.isnan(Q)) and np.array_equal(T, U)
        ok = ~np.isnan(P).any(1)
        assert np.abs(P[ok] - Q[ok]).max() < 1e-9
        assert np.isnan(P[-250 + 7]).all() and not np.isnan(P[5]).any()
        if motion is None:
            assert np.array_equal(P[5], np.zeros(3))
