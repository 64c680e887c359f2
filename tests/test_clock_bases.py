"""Sampled motion and multi-LiDAR rigs at real clock values (DESIGN.md sections 4.17 and 4.18).

Sample times, end_time and stamp offsets are usually ROS header.stamp seconds, about 1.7e9, where a double resolves
2^-22 s = 2.4e-7 s; point stamps are seconds since the scan started. A point's time s + stamp_offset rounded at that
magnitude moves it by |v + w x p| * 1.2e-7 s, up to 2.6e-5 m at 20 m/s, 2 rad/s and 100 m. The library must not round
there: every test below compares the device with an exact reference or with the same stream on a clock that starts at 0.

The reference forms each point's time on the sample clock with fractions.Fraction from the given doubles
(tau = s + o_sensor + o_motion - t_k, and the interval of that time), and the deskew T(end)^-1 T_k Exp(tau xi_k) E p with
xi_k = Log(T_k^-1 T_k+1) / (t_k+1 - t_k) in mpmath at 40 digits for a sample of points; whole clouds in float64 numpy
driven by the exact tau. Streams use a dyadic clock base and dyadic sample and scan periods, so that every clock value is
exact at both bases and a shift of the clock changes no input bit."""
import bisect
import math
from fractions import Fraction

import mpmath
import numpy as np
import pytest

from test_motion import _deskew_np, _exp_np, _oracle_deskew

EPOCH = 1_760_000_000.0  # a ROS header.stamp of 2025; integer, so every 2^-22 s step after it is exact
HZ = 8.0  # scan rate of the streams: a dyadic scan period (0.125 s)
MP_DIGITS = 40
SAMPLE = 500  # points per case checked in mpmath


# ---------------------------------------------------------------------------------------------- exact reference
def _mp_hat(w):
    return mpmath.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])


def _mp_exp(xi):
    """SE(3) Exp of a 6-vector (translation, rotation) of mpf -> (R, t)"""
    v, w = mpmath.matrix(xi[:3]), xi[3:]
    th = mpmath.sqrt(w[0] ** 2 + w[1] ** 2 + w[2] ** 2)
    K = _mp_hat(w)
    K2 = K * K
    if th < mpmath.mpf("1e-12"):
        a, b, c = 1 - th ** 2 / 6, mpmath.mpf(1) / 2 - th ** 2 / 24, mpmath.mpf(1) / 6 - th ** 2 / 120
    else:
        a, b, c = mpmath.sin(th) / th, (1 - mpmath.cos(th)) / th ** 2, (th - mpmath.sin(th)) / th ** 3
    I = mpmath.eye(3)
    return I + a * K + b * K2, (I + b * K + c * K2) * v


def _mp_log(R, t):
    """SE(3) Log of (R, t) -> 6 mpf (translation, rotation); R within rounding of a rotation, angle below pi"""
    c = (R[0, 0] + R[1, 1] + R[2, 2] - 1) / 2
    th = mpmath.acos(max(mpmath.mpf(-1), min(mpmath.mpf(1), c)))
    s = [(R[2, 1] - R[1, 2]) / 2, (R[0, 2] - R[2, 0]) / 2, (R[1, 0] - R[0, 1]) / 2]
    f = 1 + th ** 2 / 6 if th < mpmath.mpf("1e-12") else th / mpmath.sin(th)
    w = [f * x for x in s]
    th = mpmath.sqrt(w[0] ** 2 + w[1] ** 2 + w[2] ** 2)
    K = _mp_hat(w)
    b = mpmath.mpf(1) / 2 - th ** 2 / 24 if th < mpmath.mpf("1e-12") else (1 - mpmath.cos(th)) / th ** 2
    c = mpmath.mpf(1) / 6 - th ** 2 / 120 if th < mpmath.mpf("1e-12") else (th - mpmath.sin(th)) / th ** 3
    v = mpmath.lu_solve(mpmath.eye(3) + b * K + c * K * K, t)
    return [v[0], v[1], v[2], w[0], w[1], w[2]]


def _mp_pose(T):
    """a 4x4 float64 pose -> (R, t) in mpmath, exactly"""
    return mpmath.matrix(T[:3, :3].tolist()), mpmath.matrix(T[:3, 3].tolist())


def _mp_mul(a, b):
    return a[0] * b[0], a[0] * b[1] + a[1]


def _mp_inv(a):
    Rt = a[0].T
    return Rt, -(Rt * a[1])


def _frac(x) -> Fraction:
    return Fraction(float(x))


def _mpf(q: Fraction):
    return mpmath.mpf(q.numerator) / q.denominator


class ExactMotion:
    """A Motion (times, poses on the sample clock, end_time) stated exactly: the interval and tau of a point from
    Fractions, the SE(3) algebra in mpmath"""

    def __init__(self, times, poses, end_time):
        with mpmath.workdps(MP_DIGITS):
            self.F = [_frac(t) for t in times]
            self.T = [_mp_pose(P) for P in poses]
            self.xi = []
            for k in range(len(times) - 1):
                D = _mp_mul(_mp_inv(self.T[k]), self.T[k + 1])
                dt = _mpf(self.F[k + 1] - self.F[k])
                self.xi.append([x / dt for x in _mp_log(*D)])
            k, tau = self.interval(_frac(end_time))
            self.end_inv = _mp_inv(self._at(k, tau))
            self.A = [_mp_mul(self.end_inv, T) for T in self.T[:-1]]
        self.A_np = np.array([np.vstack([np.hstack([np.array(A[0].tolist(), dtype=np.float64),
                                                    np.array(A[1].tolist(), dtype=np.float64)]), [0, 0, 0, 1]])
                              for A in self.A])
        self.xi_np = np.array([[float(x) for x in xi] for xi in self.xi])

    def interval(self, u: Fraction):
        """the interval of the exact sample-clock time u (the first and last extrapolate) and tau = u - t_k"""
        k = min(max(bisect.bisect_right(self.F, u) - 1, 0), len(self.F) - 2)
        return k, u - self.F[k]

    def _at(self, k, tau: Fraction):
        return _mp_mul(self.T[k], _mp_exp([x * _mpf(tau) for x in self.xi[k]]))

    def times_of(self, stamps, *offsets):
        """exact (k, tau) of every stamp s + sum(offsets) (k = -1 for a NaN stamp); tau rounded once to float64"""
        off = sum((_frac(o) for o in offsets), Fraction(0))
        k = np.full(len(stamps), -1)
        tau = np.full(len(stamps), np.nan)
        for i, s in enumerate(stamps):
            if math.isnan(s):
                continue
            k[i], q = self.interval(_frac(s) + off)
            tau[i] = float(q)
        return k, tau

    def deskew_np(self, pts, stamps, *offsets, E=None):
        """the whole cloud in float64, driven by the exact interval and tau: A_k Exp(tau xi_k) E p"""
        p = np.asarray(pts, dtype=np.float64)
        if E is not None:
            p = p @ E[:3, :3].T + E[:3, 3]
        k, tau = self.times_of(stamps, *offsets)
        ok = k >= 0
        out = np.full_like(p, np.nan)
        X = self.A_np[k[ok]] @ _exp_np(tau[ok, None] * self.xi_np[k[ok]])
        out[ok] = np.einsum("nij,nj->ni", X[:, :3, :3], p[ok]) + X[:, :3, 3]
        return out

    def deskew_mp(self, p, s, *offsets, E=None):
        """one point in mpmath: T(end)^-1 T_k Exp(tau xi_k) E p, rounded to float64 at the end"""
        with mpmath.workdps(MP_DIGITS):
            k, tau = self.interval(_frac(s) + sum((_frac(o) for o in offsets), Fraction(0)))
            q = mpmath.matrix([float(x) for x in p])
            if E is not None:
                Rm, tm = _mp_pose(E)
                q = Rm * q + tm
            R, t = _mp_mul(self.A[k], _mp_exp([x * _mpf(tau) for x in self.xi[k]]))
            r = R * q + t
            return np.array([float(r[0]), float(r[1]), float(r[2])])


def _check_exact(got, ref_np, ref, pts, stamps, offsets, rng, E=None, tol=1e-10, sample=SAMPLE):
    """got against the float64 cloud (all points) and a sample of it in mpmath; the two references against each other
    -> the worst error of got"""
    ok = np.isfinite(ref_np).all(1)
    assert np.array_equal(ok, np.isfinite(got).all(1))
    err_np = np.abs(got[ok] - ref_np[ok]).max()
    idx = rng.choice(np.flatnonzero(ok), min(sample, int(ok.sum())), replace=False)
    mp_pts = np.array([ref.deskew_mp(pts[i], stamps[i], *offsets, E=E) for i in idx])
    err_mp = np.abs(got[idx] - mp_pts).max()
    assert np.abs(ref_np[idx] - mp_pts).max() < 1e-11  # the float64 cloud is the mpmath one to rounding
    assert err_mp < tol and err_np < tol, (err_mp, err_np)
    return max(err_mp, err_np)


# ---------------------------------------------------------------------------------------------- motions and clouds
def _twist_motion(rng, base, start, dt, m, v=20.0, w=2.0, origin=500.0):
    """m samples dt apart from base + start (dyadic start and dt: exact at any dyadic base), poses of a vehicle within
    `origin` m of the map's origin turning at up to w rad/s and moving at up to v m/s, the twist changing per interval"""
    rel = start + dt * np.arange(m)
    T = np.eye(4)
    T[:3, :3] = _exp_np(np.concatenate([np.zeros(3), rng.normal(0, 1.0, 3)]))[0][:3, :3]
    T[:3, 3] = rng.uniform(-origin, origin, 3)
    poses = [T]
    for _ in range(m - 1):
        lin = rng.normal(size=3)
        ang = rng.normal(size=3)
        xi = np.concatenate([lin / np.linalg.norm(lin) * v * rng.uniform(0.5, 1.0),
                             ang / np.linalg.norm(ang) * w * rng.uniform(0.5, 1.0)])
        poses.append(poses[-1] @ _exp_np(dt * xi)[0])
    return base + rel, np.array(poses)


def _cloud(rng, n, rmin=1.0, rmax=100.0):
    d = rng.normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(rmin, rmax, (n, 1))


# ---------------------------------------------------------------------------------------------- without a device
def test_exact_reference_matches_restatements_at_base_0(O):
    """at clock 0 the exact reference is the numpy and the oracle restatements of test_motion to 1e-12 relative"""
    rng = np.random.default_rng(40)
    times, poses = _twist_motion(rng, 0.0, 0.0, 1 / 64, 9)
    pts = _cloud(rng, 400)
    ts = np.concatenate([rng.uniform(-0.02, 0.145, 398), [times[0], times[-1]]]) - 0.01
    end = times[-1] - 1 / 256
    ref = ExactMotion(times, poses, end)
    a = ref.deskew_np(pts, ts, 0.01)
    b = _deskew_np(pts, ts, times, poses, 0.01, end)
    c = _oracle_deskew(O, pts, ts, times, poses, 0.01, end)
    scale = np.abs(b).max()
    assert np.abs(a - b).max() < 1e-12 * scale and np.abs(a - c).max() < 1e-12 * scale
    mp_pts = np.array([ref.deskew_mp(p, s, 0.01) for p, s in zip(pts[:50], ts[:50])])
    assert np.abs(mp_pts - a[:50]).max() < 1e-12 * scale


def test_exact_reference_sees_clock_rounding():
    """at clock 1.76e9 the restatements that form s + offset first lose the point's time to the clock's spacing
    (2^-22 s): they differ from the exact reference by the 1e-5 m order worked out for 20 m/s, 2 rad/s and 100 m"""
    rng = np.random.default_rng(41)
    times, poses = _twist_motion(rng, EPOCH, 0.0, 1 / 64, 9)
    pts = _cloud(rng, 4000, 50.0, 100.0)
    ts = rng.uniform(0.0, 0.125, len(pts))
    end = times[-1]
    ref = ExactMotion(times, poses, end).deskew_np(pts, ts, EPOCH)
    rounded = _deskew_np(pts, ts, times, poses, EPOCH, end)
    err = np.abs(ref - rounded).max()
    print(f"(s + offset) rounded at {EPOCH:.3g} s: worst point error {err:.2e} m")
    assert 1e-6 < err < 1e-4
    # and the same stamps as exact Fractions: (s + o) - t_k as doubles is off by up to half a clock spacing
    F = [Fraction(s) + Fraction(EPOCH) - Fraction(times[0]) for s in ts]
    assert max(abs(float(f) - ((s + EPOCH) - times[0])) for f, s in zip(F, ts)) > 2.0 ** -24


def test_synthetic_clock_base(K):
    """a clock base shifts scan_start_time, motion_samples and a rig's clock offsets by exactly the base and nothing
    else: the scans, stamps, poses and rates are the base-0 stream's"""
    from kiss_icp_b200 import synthetic
    a = synthetic.small_shape(seed=5, beams=8, cols=128, stamps="sweep", hz=HZ, shake=(0.05, 2.0))
    b = synthetic.small_shape(seed=5, beams=8, cols=128, stamps="sweep", hz=HZ, shake=(0.05, 2.0), t0=EPOCH)
    for k in (0, 3):
        assert b.scan_start_time(k) == EPOCH + a.scan_start_time(k) and b.scan_start_time(k) - EPOCH == (k - 1) / HZ
        pa, pb = a.scan(k), b.scan(k)
        assert all(np.array_equal(x, y) for x, y in zip(pa, pb))
        for rate in (64.0, 1024.0):
            sa, sb = a.motion_samples(k, rate), b.motion_samples(k, rate)
            assert np.array_equal(sb[0] - EPOCH, sa[0]) and np.array_equal(sb[0], EPOCH + sa[0])
            assert np.array_equal(sa[0], (k - 1) / HZ + np.arange(len(sa[0])) / rate)  # the dyadic grid
            assert all(np.array_equal(x, y) for x, y in zip(sa[1:], sb[1:]))
    F, R = np.eye(4), np.eye(4)
    R[:3, 3] = [-2.0, 0.0, 0.5]
    ra = synthetic.RigLidar(a, [F, R], phases=[0.0, 0.25], stamps="sweep", clock_offsets=True)
    rb = synthetic.RigLidar(b, [F, R], phases=[0.0, 0.25], stamps="sweep", clock_offsets=True)
    rel = synthetic.RigLidar(b, [F, R], phases=[0.0, 0.25], stamps="sweep")
    fa, fb, fr = ra.scan(2), rb.scan(2), rel.scan(2)
    assert fb[2] == [EPOCH + o for o in fa[2]] == [b.scan_start_time(2) + o for o in fr[2]]
    assert fr[2] == [0.0, 0.25 / HZ]


def test_motion_from_gyro_clock_invariant(K):
    """motion_from_gyro takes differences of sample times only: the same poses bit for bit at both bases"""
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=6, beams=8, cols=128, stamps="sweep", hz=HZ, shake=(0.08, 2.0))
    times, _, rates, vel = L.motion_samples(3, 1024.0)
    a = K.motion_from_gyro(times, rates, vel[0], stamp_offset=L.scan_start_time(3))
    b = K.motion_from_gyro(EPOCH + times, rates, vel[0], stamp_offset=EPOCH + L.scan_start_time(3))
    assert np.array_equal(a.poses, b.poses) and np.array_equal(b.times - EPOCH, a.times)


# ---------------------------------------------------------------------------------------------- on the device
def _with_nan(rng, ts, every=97):
    ts = ts.copy()
    ts[rng.integers(0, every):: every] = np.nan
    return ts


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["absolute", "relative", "on_samples", "imu_1khz"])
def test_deskew_exact_at_epoch(K, case):
    """kb_deskew_motion at clock 1.76e9 against the exact reference within 1e-10 m: stamps before the first sample and
    after the last, NaN stamps and points up to 100 m in every case; absolute stamps with offset 0 (exact before), per
    scan relative stamps with the scan's start as stamp_offset, stamps on the sample times, 1 kHz IMU samples. Relative
    stamps also give the same bits at clock 0."""
    rng = np.random.default_rng(["absolute", "relative", "on_samples", "imu_1khz"].index(case) + 50)
    start, dt, m = 3.0, 1 / 64, 9
    if case == "imu_1khz":
        dt, m = 1 / 1024, 129
    n = 20000
    pts = _cloud(rng, n)
    rel = rng.uniform(-0.03, m * dt + 0.02, n)  # outside the samples at both ends
    if case == "on_samples":
        rel[: 4 * m] = np.tile(dt * np.arange(m), 4)
    rel = _with_nan(rng, rel)
    worst = 0.0
    got_at = {}
    for base in (EPOCH, 0.0):
        times, poses = _twist_motion(np.random.default_rng(11), base, start, dt, m)
        end = base + start + dt * (m - 3) + 1 / 512
        if case == "absolute":
            stamps, offset = (base + start) + rel, 0.0
        else:
            stamps, offset = rel, base + start
        M = K.Motion(times, poses, stamp_offset=offset, end_time=end)
        got = K.deskew(pts, stamps, M)
        got_at[base] = got
        ref = ExactMotion(times, poses, end)
        worst = max(worst, _check_exact(got, ref.deskew_np(pts, stamps, offset), ref, pts, stamps, [offset],
                                        np.random.default_rng(7)))
        nan = np.isnan(stamps)
        assert nan.any() and np.isnan(got[nan]).all()
    if case != "absolute":
        assert got_at[EPOCH].tobytes() == got_at[0.0].tobytes()
    print(f"deskew at clock {EPOCH:.3g} s ({case}): worst point error {worst:.2e} m")


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["f32", "f64", "dev"])
def test_pipeline_deskew_exact_at_epoch(K, layout):
    """the preprocessed cloud of a first frame with a Motion at clock 1.76e9, from float32, float64 and device frames:
    the exact reference within 1e-10 m (nothing is cropped: points within 60 m)"""
    import torch
    rng = np.random.default_rng(60)
    times, poses = _twist_motion(rng, EPOCH, 0.0, 1 / 64, 9)
    pts32 = _cloud(rng, 20000, 2.0, 60.0).astype(np.float32)
    pts = pts32.astype(np.float64)
    ts = _with_nan(rng, rng.uniform(-0.01, 0.135, len(pts)))
    M = K.Motion(times, poses, stamp_offset=EPOCH, end_time=EPOCH + 0.125)
    kiss = K.KissICP(K.load_config())
    if layout == "dev":
        d, dts = torch.tensor(pts, device="cuda"), torch.tensor(ts, device="cuda")
        kiss._register_frames_raw([d.data_ptr()], [len(pts)], [dts.data_ptr()], [len(ts)], 2,
                                  motions=[M._struct(M.end_time)])
        pre, _ = kiss._last_clouds()
    else:
        pre, _ = kiss.register_frame(pts32 if layout == "f32" else pts, ts, motion=M)
    ref = ExactMotion(times, poses, M.end_time)
    full = ref.deskew_np(pts, ts, EPOCH)
    keep = np.isfinite(full).all(1)
    assert pre.shape == (int(keep.sum()), 3)
    got = np.full_like(full, np.nan)
    got[keep] = pre
    _check_exact(got, full, ref, pts, ts, [EPOCH], np.random.default_rng(61))


def _rig_sensors(rng, S):
    """S sensors: the first at the base's origin without a crop, the others with random extrinsics (a few of them
    identities) and crops"""
    from test_rig import random_extrinsic
    out = [(np.eye(4), 0.0, math.inf)]
    for i in range(1, S):
        E = random_extrinsic(rng, identity=(i % 5 == 0))
        out.append((E, float(rng.uniform(0.5, 3.0)), float(rng.uniform(60.0, 95.0)) if i % 2 else math.inf))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 2, 16])
@pytest.mark.parametrize("clock", ["sensor", "motion"])
def test_merge_rig_exact_at_epoch(K, S, clock):
    """kb_merge_rig with a Motion at clock 1.76e9 against the exact reference within 1e-10 m, for both conventions:
    "sensor": each sensor's stamp offset is its sweep's start on the clock, the motion's stamp_offset 0; "motion": small
    per-sensor clock offsets, the scan's start as the motion's stamp_offset. The same bits at clock 0; the merged stamps
    are s + offset_i."""
    rng = np.random.default_rng(70 + S + (clock == "motion"))
    sensors = _rig_sensors(rng, S)
    rig = K.Rig([K.Sensor(*s) for s in sensors])
    start = 5.0
    phases = [j / 256 for j in range(S)]  # dyadic sweep starts after the scan's start
    scans = [_cloud(rng, int(rng.integers(500, 3000))) for _ in range(S)]
    rel = [_with_nan(rng, rng.uniform(-0.01, 0.13, len(p))) for p in scans]
    got_at = {}
    worst = 0.0
    for base in (EPOCH, 0.0):
        times, poses = _twist_motion(np.random.default_rng(12), base, start, 1 / 64, 9)
        end = base + start + 0.125
        if clock == "sensor":
            offs, mo = [base + start + ph for ph in phases], 0.0
        else:
            offs, mo = list(phases), base + start
        M = K.Motion(times, poses, stamp_offset=mo, end_time=end)
        got, got_ts = K.merge_rig(scans, rig, rel, offs, M)
        got_at[base] = got
        assert np.array_equal(got_ts, np.concatenate([t + o for t, o in zip(rel, offs)]), equal_nan=True)
        ref = ExactMotion(times, poses, end)
        b = 0
        for (E, lo, hi), p, t, o in zip(sensors, scans, rel, offs):
            g = got[b: b + len(p)]
            b += len(p)
            full = ref.deskew_np(p, t, o, mo, E=E)
            if not (lo == 0.0 and hi == math.inf):
                r = np.sqrt((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2])
                full[~((r > lo) & (r < hi))] = np.nan
            worst = max(worst, _check_exact(g, full, ref, p, t, [o, mo], np.random.default_rng(13), E=E,
                                            sample=max(SAMPLE // S, 40)))
    assert got_at[EPOCH].tobytes() == got_at[0.0].tobytes()
    print(f"rig merge at clock {EPOCH:.3g} s ({S} sensors, {clock} clock): worst point error {worst:.2e} m")


# ---------------------------------------------------------------------------------------------- whole runs
N_FRAMES = 8


@pytest.fixture(scope="module")
def sweep():
    """a shaking sweep stream at 8 Hz (frames, stamps jittered off the dyadic grid so that s + clock would round)"""
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=4, beams=32, cols=512, stamps="sweep", hz=HZ, shake=(0.05, 2.0))
    rng = np.random.default_rng(80)
    frames = []
    for k in range(N_FRAMES):
        p, t = L.scan(k)
        frames.append((p, t + rng.uniform(-0.3, 0.3, len(t)) / (512 * HZ)))
    return L, frames


def _clock(L, base):
    """L's trajectory on a clock with base `base` (its scan_start_time and motion_samples; scans are never cast)"""
    from kiss_icp_b200 import synthetic
    return synthetic.small_shape(seed=L.seed, beams=8, cols=8, stamps="sweep", hz=HZ, shake=L.shake, t0=base)


def _motions(K, L, base, source):
    """per frame a Motion on the clock with base `base`: the true poses at 64 Hz ("wheel": translation scaled by 1 %,
    as wheel odometry) or motion_from_gyro of the true rates at 1 kHz ("gyro"), end_time the sweep's end"""
    C = _clock(L, base)
    out = []
    for k in range(N_FRAMES):
        end = C.scan_start_time(k) + 1 / HZ
        if source == "gyro":
            times, _, rates, vel = C.motion_samples(k, 1024.0)
            out.append(K.motion_from_gyro(times, rates, vel[0], stamp_offset=C.scan_start_time(k), end_time=end))
        else:
            times, poses, _, _ = C.motion_samples(k, 64.0)
            poses = poses.copy()
            poses[:, :3, 3] *= 1.01
            out.append(K.Motion(times, poses, stamp_offset=C.scan_start_time(k), end_time=end))
    return out


def _state(kiss):
    vox, cnt, pts = kiss.local_map.dump()
    return kiss.last_pose, kiss.last_delta, vox, cnt, pts


def _same_state(a, b):
    return all(np.array_equal(x, y) for x, y in zip(_state(a), _state(b)))


def _run(K, frames, motions, layout, queued):
    """-> (poses, iterations or None, the pipeline)"""
    import torch
    kiss = K.KissICP(K.load_config())
    pts = [f[0].astype(np.float32) if layout == "f32" else f[0] for f in frames]
    ts = [f[1] for f in frames]
    if layout == "dev":
        d = [torch.tensor(p, device="cuda") for p in pts]
        dt = [torch.tensor(t, device="cuda") for t in ts]
        P = kiss._register_frames_raw([x.data_ptr() for x in d], [len(p) for p in pts], [x.data_ptr() for x in dt],
                                      [len(t) for t in ts], 2, motions=[m._struct(m.end_time) for m in motions])
        return P, None, kiss
    if queued:
        return kiss.register_frames(pts, ts, motions=motions), None, kiss
    P, its = [], []
    for p, t, m in zip(pts, ts, motions):
        kiss.register_frame(p, t, return_clouds=False, motion=m)
        P.append(kiss.last_pose)
        its.append(kiss.last_iterations)
    return np.array(P), its, kiss


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["f64", "f32", "dev"])
@pytest.mark.parametrize("source", ["gyro", "wheel"])
def test_odometry_clock_invariant(K, sweep, source, layout):
    """a whole odometry run with Motions at clock 1.76e9 is the run at clock 0 bit for bit: poses, iteration counts,
    last_delta and the local map; queued and blocking alike"""
    L, frames = sweep
    runs = {}
    for base in (0.0, EPOCH):
        ms = _motions(K, L, base, source)
        runs[base, "q"] = _run(K, frames, ms, layout, True)
        if layout != "dev":
            runs[base, "b"] = _run(K, frames, ms, layout, False)
    ref = runs[0.0, "q"]
    for key, (P, its, kiss) in runs.items():
        assert np.array_equal(P, ref[0]) and _same_state(kiss, ref[2]), key
    if layout != "dev":
        assert runs[EPOCH, "b"][1] == runs[0.0, "b"][1]
        assert runs[EPOCH, "q"][2].motion_end_time == EPOCH + runs[0.0, "q"][2].motion_end_time


@pytest.mark.gpu
def test_veto_and_replay_clock_invariant(K, monkeypatch):
    """queued against blocking at clock 1.76e9 with frames vetoed and replayed (the minimal voxel table): the blocking
    and the queued runs at both clocks are one run bit for bit"""
    monkeypatch.setenv("KB_MAP_RESERVE_SLOTS", "0")
    rng = np.random.default_rng(8)
    xi = np.array([12.0, 1.0, 0.0, 0.0, 0.0, 1.5])
    frames, rel = [], []
    for k in range(9):
        n = 30000 if k in (0, 4, 5) else 3000
        frames.append((rng.uniform(-150, 150, size=(n, 3)) * [1.0, 1.0, 0.2], rng.uniform(0.0, 0.125, n)))
        rel.append((k - 1) / HZ + np.array([0.0, 1 / 16, 1 / 8]))
    cfg = K.load_config(max_range=300.0, voxel_size=1.0)
    out = []
    for base in (0.0, EPOCH):
        ms = [K.Motion(base + r, _exp_np(r[:, None] * xi), stamp_offset=base + r[0], end_time=base + r[-1])
              for r in rel]
        a = K.KissICP(cfg)
        P_q = a.register_frames([f[0] for f in frames], [f[1] for f in frames], motions=ms)
        assert a.grow_retries() >= 2
        b = K.KissICP(cfg)
        P_b = []
        for (p, t), m in zip(frames, ms):
            b.register_frame(p, t, return_clouds=False, motion=m)
            P_b.append(b.last_pose)
        assert np.array_equal(P_q, np.array(P_b)) and _same_state(a, b)
        out.append((P_q, a))
    assert np.array_equal(out[0][0], out[1][0]) and _same_state(out[0][1], out[1][1])


@pytest.mark.gpu
@pytest.mark.parametrize("clock", ["sensor", "motion"])
def test_rig_run_clock_invariant(K, clock):
    """a two-sensor rig run with Motions at clock 1.76e9 (sensor offsets on the clock, or the scan's start as the
    motion's stamp_offset) is the run at clock 0 bit for bit, queued and blocking"""
    from kiss_icp_b200 import synthetic
    from test_rig import _front_rear
    F, R = _front_rear()
    sensors = [(F, 4.0, math.inf), (R, 4.0, 90.0)]
    rig = K.Rig([K.Sensor(*s) for s in sensors])
    rng = np.random.default_rng(81)
    runs = []
    for base in (0.0, EPOCH):
        L = synthetic.small_shape(seed=4, beams=16, cols=256, hz=HZ, t0=base)
        RL = synthetic.RigLidar(L, [F, R], shapes=[None, (16, 128, (-20.0, 10.0))], phases=[0.0, 0.25],
                                stamps="sweep", clock_offsets=(clock == "sensor"))
        if base == 0.0:
            raw = [RL.scan(k) for k in range(6)]
            jit = [[t + rng.uniform(-0.3, 0.3, len(t)) / (256 * HZ) for t in f[1]] for f in raw]
        offs = [[L.scan_start_time(k) + ph / HZ for ph in RL.phases] if clock == "sensor" else [ph / HZ for ph in
                                                                                                 RL.phases]
                for k in range(6)]
        ms = []
        for k in range(6):
            times, poses, _, _ = L.motion_samples(k, 64.0)
            ms.append(K.Motion(times, poses, stamp_offset=0.0 if clock == "sensor" else L.scan_start_time(k),
                               end_time=L.scan_start_time(k) + 1 / HZ))
        a = K.KissICP(K.load_config())
        P = a.register_rig_frames([f[0] for f in raw], rig, jit, offs, motions=ms)
        b = K.KissICP(K.load_config())
        for f, t, o, m in zip(raw, jit, offs, ms):
            b.register_rig_frame(f[0], rig, t, o, motion=m, return_clouds=False)
        assert np.array_equal(P[-1], b.last_pose) and _same_state(a, b)
        runs.append((P, a))
    assert np.array_equal(runs[0][0], runs[1][0]) and _same_state(runs[0][1], runs[1][1])


@pytest.mark.gpu
def test_checkpoint_and_localizer_clock_invariant(K, sweep):
    """a checkpoint taken mid-run at clock 1.76e9 (motion_end_time on the clock) restores and continues as the run at
    clock 0; a localizer in that run's map tracks the stream with Motions identically at both clocks"""
    L, frames = sweep
    pts, ts = [f[0] for f in frames], [f[1] for f in frames]
    full = {}
    for base in (0.0, EPOCH):
        ms = _motions(K, L, base, "wheel")
        a = K.KissICP(K.load_config())
        a.register_frames(pts[:4], ts[:4], motions=ms[:4])
        state = a.state_dict()
        assert float(state["motion_end_time"]) == ms[3].end_time
        b = K.KissICP(K.load_config())
        b.load_state_dict(state)
        full[base] = (b.register_frames(pts[4:], ts[4:], motions=ms[4:]), b)
    assert np.array_equal(full[0.0][0], full[EPOCH][0]) and _same_state(full[0.0][1], full[EPOCH][1])
    cfg = K.load_config()
    odo = full[0.0][1]
    loc_runs = []
    for base in (0.0, EPOCH):
        prior = K.VoxelHashMap(cfg.mapping.voxel_size, 1e4, cfg.mapping.max_points_per_voxel)
        prior.load(*odo.local_map.dump())
        loc = K.KissICP(cfg, prior_map=prior)
        ms = _motions(K, L, base, "wheel")
        loc_runs.append(loc.register_frames(pts[1:], ts[1:], motions=ms[1:]))
    assert np.array_equal(loc_runs[0], loc_runs[1])


@pytest.mark.gpu
def test_default_end_time_at_epoch(K, sweep):
    """with end_time None the deskew target is max(stamps) + stamp_offset, rounded by the caller's double at the
    clock's magnitude: it moves by less than one clock spacing (2.4e-7 s), so the run at clock 1.76e9 matches the run
    at clock 0 to a pose tolerance, not bit for bit"""
    from conftest import pose_error
    L, frames = sweep
    P = []
    for base in (0.0, EPOCH):
        ms = [K.Motion(m.times, m.poses, stamp_offset=m.stamp_offset) for m in _motions(K, L, base, "wheel")]
        P.append(K.KissICP(K.load_config()).register_frames([f[0] for f in frames], [f[1] for f in frames],
                                                             motions=ms))
    worst = max(max(pose_error(a, b)) for a, b in zip(*P))
    print(f"default end_time at clock {EPOCH:.3g} s: worst pose difference {worst:.2e}")
    assert worst < 1e-6


@pytest.mark.gpu
def test_constant_velocity_rig_at_epoch_offsets(K):
    """without a Motion a rig's merged stamps are the doubles s + offset_i, which KISS-ICP normalises by the sweep's
    span as the reference does: at epoch offsets the rig run is register_frames of the host-concatenated cloud and
    stamps bit for bit"""
    from kiss_icp_b200 import synthetic
    from test_rig import _front_rear
    F, R = _front_rear()
    rig = K.Rig([K.Sensor(F, 4.0, math.inf), K.Sensor(R, 4.0, 90.0)])
    L = synthetic.small_shape(seed=4, beams=16, cols=256, hz=HZ, t0=EPOCH)
    RL = synthetic.RigLidar(L, [F, R], shapes=[None, (16, 128, (-20.0, 10.0))], phases=[0.0, 0.25], stamps="sweep",
                            clock_offsets=True)
    frames = [RL.scan(k) for k in range(6)]
    assert all(min(f[2]) > 1e9 for f in frames)
    a = K.KissICP(K.load_config())
    Pa = a.register_rig_frames([f[0] for f in frames], rig, [f[1] for f in frames], [f[2] for f in frames])
    stamps = [np.concatenate([t + o for t, o in zip(ts, offs)]) for _, ts, offs in frames]  # on the host
    merged = [K.merge_rig(f[0], rig, f[1], f[2]) for f in frames]
    assert all(np.array_equal(T, m[1]) for T, m in zip(stamps, merged))
    b = K.KissICP(K.load_config())
    Pb = b.register_frames([m[0] for m in merged], stamps)
    assert np.array_equal(Pa, Pb) and _same_state(a, b)
