"""Registration on degenerate and malformed scans, against the reference (the oracle) and a high-precision solve:
- the structured ICP solve (icp_solve_schur) declines systems whose 3x3 Schur complement is rounding noise (one
  correspondence, coincident points, two points, points on one line) and keeps solving resolved near-degenerate ones;
- deskew takes the min and max stamp exactly as std::minmax_element does, NaN included;
- the direct entry points refuse non-finite points and points beyond int voxel coordinates before any device work,
  while the pipeline keeps accepting them and crops them as the reference does."""
import math

import numpy as np
import pytest

from conftest import canon_map, pose_error
from test_device_probes import accumulate, expand, mp_solve, schur_host, solve_dev

gpu = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
OFFSETS = (1.0, 10.0, 100.0, 1000.0)


# ------------------------------------------------------------------ ICP systems
def _unit(rng):
    d = rng.normal(size=3)
    return d / np.linalg.norm(d)


def _system(S, rng):
    n = len(S)
    return accumulate(S, rng.normal(size=(n, 3)) * 0.1, rng.random(n) + 0.01)


def degenerate_systems(offset, seed=0, count=40):
    """(family, accumulators) whose Schur complement is singular in exact arithmetic, about `offset` metres out"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        c = _unit(rng) * offset
        e = _unit(rng)
        out.append(("one correspondence", _system(c[None], rng)))
        out.append(("two points", _system(c + rng.normal(size=(2, 3)) * rng.choice([0.01, 0.5, 3.0]), rng)))
        k = int(rng.integers(3, 40))
        out.append(("pole", _system(c + np.outer(rng.uniform(-1, 1, size=k), e) * rng.choice([0.1, 1.0, 3.0]), rng)))
        # one voxel's points as the voxelization leaves them: coincident
        out.append(("one voxel", _system(np.repeat(np.floor(c)[None] + rng.random(3), int(rng.integers(2, 30)), 0), rng)))
    scale = 2.0 ** round(math.log2(max(offset / 20.0, 1.0)))  # a power of two keeps the cancellation exact
    out.append(("line through the origin", accumulate(np.outer(np.arange(1, 8.0), [1.0, 2.0, 3.0]) * scale,
                                                      rng.normal(size=(7, 3)), np.ones(7))))
    return out


def resolved_systems(offset, seed=1, count=20):
    """(family, accumulators) that are near-degenerate but resolved far above rounding"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        c = _unit(rng) * offset
        e = _unit(rng)
        k = int(rng.integers(3, 40))
        pole = c + np.outer(rng.uniform(-1, 1, size=k), e) * 2.0 + rng.normal(size=(k, 3)) * 0.02
        out.append(("pole with 2 cm lateral noise", _system(pole, rng)))
        out.append(("three points", _system(c + rng.normal(size=(3, 3)) * rng.choice([0.3, 1.0, 5.0]), rng)))
        n = int(rng.integers(6, 300))
        out.append(("random", _system(rng.normal(size=(n, 3)) * 30.0 + c, rng)))
    return out


@pytest.mark.parametrize("offset", OFFSETS)
def test_schur_solve_declines_systems_it_cannot_resolve(offset):
    """the host build of icp_solve_schur: every degenerate family is declined (the loop then takes the LDL^T with
    Eigen's zero-pivot rule, as the reference solves every system)"""
    accepted = [(fam, i) for i, (fam, acc) in enumerate(degenerate_systems(offset)) if schur_host(acc)[2]]
    assert not accepted, accepted


@pytest.mark.parametrize("offset", OFFSETS)
def test_schur_solve_keeps_resolved_near_degenerate_systems(offset):
    """resolved systems stay on the structured solve and match a 50-digit solve within the condition bound of
    test_device_probes (64 cond(JTJ) eps)"""
    for fam, acc in resolved_systems(offset):
        xs, _, used = schur_host(acc)
        assert used == 1, fam
        x = mp_solve(acc)
        cond = np.linalg.cond(expand(acc)[0])
        assert np.linalg.norm(xs - x) <= 64 * cond * EPS * np.linalg.norm(x), (fam, cond)


# ------------------------------------------------------------------ std::minmax_element, restated
def minmax_element(t):
    """libstdc++'s std::minmax_element (bits/stl_algo.h, __minmax_element) on doubles with operator<: the values at
    the returned (min, max) iterators"""
    n = len(t)
    if n < 2:
        return t[0], t[0]
    lo, hi = (t[1], t[0]) if t[1] < t[0] else (t[0], t[1])
    i = 2
    while i < n:
        if i + 1 == n:
            if t[i] < lo:
                lo = t[i]
            elif not (t[i] < hi):
                hi = t[i]
            break
        a, b = t[i], t[i + 1]
        if b < a:
            if b < lo:
                lo = b
            if not (a < hi):
                hi = a
        else:
            if a < lo:
                lo = a
            if not (b < hi):
                hi = b
        i += 2
    return lo, hi


def stamp_cases(seed=3):
    """stamp vectors for an 8-point frame (and longer ones): NaN in every role, +-inf, constant, reversed, epoch
    seconds and nanoseconds"""
    rng = np.random.default_rng(seed)
    nan, inf = math.nan, math.inf
    base = np.linspace(0.0, 0.1, 8)
    cases = {
        "plain": base, "reversed": base[::-1].copy(), "constant": np.full(8, 0.25),
        "nan first": np.r_[nan, base[1:]], "nan middle": np.r_[base[:4], nan, base[5:]], "nan last": np.r_[base[:7], nan],
        "nan in the max role": np.r_[base[:2], nan, 0.01, base[4:]],  # (nan, 0.01): 0.01 is offered to the max only
        "nan paired with the min": np.r_[0.05, 0.06, nan, -1.0, base[4:]],
        "nan then larger": np.r_[base[:2], 0.2, nan, 0.3, 0.9, base[6:]],
        "all nan": np.full(8, nan), "+inf": np.r_[base[:3], inf, base[4:]], "-inf": np.r_[base[:5], -inf, base[6:]],
        "+-inf": np.r_[-inf, base[1:7], inf],
        "epoch seconds": 1.7e9 + base, "nanoseconds": 1.7e18 + np.arange(8) * 1.0e8,
        "more stamps than points": np.r_[base, 0.5, -0.5, nan],
    }
    for k in range(40):
        t = rng.random(int(rng.integers(8, 14)))
        for i in rng.choice(len(t), size=int(rng.integers(1, 4)), replace=False):
            t[i] = rng.choice([nan, inf, -inf, t[i]])
        cases[f"random {k}"] = t
    return cases


def _probe_frame():
    """8 points on the y axis; a pure translation along x deskews point i by (stamp_i - 1) metres along x"""
    return np.c_[np.zeros(8), np.linspace(5.0, 12.0, 8), np.zeros(8)]


def _translation_x():
    T = np.eye(4)
    T[0, 3] = 1.0
    return T


def test_minmax_element_restatement_matches_the_oracle(O):
    """the oracle's preprocess takes std::minmax_element of the stamps; with a pure translation as motion its
    output states the normalized stamps, which the restatement above must reproduce"""
    P, T = _probe_frame(), _translation_x()
    for name, t in stamp_cases().items():
        got = O.preprocess(P, t, T, 100.0, 0.0, True)
        lo, hi = minmax_element(t)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            s = (t[:8] - lo) / (hi - lo)
            want = P + np.outer(s - 1.0, [1.0, 0.0, 0.0])
        r = np.sqrt((want ** 2).sum(1))
        want = want[(r < 100.0) & (r > 0.0)]
        assert got.shape == want.shape, (name, got, want)
        assert np.allclose(got, want, rtol=0.0, atol=1e-12), (name, got, want)


def test_minmax_element_differs_from_a_nan_ignoring_min_and_max():
    """the cases above are not covered by a NaN-ignoring reduction or by 'NaN if the first stamp is NaN'"""
    t = np.array([0.05, 0.06, math.nan, -1.0, 0.3, 0.4])
    assert minmax_element(t) == (0.05, 0.4)  # -1.0 sits beside a NaN and is only offered as a max
    t = np.array([0.0, 0.1, 0.2, math.nan, 0.05])
    assert minmax_element(t) == (0.0, 0.05)  # the NaN took the max, then 0.05 replaced it
    assert math.isnan(minmax_element(np.array([math.nan, 0.0, 1.0]))[0])


# ------------------------------------------------------------------ argument rules of the direct entry points
def bad_point_sets():
    good = np.array([[1.0, 2.0, 3.0], [4.0, -5.0, 0.5], [0.2, 0.3, 0.4]])
    out = []
    for name, v in (("nan", math.nan), ("+inf", math.inf), ("-inf", -math.inf), ("beyond int voxels", 3e9)):
        p = good.copy()
        p[1, 2] = v
        out.append((name, p))
    return out


def test_voxel_down_sample_validates_before_device_work(K):
    """ValueError for a non-finite point, a point beyond int voxel coordinates or a bad voxel size, on a machine
    with or without a device"""
    for name, p in bad_point_sets():
        with pytest.raises(ValueError):
            K.voxel_down_sample(p, 1.0)
    for v in (0.0, -1.0, math.nan, math.inf):
        with pytest.raises(ValueError):
            K.voxel_down_sample(np.ones((3, 3)), v)


@gpu
def test_direct_entry_points_refuse_bad_points_and_write_nothing(K, O):
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=1, beams=32, cols=512)
    g = K.VoxelHashMap(1.0, 100.0, 20)
    for k in range(3):
        g.update(O.voxel_down_sample(L.scan(k)[0], 0.5), L.pose(k))
    before = g.dump()
    reg = K.Registration(500, 1e-4, 0)
    T = np.eye(4)
    T[:3, 3] = [1.0, -2.0, 0.5]
    for name, p in bad_point_sets():
        for call in (lambda: g.add_points(p), lambda: g.update(p, T), lambda: g.update(p, np.array([1.0, 2.0, 0.0])),
                     lambda: g.closest_neighbors(p), lambda: reg.align_points_to_map(p, g, T, 3.0, 1.0),
                     lambda: reg.build_system(p, g, 3.0, 1.0)):
            with pytest.raises(ValueError):
                call()
        for x, y in zip(before, g.dump()):
            assert np.array_equal(x, y), name
    with pytest.raises(ValueError):  # a finite point that the pose carries beyond int voxel coordinates
        Tf = np.eye(4)
        Tf[0, 3] = 3e9
        g.update(np.ones((2, 3)), Tf)
    with pytest.raises(ValueError):
        g.update(np.ones((2, 3)), np.array([math.nan, 0.0, 0.0]))
    for x, y in zip(before, g.dump()):
        assert np.array_equal(x, y)


# ------------------------------------------------------------------ device solve
@gpu
@pytest.mark.parametrize("offset", OFFSETS)
def test_device_solve_takes_the_host_decision_and_the_oracle_ldlt(O, offset):
    """the device declines exactly what the host declines. Where the singular directions cancel exactly (a line
    through the origin) its LDL^T is the oracle's within rounding; where they are left as rounding noise, the pivots
    of both LDL^Ts are noise and their steps agree only in being finite (the null-space part is arbitrary, also for
    the reference: the pipeline tests compare the registered points instead)"""
    fams = degenerate_systems(offset, count=15) + resolved_systems(offset, count=8)
    accs = np.array([a for _, a in fams])
    dx, used, est, _ = solve_dev(accs, 1e-4)
    for i, (fam, acc) in enumerate(fams):
        assert used[i] == schur_host(acc)[2], (fam, i)
        assert np.all(np.isfinite(dx[i])) and np.all(np.isfinite(est[i])), fam
        if fam == "line through the origin":
            J, r = expand(acc)
            xo = O.ldlt6_solve(J, -r)
            assert np.allclose(dx[i], xo, rtol=1e-11, atol=1e-13 * max(1.0, np.abs(xo).max())), (fam, dx[i], xo)


# ------------------------------------------------------------------ pipelines on degenerate frames
def _normal_run(K, O, fused=True, n=8):
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=5, beams=32, cols=512)
    g, o = K.KissICP(K.load_config(), fused=fused), O.KissICP()
    scans = [L.scan(k) for k in range(n + 1)]
    for p, t in scans[:n]:
        g.register_frame(p, t, return_clouds=False)
        o.register_frame(p, t, want_clouds=False)
    return g, o, scans[n][0]


def degenerate_frames(next_scan):
    """frames whose source after voxelization is one point, near the map's surfaces. (A few points on one pole are
    not compared: the pivots of the rotation about the pole are rounding noise in both LDL^Ts, and the registered
    points of the device and of the reference then differ by up to 0.2 m.)"""
    r = np.linalg.norm(next_scan, axis=1)
    p = next_scan[np.argmin(np.abs(r - 12.0))]
    voxel = p + np.random.default_rng(4).random((25, 3)) * 0.2
    return {"one point": p[None].copy(), "one voxel": voxel}


def _check_frame(name, Pg, Po, src_g, src_o):
    """rotations about a single point leave its residual unchanged: that part of the pose is set by
    rounding noise in the reference too, so the registered source points are compared, at the pose bar"""
    assert src_g.shape == src_o.shape, name
    a = src_g @ Pg[:3, :3].T + Pg[:3, 3]
    b = src_o @ Po[:3, :3].T + Po[:3, 3]
    assert np.abs(a - b).max() < 1e-4, (name, a, b)


@gpu
@pytest.mark.parametrize("mode", ["blocking", "queued", "modular"])
def test_pipeline_registers_degenerate_frames_as_the_reference(K, O, mode):
    for name in ("one point", "one voxel"):
        g, o, nxt = _normal_run(K, O, fused=(mode != "modular"))
        f = degenerate_frames(nxt)[name]
        _, src_o = o.register_frame(f, np.empty(0))
        if mode == "queued":
            Pg = g.register_frames([f], [np.empty(0)])[0]
            src_g = src_o  # the queue returns no clouds; the blocking modes check the source itself
            assert np.array_equal(g.last_pose, Pg)
        else:
            _, src_g = g.register_frame(f, np.empty(0))
            Pg = g.last_pose
        _check_frame(name, Pg, o.pose, src_g, src_o)


@gpu
def test_localizer_registers_degenerate_frames_as_the_reference(K, O):
    from kiss_icp_b200 import synthetic
    from test_localizer import _oracle_localize, _prior
    L = synthetic.small_shape(seed=2, beams=32, cols=512)
    cfg = K.load_config()
    prior, oprior = _prior(K, O, L, range(0, 12), 1.0)
    for name, f in degenerate_frames(L.scan(5)[0]).items():
        icp = K.KissICP(cfg, prior_map=prior)
        icp.last_pose = L.pose(0)
        scans = [L.scan(k) for k in range(5)]
        for p, t in scans:
            icp.register_frame(p, t, return_clouds=False)
        _, src_g = icp.register_frame(f, np.empty(0))
        poses, _, _ = _oracle_localize(O, oprior, cfg, scans + [(f, np.empty(0))], L.pose(0))
        src_o = O.voxel_down_sample(O.voxel_down_sample(f, 0.5), 1.5)
        _check_frame(name, icp.last_pose, poses[-1], src_g, src_o)


# ------------------------------------------------------------------ stamps
@gpu
def test_preprocessor_takes_the_reference_min_and_max_stamp(K, O):
    rng = np.random.default_rng(6)
    T = O.se3_exp([0.8, 0.05, -0.02, 0.004, -0.003, 0.03])
    for name, t in stamp_cases().items():
        n = min(len(t), 8) if name == "more stamps than points" else len(t)
        pts = rng.normal(size=(n, 3)) * 20.0
        for deskew in (True, False):
            a = K.Preprocessor(100.0, 0.5, deskew, 0).preprocess(pts, t, T)
            b = O.preprocess(pts, t, T, 100.0, 0.5, deskew)
            assert a.shape == b.shape, (name, deskew, a.shape, b.shape)
            if deskew:
                assert np.abs(a - b).max(initial=0.0) < 1e-11, name
            else:
                assert np.array_equal(a, b), name
    # a frame of realistic size: one NaN stamp among 70000, in each role
    pts = rng.normal(size=(70000, 3)) * 30.0
    for where in (0, 1, 2, 35001, 69998, 69999):
        t = np.sort(rng.random(70000))
        t[where] = math.nan
        a = K.Preprocessor(100.0, 0.5, True, 0).preprocess(pts, t, T)
        b = O.preprocess(pts, t, T, 100.0, 0.5, True)
        assert a.shape == b.shape and np.abs(a - b).max(initial=0.0) < 1e-11, where


def _stamp_stream(L, n):
    """frames of a stamped stream whose stamps are replaced, frame by frame, by a malformed variant"""
    nan = math.nan
    out = []
    for k in range(n):
        p, t = L.scan(k)
        t = t.copy()
        v = k % 8
        if v == 1:
            t[0] = nan
        elif v == 2:
            t[len(t) // 2] = nan
        elif v == 3:
            t[-1] = nan
        elif v == 4:
            t[2] = nan  # pairs (t2, t3): t3 is offered to the max only
        elif v == 5:
            t[:] = 0.5
        elif v == 6:
            t = 1.7e9 + t
        elif v == 7:
            t = np.r_[t, 0.3, nan]  # more stamps than points
        out.append((p, t))
    return out


@gpu
@pytest.mark.parametrize("mode", ["blocking", "queued", "modular"])
def test_pipeline_with_malformed_stamps_follows_the_reference(K, O, mode):
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=5, beams=32, cols=512, stamps="column")
    frames = _stamp_stream(L, 16)
    g, o = K.KissICP(K.load_config(), fused=(mode != "modular")), O.KissICP()
    ref = []
    for p, t in frames:
        o.register_frame(p, t, want_clouds=False)
        ref.append(o.pose)
    if mode == "queued":
        got = g.register_frames([p for p, _ in frames], [t for _, t in frames])
    else:
        got = []
        for p, t in frames:
            g.register_frame(p, t, return_clouds=False)
            got.append(g.last_pose)
    for k, (P, Po) in enumerate(zip(got, ref)):
        dt, dr = pose_error(P, Po)
        assert dt < 1e-4 and dr < 1e-4, (k, dt, dr)
        assert dt < 1e-6 and dr < 1e-6, (k, dt, dr)


# ------------------------------------------------------------------ coordinates the pipeline must crop
def malformed_cloud(p, rng, max_range=100.0, min_range=2.0):
    """an organized cloud with ~30 % no-return rows (NaN), +-inf, (0,0,0) returns, magnitudes that overflow (1e155)
    and underflow (1e-160) the squared norm, and points exactly at max_range and min_range"""
    p = p.copy()
    n = len(p)
    idx = rng.permutation(n)
    k = n // 10
    p[idx[:3 * k]] = math.nan
    p[idx[3 * k:3 * k + 20], rng.integers(0, 3, size=20)] = math.inf
    p[idx[3 * k + 20:3 * k + 40], rng.integers(0, 3, size=20)] = -math.inf
    p[idx[3 * k + 40:3 * k + 60]] = 0.0
    p[idx[3 * k + 60:3 * k + 70]] = rng.normal(size=(10, 3)) * 1e155
    p[idx[3 * k + 70:3 * k + 80]] = rng.normal(size=(10, 3)) * 1e-160
    p[idx[3 * k + 80]] = [0.6 * max_range, 0.8 * max_range, 0.0]
    p[idx[3 * k + 81]] = [0.0, 0.0, -max_range]
    p[idx[3 * k + 82]] = [min_range, 0.0, 0.0]
    p[idx[3 * k + 83]] = [0.0, -0.6 * min_range, 0.8 * min_range]
    return p


def _assert_maps_equal(g, o):
    """the same voxels and counts; points within the map bar of the pipeline streams (poses agree to ~1e-15)"""
    gv, gc, gp = g.dump()
    ov, oc, op = canon_map(*o.dump())
    assert np.array_equal(gv, ov) and np.array_equal(gc, oc) and np.allclose(gp, op, atol=1e-9)


@gpu
def test_preprocessor_crops_malformed_coordinates_as_the_reference(K, O):
    from kiss_icp_b200 import synthetic
    rng = np.random.default_rng(7)
    L = synthetic.small_shape(seed=5, beams=32, cols=512)
    p = malformed_cloud(L.scan(0)[0], rng)
    a = K.Preprocessor(100.0, 2.0, False, 0).preprocess(p, np.empty(0), np.eye(4))
    b = O.preprocess(p, np.empty(0), np.eye(4), 100.0, 2.0, False)
    assert np.array_equal(a, b) and np.all(np.isfinite(a))


@gpu
@pytest.mark.parametrize("mode", ["blocking", "queued", "queued f32", "modular"])
def test_pipeline_crops_malformed_coordinates_as_the_reference(K, O, mode):
    from kiss_icp_b200 import synthetic
    rng = np.random.default_rng(8)
    L = synthetic.small_shape(seed=5, beams=32, cols=512)
    frames = [malformed_cloud(L.scan(k)[0], rng) for k in range(12)]
    frames[5] = np.full((500, 3), math.nan)  # crops to empty mid-sequence; the next frames recover
    frames[6] = np.r_[np.full((100, 3), math.inf), np.zeros((10, 3))]
    if mode == "queued f32":
        frames = [f.astype(np.float32) for f in frames]
    g, o = K.KissICP(K.load_config(data__min_range=2.0), fused=(mode != "modular")), O.KissICP(min_range=2.0)
    got, ref = [], []
    for k, f in enumerate(frames):
        pre_o, _ = o.register_frame(f.astype(np.float64), np.empty(0))
        ref.append(o.pose)
        if not mode.startswith("queued"):
            pre_g, _ = g.register_frame(f, np.empty(0))
            assert np.array_equal(pre_g, pre_o), k
            got.append(g.last_pose)
    if mode.startswith("queued"):
        got = g.register_frames(frames)
    for k, (P, Po) in enumerate(zip(got, ref)):
        dt, dr = pose_error(P, Po)
        assert dt < 1e-4 and dr < 1e-4, (k, dt, dr)
        assert dt < 1e-6 and dr < 1e-6, (k, dt, dr)
    _assert_maps_equal(g.local_map, o.local_map)
