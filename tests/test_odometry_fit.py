"""KissICP(config, report_fit=True) / kb_pipeline_set_fit_reporting: an odometry pipeline that also reports, per scan,
the fit against its own map as that scan's ICP saw it (before the scan's local_map.update). Reporting only reads:
poses, iterations, threshold state and map are bit for bit those of reporting off."""
import ctypes as C
import math

import numpy as np
import pytest


def _fit_arrays(fits):
    return (np.array([f.n_correspondences for f in fits]), np.array([f.n_source for f in fits]),
            np.array([f.rmse for f in fits]), np.array([f.information for f in fits]))


def _same_fits(a, b):
    return all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


def _close(A, B, tol=1e-9):
    return np.linalg.norm(A[:3, 3] - B[:3, 3]) < tol and np.abs(A[:3, :3] - B[:3, :3]).max() < tol


def _same_map(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a.dump(), b.dump()))


def _blocking(icp, scans, fits=True):
    """per scan: pose, iterations, sigma (and the fit)"""
    out = {"poses": [], "iters": [], "sigma": [], "fits": []}
    for p, t in scans:
        icp.register_frame(p, t, return_clouds=False)
        out["poses"].append(icp.last_pose)
        out["iters"].append(icp.last_iterations)
        out["sigma"].append(icp.last_sigma)
        if fits:
            out["fits"].append(icp.last_fit)
    return out


def _queued(icp, scans, fits=True):
    icp.start_history(len(scans))
    r = icp.register_frames([p for p, _ in scans], [t for _, t in scans], return_fits=fits)
    poses, f = r if fits else (r, None)
    return poses, np.array([h.iterations for h in icp.history()]), f


def _stream(stamps, seed=3):
    from kiss_icp_b200 import synthetic
    return synthetic.small_shape(seed=seed, beams=32, cols=512, stamps=stamps)


def _check_fit_against_copy(K, icp, before, reg, src, first):
    """the pipeline's fit of the frame just registered equals build_system + closest_neighbors on `before`, a copy of
    its map taken before the frame"""
    f, P, sigma = icp.last_fit, icp.last_pose, icp.last_sigma
    assert f.n_source == len(src) > 0
    if first:  # an empty map
        assert f.n_correspondences == 0 and math.isnan(f.rmse) and not f.information.any()
        return
    mapped = src @ P[:3, :3].T + P[:3, 3]
    JTJ, _, n = reg.build_system(mapped, before, 3 * sigma, sigma)
    assert f.n_correspondences == n and n > 100
    assert np.abs(f.information - JTJ).max() <= 1e-12 * np.abs(JTJ).max()
    assert np.array_equal(f.information, f.information.T)
    _, d = before.closest_neighbors(mapped)
    sse = np.sum(d[d < 3 * sigma] ** 2)
    assert abs(f.rmse ** 2 * n - sse) <= 1e-12 * sse


def _fit_is_pre_update_map(K, cfg, scans):
    reg = K.Registration(500, 1e-4, 0)
    icp = K.KissICP(cfg, report_fit=True)
    c = cfg.mapping
    for k, (p, t) in enumerate(scans):
        before = K.VoxelHashMap(c.voxel_size, cfg.data.max_range, c.max_points_per_voxel)
        vox, cnt, pts = icp.local_map.dump()
        if len(vox):
            before.load(vox, cnt, pts)
        _, src = icp.register_frame(p, t)
        _check_fit_against_copy(K, icp, before, reg, src, k == 0)
    return icp


@pytest.mark.gpu
@pytest.mark.parametrize("stamps", ["none", "column"])
def test_reporting_changes_nothing_else(K, stamps):
    L = _stream(stamps)
    scans = [L.scan(k) for k in range(60)]
    off, on = K.KissICP(K.load_config()), K.KissICP(K.load_config(), report_fit=True)
    assert not off.report_fit and on.report_fit
    a, b = _blocking(off, scans, fits=False), _blocking(on, scans)
    for key in ("poses", "iters", "sigma"):
        assert np.array_equal(np.array(a[key]), np.array(b[key])), key
    assert _same_map(off.local_map, on.local_map)
    off, on = K.KissICP(K.load_config()), K.KissICP(K.load_config(), report_fit=True)
    pa, ia, _ = _queued(off, scans, fits=False)
    pb, ib, _ = _queued(on, scans)
    assert np.array_equal(pa, pb) and np.array_equal(ia, ib)
    assert np.array_equal(pa, np.array(a["poses"])) and np.array_equal(ia, np.array(a["iters"]))
    assert off.last_sigma == on.last_sigma == a["sigma"][-1]
    sa, sb = off.state_dict(), on.state_dict()
    assert set(sa) == set(sb) and all(sa[k].tobytes() == sb[k].tobytes() for k in sa)  # (fixed_threshold is NaN)
    assert _same_map(off.local_map, on.local_map)


@pytest.mark.gpu
def test_fit_is_against_the_map_before_the_update(K):
    L = _stream("column")
    _fit_is_pre_update_map(K, K.load_config(), [L.scan(k) for k in range(16)])


@pytest.mark.gpu
def test_fit_whole_grid_icp_path(K):
    """max_points_per_voxel 33 is above the ICP team's limit: the whole-grid loop (op_icp) runs"""
    L = _stream("none", seed=5)
    cfg = K.load_config(mapping__max_points_per_voxel=33)
    icp = K.KissICP(cfg, report_fit=True)
    icp.start_history(3)
    for k in range(3):
        icp.register_frame(*L.scan(k), return_clouds=False)
    assert all(h.team == 0 for h in icp.history())
    _fit_is_pre_update_map(K, cfg, [L.scan(k) for k in range(12)])


@pytest.mark.gpu
@pytest.mark.parametrize("stamps", ["none", "column"])
def test_queued_equals_blocking_bit_for_bit(K, stamps):
    """no stamps: the queue prefetches each next scan's front end on the CTAs the ICP team leaves idle"""
    L = _stream(stamps, seed=7)
    scans = [L.scan(k) for k in range(40)]
    a, b = K.KissICP(K.load_config(), report_fit=True), K.KissICP(K.load_config(), report_fit=True)
    r = _blocking(a, scans)
    pb, ib, fb = _queued(b, scans)
    assert np.array_equal(np.array(r["poses"]), pb) and np.array_equal(np.array(r["iters"]), ib)
    assert _same_fits(_fit_arrays(r["fits"]), fb)
    assert _same_fits(b.last_fit, r["fits"][-1])
    assert all(f.n_correspondences > 0.5 * f.n_source for f in r["fits"][1:])


@pytest.mark.gpu
def test_vetoed_frames_report_the_fit_of_their_replay(K, monkeypatch):
    """frames whose downsampled size exceeds the optimistic table sizing (every point its own voxel): the kernel vetoes
    them before any fit is computed, the host grows the table and replays them"""
    rng = np.random.default_rng(0)
    frames = [rng.uniform(-150, 150, size=(30000, 3)) * [1.0, 1.0, 0.2] for _ in range(4)]
    scans = [(p, np.empty(0)) for p in frames]
    cfg = K.load_config(max_range=300.0, voxel_size=1.0)
    reserved = K.KissICP(cfg, report_fit=True)
    ref = _blocking(reserved, scans)
    assert reserved.grow_retries() == 0
    monkeypatch.setenv("KB_MAP_RESERVE_SLOTS", "0")  # start from the minimal table instead of the sensor-sized one
    a = K.KissICP(cfg, report_fit=True)
    r = _blocking(a, scans)
    assert a.grow_retries() >= 1
    assert np.array_equal(np.array(r["poses"]), np.array(ref["poses"]))
    assert _same_fits(_fit_arrays(r["fits"]), _fit_arrays(ref["fits"]))
    b = K.KissICP(cfg, report_fit=True)
    pb, _, fb = _queued(b, scans)
    assert b.grow_retries() >= 1
    assert np.array_equal(pb, np.array(ref["poses"])) and _same_fits(fb, _fit_arrays(ref["fits"]))
    assert _same_map(reserved.local_map, a.local_map) and _same_map(reserved.local_map, b.local_map)


@pytest.mark.gpu
def test_fused_equals_modular(K):
    L = _stream("column", seed=9)
    a = K.KissICP(K.load_config(), fused=True, report_fit=True)
    b = K.KissICP(K.load_config(), fused=False, report_fit=True)
    for k in range(14):
        p, t = L.scan(k)
        a.register_frame(p, t, return_clouds=False)
        b.register_frame(p, t)
        assert _close(a.last_pose, b.last_pose)
        assert a.last_iterations == b.last_iterations
        fa, fb = a.last_fit, b.last_fit
        assert fa.n_correspondences == fb.n_correspondences and fa.n_source == fb.n_source
        assert (k == 0) == math.isnan(fa.rmse) == math.isnan(fb.rmse)
        if k:
            assert abs(fa.rmse - fb.rmse) < 1e-9
        assert np.allclose(fa.information, fb.information, rtol=1e-9, atol=1e-9)


@pytest.mark.gpu
def test_lost_track_is_visible_in_the_fit(K):
    """the pose set 1 km away mid-stream: the next scan finds no correspondences in the map, without an error; the one
    after it is registered in the map that scan started"""
    L = _stream("none", seed=11)
    icp = K.KissICP(K.load_config(), report_fit=True)
    fits = []
    for k in range(12):
        if k == 8:
            far = icp.last_pose
            far[:3, 3] += [1000.0, 0.0, 0.0]
            icp.last_pose = far
        icp.register_frame(*L.scan(k), return_clouds=False)
        fits.append(icp.last_fit)
    n = np.array([f.n_correspondences for f in fits])
    assert (n[1:8] > 0.5 * np.array([f.n_source for f in fits[1:8]])).all(), n.tolist()
    f = fits[8]
    assert f.n_correspondences == 0 and f.n_source > 0 and math.isnan(f.rmse) and not f.information.any()
    assert n[9] > 0, n.tolist()


@pytest.mark.gpu
def test_switching_and_guards(K):
    from kiss_icp_b200 import _native as N
    Lb = N.lib()
    L = _stream("none", seed=13)
    scans = [L.scan(k) for k in range(10)]
    X = (C.c_void_p * 1)(N.ptr(scans[0][0]))
    n = (N.sz * 1)(len(scans[0][0]))
    fits = (N.Fit * 1)()
    f = N.Fit()
    v = N.i32(-1)
    odo = K.KissICP(K.load_config())
    assert Lb.kb_pipeline_fit_reporting(odo._h, C.byref(v)) == N.KB_OK and v.value == 0
    N.check(Lb.kb_pipeline_set_fit_reporting(odo._h, 1))
    assert Lb.kb_pipeline_fit_reporting(odo._h, C.byref(v)) == N.KB_OK and v.value == 1
    N.check(Lb.kb_pipeline_set_fit_reporting(odo._h, 1))  # (again: a no-op)
    N.check(Lb.kb_pipeline_last_fit(odo._h, C.byref(f)))
    assert f.n_correspondences == 0 and f.n_source == 0 and not any(f.JTJ)
    N.check(Lb.kb_pipeline_register_frames_fit(odo._h, X, n, None, None, 1, 0, None, fits))
    N.check(Lb.kb_pipeline_last_fit(odo._h, C.byref(f)))
    assert f.n_source == fits[0].n_source > 0
    # on -> off: the calls fail as on a pipeline that never reported
    N.check(Lb.kb_pipeline_set_fit_reporting(odo._h, 0))
    assert Lb.kb_pipeline_fit_reporting(odo._h, C.byref(v)) == N.KB_OK and v.value == 0
    assert Lb.kb_pipeline_last_fit(odo._h, C.byref(f)) == N.KB_ERR_INVALID_ARG
    assert Lb.kb_pipeline_register_frames_fit(odo._h, X, n, None, None, 1, 0, None, fits) == N.KB_ERR_INVALID_ARG
    assert Lb.kb_pipeline_register_frames_fit(odo._h, X, n, None, None, 1, 0, None, None) == N.KB_OK
    # off -> on: the last fit starts from zeros
    N.check(Lb.kb_pipeline_set_fit_reporting(odo._h, 1))
    N.check(Lb.kb_pipeline_last_fit(odo._h, C.byref(f)))
    assert f.n_source == 0
    # a localizer always reports
    prior = K.VoxelHashMap(1.0, 1e9, 20)
    prior.update(scans[0][0], np.eye(4))
    loc = K.KissICP(K.load_config(), prior_map=prior, report_fit=False)
    assert loc.report_fit
    assert Lb.kb_pipeline_set_fit_reporting(loc._h, 0) == N.KB_ERR_INVALID_ARG
    N.check(Lb.kb_pipeline_set_fit_reporting(loc._h, 1))
    assert Lb.kb_pipeline_fit_reporting(loc._h, C.byref(v)) == N.KB_OK and v.value == 1
    del loc
    # without the keyword the Python errors stay
    with pytest.raises(ValueError):
        K.KissICP(K.load_config()).last_fit
    with pytest.raises(ValueError):
        K.KissICP(K.load_config(), fused=False).register_frames([scans[0][0]], return_fits=True)
    # the same bits from run to run at one grid size
    runs = []
    for _ in range(2):
        icp = K.KissICP(K.load_config(), report_fit=True)
        runs.append(_fit_arrays(_blocking(icp, scans)["fits"]))
    assert _same_fits(runs[0], runs[1])
    # reporting is a setting, not state: the state_dict has the keys of reporting off
    assert set(icp.state_dict()) == set(K.KissICP(K.load_config()).state_dict())


def test_fit_reporting_entry_points_without_device():
    """CPU: the entry points exist and reject NULL arguments"""
    from kiss_icp_b200 import _native as N
    L = N.lib()
    v = N.i32(0)
    assert L.kb_pipeline_set_fit_reporting(None, 1) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_set_fit_reporting(None, 0) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_fit_reporting(None, C.byref(v)) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_fit_reporting(None, None) == N.KB_ERR_INVALID_ARG
    if L.kb_device_count() == 0:
        import kiss_icp_b200 as K
        c = N.Config()
        L.kb_config_default(C.byref(c))
        h = N.vp()
        assert L.kb_pipeline_create(C.byref(c), C.byref(h)) == N.KB_ERR_NO_DEVICE
        with pytest.raises(N.NoDeviceError):
            K.KissICP(K.load_config(), report_fit=True)
