"""KissICP(config, prior_map=...) / kb_pipeline_create_localizer: RegisterFrame without the map update against a
read-only prior map, with a fit per scan. Scans are localized at fractional indices k + 0.5, so no localized scan is
in the map, which is built from integer scans at their ground-truth poses."""
import ctypes as C
import gc
import math
import threading

import numpy as np
import pytest

from conftest import pose_error


def _seed_offset(O):
    return O.se3_exp([0.5, 0.0, 0.0, 0.0, 0.0, math.radians(2.0)])


def _prior(K, O, L, ks, voxel, cap=20, crop=None):
    """a prior map (and the oracle's twin) from scans ks at their ground-truth poses: frame_downsample per scan (deskewed
    with the true motion when the stream has stamps), optionally cropped to `crop` metres around the sensor"""
    g, o = K.VoxelHashMap(voxel, 1e9, cap), O.VoxelHashMap(voxel, 1e9, cap)
    for k in ks:
        p, t = L.scan(k)
        if len(t):
            p = O.preprocess(p, t, np.linalg.inv(L.pose(k - 1)) @ L.pose(k), 1e9, 0.0, True)
        ds = O.voxel_down_sample(p, voxel * 0.5)
        if crop is not None:
            ds = ds[np.linalg.norm(ds, axis=1) < crop]
        g.update(ds, L.pose(k))
        o.update(ds, L.pose(k))
    return g, o


def _oracle_localize(O, omap, cfg, scans, seed, state=None):
    """the reference's statement (kiss_icp.py:43-75) without local_map.update, on the oracle's modules. `state`:
    (delta, model_sse, num_samples) to start from, default a new sequence's; returns the final one as a third value"""
    v, th, reg = cfg.mapping.voxel_size, cfg.adaptive_threshold, cfg.registration
    pose = np.array(seed, dtype=np.float64)
    delta, sse, ns = state if state is not None else (np.eye(4), th.initial_threshold ** 2, 1)
    poses, iters = [], []
    for p, t in scans:
        frame = O.preprocess(p, t, delta, cfg.data.max_range, cfg.data.min_range, cfg.data.deskew)
        src = O.voxel_down_sample(O.voxel_down_sample(frame, v * 0.5), v * 1.5)
        sigma = math.sqrt(sse / ns)
        guess = pose @ delta
        new, it = O.align_points_to_map(omap, src, guess, 3 * sigma, sigma, reg.max_num_iterations, reg.convergence_criterion)
        sse, ns = O.threshold_update(sse, ns, np.linalg.inv(guess) @ new, th.min_motion_th, cfg.data.max_range)
        delta = np.linalg.inv(pose) @ new
        pose = new
        poses.append(pose)
        iters.append(it)
    return np.array(poses), np.array(iters), (delta, sse, ns)


def _localize(icp, scans):
    poses, iters, fits = [], [], []
    for p, t in scans:
        icp.register_frame(p, t, return_clouds=False)
        poses.append(icp.last_pose)
        iters.append(icp.last_iterations)
        fits.append(icp.last_fit)
    return np.array(poses), np.array(iters), fits


def _fit_arrays(fits):
    return (np.array([f.n_correspondences for f in fits]), np.array([f.n_source for f in fits]),
            np.array([f.rmse for f in fits]), np.array([f.information for f in fits]))


def _same_fits(a, b):
    return all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


def _close(A, B, tol=1e-9):
    """translations within tol [m] and rotation matrices within tol elementwise (the angle of R_A^T R_B from its trace
    cannot resolve differences below ~2e-8 rad)"""
    return np.linalg.norm(A[:3, 3] - B[:3, 3]) < tol and np.abs(A[:3, :3] - B[:3, :3]).max() < tol


def _check_oracle(poses, iters, ref_poses, ref_iters, n_corr=None):
    bad = [(k, float(np.linalg.norm(P[:3, 3] - Po[:3, 3])), float(np.abs(P[:3, :3] - Po[:3, :3]).max()), int(it), int(ito),
            None if n_corr is None else int(n_corr[k]))
           for k, (P, it, Po, ito) in enumerate(zip(poses, iters, ref_poses, ref_iters)) if not (_close(P, Po) and it == ito)]
    assert not bad, bad


def _map_state(m):
    vox, cnt, pts = m.dump()
    return m.num_voxels(), m.num_points(), vox, cnt, pts


def _same_map(a, b):
    return a[0] == b[0] and a[1] == b[1] and all(np.array_equal(x, y) for x, y in zip(a[2:], b[2:]))


@pytest.fixture(scope="module")
def small():
    from kiss_icp_b200 import synthetic
    return synthetic.small_shape(seed=3, beams=32, cols=512)


@pytest.mark.gpu
def test_prior_map_is_never_written(K, O, small):
    prior, _ = _prior(K, O, small, range(0, 110, 2), 1.0)
    before = _map_state(prior)
    scans = [small.scan(k + 0.5) for k in range(100)]
    a = K.KissICP(K.load_config(), prior_map=prior)
    a.last_pose = small.pose(0.5)
    for p, t in scans:
        a.register_frame(p, t, return_clouds=False)
    assert _same_map(before, _map_state(prior))
    b = K.KissICP(K.load_config(), prior_map=prior)
    b.last_pose = small.pose(0.5)
    b.register_frames([p for p, _ in scans], [t for _, t in scans], return_fits=True)
    assert _same_map(before, _map_state(prior))
    assert np.array_equal(a.last_pose, b.last_pose)
    # the device counters too: a mutator that needs them (compact) works on the untouched map afterwards
    del a, b
    gc.collect()
    assert prior.readers() == 0
    q = np.concatenate([small.scan(k)[0] for k in (3, 50)]) @ small.pose(3)[:3, :3].T + small.pose(3)[:3, 3]
    p1, d1 = prior.closest_neighbors(q)
    prior.compact()
    assert _same_map(before, _map_state(prior))
    p2, d2 = prior.closest_neighbors(q)
    assert np.array_equal(p1, p2) and np.array_equal(d1, d2)


@pytest.mark.gpu
@pytest.mark.parametrize("stamps", ["none", "column"])
def test_localizer_matches_oracle_kitti_shape(K, O, stamps):
    import torch
    from kiss_icp_b200 import synthetic
    L = synthetic.SyntheticLidar(seed=4, beams=64, cols=1024, stamps=stamps,
                                 device="cuda" if torch.cuda.is_available() else "cpu")
    cfg = K.load_config()
    prior, oprior = _prior(K, O, L, range(0, 36), cfg.mapping.voxel_size)
    scans = [L.scan(k + 0.5) for k in range(6, 30)]
    seed = L.pose(6.5) @ _seed_offset(O)
    icp = K.KissICP(cfg, prior_map=prior)
    icp.last_pose = seed
    poses, iters, fits = _localize(icp, scans)
    ref, ref_it, _ = _oracle_localize(O, oprior, cfg, scans, seed)
    _check_oracle(poses, iters, ref, ref_it)
    assert icp.grow_retries() == 0
    # the track stays on the ground truth once the start offset is absorbed: to the map's accuracy (a map of noisy
    # scans, voxel 1 m), which is what bounds it here, not the registration (equal to the oracle within 1e-9)
    errs = np.array([pose_error(P, L.pose(k + 0.5)) for k, P in zip(range(6, 30), poses)])
    assert errs[5:, 0].max() < 0.5 and errs[5:, 1].max() < 0.01, errs
    assert all(f.n_correspondences > 0.5 * f.n_source for f in fits)


@pytest.mark.gpu
def test_localizer_whole_grid_path_and_deskew_ouster_shape(K, O):
    """131k points at voxel 0.3: the source is above the ICP team's limit, so the whole-grid loop (op_icp) runs"""
    import torch
    from kiss_icp_b200 import synthetic
    L = synthetic.ouster128_shape(seed=5, device="cuda" if torch.cuda.is_available() else "cpu")
    cfg = K.load_config(voxel_size=0.3)
    prior, oprior = _prior(K, O, L, range(0, 10), 0.3)
    scans = [L.scan(k + 0.5) for k in range(3, 8)]
    seed = L.pose(3.5) @ _seed_offset(O)
    icp = K.KissICP(cfg, prior_map=prior)
    icp.start_history(len(scans))
    icp.last_pose = seed
    poses, iters, _ = _localize(icp, scans)
    assert all(h.team == 0 for h in icp.history())  # the whole-grid path
    ref, ref_it, _ = _oracle_localize(O, oprior, cfg, scans, seed)
    _check_oracle(poses, iters, ref, ref_it)


@pytest.mark.gpu
def test_fused_localizer_equals_modular(K, O, small):
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=9, beams=32, cols=512, stamps="column")
    prior, _ = _prior(K, O, L, range(0, 20), 1.0)
    scans = [L.scan(k + 0.5) for k in range(2, 14)]
    a = K.KissICP(K.load_config(), fused=True, prior_map=prior)
    b = K.KissICP(K.load_config(), fused=False, prior_map=prior)
    assert a.local_map is prior and b.local_map is prior
    seed = L.pose(2.5) @ _seed_offset(O)
    a.last_pose = seed
    b.last_pose = seed
    for p, t in scans:
        a.register_frame(p, t, return_clouds=False)
        b.register_frame(p, t)
        assert _close(a.last_pose, b.last_pose)
        assert a.last_iterations == b.last_iterations
        fa, fb = a.last_fit, b.last_fit
        assert fa.n_correspondences == fb.n_correspondences and fa.n_source == fb.n_source
        assert abs(fa.rmse - fb.rmse) < 1e-9 and np.allclose(fa.information, fb.information, rtol=1e-9, atol=1e-9)


@pytest.mark.gpu
def test_queued_equals_blocking_bit_for_bit(K, O, small):
    """no stamps: the queue prefetches each next scan's front end on the CTAs the ICP team leaves idle"""
    prior, _ = _prior(K, O, small, range(0, 40), 1.0)
    scans = [small.scan(k + 0.5)[0] for k in range(2, 32)]
    seed = small.pose(2.5) @ _seed_offset(O)
    a = K.KissICP(K.load_config(), prior_map=prior)
    b = K.KissICP(K.load_config(), prior_map=prior)
    a.last_pose = seed
    b.last_pose = seed
    pa, _, fa = _localize(a, [(p, np.empty(0)) for p in scans])
    pb, fb = b.register_frames(scans, return_fits=True)
    assert np.array_equal(pa, pb)
    assert _same_fits(_fit_arrays(fa), fb)
    assert _same_fits(b.last_fit, fa[-1])
    plain = K.KissICP(K.load_config(), prior_map=prior)
    plain.last_pose = seed
    assert np.array_equal(plain.register_frames(scans), pb)


@pytest.mark.gpu
def test_fit_equals_build_system_and_closest_neighbors(K, O, small):
    prior, _ = _prior(K, O, small, range(0, 30), 1.0)
    reg = K.Registration(500, 1e-4, 0)
    runs = []
    for _ in range(2):
        icp = K.KissICP(K.load_config(), prior_map=prior)
        icp.last_pose = small.pose(4.5) @ _seed_offset(O)
        fits = []
        for k in range(4, 16):
            p, t = small.scan(k + 0.5)
            _, src = icp.register_frame(p, t)
            f, P, sigma = icp.last_fit, icp.last_pose, icp.last_sigma
            mapped = src @ P[:3, :3].T + P[:3, 3]
            JTJ, _, n = reg.build_system(mapped, prior, 3 * sigma, sigma)
            assert f.n_correspondences == n and f.n_source == len(src) and n > 100
            assert np.abs(f.information - JTJ).max() <= 1e-12 * np.abs(JTJ).max()
            assert np.array_equal(f.information, f.information.T)
            _, d = prior.closest_neighbors(mapped)
            sse = np.sum(d[d < 3 * sigma] ** 2)
            assert abs(f.rmse ** 2 * n - sse) <= 1e-12 * sse
            fits.append(f)
        runs.append(_fit_arrays(fits))
    assert _same_fits(runs[0], runs[1])


@pytest.mark.gpu
def test_tracking_loss_stays_with_the_oracle(K, O, small):
    """a prior map of the start of the lap only (points within 25 m of the sensor of scans 0..39) and a 30 m sensor
    range. The track leaves the mapped stretch and correspondences fall; then the pose is set 1 km away from the map
    (as a caller would after a wrong relocalization), where there are none at all. The localizer equals the oracle
    throughout and reports 0 correspondences without an error."""
    cfg = K.load_config(max_range=30.0, voxel_size=1.0)
    prior, oprior = _prior(K, O, small, range(0, 40), 1.0, crop=25.0)
    scans = [small.scan(k + 0.5) for k in range(20, 66)]
    far_scans = [small.scan(k + 0.5) for k in range(66, 76)]
    seed = small.pose(20.5)
    icp = K.KissICP(cfg, prior_map=prior)
    icp.last_pose = seed
    poses, iters, fits = _localize(icp, scans)
    ref, ref_it, state = _oracle_localize(O, oprior, cfg, scans, seed)
    far = np.array(poses[-1])
    far[:3, 3] += [1000.0, 0.0, 0.0]
    icp.last_pose = far
    poses2, iters2, fits2 = _localize(icp, far_scans)
    ref2, ref_it2, _ = _oracle_localize(O, oprior, cfg, far_scans, far, state)
    n = np.array([f.n_correspondences for f in fits + fits2])
    _check_oracle(np.concatenate([poses, poses2]), np.concatenate([iters, iters2]), np.concatenate([ref, ref2]),
                  np.concatenate([ref_it, ref_it2]), n)
    assert n[:5].min() > 400 and n[:len(scans)].min() < 0.7 * n[:5].min(), n.tolist()
    assert (n[len(scans):] == 0).all(), n.tolist()
    assert all(math.isnan(f.rmse) and f.n_source > 0 and not f.information.any() for f in fits2)


def _grid(N, blocks):
    N.check(N.lib().kb_set_grid_blocks(blocks))


@pytest.mark.gpu
def test_two_localizers_share_one_prior(K, O, small):
    """each on its own stream and grid slice, interleaved and from two host threads at once, each bit-identical to
    running alone; a batch alignment against the prior during tracking too"""
    from kiss_icp_b200 import _native as N
    prior, _ = _prior(K, O, small, range(0, 50), 1.0)
    streams = {"a": [small.scan(k + 0.5)[0] for k in range(2, 26)], "b": [small.scan(k + 0.25)[0] for k in range(20, 44)]}
    seeds = {"a": small.pose(2.5) @ _seed_offset(O), "b": small.pose(20.25)}
    _grid(N, 48)
    try:
        def make(name):
            icp = K.KissICP(K.load_config(), prior_map=prior)
            icp.last_pose = seeds[name]
            return icp
        alone = {}
        for name in streams:
            icp = make(name)
            alone[name] = icp.register_frames(streams[name], return_fits=True)
            del icp
        gc.collect()
        # interleaved blocking calls
        a, b = make("a"), make("b")
        assert prior.readers() == 2
        got = {"a": [], "b": []}
        for pa, pb in zip(streams["a"], streams["b"]):
            for name, icp, p in (("a", a, pa), ("b", b, pb)):
                icp.register_frame(p, np.empty(0), return_clouds=False)
                got[name].append((icp.last_pose, icp.last_fit))
        for name in streams:
            assert np.array_equal(np.array([g[0] for g in got[name]]), alone[name][0])
            assert _same_fits(_fit_arrays([g[1] for g in got[name]]), alone[name][1])
        # queued from two host threads at once
        a, b = make("a"), make("b")
        out, errors = {}, []

        def run(name, icp):
            try:
                out[name] = icp.register_frames(streams[name], return_fits=True)
            except Exception as e:  # (reported by the main thread)
                errors.append(e)
        threads = [threading.Thread(target=run, args=(n, i)) for n, i in (("a", a), ("b", b))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        for name in streams:
            assert np.array_equal(out[name][0], alone[name][0]) and _same_fits(out[name][1], alone[name][1])
        # a batch relocalization against the prior between tracked scans
        reg = K.Registration(500, 1e-4, 0)
        src = O.voxel_down_sample(O.voxel_down_sample(small.scan(30)[0], 0.5), 1.5)
        G = np.array([small.pose(30) @ O.se3_exp([0.3 * i, -0.2 * i, 0, 0, 0, 0.02 * i]) for i in range(6)])
        ref = reg.align_points_to_map_batch(src, prior, G, 3.0, 1.0, return_inliers=True)
        c = make("a")
        half = len(streams["a"]) // 2
        p1, f1 = c.register_frames(streams["a"][:half], return_fits=True)
        mid = reg.align_points_to_map_batch(src, prior, G, 3.0, 1.0, return_inliers=True)
        p2, f2 = c.register_frames(streams["a"][half:], return_fits=True)
        assert all(np.array_equal(x, y) for x, y in zip(ref, mid))
        assert np.array_equal(np.concatenate([p1, p2]), alone["a"][0])
        assert _same_fits([np.concatenate([x, y]) for x, y in zip(f1, f2)], alone["a"][1])
    finally:
        _grid(N, 0)


@pytest.mark.gpu
def test_prior_map_guards(K, O, small):
    from kiss_icp_b200 import _native as N
    from kiss_icp_b200.mapping import MapInUseError
    prior, _ = _prior(K, O, small, range(0, 10), 1.0)
    before = _map_state(prior)
    icp = K.KissICP(K.load_config(), prior_map=prior)
    icp2 = K.KissICP(K.load_config(), prior_map=prior)
    assert prior.readers() == 2
    pts = small.scan(3)[0]
    vox, cnt, mp = before[2:]
    for call in (prior.clear, lambda: prior.update(pts, np.eye(4)), lambda: prior.update(pts, np.zeros(3)),
                 lambda: prior.add_points(pts), lambda: prior.remove_far_away_points(np.zeros(3)), prior.compact,
                 lambda: prior.load(vox[:5], cnt[:5], mp[:int(cnt[:5].sum())])):
        with pytest.raises(MapInUseError, match="in use by 2 localizers"):
            call()
        assert _same_map(before, _map_state(prior))
    assert issubclass(MapInUseError, RuntimeError)
    L = N.lib()
    assert L.kb_map_destroy(prior._h) == N.KB_ERR_INVALID_ARG
    dv = np.zeros(3, dtype=np.int32)
    assert L.kb_map_load_dev(prior._h, N.ptr(dv), N.ptr(dv), N.ptr(np.zeros(3)), 0, 0) == N.KB_ERR_INVALID_ARG
    # read-only calls keep working
    prior.closest_neighbors(pts)
    prior.point_cloud()
    K.Registration(500, 1e-4, 0).align_points_to_map(pts[:100], prior, np.eye(4), 3.0, 1.0)
    assert _same_map(before, _map_state(prior))
    del icp
    gc.collect()
    with pytest.raises(MapInUseError, match="in use by 1 localizer:"):
        prior.clear()
    del icp2
    gc.collect()
    assert prior.readers() == 0
    prior.add_points(pts)
    prior.clear()
    assert prior.num_voxels() == 0
    # mismatched configs
    for cfg in (K.load_config(voxel_size=0.5), K.load_config(mapping__max_points_per_voxel=10)):
        with pytest.raises(ValueError, match="prior map"):
            K.KissICP(cfg, prior_map=prior)
        c = N.Config()
        L.kb_config_default(C.byref(c))
        c.voxel_size = cfg.mapping.voxel_size
        c.max_points_per_voxel = cfg.mapping.max_points_per_voxel
        h = N.vp()
        assert L.kb_pipeline_create_localizer(C.byref(c), prior._h, C.byref(h)) == N.KB_ERR_INVALID_ARG
    # an odometry pipeline has no fits, and its own map is no prior map
    odo = K.KissICP(K.load_config())
    with pytest.raises(ValueError):
        odo.last_fit
    with pytest.raises(ValueError):
        odo.register_frames([pts], return_fits=True)
    f = N.Fit()
    assert L.kb_pipeline_last_fit(odo._h, C.byref(f)) == N.KB_ERR_INVALID_ARG
    X = (C.c_void_p * 1)(N.ptr(pts))
    n = (N.sz * 1)(len(pts))
    fits = (N.Fit * 1)()
    assert L.kb_pipeline_register_frames_fit(odo._h, X, n, None, None, 1, 0, None, fits) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_register_frames_fit(odo._h, X, n, None, None, 1, 0, None, None) == N.KB_OK
    with pytest.raises(ValueError, match="own voxel map"):
        K.KissICP(K.load_config(), prior_map=odo.local_map)


@pytest.mark.gpu
def test_prior_map_on_another_device_is_rejected(K, O, small):
    from kiss_icp_b200 import _native as N
    L = N.lib()
    if L.kb_device_count() < 2:
        pytest.skip("needs two GPUs")
    prior, _ = _prior(K, O, small, range(0, 4), 1.0)
    N.check(L.kb_set_device(1))
    try:
        with pytest.raises(ValueError, match="device"):
            K.KissICP(K.load_config(), prior_map=prior)
    finally:
        N.check(L.kb_set_device(0))


@pytest.mark.gpu
def test_localizer_state_dict_has_no_map(K, O, small):
    prior, _ = _prior(K, O, small, range(0, 20), 1.0)
    icp = K.KissICP(K.load_config(), prior_map=prior)
    icp.last_pose = small.pose(2.5)
    for k in range(2, 8):
        p, t = small.scan(k + 0.5)
        icp.register_frame(p, t, return_clouds=False)
    s = icp.state_dict()
    assert not {"voxels", "counts", "points"} & set(s)
    other = K.KissICP(K.load_config(), prior_map=prior)
    other.load_state_dict(s)
    assert np.array_equal(other.last_pose, icp.last_pose)
    p, t = small.scan(8.5)
    icp.register_frame(p, t, return_clouds=False)
    other.register_frame(p, t, return_clouds=False)
    assert np.array_equal(other.last_pose, icp.last_pose) and _same_fits(other.last_fit, icp.last_fit)
    odo = K.KissICP(K.load_config())
    with pytest.raises(ValueError, match="carries no map"):
        odo.load_state_dict(s)
    with pytest.raises(ValueError, match="not part of a localizer's state"):
        other.load_state_dict(odo.state_dict())
    modular = K.KissICP(K.load_config(), fused=False, prior_map=prior)
    modular.load_state_dict(s)
    assert not {"voxels", "counts", "points"} & set(modular.state_dict())


def test_localizer_entry_points_without_device():
    """CPU: the entry points exist and reject NULL arguments; Python checks the prior map's type first"""
    from kiss_icp_b200 import _native as N
    import kiss_icp_b200 as K
    L = N.lib()
    c = N.Config()
    L.kb_config_default(C.byref(c))
    h = N.vp()
    assert L.kb_pipeline_create_localizer(C.byref(c), None, C.byref(h)) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_create_localizer(None, None, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_last_fit(None, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_map_readers(None, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_register_frames_fit(None, None, None, None, None, 1, 0, None, None) == N.KB_ERR_INVALID_ARG
    with pytest.raises(TypeError):
        K.KissICP(K.load_config(), prior_map=np.zeros((4, 3)))
    if L.kb_device_count() == 0:
        m = N.vp()
        assert L.kb_map_create(1.0, 1e9, 20, C.byref(m)) == N.KB_ERR_NO_DEVICE
        with pytest.raises(N.NoDeviceError):
            K.VoxelHashMap(1.0, 1e9, 20)
