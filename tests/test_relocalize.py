"""Registration.relocalize / KissICP.relocalize / kb_relocalize: a global pose search in a bounded region of a prior map.
The coarse scores must equal a numpy count of the documented formula, the peaks and candidates the numpy statement of
the peak rule, and the refinement align_points_to_map_batch, bit for bit."""
import ctypes as C
import gc
import math

import numpy as np
import pytest

from conftest import pose_error

TWO_PI = 6.283185307179586


def _rz(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _center(O):
    T = O.se3_exp([3.0, -2.0, 0.4, 0.02, -0.03, 0.7])
    return T


def _search(K, center, hx=2, hy=1, step=0.5, n_yaw=5, yaw_step=0.1, **kw):
    return K.RelocalizationSearch(center=center, half_cells_x=hx, half_cells_y=hy, step=step, n_yaw=n_yaw,
                                  yaw_step=yaw_step, **kw)


# ---------------------------------------------------------------------------------------------------------- CPU
def test_hypotheses_order_and_values(K, O):
    Tc = _center(O)
    for n_yaw in (1, 4, 5):
        s = _search(K, Tc, hx=3, hy=2, step=0.25, n_yaw=n_yaw, yaw_step=0.3)
        H = s.hypotheses()
        assert H.shape == (n_yaw * 5 * 7, 4, 4) and s.shape == (n_yaw, 5, 7)
        for k in range(n_yaw):
            R = _rz((k - n_yaw // 2) * 0.3) @ Tc[:3, :3]
            for j in range(-2, 3):
                for i in range(-3, 4):
                    h = (k * 5 + (j + 2)) * 7 + (i + 3)
                    assert np.abs(H[h, :3, :3] - R).max() <= 1e-15, (k, j, i)
                    assert H[h, 0, 3] == Tc[0, 3] + i * 0.25 and H[h, 1, 3] == Tc[1, 3] + j * 0.25
                    assert H[h, 2, 3] == Tc[2, 3]
                    assert np.array_equal(H[h, 3], [0.0, 0.0, 0.0, 1.0])


def test_full_circle_headings_cover_the_circle_once(K):
    s = _search(K, np.eye(4), hx=0, hy=0, n_yaw=72, yaw_step=TWO_PI / 72)
    yaw = np.arctan2(s.hypotheses()[:, 1, 0], s.hypotheses()[:, 0, 0])
    assert np.allclose(np.sort(np.mod(yaw, TWO_PI)), np.arange(72) * TWO_PI / 72, atol=1e-12)
    assert abs(yaw[36]) < 1e-15 and abs(abs(yaw[0]) - math.pi) < 1e-12  # k = n_yaw // 2 is the centre's heading


def test_hypotheses_invalid_arguments(K, O):
    from kiss_icp_b200 import _native as N
    Tc = _center(O)
    bad = [dict(hx=-1), dict(hy=-1), dict(step=0.0), dict(step=-1.0), dict(step=math.nan), dict(step=math.inf),
           dict(n_yaw=0), dict(yaw_step=0.0), dict(yaw_step=math.nan), dict(top_k=0), dict(top_k=257),
           dict(hx=2048, hy=2048, n_yaw=1), dict(hx=100, hy=100, n_yaw=500)]
    for b in bad:
        with pytest.raises(ValueError):
            _search(K, Tc, **b).hypotheses()
    assert _search(K, Tc, hx=2047, hy=2047, n_yaw=1)._struct()[1] == 4095 ** 2  # 2^24 - 2^13 + 1 <= 2^24
    notse3 = Tc.copy()
    notse3[0, 0] += 1e-3
    with pytest.raises(ValueError, match="SE\\(3\\)"):
        _search(K, notse3).hypotheses()
    inf_t = Tc.copy()
    inf_t[1, 3] = math.inf
    with pytest.raises(ValueError, match="translation"):
        _search(K, inf_t).hypotheses()
    with pytest.raises(ValueError):
        _search(K, np.eye(3)).hypotheses()
    with pytest.raises(TypeError):
        _search(K, Tc, hx=1.5).hypotheses()
    # the C entry point: status codes, two-call convention
    s, H = _search(K, Tc)._struct()
    L = N.lib()
    n = N.sz(0)
    assert L.kb_reloc_hypotheses(None, None, 0, C.byref(n)) == N.KB_ERR_INVALID_ARG
    assert L.kb_reloc_hypotheses(C.byref(s), None, 0, None) == N.KB_ERR_INVALID_ARG
    out = np.zeros((H, 4, 4))
    assert L.kb_reloc_hypotheses(C.byref(s), N.ptr(out), H - 1, C.byref(n)) == N.KB_ERR_CAPACITY and n.value == H
    assert not out.any()
    s.center[0] = 1.001
    assert L.kb_reloc_hypotheses(C.byref(s), None, 0, C.byref(n)) == N.KB_ERR_NOT_SE3


def test_relocalize_checks_arguments_before_the_device(K, O):
    """the arguments that need no handle are checked first; only then does a machine without a device answer
    KB_ERR_NO_DEVICE (handles exist only where a device does)"""
    from kiss_icp_b200 import _native as N
    L = N.lib()
    s, _ = _search(K, _center(O))._struct()
    pts = np.ones((10, 3))
    r = N.RelocResult()
    st = lambda s_, p, n, out: L.kb_relocalize(None, N.ptr(p), n, None, C.byref(s_) if s_ is not None else None,
                                              C.byref(out) if out is not None else None, None, None, None)
    assert st(None, pts, 10, r) == N.KB_ERR_INVALID_ARG
    assert st(s, pts, 10, None) == N.KB_ERR_INVALID_ARG
    assert L.kb_relocalize(None, None, 10, None, C.byref(s), C.byref(r), None, None, None) == N.KB_ERR_INVALID_ARG
    assert st(s, pts, 0, r) == N.KB_ERR_INVALID_ARG
    bad = N.RelocSearch.from_buffer_copy(s)
    bad.top_k = 0
    assert st(bad, pts, 10, r) == N.KB_ERR_INVALID_ARG
    bad = N.RelocSearch.from_buffer_copy(s)
    bad.center[1] = 0.5
    assert st(bad, pts, 10, r) == N.KB_ERR_NOT_SE3
    good = st(s, pts, 10, r)
    if L.kb_device_count() == 0:
        assert good == N.KB_ERR_NO_DEVICE
    else:
        assert good == N.KB_ERR_INVALID_ARG  # (NULL handles)
    assert r.n_hypotheses == 0 and r.inliers == 0  # nothing written
    from kiss_icp_b200.relocalization import relocalize
    with pytest.raises(TypeError):
        relocalize(None, pts, None, object())
    with pytest.raises(TypeError):
        relocalize(None, pts, object(), _search(K, np.eye(4)))


# ---------------------------------------------------------------------------------------------------------- GPU
def _map(K, O, L, ks, voxel, cap=20):
    m = K.VoxelHashMap(voxel, 1e9, cap)
    for k in ks:
        p, _ = L.scan(k)
        m.update(O.voxel_down_sample(p, voxel * 0.5), L.pose(k))
    return m


def _source(O, L, k, voxel, max_range=100.0):
    p, _ = L.scan(k)
    p = p[np.linalg.norm(p, axis=1) < max_range]
    return O.voxel_down_sample(O.voxel_down_sample(p, voxel * 0.5), voxel * 1.5)


def _numpy_scores(H, src, vmap):
    """the documented score: ((R0 x + R1 y) + R2 z) + t0 per component, then the hot path's voxel function (a
    multiply by 1 / v when v is a power of two, a division otherwise), counted against the map's voxels"""
    v = vmap_voxel_size(vmap)
    m, e = math.frexp(v)
    pow2 = m == 0.5
    vox = vmap.dump()[0].astype(np.int64)
    off = 1 << 20
    key = lambda a: ((a[..., 0] + off) << 42) | ((a[..., 1] + off) << 21) | (a[..., 2] + off)
    keys = np.sort(key(vox))
    x, y, z = src[:, 0], src[:, 1], src[:, 2]
    out = np.empty(len(H), dtype=np.int64)
    for h, T in enumerate(H):
        P = np.stack([((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)], axis=1)
        c = np.floor(P * (1.0 / v)) if pow2 else np.floor(P / v)
        q = key(c.astype(np.int64))
        i = np.minimum(np.searchsorted(keys, q), len(keys) - 1)
        out[h] = int(np.count_nonzero(keys[i] == q))
    return out


def vmap_voxel_size(vmap):
    from kiss_icp_b200 import _native as N
    vs = N.dbl(0)
    N.check(N.lib().kb_map_params(vmap._h, C.byref(vs), None, None))
    return vs.value


def _numpy_peaks(S, wrap):
    """peak rule on scores (n_yaw, Ny, Nx): no neighbour at +-1 in i, j, k with a higher score or the same score and a
    smaller index; k wraps when wrap, no padding at the edges -> peaks by (score desc, h asc)"""
    n_yaw, ny, nx = S.shape
    flat = S.ravel()
    peaks = []
    for h in range(flat.size):
        k, r = divmod(h, ny * nx)
        j, i = divmod(r, nx)
        ok = True
        for dk in (-1, 0, 1):
            k2 = k + dk
            if not 0 <= k2 < n_yaw:
                if not wrap:
                    continue
                k2 %= n_yaw
            for dj in (-1, 0, 1):
                for di in (-1, 0, 1):
                    j2, i2 = j + dj, i + di
                    if (dk, dj, di) == (0, 0, 0) or not (0 <= j2 < ny and 0 <= i2 < nx):
                        continue
                    h2 = (k2 * ny + j2) * nx + i2
                    if flat[h2] > flat[h] or (flat[h2] == flat[h] and h2 < h):
                        ok = False
        if ok:
            peaks.append(h)
    return sorted(peaks, key=lambda h: (-flat[h], h))


def _check_refinement(reg, src, vmap, search, res):
    """winner / runner-up against align_points_to_map_batch on the candidates, bit for bit"""
    P, it, inl = reg.align_points_to_map_batch(src, vmap, res.candidates, search.max_correspondence_distance,
                                               search.kernel_scale, return_inliers=True)
    w = int(np.argmax(inl))
    assert res.rank == w and np.array_equal(res.pose, P[w]) and res.iterations == it[w] and res.inliers == inl[w]
    far = []
    for c in range(len(P)):
        R = P[w][:3, :3].T @ P[c][:3, :3]
        ang = math.acos(max(-1.0, min(1.0, (np.trace(R) - 1.0) / 2.0)))
        if c != w and (math.hypot(*(P[w][:2, 3] - P[c][:2, 3])) > 2 * search.step or ang > 2 * search.yaw_step):
            far.append(c)
    if far:
        ru = max(far, key=lambda c: (inl[c], -c))
        assert res.runner_up_inliers == inl[ru] and np.array_equal(res.runner_up_pose, P[ru])
    else:
        assert res.runner_up_inliers == -1 and res.runner_up_pose is None


@pytest.fixture(scope="module")
def small():
    from kiss_icp_b200 import synthetic
    return synthetic.small_shape(seed=3, beams=32, cols=512)


@pytest.mark.gpu
@pytest.mark.parametrize("voxel", [1.0, 0.7])
def test_scores_peaks_candidates_and_refinement_exact(K, O, small, voxel):
    vmap = _map(K, O, small, range(0, 30, 2), voxel)
    reg = K.Registration(500, 1e-4, 0)
    src = _source(O, small, 12.5, voxel)
    truth = small.pose(12.5)
    for n_yaw, yaw_step in ((12, TWO_PI / 12), (12, 0.05), (13, TWO_PI / 13 + 1e-8)):  # wraps, does not, nearly does
        wrap = abs(n_yaw * yaw_step - TWO_PI) < 1e-9
        center = truth.copy()
        center[:3, :3] = _rz(0.04) @ truth[:3, :3]
        center[:2, 3] += [0.3, -0.6]
        s = _search(K, center, hx=10, hy=10, step=0.5, n_yaw=n_yaw, yaw_step=yaw_step, top_k=8)
        res = reg.relocalize(src, vmap, s, return_scores=True)
        H = s.hypotheses()
        assert res.scores.shape == s.shape and res.n_hypotheses == len(H) == res.scores.size
        ref = _numpy_scores(H, src, vmap)
        assert np.array_equal(res.scores.ravel(), ref), np.flatnonzero(res.scores.ravel() != ref)[:10]
        peaks = _numpy_peaks(res.scores, wrap)
        assert res.n_peaks == len(peaks) and len(res.candidates) == min(8, len(peaks))
        top = peaks[:8]
        assert np.array_equal(res.candidates, H[top]) and np.array_equal(res.candidate_scores, res.scores.ravel()[top])
        assert res.n_source == len(src)
        _check_refinement(reg, src, vmap, s, res)


@pytest.mark.gpu
def test_deterministic_read_only_and_rejections(K, O, small):
    from kiss_icp_b200 import _native as N
    vmap = _map(K, O, small, range(0, 20, 2), 1.0)
    before = vmap.dump()
    reg = K.Registration(500, 1e-4, 0)
    src = _source(O, small, 6.5, 1.0)
    s = _search(K, small.pose(6.5), hx=6, hy=6, step=0.5, n_yaw=8, yaw_step=0.05, top_k=6)
    a = reg.relocalize(src, vmap, s, return_scores=True)
    b = reg.relocalize(src, vmap, s, return_scores=True)
    same = lambda x, y: all(np.array_equal(getattr(x, f), getattr(y, f)) for f in x.__dataclass_fields__)
    assert same(a, b)
    assert all(np.array_equal(x, y) for x, y in zip(before, vmap.dump()))
    # while a localizer holds the map
    icp = K.KissICP(K.load_config(), prior_map=vmap)
    assert vmap.readers() == 1
    c = reg.relocalize(src, vmap, s, return_scores=True)
    assert same(a, c)
    del icp
    gc.collect()
    with pytest.raises(ValueError, match="empty source"):
        reg.relocalize(np.empty((0, 3)), vmap, s)
    with pytest.raises(ValueError, match="empty"):
        reg.relocalize(src, K.VoxelHashMap(1.0, 1e9, 20), s)
    far = np.eye(4)
    far[0, 3] = 3e9  # voxel coordinates beyond int
    with pytest.raises(ValueError, match="int range"):
        reg.relocalize(src, vmap, _search(K, far))
    bad = src.copy()
    bad[3, 1] = math.nan
    with pytest.raises(ValueError, match="not finite"):
        reg.relocalize(bad, vmap, s)
    # on error nothing is written; NULL handles are rejected
    ss, _ = s._struct()
    r = N.RelocResult()
    sc = np.full(s.shape, -7, dtype=np.int32)
    st = N.lib().kb_relocalize(reg._h, N.ptr(src), len(src), None, C.byref(ss), C.byref(r), None, None, N.ptr(sc))
    assert st == N.KB_ERR_INVALID_ARG and (sc == -7).all() and r.n_hypotheses == 0
    # odometry pipelines have no prior map to relocalize in
    with pytest.raises(ValueError, match="prior map"):
        K.KissICP(K.load_config()).relocalize(small.scan(3)[0], s)


@pytest.mark.gpu
def test_whole_grid_path_ouster_shape(K, O):
    """a source of more than 96 x 120 points: the refinement takes the whole-grid ICP path inside the batch"""
    import torch
    from kiss_icp_b200 import synthetic
    L = synthetic.ouster128_shape(seed=5, device="cuda" if torch.cuda.is_available() else "cpu")
    vmap = _map(K, O, L, range(0, 8), 0.3)
    src = O.voxel_down_sample(L.scan(3.5)[0], 0.15)
    assert len(src) > 96 * 120
    reg = K.Registration(500, 1e-4, 0)
    s = _search(K, L.pose(3.5), hx=2, hy=2, step=0.3, n_yaw=3, yaw_step=0.03, top_k=4, max_correspondence_distance=0.9,
                kernel_scale=0.3)
    res = reg.relocalize(src, vmap, s, return_scores=True)
    _check_refinement(reg, src, vmap, s, res)
    # the source is staged in chunks: the scores stay exact
    assert np.array_equal(res.scores.ravel(), _numpy_scores(s.hypotheses(), src, vmap))


# KITTI-shape recovery: a prior map of about 110 m of road, scans at k + 0.5 (none of them in the map), centres up to
# 12 m and any yaw away from the truth
POSITIONS = (20, 36, 52, 68, 84, 100)


@pytest.fixture(scope="module")
def kitti():
    import torch
    from kiss_icp_b200 import synthetic, _native as N
    if N.lib().kb_device_count() == 0:
        pytest.skip("no CUDA device")
    L = synthetic.kitti_shape(seed=0, device="cuda" if torch.cuda.is_available() else "cpu")
    import kiss_icp_b200 as K
    from oracle import oracle as O
    g, o = K.VoxelHashMap(1.0, 1e9, 20), O.VoxelHashMap(1.0, 1e9, 20)
    for k in range(0, 121):
        ds = O.voxel_down_sample(L.scan(k)[0], 0.5)
        g.update(ds, L.pose(k))
        o.update(ds, L.pose(k))
    return L, g, o


def _kitti_center(L, k, rng, flat=False):
    T = L.pose(k)
    dx, dy = rng.uniform(-12.0, 12.0, size=2)
    dyaw = rng.uniform(-math.pi, math.pi)
    C_ = T.copy()
    if flat:
        yaw = math.atan2(T[1, 0], T[0, 0])
        C_[:3, :3] = _rz(yaw + dyaw)
    else:
        C_[:3, :3] = _rz(dyaw) @ T[:3, :3]
    C_[:2, 3] += [dx, dy]
    return C_


@pytest.mark.gpu
def test_recovery_kitti_shape(K, O, kitti):
    L, vmap, _ = kitti
    reg = K.Registration(500, 1e-4, 0)
    rng = np.random.default_rng(21)
    report = []
    cases = [(k, False) for k in POSITIONS] + [(POSITIONS[2], True)]
    for k, flat in cases:
        truth = L.pose(k + 0.5)
        s = _search(K, _kitti_center(L, k + 0.5, rng, flat), hx=20, hy=20, step=1.0, n_yaw=72, yaw_step=math.radians(5.0),
                    top_k=16)
        res = reg.relocalize(_source(O, L, k + 0.5, 1.0), vmap, s)
        dt, dr = pose_error(res.pose, truth)
        report.append((k, flat, dt, math.degrees(dr), res.inliers, res.runner_up_inliers, res.n_source))
    bad = [r for r in report if not (r[2] < 0.1 and r[3] < 0.5 and r[4] > r[5])]
    assert not bad, report


def _oracle_localize(O, omap, cfg, scans, seed):
    """the reference's statement without local_map.update on the oracle's modules, from a new sequence's state"""
    v, th, reg = cfg.mapping.voxel_size, cfg.adaptive_threshold, cfg.registration
    pose, delta, sse, ns = np.array(seed, dtype=np.float64), np.eye(4), th.initial_threshold ** 2, 1
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
    return np.array(poses), np.array(iters)


def _close(A, B, tol=1e-9):
    return np.linalg.norm(A[:3, 3] - B[:3, 3]) < tol and np.abs(A[:3, :3] - B[:3, :3]).max() < tol


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False])
def test_localizer_relocalizes_then_tracks(K, O, kitti, fused):
    L, vmap, omap = kitti
    cfg = K.load_config()
    icp = K.KissICP(cfg, fused=fused, prior_map=vmap)
    assert np.array_equal(icp.last_pose, np.eye(4))
    k0 = 40
    s = _search(K, _kitti_center(L, k0 + 0.5, np.random.default_rng(5)), hx=20, hy=20, step=1.0, n_yaw=72,
                yaw_step=math.radians(5.0), top_k=16)
    p, t = L.scan(k0 + 0.5)
    sigma = 2.0  # a new sequence's threshold: initial_threshold
    res = icp.relocalize(p, s)
    dt, dr = pose_error(res.pose, L.pose(k0 + 0.5))
    assert dt < 0.1 and math.degrees(dr) < 0.5, (dt, dr)
    assert np.array_equal(icp.last_pose, res.pose) and np.array_equal(icp.last_delta, np.eye(4))
    # the search ran with (3 sigma, sigma): the same as Registration.relocalize with those thresholds
    reg = K.Registration(cfg.registration.max_num_iterations, cfg.registration.convergence_criterion, 0)
    pre = O.preprocess(p, np.empty(0), np.eye(4), cfg.data.max_range, cfg.data.min_range, False)
    src = O.voxel_down_sample(O.voxel_down_sample(pre, 0.5), 1.5)
    s3 = _search(K, s.center, hx=20, hy=20, step=1.0, n_yaw=72, yaw_step=math.radians(5.0), top_k=16,
                 max_correspondence_distance=3 * sigma, kernel_scale=sigma)
    ref = reg.relocalize(src, vmap, s3)
    assert np.array_equal(ref.pose, res.pose) and ref.inliers == res.inliers
    scans = [L.scan(k + 0.5) for k in range(k0 + 1, k0 + 31)]
    poses, iters = [], []
    for q, tq in scans:
        icp.register_frame(q, tq, return_clouds=False) if fused else icp.register_frame(q, tq)
        poses.append(icp.last_pose)
        iters.append(icp.last_iterations)
    rp, ri = _oracle_localize(O, omap, cfg, scans, res.pose)
    bad = [(k, it, ito) for k, (P, it, Po, ito) in enumerate(zip(poses, iters, rp, ri)) if not (_close(P, Po) and it == ito)]
    assert not bad, bad
