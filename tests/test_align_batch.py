"""Registration.align_points_to_map_batch / kb_registration_align_batch[_dev]: many AlignPointsToMap problems against
one map in one launch. Every hypothesis must return, bit for bit, what align_points_to_map returns for it alone."""
import ctypes as C

import numpy as np
import pytest

from conftest import pose_error


def _single(reg, clouds, vmap, guesses, md, ks):
    poses, iters = [], []
    for c, g, m, k in zip(clouds, guesses, md, ks):
        poses.append(reg.align_points_to_map(c, vmap, g, m, k))
        iters.append(reg.last_iterations)
    return np.array(poses).reshape(-1, 4, 4), np.array(iters)


def _map_by(pose, pts):
    return pts @ pose[:3, :3].T + pose[:3, 3]


@pytest.fixture(scope="module")
def lidar():
    from kiss_icp_b200 import synthetic
    return synthetic.small_shape(seed=1, beams=32, cols=512)


def _pair(K, O, lidar, n_scans):
    g, o = K.VoxelHashMap(1.0, 100.0, 20), O.VoxelHashMap(1.0, 100.0, 20)
    T0 = lidar.pose(0)
    for k in range(n_scans):
        p, _ = lidar.scan(k)
        ds = O.voxel_down_sample(p, 0.5)
        Tk = np.linalg.inv(T0) @ lidar.pose(k)
        g.update(ds, Tk)
        o.update(ds, Tk)
    return g, o


def _mixed(O, lidar):
    """~24 hypotheses: three scans of different sizes from several guesses each, per-hypothesis max_dist / kernel,
    n = 0 and n = 1, and one cloud above the team limit (96 x 120 points: the whole-grid path)"""
    rng = np.random.default_rng(7)
    T0inv = np.linalg.inv(lidar.pose(0))
    clouds, guesses = [], []
    tangents = ([0.3, -0.2, 0.05, 0.01, -0.01, 0.02], [0.0] * 6, [-0.5, 0.4, 0.0, 0.0, 0.0, -0.03],
                [1.0, -0.8, 0.1, 0.0, 0.02, 0.06], [-1.5, 1.2, 0.0, 0.01, 0.0, -0.08])
    for k, sub in ((5, 1), (6, 2), (7, 5)):
        src = O.voxel_down_sample(O.voxel_down_sample(lidar.scan(k)[0], 0.5), 1.5)[::sub]
        Tk = T0inv @ lidar.pose(k)
        for t in tangents:
            clouds.append(src)
            guesses.append(Tk @ O.se3_exp(t))
    T5 = T0inv @ lidar.pose(5)
    clouds += [np.empty((0, 3)), clouds[0][:1], clouds[0][:7]]
    guesses += [T5, T5 @ O.se3_exp([0.1, 0, 0, 0, 0, 0]), T5]
    big = np.concatenate([O.se3_act(T0inv @ lidar.pose(k), lidar.scan(k)[0]) for k in range(5, 8)])
    big = big[rng.permutation(len(big))[:12000]]  # > 96 x 120 source points
    clouds += [big, big[:600]]
    guesses += [O.se3_exp([0.2, -0.1, 0, 0, 0, 0.01]), O.se3_exp([0.1, 0, 0, 0, 0, 0])]
    B = len(clouds)
    md = 3.0 + 0.25 * (np.arange(B) % 3)
    ks = 1.0 - 0.1 * (np.arange(B) % 4)
    return clouds, np.array(guesses), md, ks


@pytest.mark.gpu
def test_batch_bit_identical_to_single_calls_and_close_to_oracle(K, O, lidar):
    g, o = _pair(K, O, lidar, 5)
    clouds, guesses, md, ks = _mixed(O, lidar)
    reg = K.Registration(500, 1e-4, 0)
    Ps, its = _single(reg, clouds, g, guesses, md, ks)
    Pb, itb = reg.align_points_to_map_batch(clouds, g, guesses, md, ks)
    assert np.array_equal(Pb, Ps) and np.array_equal(itb, its)
    assert reg.last_iterations == its[-1]
    # one cloud with overlapping / repeated ranges gives the same bits
    flat = np.concatenate([clouds[0], clouds[5]])
    n0, n1 = len(clouds[0]), len(clouds[5])
    ranges = np.array([[0, n0], [n0, n1], [0, n0], [3, n0 - 3], [n0 - 10, 20], [0, n0 + n1]])
    sub = [flat[a:a + c] for a, c in ranges]
    G = guesses[[0, 5, 1, 2, 3, 4]]
    Pr, itr = reg.align_points_to_map_batch(flat, g, G, 3.0, 1.0, ranges=ranges)
    Ps2, its2 = _single(reg, sub, g, G, [3.0] * 6, [1.0] * 6)
    assert np.array_equal(Pr, Ps2) and np.array_equal(itr, its2)
    # against the oracle, like test_align_points_to_map_matches_oracle. (Not for a single point: its 6x6 system has rank
    # 3, and the pivoted solve of a singular system turns summation-order noise into a different step.)
    bad = []
    for b, (c, G1, m, k, P, it) in enumerate(zip(clouds, guesses, md, ks, Pb, itb)):
        if len(c) == 1:
            continue
        Po, ito = O.align_points_to_map(o, c, G1, m, k)
        dt, dr = pose_error(P, Po)
        if not (dt < 1e-9 and dr < 1e-9 and it == ito):
            bad.append((b, len(c), dt, dr, int(it), ito))
    assert not bad, bad


@pytest.mark.gpu
def test_more_hypotheses_than_slots_with_unequal_lengths(K, O):
    """KITTI shape, B = 40: guesses that converge early next to far-off ones that run to max_num_iterations; slot reuse
    and tag reservation across two consecutive batch calls"""
    import torch
    from kiss_icp_b200 import synthetic
    L = synthetic.kitti_shape(seed=0, device="cuda" if torch.cuda.is_available() else "cpu")
    icp = K.KissICP(K.load_config())
    for k in range(6):
        p, t = L.scan(k)
        _, src = icp.register_frame(p, t)
    pose = icp.last_pose
    rng = np.random.default_rng(11)
    guesses = []
    for b in range(40):
        scale = 0.05 if b % 3 else 3.0  # every third one far off
        guesses.append(pose @ O.se3_exp(np.concatenate([rng.normal(size=3) * scale, rng.normal(size=3) * scale * 0.05])))
    guesses = np.array(guesses)
    reg = K.Registration(20, 1e-4, 0)
    P1, it1 = reg.align_points_to_map_batch(src, icp.local_map, guesses, 3.0, 1.0)
    P2, it2 = reg.align_points_to_map_batch(src, icp.local_map, guesses, 3.0, 1.0)
    Ps, its = _single(reg, [src] * 40, icp.local_map, guesses, [3.0] * 40, [1.0] * 40)
    assert (its == 20).any() and (its < 20).any()
    assert np.array_equal(P1, Ps) and np.array_equal(P2, Ps)
    assert np.array_equal(it1, its) and np.array_equal(it2, its)


@pytest.mark.gpu
def test_batch_degenerate_cases(K, O):
    rng = np.random.default_rng(3)
    reg = K.Registration(500, 1e-4, 0)
    guess = O.se3_exp([1, 2, 3, 0.1, 0.2, 0.3])
    G = np.array([guess, guess @ O.se3_exp([0.1, 0, 0, 0, 0, 0])])
    src = rng.normal(size=(50, 3))
    empty = K.VoxelHashMap(1.0, 100.0, 20)
    P, it = reg.align_points_to_map_batch(src, empty, G, 3.0, 1.0)
    Ps, its = _single(reg, [src, src], empty, G, [3.0] * 2, [1.0] * 2)
    assert np.array_equal(P, Ps) and np.array_equal(it, its) and (it == 0).all()
    assert np.allclose(P[0], guess, atol=1e-15)
    far = K.VoxelHashMap(1.0, 1e9, 20)
    far.add_points(rng.normal(size=(100, 3)) + 1000.0)
    P, it = reg.align_points_to_map_batch([src, np.empty((0, 3))], far, G, 3.0, 1.0)
    Ps, its = _single(reg, [src, np.empty((0, 3))], far, G, [3.0] * 2, [1.0] * 2)
    assert np.array_equal(P, Ps) and np.array_equal(it, its) and (it == 1).all()
    assert np.allclose(P[0], guess, atol=1e-15)
    near = K.VoxelHashMap(1.0, 100.0, 20)
    near.add_points(src + 0.05)
    reg1 = K.Registration(1, 1e-4, 0)
    P, it = reg1.align_points_to_map_batch(src, near, G, 3.0, 1.0)
    Ps, its = _single(reg1, [src, src], near, G, [3.0] * 2, [1.0] * 2)
    assert np.array_equal(P, Ps) and np.array_equal(it, its) and (it == 1).all()
    P, it = reg.align_points_to_map_batch(src, near, np.empty((0, 4, 4)), 3.0, 1.0)
    assert P.shape == (0, 4, 4) and it.shape == (0,)


@pytest.mark.gpu
def test_batch_validation_writes_nothing(K, O):
    from kiss_icp_b200 import _native as N
    rng = np.random.default_rng(4)
    vmap = K.VoxelHashMap(1.0, 100.0, 20)
    pts = rng.normal(size=(200, 3)) * 5
    vmap.add_points(pts)
    reg = K.Registration(500, 1e-4, 0)
    G = np.array([np.eye(4)] * 4)
    G[2] = np.diag([1.0, 1.0, -1.0, 1.0])
    with pytest.raises(ValueError):
        reg.align_points_to_map_batch(pts, vmap, G, 3.0, 1.0)
    with pytest.raises(IndexError):
        reg.align_points_to_map_batch(pts, vmap, np.array([np.eye(4)] * 2), 3.0, 1.0, ranges=[[0, 10], [150, 51]])
    # the C-ABI: sentinel-filled outputs stay untouched on every rejected call
    L = N.lib()
    off = np.array([0, 10, 20, 30], dtype=np.uint64)
    cnt = np.array([10, 10, 10, 10], dtype=np.uint64)
    md, ks = np.full(4, 3.0), np.ones(4)
    for guesses, o, c, status in ((G, off, cnt, N.KB_ERR_NOT_SE3),
                                  (np.array([np.eye(4)] * 4), off, np.array([10, 10, 10, 171], dtype=np.uint64), N.KB_ERR_INVALID_ARG),
                                  (np.array([np.eye(4)] * 4), np.array([0, 10, 201, 30], dtype=np.uint64), cnt, N.KB_ERR_INVALID_ARG)):
        poses = np.full((4, 4, 4), -7.0)
        iters = np.full(4, -7, dtype=np.int32)
        inl = np.full(4, -7, dtype=np.int32)
        st = L.kb_registration_align_batch(reg._h, N.ptr(pts), len(pts), N.ptr(o), N.ptr(c), 4, vmap._h, N.ptr(guesses),
                                           N.ptr(md), N.ptr(ks), N.ptr(poses), N.ptr(iters), N.ptr(inl))
        assert st == status
        assert (poses == -7.0).all() and (iters == -7).all() and (inl == -7).all()


@pytest.mark.gpu
def test_batch_inliers_equal_build_system(K, O, lidar):
    g, _ = _pair(K, O, lidar, 5)
    clouds, guesses, md, ks = _mixed(O, lidar)
    reg = K.Registration(500, 1e-4, 0)
    P, it, inl = reg.align_points_to_map_batch(clouds, g, guesses, md, ks, return_inliers=True)
    for c, Pb, m, k, n in zip(clouds, P, md, ks, inl):
        assert n == reg.build_system(_map_by(Pb, c), g, m, k)[2]
    assert inl[:5].min() > 100


@pytest.mark.gpu
def test_batch_device_tensors_equal_host_arrays(K, O, lidar):
    import torch
    g, _ = _pair(K, O, lidar, 5)
    clouds, guesses, md, ks = _mixed(O, lidar)
    reg = K.Registration(500, 1e-4, 0)
    P, it, inl = reg.align_points_to_map_batch(clouds, g, guesses, md, ks, return_inliers=True)
    dev = [torch.as_tensor(c, device="cuda") for c in clouds]
    Pd, itd, inld = reg.align_points_to_map_batch(dev, g, torch.as_tensor(guesses, device="cuda"), torch.as_tensor(md),
                                                 torch.as_tensor(ks), return_inliers=True)
    assert Pd.is_cuda and itd.is_cuda and inld.is_cuda
    assert np.array_equal(Pd.cpu().numpy(), P) and np.array_equal(itd.cpu().numpy(), it)
    assert np.array_equal(inld.cpu().numpy(), inl)
    flat = torch.as_tensor(np.concatenate(clouds[:5]), device="cuda")
    Pf, itf = reg.align_points_to_map_batch(flat, g, torch.as_tensor(guesses[:5], device="cuda"), 3.0, 1.0,
                                            ranges=np.array([[0, len(clouds[0])]] * 5))
    Ph, ith = reg.align_points_to_map_batch(clouds[:5], g, guesses[:5], 3.0, 1.0)
    assert np.array_equal(Pf.cpu().numpy(), Ph) and np.array_equal(itf.cpu().numpy(), ith)


@pytest.mark.gpu
def test_batch_does_not_disturb_a_pipeline(K, O):
    """a batch against a pipeline's own map (its scratch and tag sequence) between scans changes nothing"""
    from kiss_icp_b200 import synthetic
    L = synthetic.small_shape(seed=5, beams=32, cols=512)
    a, b = K.KissICP(K.load_config()), K.KissICP(K.load_config())
    pa, pb = [], []
    for k in range(30):
        p, t = L.scan(k)
        a.register_frame(p, t, return_clouds=False)
        _, src = b.register_frame(p, t)
        pa.append(a.last_pose)
        pb.append(b.last_pose)
    reg = K.Registration(500, 1e-4, 0)
    G = np.array([b.last_pose @ O.se3_exp([0.2 * i, -0.1 * i, 0, 0, 0, 0.01 * i]) for i in range(8)])
    reg.align_points_to_map_batch(src, b.local_map, G, 3.0, 1.0, return_inliers=True)
    for k in range(30, 60):
        p, t = L.scan(k)
        a.register_frame(p, t, return_clouds=False)
        b.register_frame(p, t, return_clouds=False)
        pa.append(a.last_pose)
        pb.append(b.last_pose)
    assert np.array_equal(np.array(pa), np.array(pb))
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys() and all(np.array_equal(sa[k], sb[k], equal_nan=True) for k in sa)


@pytest.mark.gpu
def test_relocalization_on_a_loaded_prior_map(K, O):
    """restore a map from a state_dict(), align scan k from a 5 x 5 grid of planar offsets, pick by inliers. The gate and
    kernel are fixed (1.0 m, 0.3 m) so that the inlier count separates converged hypotheses from the others; the true
    pose is the single call's answer from the pipeline's own pose. (With this gate and kernel instead of the pipeline's
    adaptive threshold, the optimum moves by centimetres.)"""
    from kiss_icp_b200 import synthetic
    L = synthetic.kitti_shape(seed=2)
    icp = K.KissICP(K.load_config())
    k = 8
    for j in range(k):
        p, t = L.scan(j)
        icp.register_frame(p, t, return_clouds=False)
    state = icp.state_dict()
    p, t = L.scan(k)
    _, src = icp.register_frame(p, t)
    reg = K.Registration(500, 1e-4, 0)
    prior = K.VoxelHashMap(1.0, 100.0, 20)
    prior.load(state["voxels"], state["counts"], state["points"])
    offs = np.array([-0.5, -0.25, 0.0, 0.25, 0.5])
    G = []
    for dx in offs:
        for dy in offs:
            T = icp.last_pose.copy()
            T[0, 3] += dx
            T[1, 3] += dy
            G.append(T)
    truth = reg.align_points_to_map(src, prior, icp.last_pose, 1.0, 0.3)
    P, it, inl = reg.align_points_to_map_batch(src, prior, np.array(G), 1.0, 0.3, return_inliers=True)
    best = int(np.argmax(inl))
    dt, dr = pose_error(P[best], truth)
    assert dt < 1e-4 and dr < 1e-4, (best, inl, it, dt, dr)
    dt, dr = pose_error(truth, icp.last_pose)
    assert dt < 0.2 and dr < 0.02


def test_batch_entry_points_without_device_and_null_arguments():
    """CPU: the entry points exist; without a device creating the handles fails with KB_ERR_NO_DEVICE, and NULL
    handles are rejected"""
    from kiss_icp_b200 import _native as N
    L = N.lib()
    for name in ("kb_registration_align_batch", "kb_registration_align_batch_dev"):
        fn = getattr(L, name)
        st = fn(None, None, 0, None, None, 1, None, None, None, None, None, None, None)
        assert st == N.KB_ERR_INVALID_ARG
    if L.kb_device_count() == 0:
        h = N.vp()
        assert L.kb_registration_create(500, 1e-4, 0, C.byref(h)) == N.KB_ERR_NO_DEVICE
        m = N.vp()
        assert L.kb_map_create(1.0, 100.0, 20, C.byref(m)) == N.KB_ERR_NO_DEVICE
