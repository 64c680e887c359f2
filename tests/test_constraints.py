"""Plane constraints (kb_registration_constraints, kb_pipeline_set_constraint_reporting, KissICP(report_constraints=True)):
which directions a registration pins down, from the planes of the map's voxels. Restated here in numpy; checked on
analytic scenes (corridor, room, floor); reporting changes no pose, fit or map."""
import ctypes as C

import numpy as np
import pytest


# ---------------------------------------------------------------------------------------------- numpy restatement
def _numpy_constraints(vmap, voxel_size, src, pose, max_dist, centre=None):
    """the definition, from closest_neighbors (bit-exact q) and the map's dump(); with a centre c, the lever about it:
    J = [n, (p - c) x n], summed directly (A^T H A from the sum about the origin cancels digits far from it)"""
    p = src @ pose[:3, :3].T + pose[:3, 3]
    q, d = vmap.closest_neighbors(p)
    vox, cnt, pts = vmap.dump()
    start = np.concatenate([[0], np.cumsum(cnt)])
    index = {tuple(v): i for i, v in enumerate(vox)}
    n_planes, W, S, H = 0, 0.0, 0.0, np.zeros((6, 6))
    for i in np.nonzero(d < max_dist)[0]:
        k = index[tuple(np.floor(q[i] / voxel_size).astype(np.int64))]
        X = pts[start[k]:start[k + 1]]
        if len(X) < 3:
            continue
        n_planes += 1
        mu = X.mean(0)
        D = X - mu
        lam, V = np.linalg.eigh(D.T @ D / len(X))
        a = (lam[1] - lam[0]) / lam[2] if lam[2] > 0 else 0.0
        n = V[:, 0]
        e = n @ (p[i] - q[i])
        J = np.concatenate([n, np.cross(p[i] if centre is None else p[i] - centre, n)])
        W += a
        S += a * e * e
        H += a * np.outer(J, J)
    return n_planes, W, S, H


def _raw(reg, src, vmap, pose, max_dist):
    from kiss_icp_b200 import _native as N
    c = N.Constraints()
    pts = N.points_arg(src)
    T = np.ascontiguousarray(pose, dtype=np.float64)
    N.check(N.lib().kb_registration_constraints(reg._h, N.ptr(pts), len(pts), vmap._h, N.ptr(T), float(max_dist),
                                                C.byref(c)))
    return c.n_planes, c.weight_sum, c.sum_sq_plane_residual, np.array(c.information[:]).reshape(6, 6)


def _assert_matches(got, ref):
    n, W, S, H = got
    n0, W0, S0, H0 = ref
    assert n == n0
    assert np.array_equal(H, H.T)
    assert np.abs(H - H0).max() <= 1e-10 * max(np.abs(H0).max(), 1e-300)
    assert abs(W - W0) <= 1e-12 * max(W0, 1e-300)
    assert abs(S - S0) <= 1e-12 * max(S0, 1e-300)


def _stream(stamps="none", seed=3):
    from kiss_icp_b200 import synthetic
    return synthetic.small_shape(seed=seed, beams=32, cols=512, stamps=stamps)


def _perturbed(pose, rng, t=0.1, r=0.01):
    from scipy.spatial.transform import Rotation
    D = np.eye(4)
    D[:3, :3] = Rotation.from_rotvec(rng.normal(0, r, 3)).as_matrix()
    D[:3, 3] = rng.normal(0, t, 3)
    return pose @ D


def _built_map(K, cfg, n_scans=8, seed=3):
    """an odometry run's map and a later scan's source with its pose"""
    L = _stream(seed=seed)
    icp = K.KissICP(cfg)
    for k in range(n_scans):
        icp.register_frame(*L.scan(k), return_clouds=False)
    _, src = icp.register_frame(*L.scan(n_scans))
    return icp, src, icp.last_pose


@pytest.mark.gpu
@pytest.mark.parametrize("max_points", [20, 33, 100])
def test_against_numpy(K, max_points):
    cfg = K.load_config(mapping__max_points_per_voxel=max_points)
    icp, src, pose = _built_map(K, cfg)
    reg = K.Registration(500, 1e-4, 0)
    vs = cfg.mapping.voxel_size
    rng = np.random.default_rng(max_points)
    T = _perturbed(pose, rng)
    got = _raw(reg, src, icp.local_map, T, 1.0)
    ref = _numpy_constraints(icp.local_map, vs, src, T, 1.0)
    assert ref[0] > 200
    _assert_matches(got, ref)
    # run to run: bit for bit
    again = _raw(reg, src, icp.local_map, T, 1.0)
    assert got[:3] == again[:3] and np.array_equal(got[3], again[3])
    c = reg.constraints(src, icp.local_map, T, 1.0)
    assert c.n_planes == got[0] and c.weight_sum == got[1] and np.array_equal(c.information, got[3])
    assert c.plane_rmse == np.sqrt(got[2] / got[1])


@pytest.mark.gpu
def test_sparse_empty_and_invalid(K):
    reg = K.Registration(500, 1e-4, 0)
    rng = np.random.default_rng(5)
    # voxels of 1 or 2 points: no plane terms
    vm = K.VoxelHashMap(1.0, 1000.0, 20)
    base = rng.integers(-20, 20, size=(300, 3)).astype(np.float64)
    base = np.unique(base, axis=0)
    pts = np.concatenate([base + 0.3, base[::2] + 0.6])
    vm.add_points(pts)
    src = pts[:100] + 0.01
    n, W, S, H = _raw(reg, src, vm, np.eye(4), 1.0)
    assert n == 0 and W == 0 and S == 0 and not H.any()
    c = reg.constraints(src, vm, np.eye(4), 1.0)
    assert np.isnan(c.plane_rmse) and K.covariance(c) is None
    # empty map, n = 0
    empty = K.VoxelHashMap(1.0, 1000.0, 20)
    assert _raw(reg, src, empty, np.eye(4), 1.0)[0] == 0 and not _raw(reg, src, empty, np.eye(4), 1.0)[3].any()
    n, W, S, H = _raw(reg, np.empty((0, 3)), vm, np.eye(4), 1.0)
    assert n == 0 and W == 0 and not H.any()
    bad = np.eye(4)
    bad[0, 0] = 2.0
    with pytest.raises(ValueError):
        reg.constraints(src, vm, bad, 1.0)


# ---------------------------------------------------------------------------------------------- geometry
def _grid(u, v):
    return np.stack(np.meshgrid(u, v, indexing="ij"), -1).reshape(-1, 2)


def _corridor():
    """floor z = 0, walls y = +-2, x in [-40, 40). The walls start 1 m above the floor, so that no voxel holds two
    surfaces: the points the map keeps of an edge voxel are an irregular subset of an L, whose normal would tilt along x"""
    s = np.arange(-40, 40, 0.1)
    h = np.arange(-2, 2, 0.1)
    floor = _grid(s, h)
    floor = np.column_stack([floor, np.zeros(len(floor))])
    z = np.arange(1.05, 3, 0.1)
    wall = _grid(s, z)
    walls = [np.column_stack([wall[:, 0], np.full(len(wall), y), wall[:, 1]]) for y in (-2.0, 2.0)]
    return np.concatenate([floor] + walls)


def _room():
    """a closed box room with two boxes on the floor"""
    out = []
    g = np.arange(-10, 10.001, 0.1)
    h = np.arange(0, 4.001, 0.1)
    fl = _grid(g, g)
    out += [np.column_stack([fl, np.zeros(len(fl))]), np.column_stack([fl, np.full(len(fl), 4.0)])]
    w = _grid(g, h)
    for c in (-10.0, 10.0):
        out += [np.column_stack([np.full(len(w), c), w]), np.column_stack([w[:, 0], np.full(len(w), c), w[:, 1]])]
    for cx, cy in ((3.0, -4.0), (-5.0, 6.0)):
        b = _grid(np.arange(-1, 1.001, 0.1), np.arange(0, 1.001, 0.1))
        out += [np.column_stack([np.full(len(b), cx + s), cy + b[:, 0], b[:, 1]]) for s in (-1.0, 1.0)]
        out += [np.column_stack([cx + b[:, 0], np.full(len(b), cy + s), b[:, 1]]) for s in (-1.0, 1.0)]
    return np.concatenate(out)


def _constraints_on(K, cloud, rng):
    vm = K.VoxelHashMap(1.0, 1000.0, 20)
    vm.add_points(cloud)
    src = cloud[rng.choice(len(cloud), size=min(len(cloud), 6000), replace=False)] + rng.normal(0, 0.005, (min(len(cloud), 6000), 3))
    return K.Registration(500, 1e-4, 0).constraints(src, vm, np.eye(4), 0.5)


@pytest.mark.gpu
def test_corridor_leaves_its_axis_free(K):
    c = _constraints_on(K, _corridor(), np.random.default_rng(0))
    d = K.degeneracy(c)
    lt = d.translation_eigenvalues
    assert lt[0] < 1e-9 * lt[2]
    assert abs(abs(d.translation_axes[0, 0]) - 1) < 1e-9
    assert K.covariance(c) is None


@pytest.mark.gpu
def test_room_is_well_conditioned(K):
    c = _constraints_on(K, _room(), np.random.default_rng(1))
    lt = K.degeneracy(c).translation_eigenvalues
    assert lt[0] >= 0.05 * lt[2]
    cov = K.covariance(c)
    assert cov is not None and np.all(np.linalg.eigvalsh(cov) > 0)


@pytest.mark.gpu
def test_floor_leaves_rotation_about_z_free(K):
    fl = _grid(np.arange(-20, 20, 0.1), np.arange(-20, 20, 0.1))
    c = _constraints_on(K, np.column_stack([fl, np.zeros(len(fl))]), np.random.default_rng(2))
    d = K.degeneracy(c)
    lr = d.rotation_eigenvalues
    assert lr[0] < 1e-9 * lr[2]
    assert abs(abs(d.rotation_axes[2, 0]) - 1) < 1e-9


@pytest.mark.gpu
def test_kitti_shape_stream_is_well_conditioned(K):
    L = _stream(seed=3)
    icp = K.KissICP(K.load_config(), report_constraints=True)
    assert icp.report_fit and icp.report_constraints
    scans = [L.scan(k) for k in range(30)]
    _, cons = icp.register_frames([p for p, _ in scans], [t for _, t in scans], return_constraints=True)
    ratios = []
    for k in range(1, len(scans)):
        H = cons.information[k]
        lt = np.linalg.eigvalsh(H[:3, :3])
        ratios.append(lt[0] / lt[2])
    print(f"smallest translational eigenvalue ratio over the stream: {min(ratios):.4f}")
    assert min(ratios) > 0.01


# ---------------------------------------------------------------------------------------------- pipelines
def _blocking(icp, scans):
    out = {"poses": [], "iters": [], "sigma": [], "fits": [], "cons": []}
    for p, t in scans:
        icp.register_frame(p, t, return_clouds=False)
        out["poses"].append(icp.last_pose)
        out["iters"].append(icp.last_iterations)
        out["sigma"].append(icp.last_sigma)
        if icp.report_fit:
            out["fits"].append(icp.last_fit)
        if icp.report_constraints:
            out["cons"].append(icp.last_constraints)
    return out


def _same(a, b):
    return all(np.array_equal(np.asarray(x), np.asarray(y), equal_nan=True) for x, y in zip(a, b))


def _stack_cons(cs):
    return (np.array([c.n_planes for c in cs]), np.array([c.weight_sum for c in cs]),
            np.array([c.plane_rmse for c in cs]), np.array([c.information for c in cs]))


def _same_map(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a.dump(), b.dump()))


def _prior(K, cfg, n=20, seed=3):
    L = _stream(seed=seed)
    icp = K.KissICP(cfg)
    poses = []
    for k in range(n):
        icp.register_frame(*L.scan(k), return_clouds=False)
        poses.append(icp.last_pose)
    c = cfg.mapping
    prior = K.VoxelHashMap(c.voxel_size, 1e4, c.max_points_per_voxel)
    prior.load(*icp.local_map.dump())
    return prior, L, poses


@pytest.mark.gpu
def test_localizer(K):
    cfg = K.load_config()
    prior, L, odo = _prior(K, cfg)
    scans = [L.scan(k) for k in range(2, 18)]
    a = K.KissICP(cfg, prior_map=prior)
    b = K.KissICP(cfg, prior_map=prior, report_constraints=True)
    for icp in (a, b):
        icp.last_pose = odo[1]
    ra, rb = _blocking(a, scans), _blocking(b, scans)
    for key in ("poses", "iters", "sigma"):
        assert np.array_equal(np.array(ra[key]), np.array(rb[key])), key
    assert all(_same(x, y) for x, y in zip(ra["fits"], rb["fits"]))
    # the last frame's constraints equal the stand-alone call at the reported pose, to rounding (the call rebuilds the
    # pose's quaternion from the matrix)
    reg = K.Registration(500, 1e-4, 0)
    _, src = b.register_frame(*scans[-1])
    c = b.last_constraints
    s = reg.constraints(src, prior, b.last_pose, 3 * b.last_sigma)
    assert c.n_planes == s.n_planes and c.n_planes > 100
    assert np.abs(c.information - s.information).max() <= 1e-10 * np.abs(s.information).max()
    assert abs(c.weight_sum - s.weight_sum) <= 1e-10 * s.weight_sum
    # queued equals blocking, bit for bit
    q = K.KissICP(cfg, prior_map=prior, report_constraints=True)
    q.last_pose = odo[1]
    pq, fq, cq = q.register_frames([p for p, _ in scans], [t for _, t in scans], return_fits=True,
                                   return_constraints=True)
    assert np.array_equal(pq, np.array(rb["poses"]))
    assert _same(cq, _stack_cons(rb["cons"]))
    assert _same(q.last_constraints, rb["cons"][-1])


@pytest.mark.gpu
@pytest.mark.parametrize("stamps", ["none", "column"])
def test_odometry_changes_nothing_and_is_pre_update(K, stamps):
    L = _stream(stamps, seed=7)
    scans = [L.scan(k) for k in range(30)]
    cfg = K.load_config()
    a, b = K.KissICP(cfg, report_fit=True), K.KissICP(cfg, report_constraints=True)
    ra = _blocking(a, scans)
    reg = K.Registration(500, 1e-4, 0)
    c = cfg.mapping
    rb = {"poses": [], "iters": [], "sigma": [], "fits": [], "cons": []}
    for k, (p, t) in enumerate(scans):
        before = K.VoxelHashMap(c.voxel_size, cfg.data.max_range, c.max_points_per_voxel)
        vox, cnt, pts = b.local_map.dump()
        if len(vox):
            before.load(vox, cnt, pts)
        _, src = b.register_frame(p, t)
        for key, v in (("poses", b.last_pose), ("iters", b.last_iterations), ("sigma", b.last_sigma),
                       ("fits", b.last_fit), ("cons", b.last_constraints)):
            rb[key].append(v)
        if k in (0, 5, 29):
            s = reg.constraints(src, before, b.last_pose, 3 * b.last_sigma)
            cc = b.last_constraints
            assert cc.n_planes == s.n_planes and (k == 0 or cc.n_planes > 100)
            assert np.abs(cc.information - s.information).max() <= 1e-10 * max(np.abs(s.information).max(), 1e-300)
    for key in ("poses", "iters", "sigma"):
        assert np.array_equal(np.array(ra[key]), np.array(rb[key])), key
    assert all(_same(x, y) for x, y in zip(ra["fits"], rb["fits"]))
    assert _same_map(a.local_map, b.local_map)
    sa, sb = a.state_dict(), b.state_dict()
    assert all(sa[k].tobytes() == sb[k].tobytes() for k in sa)
    # queued, bit for bit with blocking
    q = K.KissICP(cfg, report_constraints=True)
    pq, fq, cq = q.register_frames([p for p, _ in scans], [t for _, t in scans], return_fits=True,
                                   return_constraints=True)
    assert np.array_equal(pq, np.array(rb["poses"]))
    assert _same(cq, _stack_cons(rb["cons"]))
    assert _same_map(q.local_map, b.local_map)


@pytest.mark.gpu
def test_odometry_whole_grid_path_and_veto(K, monkeypatch):
    L = _stream(seed=5)
    scans = [L.scan(k) for k in range(8)]
    cfg = K.load_config(mapping__max_points_per_voxel=33)
    a, b = K.KissICP(cfg, report_fit=True), K.KissICP(cfg, report_constraints=True)
    b.start_history(3)
    ra, rb = _blocking(a, scans), _blocking(b, scans)
    assert all(h.team == 0 for h in b.history())
    assert np.array_equal(np.array(ra["poses"]), np.array(rb["poses"]))
    assert all(_same(x, y) for x, y in zip(ra["fits"], rb["fits"]))
    assert rb["cons"][-1].n_planes > 100
    # a capacity veto inside the queue: the replay's constraints
    rng = np.random.default_rng(0)
    frames = [rng.uniform(-150, 150, size=(30000, 3)) * [1.0, 1.0, 0.2] for _ in range(4)]
    vscans = [(p, np.empty(0)) for p in frames]
    vcfg = K.load_config(max_range=300.0, voxel_size=1.0)
    reserved = K.KissICP(vcfg, report_constraints=True)
    ref = _blocking(reserved, vscans)
    assert reserved.grow_retries() == 0
    monkeypatch.setenv("KB_MAP_RESERVE_SLOTS", "0")
    v = K.KissICP(vcfg, report_constraints=True)
    pv, _, cv = v.register_frames([p for p, _ in vscans], [t for _, t in vscans], return_fits=True,
                                  return_constraints=True)
    assert v.grow_retries() >= 1
    assert np.array_equal(pv, np.array(ref["poses"]))
    assert _same(cv, _stack_cons(ref["cons"]))


@pytest.mark.gpu
def test_switching_rules_and_grid_sizes(K):
    from kiss_icp_b200 import _native as N
    Lb = N.lib()
    L = _stream(seed=13)
    scans = [L.scan(k) for k in range(12)]
    cfg = K.load_config()
    plain = K.KissICP(cfg)
    ref = _blocking(plain, scans)
    icp = K.KissICP(cfg)
    h = icp._h
    c = N.Constraints()
    assert Lb.kb_pipeline_set_constraint_reporting(h, 1) == N.KB_ERR_INVALID_ARG  # no fits
    assert Lb.kb_pipeline_last_constraints(h, C.byref(c)) == N.KB_ERR_INVALID_ARG
    assert Lb.kb_pipeline_set_constraint_reporting(None, 1) == N.KB_ERR_INVALID_ARG
    assert Lb.kb_pipeline_last_constraints(h, None) == N.KB_ERR_INVALID_ARG
    assert Lb.kb_pipeline_set_fit_reporting(h, 1) == 0
    assert Lb.kb_pipeline_set_constraint_reporting(h, 1) == 0
    assert Lb.kb_pipeline_set_constraint_reporting(h, 1) == 0  # no-op
    assert Lb.kb_pipeline_last_constraints(h, C.byref(c)) == 0 and c.n_planes == 0 and not any(c.information)
    assert Lb.kb_pipeline_set_fit_reporting(h, 0) == N.KB_ERR_INVALID_ARG  # plane reporting needs the fits
    poses = []
    for k, (p, t) in enumerate(scans):
        if k == 4:
            assert Lb.kb_pipeline_set_constraint_reporting(h, 0) == 0
            assert Lb.kb_pipeline_last_constraints(h, C.byref(c)) == N.KB_ERR_INVALID_ARG
        if k == 8:
            assert Lb.kb_pipeline_set_constraint_reporting(h, 1) == 0
        icp.register_frame(p, t, return_clouds=False)
        poses.append(icp.last_pose)
    assert np.array_equal(np.array(poses), np.array(ref["poses"]))
    assert Lb.kb_pipeline_last_constraints(h, C.byref(c)) == 0 and c.n_planes > 100
    # a non-NULL constraints_out without reporting
    X = (C.c_void_p * 1)(None)
    n = (N.sz * 1)(0)
    assert Lb.kb_pipeline_register_frames_constraints(plain._h, X, n, None, None, 1, 0, None, None, C.byref(c)) == \
        N.KB_ERR_INVALID_ARG
    with pytest.raises(ValueError):
        _ = plain.last_constraints
    with pytest.raises(ValueError):
        plain.register_frames([scans[0][0]], return_constraints=True)
    # two grid sizes agree to rounding
    icp2, src, pose = _built_map(K, cfg)
    reg = K.Registration(500, 1e-4, 0)
    full = _raw(reg, src, icp2.local_map, pose, 1.0)
    assert Lb.kb_set_grid_blocks(40) == 0
    try:
        m2 = K.VoxelHashMap(cfg.mapping.voxel_size, cfg.data.max_range, cfg.mapping.max_points_per_voxel)
        m2.load(*icp2.local_map.dump())
        part = _raw(reg, src, m2, pose, 1.0)
    finally:
        Lb.kb_set_grid_blocks(0)
    assert full[0] == part[0]
    assert np.abs(full[3] - part[3]).max() <= 1e-12 * np.abs(full[3]).max()
    assert abs(full[1] - part[1]) <= 1e-12 * full[1] and abs(full[2] - part[2]) <= 1e-12 * full[2]


def test_entry_points_without_device():
    """CPU: the entry points exist and reject NULL arguments before any work"""
    from kiss_icp_b200 import _native as N
    L = N.lib()
    c = N.Constraints()
    assert L.kb_pipeline_set_constraint_reporting(None, 1) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_last_constraints(None, C.byref(c)) == N.KB_ERR_INVALID_ARG
    assert L.kb_registration_constraints(None, None, 0, None, None, 1.0, C.byref(c)) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_register_frames_constraints(None, None, None, None, None, 0, 0, None, None, None) == \
        N.KB_ERR_INVALID_ARG
    assert L.kb_debug_sym3_eig(None, None, None) == N.KB_ERR_INVALID_ARG


def test_degeneracy_and_covariance_helpers():
    import kiss_icp_b200 as K
    H = np.diag([4.0, 2.0, 1e-14, 3.0, 3.0, 3.0])
    c = K.Constraints(10, 5.0, 0.1, H)
    d = K.degeneracy(c)
    assert np.allclose(d.translation_eigenvalues, [1e-14, 2.0, 4.0]) and abs(d.translation_axes[2, 0]) == 1.0
    assert K.covariance(c) is None
    c = K.Constraints(10, 5.0, 0.1, np.diag([4.0, 2.0, 1.0, 3.0, 3.0, 3.0]))
    assert np.allclose(K.covariance(c), 0.01 * np.diag([0.25, 0.5, 1.0, 1 / 3, 1 / 3, 1 / 3]))
