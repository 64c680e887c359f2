"""Degeneracy-aware ICP (kb_pipeline_set_degeneracy_ratio, KissICP(config, degeneracy_ratio=...)): before ICP the plane
information at the initial guess, centred at its position, is eigen-decomposed blockwise; axes below ratio * the block's
largest eigenvalue are held and every ICP step is projected off them. Restated here in numpy; checked in an analytic
tunnel (the axis is held, x advances by the prediction), on well-conditioned streams (nothing held, bit for bit the
plain pipeline), across paths, grid sizes and checkpoints."""
import ctypes as C

import numpy as np
import pytest

from test_constraints import _numpy_constraints, _same_map


# ---------------------------------------------------------------------------------------------- numpy restatement
def _cross_matrix(c):
    return np.array([[0.0, -c[2], c[1]], [c[2], 0.0, -c[0]], [-c[1], c[0], 0.0]])


def _A(c):
    A = np.eye(6)
    A[:3, 3:] = _cross_matrix(c)
    return A


def _centred(H, c):
    """H_c = A^T H A: the information of J_c = [n, (p - c) x n] from that of J = [n, p x n]"""
    A = _A(c)
    return A.T @ H @ A


def _projector(Hc, ratio, n_planes):
    """-> (P (6x6, centred coordinates), held_t, held_r, (lt, vt, lr, vr)): the definition of the header"""
    P = np.zeros((6, 6))
    held, eig = [], []
    for b in (slice(0, 3), slice(3, 6)):
        lam, V = np.linalg.eigh(Hc[b, b])
        h = (n_planes > 0) & (lam[2] > 0) & (lam < ratio * lam[2])
        P[b, b] = V @ np.diag(np.where(h, 0.0, 1.0)) @ V.T
        held.append(h)
        eig += [lam, V]
    return P, held[0], held[1], tuple(eig)


def _step(P, c, dx):
    """the projected step about the map origin: A P A^-1 dx"""
    A = _A(c)
    return A @ P @ np.linalg.solve(A, dx)


def _se3_exp(dx):
    """SE3::exp of (v, w), translation first: [R(w), V(w) v]"""
    v, w = np.asarray(dx[:3]), np.asarray(dx[3:])
    th = float(np.linalg.norm(w))
    W = _cross_matrix(w)
    if th < 1e-10:
        R, V = np.eye(3) + W, np.eye(3) + 0.5 * W
    else:
        R = np.eye(3) + np.sin(th) / th * W + (1 - np.cos(th)) / th ** 2 * W @ W
        V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * W + (th - np.sin(th)) / th ** 3 * W @ W
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, V @ v
    return T


def _align(O, vmap, src, guess, max_dist, kscale, proj=None, max_iter=500, conv=1e-4):
    """AlignPointsToMap (Registration.cpp:138-167) over the oracle's DataAssociation + BuildLinearSystem, with every
    step dx replaced by proj @ dx before Exp and the convergence test when proj is given"""
    pts = np.asarray(src) @ guess[:3, :3].T + guess[:3, 3]
    T_icp = np.eye(4)
    for _ in range(max_iter):
        JTJ, JTr, _ = O.build_system(vmap, pts, max_dist, kscale)
        dx = np.linalg.solve(JTJ, -JTr)
        if proj is not None:
            dx = proj @ dx
        E = _se3_exp(dx)
        pts = pts @ E[:3, :3].T + E[:3, 3]
        T_icp = E @ T_icp
        if np.linalg.norm(dx) < conv:
            break
    return T_icp @ guess


def test_align_restatement_matches_the_oracle(O):
    """the restated loop without a projector is the oracle's AlignPointsToMap, to rounding"""
    rng = np.random.default_rng(2)
    g = np.arange(-8, 8, 0.25)
    floor = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
    cloud = np.concatenate([np.column_stack([floor, np.zeros(len(floor))]),
                            np.column_stack([floor[:, 0], np.full(len(floor), 3.0), floor[:, 1] / 4 + 2]),
                            np.column_stack([np.full(len(floor), -4.0), floor[:, 0], floor[:, 1] / 4 + 2])])
    vm = O.VoxelHashMap(1.0, 100.0, 20)
    vm.add_points(cloud)
    src = cloud[rng.choice(len(cloud), 1500, replace=False)] + rng.normal(0, 0.01, (1500, 3))
    G = _se3_exp([0.05, -0.04, 0.02, 0.002, -0.003, 0.01])
    ref, _ = O.align_points_to_map(vm, src, G, 1.0, 0.3)
    assert np.abs(_align(O, vm, src, G, 1.0, 0.3) - ref).max() < 1e-9
    # a projector that removes x keeps the guess's x (to second order in the step)
    P = np.eye(6)
    P[0, 0] = 0.0
    held = _align(O, vm, src, G, 1.0, 0.3, P)
    assert abs(held[0, 3] - G[0, 3]) < 1e-3 and abs(ref[0, 3] - G[0, 3]) > 1e-2


def test_centred_information_equals_the_direct_centred_sum():
    rng = np.random.default_rng(0)
    c = np.array([1234.5, -87.25, 3.0])
    H, Hc = np.zeros((6, 6)), np.zeros((6, 6))
    for _ in range(200):
        n = rng.normal(size=3)
        n /= np.linalg.norm(n)
        p = c + rng.normal(0, 20, 3)
        a = rng.uniform()
        J = np.concatenate([n, np.cross(p, n)])
        Jc = np.concatenate([n, np.cross(p - c, n)])
        H += a * np.outer(J, J)
        Hc += a * np.outer(Jc, Jc)
    assert np.abs(_centred(H, c) - Hc).max() <= 1e-9 * np.abs(Hc).max()
    # the translation block does not depend on the centre
    assert np.array_equal(_centred(H, c)[:3, :3], H[:3, :3])


def test_projector_definition():
    rng = np.random.default_rng(1)
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    # a corridor along R[:, 0]: one translation held, nothing in the rotation block
    Hc = np.zeros((6, 6))
    Hc[:3, :3] = R @ np.diag([1e-9, 5.0, 9.0]) @ R.T
    Hc[3:, 3:] = np.diag([2.0, 3.0, 4.0])
    P, ht, hr, _ = _projector(Hc, 0.02, 100)
    assert ht.tolist() == [True, False, False] and not hr.any()
    assert np.allclose(P[:3, :3], np.eye(3) - np.outer(R[:, 0], R[:, 0]), atol=1e-12)
    assert np.allclose(P[3:, 3:], np.eye(3), atol=1e-12)
    # a step along the held axis vanishes, one across it stays; about a centre, a pure rotation keeps the centre fixed
    c = np.array([50.0, -3.0, 1.0])
    dx = np.concatenate([R[:, 0], np.zeros(3)])
    assert np.abs(_step(P, c, dx)).max() < 1e-12
    w = np.array([0.0, 0.0, 0.01])
    dx = np.concatenate([-np.cross(w, c), w])  # rotation about c
    assert np.allclose(_step(P, c, dx), dx, atol=1e-12)
    # the identity cases: no plane term, a block without information, nothing below the ratio
    assert not np.any(_projector(Hc, 0.02, 0)[1]) and np.allclose(_projector(Hc, 0.02, 0)[0], np.eye(6), atol=1e-12)
    Z = Hc.copy()
    Z[:3, :3] = 0.0
    _, ht, hr, _ = _projector(Z, 0.5, 100)
    assert not ht.any() and hr.tolist() == [False, False, False]
    _, ht, hr, _ = _projector(Hc, 1e-12, 100)
    assert not ht.any() and not hr.any()
    # ratio is strict: an eigenvalue equal to ratio * l_max is kept
    _, ht, _, _ = _projector(np.diag([1.0, 2.0, 4.0, 1.0, 1.0, 1.0]), 0.25, 1)
    assert not ht.any()


def test_arguments_without_device():
    import kiss_icp_b200 as K
    from kiss_icp_b200 import _native as N
    L = N.lib()
    d, r = N.Degeneracy(), N.dbl(0)
    assert L.kb_pipeline_set_degeneracy_ratio(None, 0.1) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_degeneracy_ratio(None, C.byref(r)) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_last_degeneracy(None, C.byref(d)) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_register_frames_degeneracy(None, None, None, None, None, 0, 0, None, None, None, None) == \
        N.KB_ERR_INVALID_ARG
    for bad in (float("nan"), -0.1, 1.0, 2.0, float("inf")):
        with pytest.raises(ValueError):
            K.KissICP(K.load_config(), degeneracy_ratio=bad)
    with pytest.raises(ValueError):
        K.KissICP(K.load_config(), fused=False, degeneracy_ratio=0.02)
    assert 0.0 < K.RECOMMENDED_DEGENERACY_RATIO < 1.0


# ---------------------------------------------------------------------------------------------- device
def _tunnel():
    from kiss_icp_b200 import synthetic
    return synthetic.Tunnel(seed=0)


def _entering(icp, T):
    """the track enters at scan 0 with the true velocity: the first guess is the true pose of scan 0"""
    icp.last_pose = T.pose(-1)
    icp.last_delta = T.pose(1)


def _yaw(R):
    return float(np.arctan2(R[1, 0], R[0, 0]))


@pytest.mark.gpu
def test_tunnel_holds_the_axis_and_keeps_the_prediction(K):
    T = _tunnel()
    n = 48
    scans = [T.scan(k) for k in range(n)]
    rho = K.RECOMMENDED_DEGENERACY_RATIO
    on, off = K.KissICP(K.load_config(), degeneracy_ratio=rho), K.KissICP(K.load_config())
    assert on.degeneracy_ratio == rho and on.report_fit and off.degeneracy_ratio == 0.0
    for icp in (on, off):
        _entering(icp, T)
    xs_on, xs_off, along, tilt, ratios, rot_held = [], [], [], [], [], 0
    for k, (p, t) in enumerate(scans):
        G = on.last_pose @ on.last_delta
        on.register_frame(p, t, return_clouds=False)
        off.register_frame(p, t, return_clouds=False)
        A = on.last_pose
        xs_on.append(A[0, 3])
        xs_off.append(off.last_pose[0, 3])
        d = on.last_degeneracy
        if k > 0:
            assert d.translation_held.tolist() == [True, False, False], k
            # rotational information grows with the lever squared: against pitch and yaw from the far walls, roll
            # about the axis (levers <= the tunnel's half size) may fall below the ratio, and is then held too
            for i in np.nonzero(d.rotation_held)[0]:
                assert abs(d.rotation_axes[0, i]) > 0.9, k
            rot_held += int(d.rotation_held.any())
            ratios.append(d.translation_eigenvalues[0] / d.translation_eigenvalues[2])
            axis = d.translation_axes[:, 0]
            tilt.append(float(np.arccos(min(1.0, abs(axis[0])))))
            along.append(abs((A[:3, 3] - G[:3, 3]) @ axis))  # the prediction is kept along the held axis
        else:
            assert d.n_planes == 0 and not d.translation_held.any()  # empty map: no evidence, nothing held
        # lateral position, height and yaw stay near the truth. (The held axis, estimated from the voxel planes of a
        # ring-sampled floor, tilts toward the floor normal: ICP's pull along the tunnel leaks into the height.)
        assert abs(A[1, 3]) < 0.05 and abs(A[2, 3]) < 0.15 and abs(_yaw(A[:3, :3])) < 2e-3, k
    steps = np.diff(xs_on)
    print(f"held: final y {A[1, 3]:.4f} z {A[2, 3]:.4f}; x after {n - 1} steps {xs_on[-1]:.6f} (true {T.pose(n - 1)[0, 3]}), largest step error "
          f"{np.abs(steps - T.step).max():.3e}, largest move along the held axis {max(along):.3e}, largest tilt of "
          f"the held axis from x {max(tilt):.4f} rad, largest ratio on it {max(ratios):.4f}, scans holding a rotation {rot_held}; plain ICP: x = {xs_off[-1]:.3f}")
    assert max(along) < 1e-5
    # the held axis is estimated from the map's voxel planes, within a few degrees of x: a correction across it (in z,
    # say) moves x by that much of it
    assert max(tilt) < 0.05
    assert np.abs(steps - T.step).max() < 1e-3
    assert abs(xs_on[-1] - T.pose(n - 1)[0, 3]) < 0.02
    # without the mode, point-to-point ICP pulls every scan back toward the previous ring pattern
    assert T.pose(n - 1)[0, 3] - xs_off[-1] > 2.0


@pytest.mark.gpu
def test_tunnel_localizer(K):
    T = _tunnel()
    cfg = K.load_config()
    c = cfg.mapping
    prior = K.VoxelHashMap(c.voxel_size, 1e4, c.max_points_per_voxel)
    for k in range(0, 60):
        p, _ = T.scan(1000 + k)
        prior.update(K.voxel_down_sample(p, 0.5 * c.voxel_size), T.pose(k))
    loc = K.KissICP(cfg, prior_map=prior, degeneracy_ratio=K.RECOMMENDED_DEGENERACY_RATIO)
    _entering(loc, T)
    scans = [T.scan(k) for k in range(40)]
    poses, degs = loc.register_frames([p for p, _ in scans], [t for _, t in scans], return_degeneracy=True)
    assert degs.translation_held[:, 0].all() and not degs.translation_held[:, 1:].any()
    print(f"localizer: largest step error {np.abs(np.diff(poses[:, 0, 3]) - T.step).max():.3e}")
    assert np.abs(np.diff(poses[:, 0, 3]) - T.step).max() < 1e-3
    assert np.abs(poses[:, 1, 3]).max() < 0.05 and np.abs(poses[:, 2, 3]).max() < 0.15


def _run(K, cfg, scans, rho, queued=False, **kw):
    icp = K.KissICP(cfg, report_fit=True, degeneracy_ratio=rho, **kw)
    if queued:
        out = icp.register_frames([p for p, _ in scans], [t for _, t in scans], return_fits=True,
                                  return_degeneracy=rho > 0)
        return icp, out
    poses, fits, degs = [], [], []
    for p, t in scans:
        icp.register_frame(p, t, return_clouds=False)
        poses.append(icp.last_pose)
        fits.append(icp.last_fit)
        if rho > 0:
            degs.append(icp.last_degeneracy)
    return icp, (np.array(poses), fits, degs)


def _ratios(degs):
    lt = np.array([d.translation_eigenvalues for d in degs if d.n_planes > 0])
    lr = np.array([d.rotation_eigenvalues for d in degs if d.n_planes > 0])
    return (lt[:, 0] / lt[:, 2]).min(), (lr[:, 0] / lr[:, 2]).min()


@pytest.mark.gpu
@pytest.mark.parametrize("stream", ["small", "kitti"])
def test_no_change_where_nothing_is_held(K, stream):
    from kiss_icp_b200 import synthetic
    if stream == "small":
        L, n = synthetic.small_shape(seed=3, beams=32, cols=512), 30
    else:
        L, n = synthetic.kitti_shape(seed=0, device="cuda"), 20
    scans = [L.scan(k) for k in range(n)]
    cfg = K.load_config()
    rho = K.RECOMMENDED_DEGENERACY_RATIO
    a, (pa, fa, _) = _run(K, cfg, scans, 0.0)
    b, (pb, fb, db) = _run(K, cfg, scans, rho)
    rt, rr = _ratios(db)
    print(f"{stream}: smallest eigenvalue ratio, translation {rt:.4f}, rotation {rr:.4f}")
    assert rt > rho and rr > rho
    assert not any(d.translation_held.any() or d.rotation_held.any() for d in db)
    assert np.array_equal(pa, pb)
    assert all(np.array_equal(x.information, y.information) and x.n_correspondences == y.n_correspondences and
               np.array_equal(x.rmse, y.rmse, equal_nan=True) for x, y in zip(fa, fb))
    assert _same_map(a.local_map, b.local_map)


@pytest.mark.gpu
def test_parity_with_the_numpy_restatement(K, O):
    T = _tunnel()
    cfg = K.load_config()
    c = cfg.mapping
    rho = K.RECOMMENDED_DEGENERACY_RATIO
    icp = K.KissICP(cfg, degeneracy_ratio=rho)
    _entering(icp, T)
    checked, worst = 0, 0.0
    for k in range(12):
        p, t = T.scan(k)
        before = K.VoxelHashMap(c.voxel_size, cfg.data.max_range, c.max_points_per_voxel)
        vox, cnt, pts = icp.local_map.dump()
        if len(vox):
            before.load(vox, cnt, pts)
        G = icp.last_pose @ icp.last_delta
        sigma = icp.adaptive_threshold.get_threshold()
        _, src = icp.register_frame(p, t)
        d = icp.last_degeneracy
        if not len(vox):
            continue
        n_planes, W, _, H = _numpy_constraints(before, c.voxel_size, src, G, 3 * sigma)
        Hc = _centred(H, G[:3, 3])
        P, ht, hr, (lt, vt, lr, vr) = _projector(Hc, rho, n_planes)
        assert d.n_planes == n_planes and abs(d.weight_sum - W) <= 1e-12 * W
        for lam, V, glam, gV, gh, h in ((lt, vt, d.translation_eigenvalues, d.translation_axes, d.translation_held, ht),
                                        (lr, vr, d.rotation_eigenvalues, d.rotation_axes, d.rotation_held, hr)):
            assert np.abs(glam - lam).max() <= 1e-10 * lam[2], k
            assert np.array_equal(gh, h), k
            for i in range(3):
                gap = min(abs(lam[i] - lam[j]) for j in range(3) if j != i)
                if gap > 1e-6 * lam[2]:  # (an axis is defined to the accuracy of its eigenvalue gap)
                    assert abs(abs(gV[:, i] @ V[:, i]) - 1) < 1e-10 * lam[2] / gap, (k, i)
        # the held direction of the step: the pose moved from the guess only across the held axis (to second order)
        axis = vt[:, 0]
        assert abs((icp.last_pose[:3, 3] - G[:3, 3]) @ axis) < 1e-5
        # the restated loop over the oracle's linear systems, every step projected by A P A^-1 (none when nothing is
        # held), in the same map
        om = O.VoxelHashMap(c.voxel_size, cfg.data.max_range, c.max_points_per_voxel)
        om.add_points(pts)
        A = _A(G[:3, 3])
        proj = A @ P @ np.linalg.inv(A) if (ht.any() or hr.any()) else None
        ref = _align(O, om, src, G, 3 * sigma, sigma, proj)
        worst = max(worst, np.abs(icp.last_pose - ref).max())
        checked += 1
    print(f"largest pose difference to the projected restatement: {worst:.3e}")
    assert worst < 1e-6
    assert checked == 11


@pytest.mark.gpu
def test_paths_grid_sizes_and_repeats_agree(K, monkeypatch):
    from kiss_icp_b200 import _native as N
    T = _tunnel()
    scans = [T.scan(k) for k in range(16)]
    cfg = K.load_config()
    rho = K.RECOMMENDED_DEGENERACY_RATIO

    def run(queued):
        icp = K.KissICP(cfg, degeneracy_ratio=rho)
        _entering(icp, T)
        icp.start_history(len(scans))
        if queued:
            poses, degs = icp.register_frames([p for p, _ in scans], [t for _, t in scans], return_degeneracy=True)
            return icp, poses, degs
        poses, degs = [], []
        for p, t in scans:
            icp.register_frame(p, t, return_clouds=False)
            poses.append(icp.last_pose)
            degs.append(icp.last_degeneracy)
        return icp, np.array(poses), degs

    a, pa, da = run(False)
    b, pb, db = run(True)
    c, pc, _ = run(True)
    assert all(h.team > 0 for h in a.history()[1:])
    assert np.array_equal(pa, pb) and np.array_equal(pb, pc)
    assert np.array_equal(np.array([d.translation_eigenvalues for d in da]), db.translation_eigenvalues)
    assert np.array_equal(np.array([d.rotation_axes for d in da]), db.rotation_axes)
    assert np.array_equal(np.array([d.translation_held for d in da]), db.translation_held)
    assert _same_map(a.local_map, b.local_map)
    # the whole-grid ICP loop
    monkeypatch.setenv("KB_ICP_TEAM_Q", "0")
    w, pw, _ = run(True)
    assert all(h.team == 0 for h in w.history())
    monkeypatch.delenv("KB_ICP_TEAM_Q")
    assert np.abs(pw - pa).max() < 1e-6
    # another grid size
    assert N.lib().kb_set_grid_blocks(40) == 0
    try:
        g, pg, dg = run(True)
    finally:
        N.lib().kb_set_grid_blocks(0)
    assert np.abs(pg - pa).max() < 1e-6
    assert np.array_equal(dg.translation_held, db.translation_held)


@pytest.mark.gpu
def test_switching_rules(K):
    from kiss_icp_b200 import _native as N
    L = N.lib()
    icp = K.KissICP(K.load_config())
    h = icp._h
    r, d = N.dbl(0), N.Degeneracy()
    assert L.kb_pipeline_degeneracy_ratio(h, C.byref(r)) == 0 and r.value == 0.0
    assert L.kb_pipeline_set_degeneracy_ratio(h, 0.1) == N.KB_ERR_INVALID_ARG  # no fits
    assert L.kb_pipeline_last_degeneracy(h, C.byref(d)) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_set_fit_reporting(h, 1) == 0
    assert L.kb_pipeline_set_degeneracy_ratio(h, 0.1) == 0
    for bad in (float("nan"), -1e-3, 1.0, float("inf")):
        assert L.kb_pipeline_set_degeneracy_ratio(h, bad) == N.KB_ERR_INVALID_ARG
        assert L.kb_pipeline_degeneracy_ratio(h, C.byref(r)) == 0 and r.value == 0.1
    assert L.kb_pipeline_last_degeneracy(h, C.byref(d)) == 0 and d.n_planes == 0 and not any(d.translation_held)
    assert L.kb_pipeline_set_fit_reporting(h, 0) == N.KB_ERR_INVALID_ARG  # the mode runs next to the fit
    assert L.kb_pipeline_set_degeneracy_ratio(h, 0.0) == 0
    assert L.kb_pipeline_last_degeneracy(h, C.byref(d)) == N.KB_ERR_INVALID_ARG
    assert L.kb_pipeline_set_fit_reporting(h, 0) == 0
    X = (C.c_void_p * 1)(None)
    n = (N.sz * 1)(0)
    assert L.kb_pipeline_register_frames_degeneracy(h, X, n, None, None, 1, 0, None, None, None, C.byref(d)) == \
        N.KB_ERR_INVALID_ARG
    with pytest.raises(ValueError):
        _ = icp.last_degeneracy
    with pytest.raises(ValueError):
        icp.register_frames([np.zeros((10, 3))], return_degeneracy=True)


@pytest.mark.gpu
def test_checkpoint_continues_bit_for_bit(K):
    T = _tunnel()
    scans = [T.scan(k) for k in range(20)]
    cfg = K.load_config()
    rho = K.RECOMMENDED_DEGENERACY_RATIO
    a = K.KissICP(cfg, degeneracy_ratio=rho)
    _entering(a, T)
    for p, t in scans[:10]:
        a.register_frame(p, t, return_clouds=False)
    b = K.KissICP(cfg, degeneracy_ratio=rho)
    b.load_state_dict(a.state_dict())
    pa = a.register_frames([p for p, _ in scans[10:]], [t for _, t in scans[10:]])
    pb = b.register_frames([p for p, _ in scans[10:]], [t for _, t in scans[10:]])
    assert np.array_equal(pa, pb)
    assert np.abs(np.diff(pa[:, 0, 3]) - T.step).max() < 1e-3
