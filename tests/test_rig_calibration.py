"""Rig extrinsic calibration (kb_calibrate_rig, calibrate_rig, DESIGN.md section 4.19): the C-ABI's argument checks, a
numpy restatement of the calibration over the oracle, and on the device the report against kb_registration_build_system,
the restatement, recovery of perturbed extrinsics with true and odometry poses, determinism across layouts, the
observability report in a tunnel and a map held by a localizer."""
import ctypes as C
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation


def _mounts():
    F = np.eye(4)
    F[:3, 3] = [2.0, 0.0, 0.0]
    R = np.diag([-1.0, -1.0, 1.0, 1.0])
    R[:3, 3] = [-2.0, 0.0, 0.0]
    return F, R


def _perturb(E, dt, drot_deg, seed):
    """E Exp(d): a right perturbation in the sensor frame, |translation| = dt, |rotation| = drot_deg"""
    rng = np.random.default_rng(seed)
    u, w = rng.normal(size=3), rng.normal(size=3)
    D = np.eye(4)
    D[:3, :3] = Rotation.from_rotvec(w / np.linalg.norm(w) * math.radians(drot_deg)).as_matrix()
    D[:3, 3] = u / np.linalg.norm(u) * dt
    return E @ D


def _error(E, E_true):
    D = np.linalg.inv(E_true) @ E
    return float(np.linalg.norm(D[:3, 3])), math.degrees(float(Rotation.from_matrix(D[:3, :3]).magnitude()))


def _transform(M, p):
    return p @ M[:3, :3].T + M[:3, 3]


def _hat(p):
    Z = np.zeros(len(p))
    return np.stack([np.stack([Z, -p[:, 2], p[:, 1]], -1), np.stack([p[:, 2], Z, -p[:, 0]], -1),
                     np.stack([-p[:, 1], p[:, 0], Z], -1)], 1)


def system_np(P, Q, kscale):
    """KISS-ICP's BuildLinearSystem (Registration.cpp:80-121) with source P and target Q: J = [I, -[p]x],
    w = k^2 / (k + |r|^2)^2 -> (JTJ, JTr)"""
    r = P - Q
    w = kscale * kscale / (kscale + np.sum(r * r, 1)) ** 2
    J = np.concatenate([np.broadcast_to(np.eye(3), (len(P), 3, 3)), -_hat(P)], 2)
    return np.einsum("nij,nik,n->jk", J, J, w), np.einsum("nij,ni,n->j", J, r, w)


def oracle_calibrate(O, omap, poses, E0, scans, max_dist, kscale, max_iter, conv):
    """The calibration of one sensor restated over the oracle: each iteration, every frame's points p (cropped) at
    T_k E, their nearest map points q kept below max_dist, the system with source p and target (T_k E)^-1 q, the
    oracle's LDL^T and E <- E Exp(dx); stops at |dx| < conv. -> (E, iterations, first step)"""
    E = np.array(E0, dtype=np.float64)
    first = None
    it = 0
    while it < max_iter:
        Ps, Qs = [], []
        for k, p in enumerate(scans):
            if not len(p):
                continue
            M = O.se3_mul(poses[k], E)
            q, d = omap.closest_neighbors(O.se3_act(M, p))
            keep = d < max_dist
            Ps.append(p[keep])
            Qs.append(O.se3_act(O.se3_inverse(M), q[keep]))
        JTJ, JTr = system_np(np.concatenate(Ps), np.concatenate(Qs), kscale)
        dx = O.ldlt6_solve(JTJ, -JTr)
        E = O.se3_mul(E, O.se3_exp(dx))
        it += 1
        if first is None:
            first = E.copy()
        if np.linalg.norm(dx) < conv:
            break
    return E, it, first


def _small_run(K, n=20, seed=0, device="cpu"):
    from kiss_icp_b200 import synthetic
    L = synthetic.SyntheticLidar(seed=seed, beams=32, cols=512, stamps="none", device=device)
    F, R = _mounts()
    rig = synthetic.RigLidar(L, [F, R])
    frames = [rig.scan(k)[0] for k in range(n)]
    return frames, np.array([L.pose(k) for k in range(n)]), (F, R)


def _oracle_setup(O, frames, poses, F):
    omap = O.VoxelHashMap(1.0, 100.0, 20)
    for k, f in enumerate(frames):
        omap.add_points(O.se3_act(poses[k] @ F, O.voxel_down_sample(f[0], 0.5)))
    srcs = [O.voxel_down_sample(O.voxel_down_sample(f[1], 0.5), 1.5) for f in frames]
    return omap, srcs


STAGES = ((3.0, 1.0), (1.0, 1.0 / 3.0))  # DEFAULT_STAGES_VOXELS at a 1 m voxel
# (m, deg) after calibration on the front/rear rig, 100 KITTI-shape scans: measured on an H100 3.0 mm / 0.010 deg with
# true poses and 4.5 mm / 0.020 deg with odometry poses (DESIGN.md section 4.19)
TRUE_POSE_BOUND = (0.01, 0.05)
ODOMETRY_POSE_BOUND = (0.02, 0.1)


# ---------------------------------------------------------------------------------------------------------- no device
def test_argument_errors_write_nothing():
    from kiss_icp_b200 import _native as N
    L = N.lib()
    F, R = _mounts()
    sensors = (N.Sensor * 2)()
    for s, E in zip(sensors, (F, R)):
        s.extrinsic[:] = list(E.reshape(-1))
        s.min_range, s.max_range = 0.0, math.inf
    pts = [np.random.default_rng(i).normal(size=(50, 3)) for i in range(4)]
    poses = np.ascontiguousarray(np.stack([np.eye(4)] * 2))

    def call(sens=sensors, S=2, poses=poses, K=2, refine=None, xyz=None, n=None, layout=0, opt="ok", E="ok", rep="ok"):
        X = (C.c_void_p * 4)(*[a.ctypes.data for a in pts]) if xyz is None else xyz
        nn = (N.sz * 4)(*[len(a) for a in pts]) if n is None else n
        o = N.RigCalibrationOptions(3.0, 1.0, 10, 1e-4) if opt == "ok" else opt
        Eo = np.full((2, 4, 4), 1234.5)
        Ro = (N.SensorCalibration * 2)()
        C.memset(Ro, 0xAB, C.sizeof(Ro))
        before = bytes(Ro)
        st = L.kb_calibrate_rig(None, None if poses is None else N.ptr(poses), K, sens, S, refine, X, nn, layout,
                                None if o is None else C.byref(o), N.ptr(Eo) if E == "ok" else None,
                                Ro if rep == "ok" else None)
        assert np.all(Eo == 1234.5) and bytes(Ro) == before
        return st, L.kb_last_error().decode()

    st, msg = call()  # every argument valid: the NULL map is the error
    assert st == N.KB_ERR_INVALID_ARG and "map" in msg
    bad_opts = [None, N.RigCalibrationOptions(math.nan, 1.0, 10, 1e-4), N.RigCalibrationOptions(0.0, 1.0, 10, 1e-4),
                N.RigCalibrationOptions(math.inf, 1.0, 10, 1e-4), N.RigCalibrationOptions(3.0, 0.0, 10, 1e-4),
                N.RigCalibrationOptions(3.0, math.nan, 10, 1e-4), N.RigCalibrationOptions(3.0, math.inf, 10, 1e-4),
                N.RigCalibrationOptions(3.0, 1.0, -1, 1e-4), N.RigCalibrationOptions(3.0, 1.0, 10, math.nan),
                N.RigCalibrationOptions(3.0, 1.0, 10, -1e-4), N.RigCalibrationOptions(3.0, 1.0, 10, math.inf)]
    for o in bad_opts:
        st, msg = call(opt=o)
        assert st == N.KB_ERR_INVALID_ARG and "map" not in msg, msg
    # the rig (kb_rig_check)
    assert call(S=0)[0] == N.KB_ERR_INVALID_ARG
    assert call(S=17)[0] == N.KB_ERR_INVALID_ARG
    assert call(sens=None)[0] == N.KB_ERR_INVALID_ARG
    bad = (N.Sensor * 2)()
    C.memmove(bad, sensors, C.sizeof(bad))
    bad[1].extrinsic[0] = 2.0
    assert call(sens=bad)[0] == N.KB_ERR_NOT_SE3
    C.memmove(bad, sensors, C.sizeof(bad))
    bad[0].min_range = math.nan
    assert call(sens=bad)[0] == N.KB_ERR_INVALID_ARG
    # refine, layout, outputs
    for r in ((N.i32 * 2)(0, 2), (N.i32 * 2)(-1, 1)):
        assert call(refine=r)[0] == N.KB_ERR_INVALID_ARG
    for layout in (3, -1):
        assert call(layout=layout)[0] == N.KB_ERR_INVALID_ARG
    assert call(E=None)[0] == N.KB_ERR_INVALID_ARG
    assert call(rep=None)[0] == N.KB_ERR_INVALID_ARG
    # poses
    for v in (math.nan, math.inf, 2.0):
        P = poses.copy()
        P[1, 0, 0] = v
        st, msg = call(poses=P)
        assert st == N.KB_ERR_NOT_SE3, msg
    P = poses.copy()
    P[0, 3, :] = [0.0, 0.0, 1.0, 1.0]
    assert call(poses=P)[0] == N.KB_ERR_NOT_SE3
    assert call(poses=None)[0] == N.KB_ERR_INVALID_ARG
    # arrays: NULL arrays of frames with points, too many points
    X = (C.c_void_p * 4)(*[a.ctypes.data for a in pts])
    X[3] = None
    assert call(xyz=X)[0] == N.KB_ERR_INVALID_ARG
    assert call(xyz=X, refine=(N.i32 * 2)(1, 0))[1] != ""  # sensor 1 not refined: its NULL array is not read
    assert "map" in call(xyz=X, refine=(N.i32 * 2)(1, 0))[1]
    for big in ((1 << 31), (1 << 30)):
        n = (N.sz * 4)(50, big, 50, big)
        st, msg = call(n=n)
        assert st == N.KB_ERR_INVALID_ARG and "2^31" in msg


def test_oracle_restatement_recovers_a_perturbed_rear_extrinsic(O):
    """the calibration's maths without the device: the numpy system equals the oracle's BuildLinearSystem at T = E = I,
    and the restated loop recovers a perturbed rear extrinsic from 20 frames at true poses"""
    frames, poses, (F, Rm) = _small_run(None)
    omap, srcs = _oracle_setup(O, frames, poses, F)
    p = O.se3_act(poses[3] @ Rm, srcs[3])
    q, d = omap.closest_neighbors(p)
    keep = d < 3.0
    JTJ, JTr = system_np(p[keep], q[keep], 1.0)
    JTJ_o, JTr_o, nc = O.build_system(omap, p, 3.0, 1.0)
    assert nc == keep.sum()
    assert np.allclose(JTJ, JTJ_o, rtol=1e-9, atol=1e-9 * np.abs(JTJ_o).max())
    assert np.allclose(JTr, JTr_o, rtol=1e-9, atol=1e-9 * np.abs(JTr_o).max())
    E0 = _perturb(Rm, 0.2, 2.0, 0)
    E = E0
    for d, k in STAGES:
        E, it, _ = oracle_calibrate(O, omap, poses, E, srcs, d, k, 500, 1e-4)
        assert 0 < it < 500
    t0, r0 = _error(E0, Rm)
    t1, r1 = _error(E, Rm)
    assert t1 < 0.05 and r1 < 0.25 and t1 < t0 / 10 and r1 < r0 / 10, (t0, r0, t1, r1)


# -------------------------------------------------------------------------------------------------------------- device
@pytest.fixture(scope="module")
def kitti_run():
    """the front/rear rig of tools/rig_accuracy.py on the KITTI-shape run, 100 scans, no body"""
    from kiss_icp_b200 import synthetic
    L = synthetic.SyntheticLidar(seed=0, beams=64, cols=1024, elev_deg=(-24.8, 2.0), stamps="none", device="cuda")
    F, R = _mounts()
    rig = synthetic.RigLidar(L, [F, R])
    frames = [rig.scan(k)[0] for k in range(100)]
    return frames, np.array([L.pose(k) for k in range(100)]), (F, R)


def _gpu_map(K, frames, poses, F, v=1.0):
    vmap = K.VoxelHashMap(v, 100.0, 20)
    for k, f in enumerate(frames):
        vmap.add_points(_transform(poses[k] @ F, K.voxel_down_sample(f[0], 0.5 * v)))
    return vmap


def _sources(K, frames, j):
    kiss = K.KissICP(K.load_config())
    return [kiss.voxelize(f[j])[0] for f in frames]


def _raw(K, vmap, poses, rig, srcs_by_frame, stage, max_iter=500, layout=0, ptrs=None, refine=(0, 1)):
    from kiss_icp_b200.calibration import _calibrate
    flat = [a for f in srcs_by_frame for a in f]
    if ptrs is None:
        ptrs = [a.ctypes.data if len(a) else None for a in flat]
    return _calibrate(vmap, poses, rig, ptrs, [len(a) for a in flat], layout, refine, stage[0], stage[1], max_iter, 1e-4)


def _rep_tuple(r):
    return (r.iterations, r.converged, r.fit.n_correspondences, r.fit.n_source, r.fit.sum_sq_residual,
            tuple(r.fit.JTJ), r.constraints.n_planes, r.constraints.weight_sum, r.constraints.sum_sq_plane_residual,
            tuple(r.constraints.information))


def _adjoint(T):
    R, t = T[:3, :3], T[:3, 3]
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = R
    A[:3, 3:] = _hat(t[None])[0] @ R
    return A


@pytest.mark.gpu
def test_report_at_the_given_extrinsics_matches_build_system(K, kitti_run):
    frames, poses, (F, Rm) = kitti_run
    vmap = _gpu_map(K, frames[:10], poses[:10], F)
    reg = K.Registration(500, 1e-4, 0)
    src = _sources(K, [frames[5]], 1)[0]
    one = K.Rig([K.Sensor(np.eye(4))])
    # T = I, E = I: the sensor points are map points
    E, rep = _raw(K, vmap, np.eye(4)[None], one, [[src]], (3.0, 1.0), max_iter=0, refine=(1,))
    JTJ, _, nc = reg.build_system(src, vmap, 3.0, 1.0)
    assert rep[0].iterations == 0 and rep[0].fit.n_correspondences == nc == rep[0].fit.n_correspondences
    assert rep[0].fit.n_source == len(src)
    assert np.abs(np.array(rep[0].fit.JTJ).reshape(6, 6) - JTJ).max() <= 1e-12 * np.abs(JTJ).max()
    assert np.array_equal(E[0], np.eye(4))
    # general T and E: H_sensor = Ad^T H_map Ad, Ad the adjoint of T E
    rig = K.Rig([K.Sensor(F), K.Sensor(Rm)])
    E, rep = _raw(K, vmap, poses[5][None], rig, [[np.empty((0, 3)), src]], (3.0, 1.0), max_iter=0)
    M = poses[5] @ Rm
    JTJm, _, ncm = reg.build_system(_transform(M, src), vmap, 3.0, 1.0)
    Ad = _adjoint(M)
    H = Ad.T @ JTJm @ Ad
    assert rep[1].fit.n_correspondences == ncm > 0
    assert np.abs(np.array(rep[1].fit.JTJ).reshape(6, 6) - H).max() <= 1e-9 * np.abs(H).max()
    assert rep[1].constraints.n_planes > 0
    assert np.array_equal(E, np.stack([F, Rm]))  # nothing moved: the given bits
    assert _rep_tuple(rep[0]) == _rep_tuple(type(rep[0])())


@pytest.mark.gpu
def test_device_matches_the_oracle_restatement(K, O):
    frames, poses, (F, Rm) = _small_run(K)
    omap, srcs = _oracle_setup(O, frames, poses, F)
    vmap = K.VoxelHashMap(1.0, 100.0, 20)
    for k, f in enumerate(frames):
        vmap.add_points(O.se3_act(poses[k] @ F, O.voxel_down_sample(f[0], 0.5)))
    E0 = _perturb(Rm, 0.2, 2.0, 0)
    by_frame = [[np.empty((0, 3)), s] for s in srcs]
    E_dev = E_or = E0
    for stage in STAGES:
        rig = K.Rig([K.Sensor(F), K.Sensor(E_dev)])
        E1, _ = _raw(K, vmap, poses, rig, by_frame, stage, max_iter=1)
        E_o, it_o, first = oracle_calibrate(O, omap, poses, E_or, srcs, stage[0], stage[1], 500, 1e-4)
        assert np.abs(E1[1] - first).max() < 1e-9
        E, rep = _raw(K, vmap, poses, rig, by_frame, stage)
        assert rep[1].iterations == it_o and rep[1].converged
        assert np.abs(E[1] - E_o).max() < 1e-9
        E_dev, E_or = E[1], E_o


CASES = [(0.3, 0.0), (0.0, 3.0), (0.3, 3.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1])
def test_recovery_with_true_poses(K, kitti_run, seed):
    frames, poses, (F, Rm) = kitti_run
    for dt, dr in CASES:
        E0 = _perturb(Rm, dt, dr, seed)
        cal = K.calibrate_rig(frames, K.Rig([K.Sensor(F), K.Sensor(E0)]), poses=poses)
        t0, r0 = _error(E0, Rm)
        t1, r1 = _error(cal.extrinsics[1], Rm)
        print(f"true poses seed {seed} perturbation ({dt} m, {dr} deg): error {t1:.4f} m {r1:.4f} deg, "
              f"iterations {cal.sensors[1].iterations}")
        assert t1 < TRUE_POSE_BOUND[0] and r1 < TRUE_POSE_BOUND[1]
        assert (t0 == 0 or t1 < t0 / 10) and (r0 == 0 or r1 < r0 / 10)
        assert cal.sensors[1].converged and np.array_equal(cal.extrinsics[0], F)


@pytest.mark.gpu
def test_recovery_with_odometry_poses(K, kitti_run):
    frames, _, (F, Rm) = kitti_run
    for seed in (0, 1):
        for dt, dr in CASES:
            E0 = _perturb(Rm, dt, dr, seed)
            cal = K.calibrate_rig(frames, K.Rig([K.Sensor(F), K.Sensor(E0)]))
            t1, r1 = _error(cal.extrinsics[1], Rm)
            print(f"odometry poses seed {seed} perturbation ({dt} m, {dr} deg): error {t1:.4f} m {r1:.4f} deg")
            assert t1 < ODOMETRY_POSE_BOUND[0] and r1 < ODOMETRY_POSE_BOUND[1]


@pytest.mark.gpu
def test_true_extrinsics_stay_and_unrefined_sensors_pass_through(K, kitti_run):
    frames, poses, (F, Rm) = kitti_run
    side = F @ np.array([[0.0, -1.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.3], [0.0, 0.0, 1.0, 0.1], [0.0, 0.0, 0.0, 1.0]])
    frames3 = [f + [f[0]] for f in frames[:40]]
    rig = K.Rig([K.Sensor(F, 0.5, 90.0), K.Sensor(Rm, 0.0, 80.0), K.Sensor(side, 1.0, 50.0)])
    cal = K.calibrate_rig(frames3, rig, poses=poses[:40], refine=[1])
    t, r = _error(cal.extrinsics[1], Rm)
    print(f"from the true extrinsic: moved {t:.4f} m {r:.4f} deg")
    assert t < TRUE_POSE_BOUND[0] and r < TRUE_POSE_BOUND[1]
    for j, E in ((0, F), (2, side)):
        assert np.array_equal(cal.extrinsics[j], E) and np.array_equal(cal.rig.sensors[j].extrinsic, E)
        s = cal.sensors[j]
        assert s.iterations == 0 and not s.converged and s.fit.n_source == 0 and s.constraints.n_planes == 0
        assert not s.fit.information.any() and not s.constraints.information.any()
    assert [(s.min_range, s.max_range) for s in cal.rig.sensors] == [(0.5, 90.0), (0.0, 80.0), (1.0, 50.0)]


@pytest.mark.gpu
def test_bit_identical_across_calls_and_layouts(K, kitti_run):
    import torch
    frames, poses, (F, Rm) = kitti_run
    n = 30
    vmap = _gpu_map(K, frames[:n], poses[:n], F)
    src = _sources(K, frames[:n], 1)
    by_frame = [[np.empty((0, 3)), s] for s in src]
    rig = K.Rig([K.Sensor(F), K.Sensor(_perturb(Rm, 0.2, 2.0, 3), 0.0, 60.0)])
    A = _raw(K, vmap, poses[:n], rig, by_frame, (3.0, 1.0))
    B = _raw(K, vmap, poses[:n], rig, by_frame, (3.0, 1.0))
    f32 = [[a.astype(np.float32) for a in f] for f in by_frame]
    assert all(np.array_equal(a.astype(np.float64), b) for f, g in zip(f32, by_frame) for a, b in zip(f, g))
    Cf = _raw(K, vmap, poses[:n], rig, f32, (3.0, 1.0), layout=1)
    dev = [torch.from_numpy(a).cuda() for f in by_frame for a in f]
    torch.cuda.synchronize()
    D = _raw(K, vmap, poses[:n], rig, by_frame, (3.0, 1.0), layout=2,
             ptrs=[t.data_ptr() if t.numel() else None for t in dev])
    for X in (B, Cf, D):
        assert np.array_equal(A[0], X[0])
        assert [_rep_tuple(r) for r in A[1]] == [_rep_tuple(r) for r in X[1]]
    assert A[1][1].iterations > 1


@pytest.mark.gpu
def test_tunnel_leaves_the_rear_offset_along_the_axis_unconstrained(K, kitti_run):
    from kiss_icp_b200 import synthetic
    T = synthetic.Tunnel(seed=0)
    lag = 4
    E_rear = np.eye(4)
    E_rear[0, 3] = -lag * T.step
    ks = range(lag, lag + 60)
    frames = [[T.scan(k)[0], T.scan(k - lag)[0]] for k in ks]
    poses = np.array([T.pose(k) for k in ks])
    cal = K.calibrate_rig(frames, K.Rig([K.Sensor(np.eye(4)), K.Sensor(E_rear)]), poses=poses)
    d = K.degeneracy(cal.sensors[1].constraints)
    axis = d.translation_axes[:, 0]
    assert math.degrees(math.acos(min(1.0, abs(axis[0])))) < 5.0
    ratio = d.translation_eigenvalues[0] / d.translation_eigenvalues[2]
    # the KITTI-shape rig's rear sensor, calibrated at its true extrinsic
    frames_k, poses_k, (F, Rm) = kitti_run
    ck = K.calibrate_rig(frames_k, K.Rig([K.Sensor(F), K.Sensor(Rm)]), poses=poses_k)
    dk = K.degeneracy(ck.sensors[1].constraints)
    kitti = np.concatenate([dk.translation_eigenvalues / dk.translation_eigenvalues[2],
                            dk.rotation_eigenvalues / dk.rotation_eigenvalues[2]])
    print(f"tunnel rear translation ratio {ratio:.3e}; KITTI-shape rear ratios {np.array2string(kitti, precision=3)}")
    assert ratio < kitti.min()


@pytest.mark.gpu
def test_calibration_against_a_map_held_by_a_localizer(K, kitti_run):
    frames, poses, (F, Rm) = kitti_run
    n = 40
    vmap = _gpu_map(K, frames[:n], poses[:n], F)
    loc = K.KissICP(K.load_config(), prior_map=vmap)
    assert vmap.readers() == 1
    before = vmap.dump()
    E0 = _perturb(Rm, 0.2, 2.0, 5)
    cal = K.calibrate_rig(frames[:n], K.Rig([K.Sensor(F), K.Sensor(E0)]), poses=poses[:n], voxel_map=vmap)
    after = vmap.dump()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    t, r = _error(cal.extrinsics[1], Rm)
    assert t < 0.05 and r < 0.25
    del loc
